"""Hand-computed known-answer boards of the multi-robot warehouse (DESIGN.md Appendix B), shared by the oracle test (tests/test_rware.py)
and the kernel test (tests/test_rware_gpu.py).

All boards are rware-tiny (11 rows x 10 columns, column_height 8): highways are the columns x = 0, 3, 6, 9, the rows y = 0, 9, 10 and the
queuing box x = 4, 5 below row 0; shelves 1..32 sit on x = 1, 2, 7, 8 for y = 1..8, id = 4 * (y - 1) + (1, 2, 3, 4)[x in (1, 2, 7, 8)];
the goals are (4, 10) and (5, 10).  An agent is (x, y, dir, carried shelf); dir UP 0, DOWN 1, LEFT 2, RIGHT 3; actions NOOP 0, FORWARD 1,
LEFT 2, RIGHT 3, TOGGLE_LOAD 4.  `moved` places shelves away from their home cell (a carried shelf sits at its carrier's cell; None: the
shelf is off the board's grid layer, i.e. nowhere).  A move graph on a grid is bipartite, so it has no cycle of odd length: the boards
rotate 4- and 6-cycles.
"""
from __future__ import annotations

import numpy as np

U, D, L, R = 0, 1, 2, 3
NOOP, FWD, TL, TR, TOG = range(5)


def shelf_id(x, y):
    return 4 * (y - 1) + {1: 1, 2: 2, 7: 3, 8: 4}[x]


EMPTY = [0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0]   # no agent (direction written as UP), no shelf


def _cell(agent=None, shelf=None, req=False):
    a = [0.0, 1.0, 0.0, 0.0, 0.0] if agent is None else [1.0] + [float(agent == k) for k in range(4)]
    return a + ([1.0, float(req)] if shelf else [0.0, 0.0])


KATS = [
    dict(name="move into an empty cell", agents=[(3, 5, U, 0)], actions=[FWD], want=[(3, 4, U, 0)]),
    dict(name="chain of three moves together", agents=[(3, 2, U, 0), (3, 3, U, 0), (3, 4, U, 0)], actions=[FWD] * 3,
         want=[(3, 1, U, 0), (3, 2, U, 0), (3, 3, U, 0)]),
    dict(name="two into one empty cell: the longer chain wins", agents=[(2, 0, R, 0), (4, 0, L, 0), (5, 0, L, 0)], actions=[FWD] * 3,
         want=[(2, 0, R, 0), (3, 0, L, 0), (4, 0, L, 0)]),
    dict(name="two into one empty cell: equal chains, the lower index wins", agents=[(2, 0, R, 0), (4, 0, L, 0)], actions=[FWD] * 2,
         want=[(3, 0, R, 0), (4, 0, L, 0)]),
    dict(name="equal chains: the agent whose cell entered the graph first wins", agents=[(5, 0, L, 0), (2, 0, R, 0), (4, 0, L, 0), (1, 0, R, 0)],
         actions=[FWD] * 4, want=[(4, 0, L, 0), (2, 0, R, 0), (3, 0, L, 0), (1, 0, R, 0)]),
    dict(name="swap is blocked", agents=[(3, 0, R, 0), (4, 0, L, 0)], actions=[FWD] * 2, want=[(3, 0, R, 0), (4, 0, L, 0)]),
    dict(name="4-cycle rotates", agents=[(3, 0, R, 0), (4, 0, D, 0), (4, 1, L, 0), (3, 1, U, 0)], actions=[FWD] * 4,
         want=[(4, 0, R, 0), (4, 1, D, 0), (3, 1, L, 0), (3, 0, U, 0)]),
    dict(name="6-cycle rotates", agents=[(3, 0, R, 0), (4, 0, R, 0), (5, 0, D, 0), (5, 1, L, 0), (4, 1, L, 0), (3, 1, U, 0)], actions=[FWD] * 6,
         want=[(4, 0, R, 0), (5, 0, R, 0), (5, 1, D, 0), (4, 1, L, 0), (3, 1, L, 0), (3, 0, U, 0)]),
    dict(name="a tail into a cycle stays", agents=[(3, 0, R, 0), (4, 0, D, 0), (4, 1, L, 0), (3, 1, U, 0), (2, 0, R, 0)], actions=[FWD] * 5,
         want=[(4, 0, R, 0), (4, 1, D, 0), (3, 1, L, 0), (3, 0, U, 0), (2, 0, R, 0)]),
    dict(name="queueing behind a turning agent", agents=[(3, 3, U, 0), (3, 4, U, 0), (3, 5, U, 0)], actions=[TL, FWD, FWD],
         want=[(3, 3, L, 0), (3, 4, U, 0), (3, 5, U, 0)]),
    dict(name="turns: RIGHT steps UP -> RIGHT -> DOWN -> LEFT, LEFT steps back", agents=[(0, 1, U, 0), (0, 3, L, 0), (0, 5, U, 0), (0, 7, R, 0)],
         actions=[TR, TR, TL, TL], want=[(0, 1, R, 0), (0, 3, U, 0), (0, 5, L, 0), (0, 7, U, 0)]),
    dict(name="wall clamp", agents=[(0, 5, L, 0), (9, 0, U, 0), (9, 10, D, 0), (8, 10, D, 0)], actions=[FWD] * 4,
         want=[(0, 5, L, 0), (9, 0, U, 0), (9, 10, D, 0), (8, 10, D, 0)]),
    dict(name="a loaded agent is blocked by a resting shelf", agents=[(3, 3, L, 6)], moved={6: (3, 3)}, actions=[FWD], want=[(3, 3, L, 6)]),
    dict(name="a loaded agent follows a loaded agent into its cell", agents=[(3, 3, U, 6), (3, 4, U, 10)], moved={6: (3, 3), 10: (3, 4)},
         actions=[FWD, FWD], want=[(3, 2, U, 6), (3, 3, U, 10)], want_moved={6: (3, 2), 10: (3, 3)}),
    dict(name="a loaded agent is blocked by an unloaded agent standing under a shelf", agents=[(3, 1, L, 5), (2, 1, U, 0)], moved={5: (3, 1)},
         actions=[FWD, NOOP], want=[(3, 1, L, 5), (2, 1, U, 0)]),
    dict(name="an unloaded agent walks under shelves", agents=[(1, 1, D, 0), (2, 4, U, 0)], actions=[FWD, FWD], want=[(1, 2, D, 0), (2, 3, U, 0)]),
    dict(name="pickup", agents=[(1, 1, U, 0), (0, 1, U, 0)], actions=[TOG, TOG], want=[(1, 1, U, 1), (0, 1, U, 0)]),
    dict(name="drop refused on a highway", agents=[(3, 1, U, 1)], moved={1: (3, 1)}, actions=[TOG], want=[(3, 1, U, 1)]),
    dict(name="drop on a free shelf cell", agents=[(1, 1, U, 5)], moved={1: None, 5: (1, 1)}, actions=[TOG], want=[(1, 1, U, 0)]),
    dict(name="delivery pays only the agent on the goal", agents=[(4, 9, D, 3), (3, 10, U, 0)], moved={3: (4, 9)}, requested=[3, 20],
         actions=[FWD, NOOP], want=[(4, 10, D, 3), (3, 10, U, 0)], want_moved={3: (4, 10)}, rewards=[1.0, 0.0], delivered=[3]),
    dict(name="two simultaneous deliveries, goals in order", agents=[(5, 10, D, 3), (4, 10, D, 4), (6, 10, U, 0)], moved={3: (5, 10), 4: (4, 10)},
         requested=[3, 4, 30], actions=[NOOP] * 3, want=[(5, 10, D, 3), (4, 10, D, 4), (6, 10, U, 0)], rewards=[1.0, 1.0, 0.0], delivered=[4, 3]),
    dict(name="an unrequested shelf on a goal pays nothing", agents=[(4, 10, D, 3)], moved={3: (4, 10)}, requested=[20], actions=[NOOP],
         want=[(4, 10, D, 3)], rewards=[0.0], inactive=3, want_inactive=4),
    dict(name="termination at max_steps", agents=[(3, 5, U, 0)], actions=[NOOP], step=499, want=[(3, 5, U, 0)], done=True),
    dict(name="no termination the step before max_steps", agents=[(3, 5, U, 0)], actions=[NOOP], step=498, want=[(3, 5, U, 0)], done=False),
    dict(name="termination at max_inactivity_steps", cfg=dict(max_inactivity_steps=5), agents=[(3, 5, U, 0)], actions=[NOOP], inactive=4,
         want=[(3, 5, U, 0)], done=True),
    dict(name="a delivery restarts the inactivity count", cfg=dict(max_inactivity_steps=5), agents=[(4, 10, D, 3)], moved={3: (4, 10)},
         requested=[3], inactive=4, actions=[NOOP], want=[(4, 10, D, 3)], rewards=[1.0], delivered=[3], want_inactive=0, done=False),
    dict(name="observation at the corner (0, 0): padding and the empty-cell direction", agents=[(0, 0, U, 0)], requested=[1], actions=[NOOP],
         want=[(0, 0, U, 0)],
         obs={0: [0, 0, 0, 1, 0, 0, 0, 1] + EMPTY * 3 + EMPTY + _cell(U) + EMPTY + EMPTY + EMPTY + _cell(None, 1, True)}),
    dict(name="observation at the corner (9, 0) with a neighbour facing DOWN", agents=[(9, 0, R, 0), (8, 1, D, 0)], actions=[NOOP, NOOP],
         want=[(9, 0, R, 0), (8, 1, D, 0)],
         obs={0: [9, 0, 0, 0, 0, 0, 1, 1] + EMPTY * 3 + EMPTY + _cell(R) + EMPTY + _cell(D, 4) + EMPTY + EMPTY}),
    dict(name="observation at the corner (0, 10), carrying", agents=[(0, 10, L, 29)], moved={29: (0, 10)}, actions=[NOOP], want=[(0, 10, L, 29)],
         obs={0: [0, 10, 1, 0, 0, 1, 0, 1] + EMPTY + EMPTY + EMPTY + EMPTY + _cell(L, 29) + EMPTY + EMPTY * 3}),
    dict(name="observation at the corner (9, 10)", agents=[(9, 10, D, 0)], actions=[NOOP], want=[(9, 10, D, 0)],
         obs={0: [9, 10, 0, 0, 1, 0, 0, 1] + EMPTY * 3 + EMPTY + _cell(D) + EMPTY + EMPTY * 3}),
    dict(name="observation on a shelf cell, under a requested shelf", agents=[(7, 4, U, 0)], requested=[15], actions=[NOOP], want=[(7, 4, U, 0)],
         obs={0: [7, 4, 0, 1, 0, 0, 0, 0] + EMPTY + _cell(None, 11) + _cell(None, 12) + EMPTY + _cell(U, 15, True) + _cell(None, 16)
              + EMPTY + _cell(None, 19) + _cell(None, 20)}),
]


def materialise(kat):
    """(cfg, shelves uint8 [rows*cols], agents uint8 [N][4], requested int32 [8], step, inactive) of a board."""
    from codebase_b200.rware import parse_rware_id
    from oracle import rware_ref

    n = len(kat["agents"])
    cfg = parse_rware_id(f"rware-tiny-{n}ag-v2", 0, **kat.get("cfg", {}))
    cfg.request_queue_size = max(1, len(kat.get("requested", [20])))
    shelves = rware_ref.home_shelves(cfg)
    for s, where in kat.get("moved", {}).items():
        shelves[shelves == s] = 0
        if where is not None:
            shelves[where[1] * cfg.cols + where[0]] = s
    req = np.zeros(8, np.uint32)
    for s in kat.get("requested", [20]):
        req[s >> 5] |= np.uint32(1 << (s & 31))
    return cfg, shelves, np.array(kat["agents"], np.uint8).reshape(n, 4), req.view(np.int32), kat.get("step", 0), kat.get("inactive", 0)


def expected_shelves(kat, cfg):
    from oracle import rware_ref

    shelves = rware_ref.home_shelves(cfg)
    for s, where in {**kat.get("moved", {}), **kat.get("want_moved", {})}.items():
        shelves[shelves == s] = 0
        if where is not None:
            shelves[where[1] * cfg.cols + where[0]] = s
    return shelves
