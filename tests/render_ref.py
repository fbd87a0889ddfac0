"""numpy restatement of the frame rasteriser (DESIGN.md §4.8), the oracle of lbf_render_kernel and rware_render_kernel.

Written from the specification, not from the kernels: a frame is composed cell by cell from tiles, each tile layered from whole-tile masks,
where the kernels evaluate one pixel at a time.  Integer arithmetic only, so frames compare bit for bit.
"""
from __future__ import annotations

import functools

import numpy as np

WHITE, BLACK = (255, 255, 255), (0, 0, 0)
LBF = dict(cell=50, food_r=16, agent_r=20, badge_c=37, badge_r=11, badge_line=2, food=(197, 58, 50), agent=(46, 104, 190))
RWARE = dict(cell=30, shelf_pad=2, agent_r=10, dir_line=2, goal=(60, 60, 60), shelf=(72, 61, 139), shelf_requested=(0, 128, 128),
             agent=(255, 140, 0), agent_loaded=(255, 0, 0), dir=(0, 0, 0))
FONT_SCALE, DIGIT_GAP = 2, 2
FONT = {
    0: ("###", "#.#", "#.#", "#.#", "###"), 1: (".#.", "##.", ".#.", ".#.", "###"), 2: ("###", "..#", "###", "#..", "###"),
    3: ("###", "..#", "###", "..#", "###"), 4: ("#.#", "#.#", "###", "..#", "..#"), 5: ("###", "#..", "###", "..#", "###"),
    6: ("###", "#..", "###", "#.#", "###"), 7: ("###", "..#", "..#", "..#", "..#"), 8: ("###", "#.#", "###", "#.#", "###"),
    9: ("###", "#.#", "###", "..#", "###"),
}
UP, DOWN, LEFT, RIGHT = 0, 1, 2, 3


def frame_shape(rows, cols, cell):
    return 1 + rows * (cell + 1), 1 + cols * (cell + 1), 3


def disc(g, cx, cy, r):
    """Pixels of a g x g tile whose centres lie within r of corner (cx, cy), in half pixels."""
    ly, lx = np.mgrid[0:g, 0:g]
    return (2 * (lx - cx) + 1) ** 2 + (2 * (ly - cy) + 1) ** 2 <= 4 * r * r


def rect(g, x0, y0, x1, y1):
    m = np.zeros((g, g), bool)
    m[max(y0, 0):max(y1, 0), max(x0, 0):max(x1, 0)] = True
    return m


def text(g, value, cx, cy):
    """Inked pixels of `value` in decimal, the text box centred on corner (cx, cy)."""
    glyphs = [np.kron(np.array([[ch == "#" for ch in row] for row in FONT[int(d)]]), np.ones((FONT_SCALE, FONT_SCALE), bool)) for d in str(value)]
    gap = np.zeros((5 * FONT_SCALE, DIGIT_GAP), bool)
    box = glyphs[0]
    for gl in glyphs[1:]:
        box = np.concatenate([box, gap, gl], axis=1)
    m = np.zeros((g, g), bool)
    top, left = cy - box.shape[0] // 2, cx - box.shape[1] // 2
    for (y, x) in zip(*np.nonzero(box)):
        if 0 <= top + y < g and 0 <= left + x < g:
            m[top + y, left + x] = True
    return m


def paint(tile, mask, colour):
    tile[mask] = colour


def compose(tiles, rows, cols, cell):
    """Frame from a dict (row, col) -> tile; cells not in it are white; grid lines black."""
    H, W, _ = frame_shape(rows, cols, cell)
    f = np.zeros((H, W, 3), np.uint8)
    blank = np.full((cell, cell, 3), WHITE, np.uint8)
    for r in range(rows):
        for c in range(cols):
            y, x = 1 + r * (cell + 1), 1 + c * (cell + 1)
            f[y:y + cell, x:x + cell] = tiles.get((r, c), blank)
    return f


@functools.lru_cache(maxsize=None)
def lbf_tile(food, agent, level):
    """Cell with a food of level `food` (0: none), an agent (True / False), and the badge of `level`."""
    P = LBF
    g, m = P["cell"], P["cell"] // 2
    t = np.full((g, g, 3), WHITE, np.uint8)
    if food:
        paint(t, disc(g, m, m, P["food_r"]), P["food"])
    if agent:
        paint(t, disc(g, m, m, P["agent_r"]), P["agent"])
    bc = P["badge_c"]
    paint(t, disc(g, bc, bc, P["badge_r"]), BLACK)
    paint(t, disc(g, bc, bc, P["badge_r"] - P["badge_line"]), WHITE)
    paint(t, text(g, level, bc, bc) & disc(g, bc, bc, P["badge_r"]), BLACK)
    return t


def lbf_frame(field, players):
    """field: int [rows, cols] food levels (0: none); players: int [N, 3] (row, col, level).  The badge shows the level of the highest-index
    agent on the cell, else the food's."""
    field = np.asarray(field).astype(np.int64) & 0xFF
    rows, cols = field.shape
    top = {}
    for i, (r, c, _) in enumerate(np.asarray(players)):
        top[(int(r), int(c))] = i
    tiles = {}
    for r, c in set(zip(*np.nonzero(field))) | set(top):
        r, c = int(r), int(c)
        who = top.get((r, c))
        level = int(players[who][2]) if who is not None else int(field[r, c])
        tiles[(r, c)] = lbf_tile(int(field[r, c]), who is not None, level)
    return compose(tiles, rows, cols, LBF["cell"])


@functools.lru_cache(maxsize=None)
def rware_tile(goal, shelf, agent, direction):
    """goal: bool; shelf: 0 none, 1 shelf, 2 requested shelf; agent: 0 none, 1 unloaded, 2 loaded; direction 0..3."""
    P = RWARE
    g, m, r = P["cell"], P["cell"] // 2, P["agent_r"]
    t = np.full((g, g, 3), WHITE, np.uint8)
    if goal:
        t[:] = P["goal"]
    if shelf:
        pad = P["shelf_pad"]
        paint(t, rect(g, pad, pad, g - pad, g - pad), P["shelf_requested"] if shelf == 2 else P["shelf"])
    if agent:
        paint(t, disc(g, m, m, r), P["agent_loaded"] if agent == 2 else P["agent"])
        w, h = P["dir_line"], P["dir_line"] // 2
        line = {UP: rect(g, m - h, m - r, m - h + w, m), DOWN: rect(g, m - h, m, m - h + w, m + r),
                LEFT: rect(g, m - r, m - h, m, m - h + w), RIGHT: rect(g, m, m - h, m + r, m - h + w)}[direction]
        paint(t, line, P["dir"])
    return t


def rware_goals(rows, cols):
    return {(rows - 1, cols // 2 - 1), (rows - 1, cols // 2)}


def rware_frame(shelves, agents, requested):
    """shelves: int [rows, cols] shelf id at its current cell (0: none); agents: int [N, 4] (x, y, dir, carried shelf id); requested: uint32 [8],
    bit k of the 256-bit mask = shelf k requested."""
    shelves = np.asarray(shelves).astype(np.int64)
    rows, cols = shelves.shape
    req = np.asarray(requested).astype(np.uint64)
    is_req = lambda s: bool((int(req[s >> 5]) >> (s & 31)) & 1)   # noqa: E731
    top = {(int(a[1]), int(a[0])): a for a in np.asarray(agents)}
    goals = rware_goals(rows, cols)
    tiles = {}
    for r, c in set(zip(*np.nonzero(shelves))) | set(top) | goals:
        r, c = int(r), int(c)
        sid = int(shelves[r, c])
        a = top.get((r, c))
        agent = 0 if a is None else (2 if int(a[3]) else 1)
        tiles[(r, c)] = rware_tile((r, c) in goals, 0 if not sid else (2 if is_req(sid) else 1), agent, 0 if a is None else int(a[2]))
    return compose(tiles, rows, cols, RWARE["cell"])
