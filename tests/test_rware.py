"""CPU: the multi-robot warehouse oracle (oracle/rware_ref.py) against hand-computed boards, its closed-form move resolution against a
literal transcription of upstream's networkx resolution, and the id parser's layouts and refusals (DESIGN.md Appendix B)."""
import numpy as np
import pytest

from codebase_b200.rware import RwareConfig, parse_rware_id
from oracle import rware_ref as R
from tests.rware_kats import KATS, expected_shelves, materialise


@pytest.mark.parametrize("kat", KATS, ids=[k["name"] for k in KATS])
def test_known_answer_boards(kat):
    cfg, shelves, agents, req, step, inactive = materialise(kat)
    wh = R.Warehouse(cfg)
    wh.load(shelves, agents, req, step, inactive)
    before = set(np.nonzero(wh.requested)[0])
    rew, done = wh.step(kat["actions"], seed=7, env_gid=3, episode=0)
    assert [tuple(a) for a in wh.agents] == [tuple(a) for a in kat["want"]]
    assert np.array_equal(wh.shelves, expected_shelves(kat, cfg))
    assert rew == kat.get("rewards", [0.0] * len(kat["agents"]))
    assert done == kat.get("done", False)
    after = set(np.nonzero(wh.requested)[0])
    gone = before - after
    assert sorted(gone) == sorted(kat.get("delivered", [])) and len(after) == len(before)
    assert not (after - before) & before   # replacements come from the shelves that were not requested
    if "want_inactive" in kat:
        assert wh.inactive == kat["want_inactive"]
    for i, want in kat.get("obs", {}).items():
        assert np.array_equal(wh.obs(i), np.array(want, np.float32)), kat["name"]


def test_enough_known_answer_boards():
    assert len(KATS) >= 20


def _random_board(rng, cfg, N):
    RC = cfg.rows * cfg.cols
    if rng.random() < 0.7:   # crowd the agents into a window so that chains, merges and cycles are frequent
        w = min(RC, int(rng.integers(N, 3 * N + 4)))
        cells = int(rng.integers(0, RC - w + 1)) + rng.choice(w, N, replace=False)
    else:
        cells = rng.choice(RC, N, replace=False)
    home = R.home_shelves(cfg)
    shelves = np.where(rng.random(RC) < 0.5, home, 0).astype(np.uint8)
    agents = []
    for c in cells:
        carry = int(rng.integers(1, 250)) if rng.random() < 0.4 else 0
        if carry:
            shelves[c] = carry
        agents.append([int(c % cfg.cols), int(c // cfg.cols), int(rng.integers(0, 4)), carry])
    actions = rng.choice(5, N, p=[0.1, 0.6, 0.1, 0.1, 0.1])
    return agents, shelves, actions


def test_closed_form_resolution_equals_networkx():
    """100 000 random boards over the four sizes and 1..19 agents.  networkx breaks a tie between two equally long chains by the iteration
    order of the component's node set (a Python set of (x, y) tuples); the closed form takes the cell that entered the graph first.  So the
    two must agree exactly when the closed form is given networkx's order, and may differ only on boards with such a tie."""
    pytest.importorskip("networkx")
    rng = np.random.default_rng(2024)
    n = ties = 0
    for size in ("tiny", "small", "medium", "large"):
        for N in range(1, 20):
            cfg = parse_rware_id(f"rware-{size}-{N}ag-v2")
            for _ in range(1316):
                agents, shelves, actions = _random_board(rng, cfg, N)
                want, node_pos = R.resolve_moves_networkx(cfg, agents, shelves, actions)
                assert R.resolve_moves(cfg, agents, shelves, actions, tie_rank=node_pos) == want, (size, N, agents, list(actions))
                ties += R.resolve_moves(cfg, agents, shelves, actions) != want
                n += 1
    assert n >= 100_000
    assert ties < 0.1 * n


@pytest.mark.parametrize("size,rows,cols,shelves", [("tiny", 11, 10, 32), ("small", 20, 10, 80), ("medium", 20, 16, 144), ("large", 29, 16, 224)])
def test_layout(size, rows, cols, shelves):
    cfg = parse_rware_id(f"rware:rware-{size}-2ag-v2")
    assert (cfg.rows, cfg.cols) == (rows, cols) and R.n_shelves(cfg) == shelves
    assert R.goals(cfg) == [(cols // 2 - 1, rows - 1), (cols // 2, rows - 1)]
    home = R.home_shelves(cfg)
    assert sorted(home[home > 0]) == list(range(1, shelves + 1))   # ids 1.. in row-major order
    assert list(home[home > 0]) == list(range(1, shelves + 1))
    for y in range(rows):
        for x in range(cols):
            hw = x % 3 == 0 or y % 9 == 0 or y == rows - 1 or (y > rows - 11 and x in (cols // 2 - 1, cols // 2))
            assert R.is_highway(cfg, x, y) == hw and (home[y * cols + x] == 0) == hw
    for g in R.goals(cfg):
        assert R.is_highway(cfg, *g)


def test_ids_and_request_sizes():
    assert parse_rware_id("rware-tiny-4ag-v2").request_queue_size == 4
    assert parse_rware_id("rware:rware-small-2ag-easy-v2").request_queue_size == 4
    assert parse_rware_id("rware-medium-6ag-hard-v2").request_queue_size == 3
    assert parse_rware_id("rware-large-19ag-hard-v2").request_queue_size == 9
    assert parse_rware_id("rware-large-1ag-hard-v2").request_queue_size == 0   # as upstream computes it; the native handle refuses 0
    c = parse_rware_id("rware-tiny-4ag-v2", 500)
    assert (c.column_height, c.sensor_range, c.max_steps, c.max_inactivity_steps, c.time_limit) == (8, 1, 500, 0, 500)
    assert c.obs_dim == 71 and c.n_actions == 5
    assert RwareConfig(n_agents=3, observe_id=1).obs_dim == 74
    c = parse_rware_id("rware-tiny-2ag-v2", 0, column_height=4, shelf_columns=5, max_inactivity_steps=100, sensor_range=2)
    assert (c.rows, c.cols, c.max_inactivity_steps, c.obs_dim) == (7, 16, 100, 8 + 7 * 25)


@pytest.mark.parametrize("name,kw,match", [
    ("rware-tiny-4ag-v1", {}, "v2"),
    ("rware-tiny-4ag-v2", dict(msg_bits=2), "msg_bits"),
    ("rware-tiny-4ag-v2", dict(observation_type="image"), "observation_type"),
    ("rware-tiny-4ag-v2", dict(observation_type="dict"), "observation_type"),
    ("rware-tiny-4ag-v2", dict(reward_type="global"), "reward_type"),
    ("rware-huge-4ag-v2", {}, "size"),
    ("rware-tiny-20ag-v2", {}, "agents"),
    ("rware-tiny-4ag-medium-v2", {}, "unsupported RWARE id"),
])
def test_refusals(name, kw, match):
    with pytest.raises(ValueError, match=match):
        parse_rware_id(name, 0, **kw)
    with pytest.raises(TypeError):
        parse_rware_id("rware-tiny-4ag-v2", 0, colour="blue")


def test_make_env_dispatch_refuses_before_any_native_call():
    from codebase_b200.utils.envs import make_env

    with pytest.raises(ValueError, match="v2"):
        make_env(0, name="rware:rware-tiny-2ag-v1", time_limit=500)
    with pytest.raises(ValueError, match="Level-Based Foraging"):
        make_env(0, name="smaclite:3m", time_limit=500)


def test_oracle_reset_and_episode():
    """Reset draws distinct cells and exactly request_queue_size requests; the request set keeps its size through deliveries."""
    cfg = parse_rware_id("rware-tiny-4ag-v2", 60)
    venv = R.OracleVecRware(cfg, 16, seed=3)
    obs = venv.reset()
    assert obs.shape == (16, 4, 71)
    rng = np.random.default_rng(0)
    for _ in range(120):
        for w in venv.envs:
            cells = {(a[0], a[1]) for a in w.env.agents}
            assert len(cells) == 4 and w.env.requested.sum() == 4 and not w.env.requested[0]
        venv.step(rng.integers(0, 5, size=(16, 4)), autoreset=True)
    assert venv.episode_idx.min() >= 2
