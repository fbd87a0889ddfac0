"""CPU: the repeated matrix games (DESIGN.md Appendix C): id parsing, constructor overrides and refusals (codebase_b200/matrix.py), known
answers of the oracle (oracle/matrix_ref.py) under the wrapper stack, and make_env's dispatch between the env families."""
import numpy as np
import pytest

from codebase_b200 import matrix as M
from codebase_b200.lbf import LbfConfig
from codebase_b200.matrix import MatrixConfig, is_matrix_id, parse_matrix_id
from codebase_b200.rware import RwareConfig
from oracle import matrix_ref as R

GAMES = ["climbing"] + [f"penalty-{k}" for k in (0, 25, 50, 75, 100)]
IDS = [f"{g}{s}-v0" for g in GAMES for s in ("", "-nostate")]
CLIMBING = np.array([[11, -30, 0], [-30, 7, 6], [0, 0, 5]])


def test_twelve_registered_ids():
    assert len(IDS) == 12


@pytest.mark.parametrize("prefix", ["", "matrixgames:"])
@pytest.mark.parametrize("name", IDS)
def test_id_parsing(name, prefix):
    assert is_matrix_id(prefix + name)
    cfg = parse_matrix_id(prefix + name, 30)
    game = name.split("-nostate")[0].removesuffix("-v0")
    k = int(game.split("-")[1]) if game.startswith("penalty") else None
    want = CLIMBING if k is None else np.array([[-k, 0, 10], [0, 2, 0], [10, 0, -k]])
    assert cfg.payoff.dtype == np.float64 and np.array_equal(cfg.payoff, want)
    assert (cfg.n_agents, cfg.n_actions, cfg.ep_length, cfg.time_limit) == (2, 3, 25, 30)
    assert cfg.last_action_state == int("-nostate" not in name)
    assert cfg.obs_dim == (6 if cfg.last_action_state else 1) and cfg.obs_bounds == (0.0, 1.0)


def test_overrides():
    cfg = parse_matrix_id("matrixgames:climbing-v0", 0, ep_length=7, last_action_state=False, payoff_matrix=[[1, 2], [3, 4]])
    assert (cfg.ep_length, cfg.last_action_state, cfg.n_agents, cfg.n_actions, cfg.obs_dim) == (7, 0, 2, 2, 1)
    cfg = parse_matrix_id("penalty-0-nostate-v0", 0, last_action_state=True, payoff_matrix=np.arange(27).reshape(3, 3, 3) * 0.5)
    assert (cfg.n_agents, cfg.n_actions, cfg.obs_dim) == (3, 3, 9) and cfg.payoff[2, 1, 0] == 10.5
    with pytest.raises(TypeError, match="unknown matrix game option"):
        parse_matrix_id("climbing-v0", 0, n_agents=3)
    with pytest.raises(ValueError, match="ep_length"):
        parse_matrix_id("climbing-v0", 0, ep_length=0)


@pytest.mark.parametrize("name,over,match", [
    ("matrixgames:prisoners-v0", {}, "unsupported matrix game id"),
    ("matrixgames:penalty-30-v0", {}, "unsupported matrix game id"),
    ("climbing-v1", {}, "v0"),
    ("matrixgames:penalty-100-nostate-v2", {}, "v0"),
    ("climbing-v0", dict(payoff_matrix=[[1, 2], [3]]), "rectangular"),
    ("climbing-v0", dict(payoff_matrix=np.zeros((2, 3))), "same number of actions"),
    ("climbing-v0", dict(payoff_matrix=np.zeros((9, 9))), "1..8"),
    ("climbing-v0", dict(payoff_matrix=np.zeros((8,) * 6)), "65536"),
    ("climbing-v0", dict(payoff_matrix=np.zeros((2,) * 17)), "65536"),
    ("climbing-v0", dict(payoff_matrix=5), "one dimension per player"),
])
def test_refusals(name, over, match):
    with pytest.raises(ValueError, match=match):
        parse_matrix_id(name, 25, **over)


def test_limits_at_the_edge():
    assert parse_matrix_id("climbing-v0", 0, payoff_matrix=np.zeros((4,) * 8)).payoff.size == 65536
    assert parse_matrix_id("climbing-v0", 0, payoff_matrix=np.zeros((8, 8))).n_actions == 8
    assert parse_matrix_id("climbing-v0", 0, payoff_matrix=np.zeros((1,) * 32)).n_agents == 32


def test_obs_dim():
    for state, oid, want in ((1, 0, 6), (0, 0, 1), (1, 1, 8), (0, 1, 3)):
        assert MatrixConfig(last_action_state=state, observe_id=oid).obs_dim == want
    assert MatrixConfig(payoff=np.zeros((2, 2, 2))).obs_dim == 6


def test_is_matrix_id_leaves_other_families_alone():
    assert not any(is_matrix_id(n) for n in ("smaclite:3m", "lbforaging:Foraging-8x8-2p-3f-v3", "rware:rware-tiny-2ag-v2", "Foraging-8x8-2p-3f-v3"))
    assert is_matrix_id("matrixgames:anything-v0") and not is_matrix_id("anything-v0")


def _cfg(name="climbing-v0", tl=0, **wrap):
    cfg = parse_matrix_id(name, tl)
    for k, v in wrap.items():
        setattr(cfg, k, v)
    return cfg


def test_every_climbing_cell_pays_its_entry_to_both_players():
    w = R.WrappedMatrixGame(_cfg(), payoff=CLIMBING)   # int64, as the package registers it
    for a0 in range(3):
        for a1 in range(3):
            w.reset()
            obs, rew, done, trunc, _ = w.step([a0, a1])
            assert rew.dtype == np.float32 and list(rew) == [CLIMBING[a0, a1]] * 2
            assert not done and not trunc
    _, raw, _ = R.MatrixGame(CLIMBING).step([0, 1])
    assert raw == [-30, -30] and raw[0].dtype == np.int64


def test_one_hot_observation_after_a_step_and_zeros_at_reset():
    w = R.WrappedMatrixGame(_cfg())
    assert np.array_equal(w.reset(), np.zeros((2, 6), np.float32))
    obs, *_ = w.step([2, 0])
    assert np.array_equal(obs, np.array([[0, 0, 1, 1, 0, 0]] * 2, np.float32))
    obs, *_ = w.step([1, 1])
    assert np.array_equal(obs, np.array([[0, 1, 0, 0, 1, 0]] * 2, np.float32))
    assert np.array_equal(w.reset(), np.zeros((2, 6), np.float32))
    w = R.WrappedMatrixGame(_cfg("climbing-nostate-v0"))
    assert np.array_equal(w.reset(), np.zeros((2, 1), np.float32))
    assert np.array_equal(w.step([2, 0])[0], np.zeros((2, 1), np.float32))


def test_terminates_at_ep_length_and_never_truncates_itself():
    w = R.WrappedMatrixGame(_cfg())
    w.reset()
    for t in range(1, 26):
        _, _, done, trunc, info = w.step([0, 0])
        assert done == (t == 25) and not trunc
    assert info["episode_length"] == 25 and list(info["episode_returns"]) == [275.0, 275.0]


@pytest.mark.parametrize("tl,done_at,trunc_at", [(10, None, 10), (25, 25, 25), (40, 25, None)])
def test_time_limit_below_equal_and_above_ep_length(tl, done_at, trunc_at):
    w = R.WrappedMatrixGame(_cfg(tl=tl))
    w.reset()
    end = min(tl, 25)
    for t in range(1, end + 1):
        _, _, done, trunc, info = w.step([1, 2])
        assert done == (t == done_at) and trunc == (t == trunc_at), t
    assert info["episode_length"] == end and list(info["episode_returns"]) == [6.0 * end] * 2


def test_cooperative_reward_pays_n_times_the_payoff():
    w = R.WrappedMatrixGame(_cfg(cooperative_reward=1))
    w.reset()
    _, rew, _, _, info = w.step([0, 1])
    assert list(rew) == [-60.0, -60.0]
    table = np.arange(8).reshape(2, 2, 2)
    w = R.WrappedMatrixGame(MatrixConfig(payoff=table.astype(np.float64), cooperative_reward=1), payoff=table)
    w.reset()
    assert list(w.step([1, 0, 1])[1]) == [15.0] * 3


def test_standardise_reward_sees_the_raw_payoff_and_the_statistics_keep_the_raw_return():
    w = R.WrappedMatrixGame(_cfg(standardise_rewards=1))
    w.reset()
    assert list(w.step([0, 0])[1]) == [11.0, 11.0]   # the first reward passes unchanged
    _, rew, _, _, _ = w.step([0, 1])
    assert np.all(rew < 0) and rew[0] == rew[1]
    assert list(w.episode_reward) == [-19.0, -19.0]


def test_observe_id_layout():
    w = R.WrappedMatrixGame(_cfg(observe_id=1))
    assert w.cfg.obs_dim == 8
    w.reset()
    obs, *_ = w.step([1, 2])
    assert np.array_equal(obs, np.array([[1, 0, 0, 1, 0, 0, 0, 1], [0, 1, 0, 1, 0, 0, 0, 1]], np.float32))
    w = R.WrappedMatrixGame(_cfg("penalty-50-nostate-v0", observe_id=1))
    assert np.array_equal(w.reset(), np.array([[1, 0, 0], [0, 1, 0]], np.float32))


def test_vector_oracle_autoreset_inactive_envs_and_state():
    orc = R.OracleVecMatrix(_cfg(tl=3), 3)
    orc.reset()
    a = np.array([[0, 0], [5, -1], [2, 2]])   # out-of-range actions are played as action 0
    _, rew, *_ = orc.step(a)
    assert list(rew[:, 0]) == [11.0, 11.0, 5.0]
    orc.step(a)
    obs, rew, done, trunc, fret, flen = orc.step(a, autoreset=False)
    assert list(trunc) == [1, 1, 1] and list(done) == [0, 0, 0] and list(flen) == [3, 3, 3] and list(fret[:, 1]) == [33.0, 33.0, 15.0]
    obs, rew, done, trunc, fret, flen = orc.step(a)
    assert list(done) == [1, 1, 1] and not rew.any() and not flen.any()   # inactive envs: done, no reward, frozen observation
    assert np.array_equal(obs[2], np.array([[0, 0, 1, 0, 0, 1]] * 2, np.float32))
    st = orc.state()
    assert st["last_action"].tolist() == [[0, 0], [0, 0], [2, 2]] and list(st["step"]) == [3, 3, 3] and list(st["active"]) == [0, 0, 0]
    obs = orc.reset(np.array([1, 0, 0], bool))
    assert not obs[0].any() and obs[2].any() and list(orc.episode_idx) == [2, 1, 1]


def test_make_env_dispatch(monkeypatch):
    from codebase_b200.utils import envs

    monkeypatch.setattr(envs, "B200VecEnv", lambda cfg, *a, **k: cfg)
    cfg = envs.make_env(0, name="matrixgames:climbing-nostate-v0", time_limit=25, wrappers=["CooperativeReward"], observe_id=True)
    assert isinstance(cfg, MatrixConfig) and (cfg.cooperative_reward, cfg.observe_id, cfg.last_action_state, cfg.obs_dim) == (1, 1, 0, 3)
    assert isinstance(envs.make_env(0, name="penalty-25-v0", time_limit=25, ep_length=10), MatrixConfig)
    assert isinstance(envs.make_env(0, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=25), LbfConfig)
    assert isinstance(envs.make_env(0, name="rware:rware-tiny-2ag-v2", time_limit=500), RwareConfig)
    with pytest.raises(ValueError, match="Level-Based Foraging"):
        envs.make_env(0, name="smaclite:3m", time_limit=500)
    with pytest.raises(ValueError, match="v0"):
        envs.make_env(0, name="matrixgames:climbing-v1", time_limit=25)


def test_recalled_constants_are_named():
    assert M.EP_LENGTH == 25 and M.PENALTY_KS == (0, 25, 50, 75, 100) and M.CLIMBING == tuple(map(tuple, CLIMBING.tolist()))


def test_matrix_config_round_trips_through_the_native_struct():
    cfg = MatrixConfig(payoff=np.arange(27.0).reshape(3, 3, 3), ep_length=9, last_action_state=0, observe_id=1)
    n = cfg.to_native()
    assert (n.n_agents, n.n_actions, n.ep_length, n.last_action_state, n.observe_id) == (3, 3, 9, 0, 1) and n.payoff[26] == 26.0
