"""CPU: Level-Based Foraging grid observations (`Foraging-grid[-Ks]-*` ids) -- id parsing and refusals, the observation width through every
layer (Python, ctypes, marl_lbf_obs_dim), hand-computed boards, the literal transcription of upstream against the C restatement, and (where
`lbforaging` imports) upstream itself."""
import ctypes as C

import numpy as np
import pytest

from tests.lbf_grid_kats import KATS, expected, materialise
from tests.lbf_grid_ref import RECALLED, flat_upstream, grid_obs_c


# ---- ids -------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,want", [
    ("lbforaging:Foraging-grid-8x8-2p-3f-v3", dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=8, force_coop=0, penalty=0.0)),
    ("Foraging-grid-2s-8x8-2p-3f-v3", dict(rows=8, cols=8, sight=2)),
    ("lbforaging:Foraging-grid-1s-10x10-3p-3f-coop-v3", dict(rows=10, n_agents=3, sight=1, force_coop=1)),
    ("Foraging-grid-3s-15x15-4p-5f-pen-v3", dict(rows=15, n_agents=4, max_num_food=5, sight=3, penalty=0.1)),
    ("Foraging-grid-8s-8x8-2p-3f-coop-pen-v3", dict(sight=8, force_coop=1, penalty=0.1)),
    ("Foraging-grid-2s-8x8-2p-3f-v2", dict(sight=2, max_player_level=3)),
])
def test_grid_ids_parse(name, want):
    from codebase_b200.lbf import parse_env_id

    cfg = parse_env_id(name, 25)
    assert cfg.grid_observation == 1 and cfg.observe_id == 0 and cfg.time_limit == 25
    for k, v in want.items():
        assert getattr(cfg, k) == v, (k, getattr(cfg, k), v)


@pytest.mark.parametrize("s", [5, 8, 12])
def test_every_registered_grid_sight_parses(s):
    from codebase_b200.lbf import parse_env_id

    for k in RECALLED["grid_sights"](s):
        cfg = parse_env_id(f"lbforaging:Foraging-grid-{k}s-{s}x{s}-2p-3f-v3")
        assert cfg.sight == k and cfg.obs_dim == 3 * (2 * k + 1) ** 2


def test_sight_override_and_vector_ids_unchanged():
    from codebase_b200.lbf import parse_env_id

    assert parse_env_id("Foraging-grid-2s-8x8-2p-3f-v3", sight=1).sight == 1   # env.sight=<k>
    v = parse_env_id("lbforaging:Foraging-2s-8x8-2p-3f-v3")
    assert v.grid_observation == 0 and v.sight == 2 and v.obs_dim == 15
    assert parse_env_id("lbforaging:Foraging-8x8-2p-3f-v3").sight == 8
    with pytest.raises(ValueError, match="unsupported environment id"):   # vector ids keep taking -2s only
        parse_env_id("lbforaging:Foraging-3s-8x8-2p-3f-v3")


@pytest.mark.parametrize("name", ["Foraging-grid-0s-8x8-2p-3f-v3", "Foraging-grid-9s-8x8-2p-3f-v3", "Foraging-grid-12s-10x10-2p-3f-v3"])
def test_grid_sight_out_of_range_refused(name):
    from codebase_b200.lbf import parse_env_id

    with pytest.raises(ValueError, match="sight 1 <= k <="):
        parse_env_id(name)


def test_make_env_needs_flatten_and_refuses_observe_id():
    from codebase_b200.utils.envs import make_env

    with pytest.raises(ValueError, match="FlattenObservation"):
        make_env(0, name="lbforaging:Foraging-grid-2s-8x8-2p-3f-v3", time_limit=25, parallel_envs=4)
    with pytest.raises(ValueError, match="ObserveID wrapper assumes a flattened observation space"):
        make_env(0, name="lbforaging:Foraging-grid-2s-8x8-2p-3f-v3", time_limit=25, parallel_envs=4, observe_id=True,
                 wrappers=["FlattenObservation"])
    with pytest.raises(NotImplementedError):   # other wrappers are still refused
        make_env(0, name="lbforaging:Foraging-grid-2s-8x8-2p-3f-v3", time_limit=25, wrappers=["FlattenObservation", "ClearInfo"])


# ---- observation width in every layer ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sight,D", [(1, 27), (2, 75), (3, 147), (5, 363), (8, 867), (127, 195075)])
def test_obs_dim_python_ctypes_and_c(sight, D):
    from codebase_b200 import _native as nat
    from codebase_b200.lbf import LbfConfig
    from tests import lbf_grid_ref

    cfg = LbfConfig(rows=8, cols=8, sight=sight, grid_observation=1)
    assert cfg.obs_dim == D
    ncfg = cfg.to_native()
    assert ncfg.grid_observation == 1 and C.sizeof(ncfg) == 80
    assert nat.lib().marl_lbf_obs_dim(C.byref(ncfg)) == D
    assert lbf_grid_ref.lib().lbf_grid_obs_dim(C.c_int(sight)) == D
    ncfg.grid_observation = 0
    assert nat.lib().marl_lbf_obs_dim(C.byref(ncfg)) == 3 * 3 + 3 * 2   # the vector width is untouched


def test_obs_dim_refuses_grid_sight_out_of_range():
    from codebase_b200 import _native as nat
    from codebase_b200.lbf import LbfConfig

    for sight in (0, 128):
        ncfg = LbfConfig(sight=sight, grid_observation=1).to_native()
        assert nat.lib().marl_lbf_obs_dim(C.byref(ncfg)) < 0


# ---- known answers -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kat", [k for k in KATS if not any(k["actions"])], ids=lambda k: k["name"])
def test_known_answer_boards(kat):
    cfgkw, field, players, _, _ = materialise(kat)
    want = expected(kat)
    R, Cc, k = cfgkw["rows"], cfgkw["cols"], cfgkw["sight"]
    assert np.array_equal(flat_upstream(field.reshape(R, Cc), players, k), want)
    assert np.array_equal(grid_obs_c(R, Cc, k, field[None], players[None])[0], want)


@pytest.mark.parametrize("kat", [k for k in KATS if any(k["actions"])], ids=lambda k: k["name"])
def test_known_answer_transitions_through_the_oracle_step(kat):
    """The boards with moves or loads: the C oracle's transition, then both grid restatements of the state it leaves."""
    from tests.lbf_grid_ref import GridOracleVecEnv

    cfgkw, field, players, step, actions = materialise(kat)
    orc = GridOracleVecEnv(cfgkw, 1, 0)
    orc.set_state(field[None], players[None], np.array([step], np.int32))
    obs, rew, done, _, _, _ = orc.step(actions[None])
    assert not done[0]
    assert np.array_equal(obs[0], expected(kat))
    assert np.array_equal(flat_upstream(orc.field[0].reshape(cfgkw["rows"], cfgkw["cols"]), orc.players[0], cfgkw["sight"]), expected(kat))


# ---- the two restatements against each other ---------------------------------------------------------------------------------------------------
def _random_states(rng, R, Cc, N, n_states):
    """Random states: foods and players on distinct cells, levels 1..3; in one state of ten the last player stands on the first one's cell
    (reachable: a player enters the cell of one whose own move collided)."""
    fields = np.zeros((n_states, R * Cc), np.int8)
    players = np.zeros((n_states, N, 4), np.int8)
    for s in range(n_states):
        cells = rng.choice(R * Cc, size=N + rng.integers(0, min(6, R * Cc - N) + 1), replace=False)
        for i in range(N):
            players[s, i, :3] = (cells[i] // Cc, cells[i] % Cc, rng.integers(1, 4))
        for c in cells[N:]:
            fields[s, c] = rng.integers(1, 4)
        if N > 1 and s % 10 == 0:
            players[s, N - 1, :2] = players[s, 0, :2]
    return fields, players


@pytest.mark.parametrize("R,Cc,N,sights", [(5, 5, 2, (1, 2, 5)), (8, 8, 2, (1, 2, 3, 8)), (10, 10, 3, (1, 2)), (15, 15, 4, (3,)),
                                           (7, 11, 5, (2, 11)), (20, 20, 9, (2,)), (16, 16, 20, (2,))])
def test_literal_transcription_matches_c_restatement(R, Cc, N, sights):
    """>= 10^5 (state, agent) pairs over all parameter sets."""
    rng = np.random.default_rng(R * 100 + N)
    n_states = max(2000, 16000 // N)
    fields, players = _random_states(rng, R, Cc, N, n_states)
    for k in sights:
        got = grid_obs_c(R, Cc, k, fields, players)
        for s in range(n_states):
            assert np.array_equal(flat_upstream(fields[s].reshape(R, Cc), players[s], k), got[s]), (k, s)


# ---- upstream, where it is installed -----------------------------------------------------------------------------------------------------------
def test_upstream_grid_ids_and_observations():
    lbforaging = pytest.importorskip("lbforaging")
    import gymnasium as gym

    from lbforaging.foraging.environment import ForagingEnv  # noqa: F401

    from codebase_b200.lbf import parse_env_id

    for name in ("Foraging-grid-8x8-2p-3f-v3", "Foraging-grid-2s-8x8-2p-3f-v3", "Foraging-grid-1s-10x10-3p-3f-coop-v3"):
        spec = gym.spec(name)
        cfg = parse_env_id(name)
        assert spec.kwargs["grid_observation"] and spec.kwargs["sight"] == cfg.sight, name
    rng = np.random.default_rng(0)
    env = gym.make("Foraging-grid-2s-8x8-2p-3f-v3").unwrapped
    env.reset(seed=0)
    fields, players = _random_states(rng, 8, 8, 2, 500)
    for s in range(len(fields)):
        env.field = fields[s].reshape(8, 8).astype(np.int32).copy()
        for i, p in enumerate(env.players):
            p.position, p.level = (int(players[s, i, 0]), int(players[s, i, 1])), int(players[s, i, 2])
        obs = env._make_gym_obs()
        got = np.stack([np.asarray(o, np.float32).reshape(-1) for o in obs])
        assert np.array_equal(got, grid_obs_c(8, 8, 2, fields[s:s + 1], players[s:s + 1])[0]), (lbforaging.__name__, s)
