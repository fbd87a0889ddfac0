"""GPU: the LBF grid observation (lbf_step_kernel<true>, lbf_grid_obs_kernel) bit for bit against the C restatement on the C oracle's states --
known answers, random rollouts with autoreset, the reset path with its trajectory row, the fused rollouts with trajectory writes -- and the
B200VecEnv surface and the drivers on `Foraging-grid-*` ids."""
import numpy as np
import pytest
import torch

from oracle import policy_ref
from tests.lbf_grid_kats import KATS, expected, materialise
from tests.lbf_grid_ref import GridOracleVecEnv

pytestmark = pytest.mark.gpu


def _native(cfgkw, E, seed, gid0=0):
    from codebase_b200.lbf import LbfConfig, NativeLbf

    return NativeLbf(LbfConfig(**{**cfgkw, "grid_observation": 1}), E, seed, gid0)


def _state_equal(env, orc):
    st = {k: v.cpu().numpy() for k, v in env.get_state().items()}
    return (np.array_equal(st["field"], orc.field) and np.array_equal(st["players"], orc.players) and np.array_equal(st["step"], orc.step_count)
            and np.array_equal(st["episode_idx"].astype(np.uint32), orc.episode_idx))


@pytest.mark.parametrize("kat", KATS, ids=lambda k: k["name"])
def test_known_answer_boards(kat):
    cfgkw, field, players, step, actions = materialise(kat)
    env = _native(cfgkw, 3, 0)   # the same board in three envs
    env.set_state(torch.tensor(np.tile(field, (3, 1))), torch.tensor(np.tile(players, (3, 1, 1))), torch.tensor([step] * 3, dtype=torch.int32))
    obs = env.step(torch.tensor(np.tile(actions, (3, 1)), device="cuda"))[0].cpu().numpy()
    for e in range(3):
        assert np.array_equal(obs[e], expected(kat)), (kat["name"], e)


CONFIGS = [   # (cfg, E, steps): >= 200 000 env-steps each
    (dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=2), 4096, 50),                                                   # D 75
    (dict(rows=10, cols=10, n_agents=3, max_num_food=3, sight=1, force_coop=1, cooperative_reward=1, standardise_rewards=1), 4096, 50),   # D 27
    (dict(rows=15, cols=15, n_agents=4, max_num_food=5, sight=3), 4096, 50),                                                 # D 147
    (dict(rows=20, cols=20, n_agents=9, max_num_food=6, sight=2), 4000, 50),                                                 # G = 16, ragged last CTA
    (dict(rows=5, cols=5, n_agents=2, max_num_food=1, sight=5), 4096, 50),                                                   # D 363
    (dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=8), 4096, 50),                                                   # D 867
    (dict(rows=16, cols=16, n_agents=20, max_num_food=5, sight=2, penalty=0.1), 4096, 50),                                   # 20 agents, G = 32
]


@pytest.mark.parametrize("cfgkw,E,T", CONFIGS, ids=lambda x: str(x) if not isinstance(x, dict) else f"{x['rows']}x{x['cols']}-{x['n_agents']}p-k{x['sight']}")
def test_random_rollouts_bit_exact(cfgkw, E, T):
    rng = np.random.default_rng(7)
    seed, gid0 = 0xC0FFEE1234, 500
    env = _native(cfgkw, E, seed, gid0)
    orc = GridOracleVecEnv(cfgkw, E, seed, gid0)
    assert env.D == orc.D
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())
    N, finished = orc.N, 0
    for t in range(T):
        acts = rng.integers(0, 6, size=(E, N)).astype(np.int32)
        acts[rng.random(acts.shape) < 0.35] = 5
        o, r, d, tr = env.step(torch.tensor(acts, device="cuda"), autoreset=True)
        oo, rr, dd, tt, _, flen = orc.step(acts, autoreset=True)
        assert np.array_equal(o.cpu().numpy(), oo), t
        assert np.array_equal(r.cpu().numpy(), rr), t
        assert np.array_equal(d.cpu().numpy(), dd) and np.array_equal(tr.cpu().numpy(), tt), t
        finished += int((flen > 0).sum())
    assert finished > 0 and _state_equal(env, orc)
    assert E * T >= 200_000


def test_reset_observations_and_trajectory_rows():
    """marl_lbf_reset: obs_out for every env, init_episode's row 0 for the masked envs only, through a wrapping ring."""
    from codebase_b200.lbf import TrajStore

    cfgkw = dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=2)
    E, seed, T = 1000, 3, 25
    env, orc = _native(cfgkw, E, seed), GridOracleVecEnv(cfgkw, E, seed)
    cap, slot0 = E + 13, 40
    traj = TrajStore(cap, 2, T, orc.D, env.device)
    assert np.array_equal(env.reset(traj=traj, slot0=slot0).cpu().numpy(), orc.reset())
    want = np.zeros((cap, 2, T + 1, orc.D), np.float32)
    slots = (slot0 + np.arange(E)) % cap
    want[slots, :, 0] = orc.obs()
    assert np.array_equal(traj.obs.cpu().numpy(), want)
    mask = (np.arange(E) % 3 == 0).astype(np.uint8)
    got = env.reset(torch.tensor(mask, device="cuda"), traj=traj, slot0=slot0).cpu().numpy()
    oo = orc.reset(mask)
    assert np.array_equal(got, oo)
    want[slots[mask == 1], :, 0] = oo[mask == 1]
    assert np.array_equal(traj.obs.cpu().numpy(), want)


@pytest.mark.parametrize("cfgkw", [dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=1),
                                   dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=8),
                                   dict(rows=12, cols=12, n_agents=6, max_num_food=4, sight=3)])
@pytest.mark.parametrize("proper", [False, True])
def test_fused_eps_greedy_rollout_and_replay_writes(cfgkw, proper):
    from codebase_b200.lbf import TrajStore

    rng = np.random.default_rng(3)
    E, seed, gid0, T, A = 512, 77, 64, 25, 6
    env, orc = _native(cfgkw, E, seed, gid0), GridOracleVecEnv(cfgkw, E, seed, gid0)
    N, D = orc.N, orc.D
    cap, slot0 = E + 37, 30
    traj = TrajStore(cap, N, T, D, env.device)
    ref = dict(obs=np.zeros((cap, N, T + 1, D), np.float32), act=np.zeros((cap, N, T), np.int32), rew=np.zeros((cap, N, T), np.float32),
               done=np.zeros((cap, T + 1), np.uint8), filled=np.zeros((cap, T), np.uint8))
    slots = (slot0 + np.arange(E)) % cap
    gids = gid0 + np.arange(E)
    for it in range(2):
        assert np.array_equal(env.reset(traj=traj, slot0=slot0).cpu().numpy(), orc.reset())
        ref["obs"][slots, :, 0] = orc.obs()
        for t in range(T):
            q = rng.standard_normal((E, N, A)).astype(np.float32)
            ep_cur, step0, act0 = orc.episode_idx - 1, orc.step_count.copy(), orc.active.copy().astype(bool)
            want_a = np.where(act0[:, None], policy_ref.eps_greedy(q, 0.3, seed, gids, ep_cur, step0), 0)
            env.rollout_step(torch.tensor(q, device="cuda"), policy=1, epsilon=0.3, traj=traj, slot0=slot0, use_proper_termination=proper)
            assert np.array_equal(env.actions.cpu().numpy(), want_a), (it, t)
            oo, rr, dd, tt, _, _ = orc.step(want_a, autoreset=False)
            assert np.array_equal(env.obs.cpu().numpy(), oo) and np.array_equal(env.rew.cpu().numpy(), rr)
            s = slots[act0]
            ref["act"][s, :, step0[act0]] = want_a[act0]
            ref["rew"][s, :, step0[act0]] = rr[act0]
            ref["obs"][s, :, step0[act0] + 1] = oo[act0]
            ref["done"][s, step0[act0] + 1] = (dd[act0] if proper else (dd[act0] | tt[act0]))
            ref["filled"][s, step0[act0]] = 1
        for k in ref:
            assert np.array_equal(getattr(traj, k).cpu().numpy(), ref[k]), (it, k)
    assert ref["filled"].sum() > 0


def test_fused_categorical_rollout_with_batch_writes():
    """policy 2 (IA2C / IPPO's batch_* writes): actions as the oracle samples them, observations and trajectory rows bit for bit."""
    from codebase_b200.lbf import TrajStore

    rng = np.random.default_rng(9)
    cfgkw = dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=2)
    E, seed, T = 2048, 5, 10
    env, orc = _native(cfgkw, E, seed), GridOracleVecEnv(cfgkw, E, seed)
    traj = TrajStore(E, 2, T, orc.D, env.device)
    env.reset(traj=traj)
    want_obs = np.zeros((E, 2, T + 1, orc.D), np.float32)
    want_obs[:, :, 0] = orc.reset()
    bad_total = 0
    for t in range(T):
        logits = (2.0 * rng.standard_normal((E, 2, 6))).astype(np.float32)
        want, margin = policy_ref.categorical(logits, seed, np.arange(E), orc.episode_idx - 1, orc.step_count)
        act0 = orc.active.copy().astype(bool)
        step0 = orc.step_count.copy()
        env.rollout_step(torch.tensor(logits, device="cuda"), policy=2, traj=traj)
        got = env.actions.cpu().numpy()
        bad = (got != want) & act0[:, None]
        assert np.all(margin[bad] < 1e-5)   # expf differs by an ulp between libm and CUDA: only samples on a CDF edge may differ
        bad_total += int(bad.sum())
        oo = orc.step(got, autoreset=False)[0]
        assert np.array_equal(env.obs.cpu().numpy(), oo)
        want_obs[np.nonzero(act0)[0], :, step0[act0] + 1] = oo[act0]
    assert bad_total < 5
    assert np.array_equal(traj.obs.cpu().numpy(), want_obs)


def test_vecenv_surface():
    from codebase_b200.utils.envs import make_env

    E = 64
    env = make_env(4, name="lbforaging:Foraging-grid-2s-8x8-2p-3f-v3", time_limit=25, parallel_envs=E, wrappers=["FlattenObservation"])
    sp = env.single_observation_space[0]
    assert sp.shape == (75,) and sp.low == -np.inf and sp.high == np.inf and env.observation_space[0].shape == (E, 75)
    assert len(env.single_action_space) == 2 and env.single_action_space[0].n == 6
    orc = GridOracleVecEnv(dict(rows=8, cols=8, n_agents=2, max_num_food=3, sight=2, time_limit=25), E, 4)
    obs, info = env.reset()
    want = orc.reset()
    assert len(obs) == 2 and all(np.array_equal(obs[i], want[:, i]) for i in range(2)) and info == {}
    rng = np.random.default_rng(0)
    seen_final = False
    for t in range(30):
        a = rng.integers(0, 6, size=(2, E))
        obs, rew, done, trunc, info = env.step(a)
        oo, rr, dd, tt, fret, flen = orc.step(a.T.astype(np.int32), autoreset=True)
        assert all(np.array_equal(obs[i], oo[:, i]) for i in range(2)) and np.array_equal(rew, rr)
        assert np.array_equal(done, dd.astype(bool)) and np.array_equal(trunc, tt.astype(bool))
        if "final_info" in info:
            seen_final = True
            for i in np.nonzero(info["_final_info"])[0]:
                fi = info["final_info"][i]
                assert fi["episode_length"] == flen[i] and np.array_equal(fi["episode_returns"], fret[i])
    assert seen_final
    env.close()
    # on a vector id the wrapper only unbounds the Box
    v = make_env(4, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=25, parallel_envs=8, wrappers=["CooperativeReward", "FlattenObservation"])
    assert v.single_observation_space[0].shape == (15,) and v.single_observation_space[0].low == -np.inf and v.cfg.cooperative_reward == 1
    w = make_env(4, name="lbforaging:Foraging-8x8-2p-3f-v3", time_limit=25, parallel_envs=8, wrappers=["CooperativeReward"])
    assert np.array_equal(v.reset()[0][0], w.reset()[0][0]) and w.single_observation_space[0].low == -1.0


def test_create_refusals_name_the_limit():
    from codebase_b200 import _native as nat
    from codebase_b200.lbf import LbfConfig, NativeLbf

    with pytest.raises(nat.NativeError, match="observe_id"):
        NativeLbf(LbfConfig(grid_observation=1, sight=2, observe_id=1), 4, 0)
    with pytest.raises(nat.NativeError, match="shared memory per CTA"):
        NativeLbf(LbfConfig(rows=60, cols=60, n_agents=2, sight=2, grid_observation=1), 4, 0)


@pytest.mark.parametrize("alg,env,wrappers,extra", [
    ("ia2c", "Foraging-grid-2s-8x8-2p-3f-v3", "[FlattenObservation]", []),
    ("ippo", "Foraging-grid-2s-8x8-2p-3f-v3", "[FlattenObservation]", []),
    ("maa2c", "Foraging-grid-1s-8x8-2p-3f-v3", "[FlattenObservation]", []),
    ("idqn", "Foraging-grid-1s-8x8-2p-3f-v3", "[FlattenObservation]", ["algorithm.batch_size=128", "algorithm.buffer_size=4096"]),
    ("vdn", "Foraging-grid-1s-8x8-2p-3f-v3", "[CooperativeReward,FlattenObservation]", ["algorithm.batch_size=128", "algorithm.buffer_size=4096"]),
    ("qmix", "Foraging-grid-1s-8x8-2p-3f-v3", "[FlattenObservation]", ["algorithm.batch_size=128", "algorithm.buffer_size=4096"]),
])
def test_drivers_and_checkpoint_eval(tmp_path, monkeypatch, alg, env, wrappers, extra):
    import pandas as pd

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    run.main([f"+algorithm={alg}", f"env.name=lbforaging:{env}", f"env.wrappers={wrappers}", "env.time_limit=25", "env.parallel_envs=64", "seed=0",
              "algorithm.total_steps=20000", "algorithm.eval_interval=10000", "algorithm.save_interval=10000", f"run_dir={out}"] + extra)
    df = pd.read_csv(f"{out}/results.csv")
    assert len(df) >= 1 and np.isfinite(df["loss"]).all()
    monkeypatch.chdir(tmp_path)
    res = ev.main([f"path={out}", "episodes=16", "seed=3"])
    assert res["episodes"] == 16 and np.isfinite(res["mean_episode_returns"]) and 0.0 <= res["mean_episode_returns"] <= 1.0 + 1e-6
