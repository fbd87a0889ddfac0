"""GPU: the CUDA multi-robot warehouse (marl_rware_* through codebase_b200.rware) BIT-EXACT against the CPU oracle (oracle/rware_ref.py):
known-answer boards, random rollouts with autoreset and the wrappers, the fused categorical rollout with trajectory writes, sharding, the
vector-env surface; one IPPO update on an RWARE batch against the learner oracle; the IA2C / IPPO drivers and checkpoint evaluation."""
import numpy as np
import pytest
import torch

from codebase_b200.rware import NativeRware, parse_rware_id
from oracle import learner_ref as lr
from oracle import policy_ref
from oracle.rware_ref import OracleVecRware
from tests.helpers import ac_model, ac_oracle_batch, traj_store
from tests.rware_kats import KATS, expected_shelves, materialise

pytestmark = pytest.mark.gpu


def _assert_state_equal(env, orc, what=""):
    got = {k: v.cpu().numpy() for k, v in env.get_state().items()}
    want = orc.state()
    for k in want:
        assert np.array_equal(got[k], want[k]), (what, k)


def test_known_answer_boards():
    for kat in KATS:
        cfg, shelves, agents, req, step, inactive = materialise(kat)
        env = NativeRware(cfg, 1, seed=7, env_gid0=3)
        orc = OracleVecRware(cfg, 1, seed=7, gid0=3)
        orc.envs[0].n_resets = 1
        orc.envs[0].env.load(shelves, agents, req, step, inactive)
        env.set_state(torch.tensor(shelves[None]), torch.tensor(agents[None]), torch.tensor(req[None]), torch.tensor([step]), torch.tensor([inactive]))
        obs, rew, done, trunc = env.step(torch.tensor([kat["actions"]], dtype=torch.int32, device="cuda"))
        oo, rr, dd, tt, _, _ = orc.step(np.array([kat["actions"]]))
        st = {k: v.cpu().numpy() for k, v in env.get_state().items()}
        assert [tuple(a) for a in st["agents"][0]] == [tuple(a) for a in kat["want"]], kat["name"]
        assert np.array_equal(st["shelves"][0], expected_shelves(kat, cfg)), kat["name"]
        assert list(rew.cpu().numpy()[0]) == kat.get("rewards", [0.0] * len(kat["agents"])), kat["name"]
        assert bool(done.cpu()[0]) == kat.get("done", False), kat["name"]
        for i, want in kat.get("obs", {}).items():
            assert np.array_equal(obs.cpu().numpy()[0, i], np.array(want, np.float32)), kat["name"]
        assert np.array_equal(obs.cpu().numpy(), oo) and np.array_equal(rew.cpu().numpy(), rr), kat["name"]
        assert np.array_equal(st["requested"], orc.state()["requested"]) and np.array_equal(st["inactive"], orc.state()["inactive"]), kat["name"]
        env.close()


# (id, env overrides, wrappers, E, steps): >= 200 000 env-steps in all, every config ending episodes (autoreset) several times
CONFIGS = [
    ("rware-tiny-4ag-v2", dict(time_limit=40), dict(cooperative_reward=1), 700, 130),
    ("rware-small-2ag-easy-v2", dict(max_inactivity_steps=30), dict(observe_id=1, standardise_rewards=1), 600, 130),
    ("rware-medium-6ag-hard-v2", dict(max_steps=50), dict(), 256, 110),
    ("rware-large-19ag-v2", dict(time_limit=35), dict(standardise_rewards=1, cooperative_reward=1, observe_id=1), 64, 80),
]


@pytest.mark.parametrize("name,over,wrap,E,steps", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_random_rollouts_bit_exact(name, over, wrap, E, steps):
    over = dict(over)
    tl = over.pop("time_limit", 0)
    cfg = parse_rware_id(name, tl, **over)
    for k, v in wrap.items():
        setattr(cfg, k, v)
    seed, gid0 = 0xC0FFEE1234567, 500
    env = NativeRware(cfg, E, seed, gid0)
    orc = OracleVecRware(cfg, E, seed, gid0)
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())
    _assert_state_equal(env, orc, "reset")
    rng = np.random.default_rng(5)
    ended = 0
    for t in range(steps):
        acts = rng.choice(6, size=(E, cfg.n_agents), p=[0.1, 0.45, 0.1, 0.1, 0.2, 0.05]).astype(np.int32)   # 5: out of range -> NOOP
        o, r, d, tr = env.step(torch.tensor(acts, device="cuda"), autoreset=True)
        oo, rr, dd, tt, fret, flen = orc.step(acts, autoreset=True)
        assert np.array_equal(o.cpu().numpy(), oo), t
        assert np.array_equal(r.cpu().numpy(), rr), t
        assert np.array_equal(d.cpu().numpy(), dd) and np.array_equal(tr.cpu().numpy(), tt), t
        fin = flen > 0
        assert np.array_equal(env.final_len.cpu().numpy()[fin], flen[fin]) and np.array_equal(env.final_ret.cpu().numpy()[fin], fret[fin]), t
        ended += fin.sum()
        if t % 20 == 0:
            _assert_state_equal(env, orc, t)
    _assert_state_equal(env, orc, "end")
    assert ended >= 2 * E
    env.close()


def test_fused_categorical_rollout_and_batch_writes():
    """marl_rware_rollout_step == policy_ref.categorical + the oracle step + the on-policy batch writes, with episodes ending early."""
    from codebase_b200.lbf import TrajStore

    cfg = parse_rware_id("rware-tiny-4ag-v2", 0, max_inactivity_steps=12)
    E, seed, gid0, T, N, D, A = 384, 91, 7, 30, 4, 71, 5
    env = NativeRware(cfg, E, seed, gid0)
    orc = OracleVecRware(cfg, E, seed, gid0)
    traj = TrajStore(E, N, T, D, env.device)
    ref = dict(obs=np.zeros((E, N, T + 1, D), np.float32), act=np.zeros((E, N, T), np.int32), rew=np.zeros((E, N, T), np.float32),
               done=np.zeros((E, T + 1), np.uint8), filled=np.zeros((E, T), np.uint8))
    rng = np.random.default_rng(4)
    ref["obs"][:, :, 0] = orc.reset()
    assert np.array_equal(env.reset(traj=traj).cpu().numpy(), ref["obs"][:, :, 0])
    gids, loose = gid0 + np.arange(E), 0
    for t in range(T):
        logits = (1.5 * rng.standard_normal((E, N, A))).astype(np.float32)
        act0, step0 = orc.active.astype(bool), orc.step_count.copy()
        want, margin = policy_ref.categorical(logits, seed, gids, orc.episode_idx - 1, step0)
        env.rollout_step(torch.tensor(logits, device="cuda"), policy=2, traj=traj)
        got = env.actions.cpu().numpy()
        bad = (got != want) & act0[:, None]
        assert np.all(margin[bad] < 1e-5)   # expf differs by an ulp between libm and CUDA: only thresholds on a CDF edge may differ
        loose += bad.sum()
        got = np.where(act0[:, None], got, 0)
        oo, rr, dd, tt, _, _ = orc.step(got, autoreset=False)
        assert np.array_equal(env.obs.cpu().numpy(), oo) and np.array_equal(env.rew.cpu().numpy(), rr) and np.array_equal(env.done.cpu().numpy(), dd)
        s = np.nonzero(act0)[0]
        ref["act"][s, :, step0[s]] = got[s]
        ref["rew"][s, :, step0[s]] = rr[s]
        ref["obs"][s, :, step0[s] + 1] = oo[s]
        ref["done"][s, step0[s] + 1] = dd[s] | tt[s]
        ref["filled"][s, step0[s]] = 1
    for k in ref:
        assert np.array_equal(getattr(traj, k).cpu().numpy(), ref[k]), k
    assert loose < 5 and 0 < ref["filled"].sum() < E * T   # some episodes ended before T
    with pytest.raises(Exception, match="epsilon-greedy"):
        env.rollout_step(torch.zeros(E, N, A, device="cuda"), policy=1, epsilon=0.1)


def test_sharding_reproduces_one_unsharded_run():
    cfg = parse_rware_id("rware-tiny-4ag-v2", 25)
    E, seed = 512, 17
    whole, lo, hi = NativeRware(cfg, E, seed, 0), NativeRware(cfg, E // 2, seed, 0), NativeRware(cfg, E // 2, seed, E // 2)
    rng = np.random.default_rng(8)
    o = whole.reset().cpu().numpy()
    assert np.array_equal(o, np.concatenate([lo.reset().cpu().numpy(), hi.reset().cpu().numpy()]))
    for _ in range(60):
        a = torch.tensor(rng.integers(0, 5, size=(E, 4)).astype(np.int32), device="cuda")
        o, r, d, _ = whole.step(a, autoreset=True)
        o1, r1, d1, _ = lo.step(a[: E // 2].contiguous(), autoreset=True)
        o2, r2, d2, _ = hi.step(a[E // 2:].contiguous(), autoreset=True)
        assert torch.equal(o, torch.cat([o1, o2])) and torch.equal(r, torch.cat([r1, r2])) and torch.equal(d, torch.cat([d1, d2]))


def test_vecenv_protocol_matches_oracle():
    from codebase_b200.utils.envs import make_env

    P, seed, T = 6, 5, 30
    env = make_env(seed, name="rware:rware-tiny-2ag-v2", time_limit=T, parallel_envs=P, wrappers=["CooperativeReward"])
    cfg = parse_rware_id("rware-tiny-2ag-v2", T)
    cfg.cooperative_reward = 1
    orc = OracleVecRware(cfg, P, seed)
    assert env.single_observation_space[0].shape == (71,) and env.single_action_space[0].n == 5 and env.observation_space[0].shape == (P, 71)
    obs, info = env.reset()
    want = orc.reset()
    assert info == {} and all(np.array_equal(obs[i], want[:, i]) for i in range(2))
    rng = np.random.default_rng(0)
    finished = 0
    for _ in range(70):
        acts = rng.integers(0, 5, size=(2, P))
        obs, rew, done, trunc, info = env.step(acts.tolist())
        oo, rr, dd, tt, fret, flen = orc.step(acts.T, autoreset=True)
        assert np.array_equal(rew, rr) and np.array_equal(done, dd.astype(bool)) and np.array_equal(trunc, tt.astype(bool))
        assert all(np.array_equal(obs[i], oo[:, i]) for i in range(2))
        for e in np.nonzero(flen)[0]:
            fi = info["final_info"][e]
            finished += 1
            assert np.array_equal(fi["episode_returns"], fret[e]) and fi["episode_length"] == flen[e] == T
            assert fi["agent1/episode_returns"] == fret[e, 1]
    assert finished == 2 * P
    env.close()


def test_ippo_update_on_an_rware_batch_matches_oracle():
    """One PPONetwork update on a collected RWARE batch (71 features, T = 500), at test_ppo.py's tolerances."""
    from codebase_b200.ac.train import Collector
    from codebase_b200.utils.envs import make_env

    P, N, D, A, T = 24, 4, 71, 5, 500
    hp = lr.A2CHP(target_update_interval_or_tau=2)
    m = ac_model(hp, N, D, P, T, A=A, cls="PPONetwork", num_epochs=4)
    envs = make_env(3, name="rware-tiny-4ag-v2", time_limit=T, parallel_envs=P)
    coll = Collector(envs, m, T)
    ln, _ = coll.collect()
    assert int(ln.min()) == T
    s = {k: getattr(coll.batch, k).cpu().numpy() for k in ("obs", "act", "rew", "done", "filled")}
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), list(range(N)), list(range(N)), D, A)
    want = lr.ppo_update(st, ac_oracle_batch(s), hp, 0, 4, 0.2)
    met = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, 0))
    got, exp = [met["loss"], met["actor_loss"], met["value_loss"], met["entropy"]], [want["loss"], want["actor_loss"], want["value_loss"], want["entropy"]]
    assert np.allclose(got, exp, rtol=2e-5, atol=2e-5), (got, exp)
    d = np.abs(m.theta.cpu().numpy() - np.concatenate([st.actor.numpy(), st.critic.numpy()]))
    assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * 4 + 1e-6, (np.quantile(d, 0.999), d.max())


@pytest.mark.parametrize("alg", ["ia2c", "ippo"])
def test_drivers_and_checkpoint_eval(tmp_path, monkeypatch, alg):
    import pandas as pd

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    run.main([f"+algorithm={alg}", "env.name=rware:rware-tiny-4ag-v2", "env.time_limit=500", "env.parallel_envs=64", "seed=0",
              "algorithm.total_steps=64000", "algorithm.eval_interval=30000", "algorithm.save_interval=30000", f"run_dir={out}"])
    df = pd.read_csv(f"{out}/results.csv")
    for col in ("environment_steps", "loss", "value_loss", "entropy", "mean_episode_returns", "mean_episode_length", "agent3/mean_episode_returns", "updates"):
        assert col in df.columns, col
    assert len(df) >= 2 and np.isfinite(df["loss"]).all() and (df["mean_episode_length"] == 500).all()
    monkeypatch.chdir(tmp_path)
    res = ev.main([f"path={out}", "episodes=16", "seed=3"])
    assert res["episodes"] == 16 and np.isfinite(res["mean_episode_returns"]) and res["mean_episode_returns"] >= 0.0


def test_idqn_on_rware_keeps_the_32_feature_refusal(tmp_path, monkeypatch):
    from codebase_b200 import _native as nat
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    with pytest.raises(nat.NativeError, match=r"observation width 71 not supported \(1\.\.32\)"):
        run.main(["+algorithm=idqn", "env.name=rware:rware-tiny-4ag-v2", "env.time_limit=500", "env.parallel_envs=64", "seed=0",
                  "algorithm.total_steps=1000", f"run_dir={tmp_path}/out"])
