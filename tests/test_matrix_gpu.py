"""GPU: the CUDA matrix games (marl_matrix_* through codebase_b200.matrix) BIT-EXACT against the CPU oracle (oracle/matrix_ref.py): random
explicit actions with and without autoreset over every wrapper combination, the fused epsilon-greedy and categorical rollouts with trajectory
writes, sharding, set_state / get_state, the vector-env surface and the frames; one IDQN, one QMIX and one IPPO update on a collected
matrix-game batch against the learner oracles; all seven drivers, checkpoint evaluation and a training video."""
import copy
import itertools
import os
import types

import numpy as np
import pytest
import torch

from codebase_b200.matrix import NativeMatrix, parse_matrix_id
from oracle import learner_ref as lr
from oracle import policy_ref
from oracle.matrix_ref import OracleVecMatrix
from tests.helpers import ac_model, ac_oracle_batch, assert_grad_close, check_margin, redraw_on_near_tie, space
from tests.matrix_render_ref import matrix_frame

pytestmark = pytest.mark.gpu

WRAPPERS = list(itertools.product((0, 1), repeat=3))   # (observe_id, standardise_rewards, cooperative_reward)


def _cfg(name, tl=0, wrap=(0, 0, 0), **over):
    cfg = parse_matrix_id(name, tl, **over)
    cfg.observe_id, cfg.standardise_rewards, cfg.cooperative_reward = wrap
    return cfg


def _assert_state_equal(env, orc, what=""):
    got = {k: v.cpu().numpy() for k, v in env.get_state().items()}
    want = orc.state()
    for k in want:
        assert np.array_equal(got[k], want[k]), (what, k, got[k][:4], want[k][:4])


def _run(cfg, E, steps, autoreset, seed):
    env, orc = NativeMatrix(cfg, E, seed=11, env_gid0=3), OracleVecMatrix(cfg, E)
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())
    _assert_state_equal(env, orc, "reset")
    rng = np.random.default_rng(seed)
    ended = 0
    for t in range(steps):
        acts = rng.integers(-1, cfg.n_actions + 1, size=(E, cfg.n_agents)).astype(np.int32)   # -1 and A: out of range -> action 0
        o, r, d, tr = env.step(torch.tensor(acts, device="cuda"), autoreset=autoreset)
        oo, rr, dd, tt, fret, flen = orc.step(acts, autoreset=autoreset)
        assert np.array_equal(o.cpu().numpy(), oo), t
        assert np.array_equal(r.cpu().numpy(), rr), t
        assert np.array_equal(d.cpu().numpy(), dd) and np.array_equal(tr.cpu().numpy(), tt), t
        fin = flen > 0
        assert np.array_equal(env.final_len.cpu().numpy()[fin], flen[fin]) and np.array_equal(env.final_ret.cpu().numpy()[fin], fret[fin]), t
        ended += fin.sum()
        if t % 7 == 0:
            _assert_state_equal(env, orc, t)
    _assert_state_equal(env, orc, "end")
    env.close()
    return ended


@pytest.mark.parametrize("tl", [10, 25, 40])
@pytest.mark.parametrize("name", ["climbing-v0", "climbing-nostate-v0", "penalty-100-v0", "penalty-25-nostate-v0"])
def test_random_actions_bit_exact_every_wrapper_combination(name, tl):
    """time_limit below, equal to and above ep_length = 25; 60 steps: autoreset ends two or more episodes per env, and without it the finished
    envs stay frozen for the rest of the run"""
    for wrap in WRAPPERS:
        for autoreset in (True, False):
            cfg = _cfg(name, tl, wrap)
            ended = _run(cfg, 48, 60, autoreset, seed=sum(wrap) + 10 * tl)
            assert ended == (48 * (60 // min(tl, 25)) if autoreset else 48), (wrap, autoreset)


@pytest.mark.parametrize("state", [1, 0])
def test_custom_three_player_payoff_bit_exact(state):
    rng = np.random.default_rng(2)
    table = np.round(rng.standard_normal((4, 4, 4)) * 7.3, 3)   # float64 payoffs
    for wrap in [(0, 0, 0), (1, 1, 1), (0, 1, 0), (0, 0, 1)]:
        cfg = _cfg("climbing-v0", 9, wrap, payoff_matrix=table, ep_length=13, last_action_state=state)
        assert (cfg.n_agents, cfg.n_actions) == (3, 4)
        assert _run(cfg, 40, 50, True, seed=7) == 40 * (50 // 9)
        _run(cfg, 40, 20, False, seed=8)


def test_wide_games_bit_exact():
    """group widths G = 1, 8 and 32: one player, five players of 8 actions (32 768 entries), 32 players of one action"""
    for table, tl in ((np.arange(5.0) - 2.0, 6), (np.arange(8 ** 5, dtype=np.float64).reshape((8,) * 5) % 97 - 48, 11), (np.full((1,) * 32, 2.5), 4)):
        for wrap in [(0, 0, 0), (1, 1, 1)]:
            cfg = _cfg("climbing-v0", tl, wrap, payoff_matrix=table)
            _run(cfg, 70, 14, True, seed=3)


@pytest.mark.parametrize("tl,proper", [(20, False), (20, True), (25, False), (25, True)])
def test_fused_eps_greedy_rollout_and_replay_writes(tl, proper):
    from codebase_b200.native_env import TrajStore

    rng = np.random.default_rng(3)
    cfg = _cfg("climbing-v0", tl, (1, 1, 1))
    E, seed, gid0, T, N, D, A = 300, 77, 64, 25, 2, cfg.obs_dim, 3
    env, orc = NativeMatrix(cfg, E, seed, gid0), OracleVecMatrix(cfg, E)
    cap, slot0 = E + 37, 200
    traj = TrajStore(cap, N, T, D, env.device)
    ref = dict(obs=np.zeros((cap, N, T + 1, D), np.float32), act=np.zeros((cap, N, T), np.int32), rew=np.zeros((cap, N, T), np.float32),
               done=np.zeros((cap, T + 1), np.uint8), filled=np.zeros((cap, T), np.uint8))
    slots, gids = (slot0 + np.arange(E)) % cap, gid0 + np.arange(E)
    for it in range(2):
        oo = orc.reset()
        assert np.array_equal(env.reset(traj=traj, slot0=slot0).cpu().numpy(), oo)
        ref["obs"][slots, :, 0] = oo
        for t in range(T):
            q = rng.standard_normal((E, N, A)).astype(np.float32)
            q[rng.random((E, N)) < 0.2] = 0.0
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
            ref["done"][s, step0[act0] + 1] = dd[act0] if proper else (dd[act0] | tt[act0])
            ref["filled"][s, step0[act0]] = 1
        for k in ref:
            assert np.array_equal(getattr(traj, k).cpu().numpy(), ref[k]), (it, k)
    assert ref["filled"].sum() == E * min(tl, T) and ref["done"].sum() == (0 if proper and tl < 25 else E)
    with pytest.raises(Exception, match="n_actions 4 does not match"):
        env.rollout_step(torch.zeros(E, N, 4, device="cuda"), policy=1, epsilon=0.1)


@pytest.mark.parametrize("proper", [False, True])
def test_fused_categorical_rollout_and_batch_writes(proper):
    from codebase_b200.native_env import TrajStore

    cfg = _cfg("penalty-50-v0", 18, (0, 0, 1))
    E, seed, gid0, T, N, D, A = 384, 91, 7, 25, 2, 6, 3
    env, orc = NativeMatrix(cfg, E, seed, gid0), OracleVecMatrix(cfg, E)
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
        env.rollout_step(torch.tensor(logits, device="cuda"), policy=2, traj=traj, use_proper_termination=proper)
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
        ref["done"][s, step0[s] + 1] = dd[s] if proper else (dd[s] | tt[s])
        ref["filled"][s, step0[s]] = 1
    for k in ref:
        assert np.array_equal(getattr(traj, k).cpu().numpy(), ref[k]), k
    assert loose < 5 and ref["filled"].sum() == E * 18


def test_sharding_reproduces_one_unsharded_run():
    cfg = _cfg("climbing-v0", 20, (1, 1, 0))
    E = 512
    whole, lo, hi = NativeMatrix(cfg, E, 17, 0), NativeMatrix(cfg, E // 2, 17, 0), NativeMatrix(cfg, E // 2, 17, E // 2)
    rng = np.random.default_rng(8)
    assert torch.equal(whole.reset(), torch.cat([lo.reset(), hi.reset()]))
    for _ in range(45):
        logits = torch.tensor(rng.standard_normal((E, 2, 3)).astype(np.float32), device="cuda")
        whole.rollout_step(logits, policy=2, autoreset=True)
        lo.rollout_step(logits[: E // 2].contiguous(), policy=2, autoreset=True)
        hi.rollout_step(logits[E // 2:].contiguous(), policy=2, autoreset=True)
        for k in ("obs", "rew", "done", "trunc", "actions"):
            assert torch.equal(getattr(whole, k), torch.cat([getattr(lo, k), getattr(hi, k)])), k


def test_set_state_get_state_round_trip():
    cfg = _cfg("penalty-75-v0", 0, (1, 0, 0))
    E = 200
    env, orc = NativeMatrix(cfg, E, 3), OracleVecMatrix(cfg, E)
    env.reset(); orc.reset()
    rng = np.random.default_rng(6)
    last = rng.integers(0, 3, size=(E, 2)).astype(np.int8)
    last[rng.random(E) < 0.3] = -1   # a previous action for both players or for neither
    step = rng.integers(0, 25, size=E).astype(np.int32)
    env.set_state(torch.tensor(last), torch.tensor(step))
    orc.load(last, step)
    _assert_state_equal(env, orc, "after set_state")
    st = env.get_state()
    assert np.array_equal(st["last_action"].cpu().numpy(), last) and np.array_equal(st["step"].cpu().numpy(), step)
    for t in range(30):
        acts = rng.integers(0, 3, size=(E, 2)).astype(np.int32)
        o, r, d, tr = env.step(torch.tensor(acts, device="cuda"), autoreset=True)
        oo, rr, dd, tt, _, _ = orc.step(acts, autoreset=True)
        assert np.array_equal(o.cpu().numpy(), oo) and np.array_equal(r.cpu().numpy(), rr) and np.array_equal(d.cpu().numpy(), dd), t
    _assert_state_equal(env, orc, "end")
    again = NativeMatrix(cfg, E, 3)
    again.set_state(env.get_state()["last_action"], env.get_state()["step"])
    assert torch.equal(again.get_state()["last_action"], env.get_state()["last_action"])


def test_vecenv_protocol_matches_oracle():
    from codebase_b200.utils.envs import make_env

    P, T = 6, 25
    env = make_env(5, name="matrixgames:climbing-v0", time_limit=T, parallel_envs=P, wrappers=["CooperativeReward"])
    cfg = _cfg("climbing-v0", T, (0, 0, 1))
    orc = OracleVecMatrix(cfg, P)
    assert env.single_observation_space[0].shape == (6,) and env.single_action_space[0].n == 3 and env.observation_space[0].shape == (P, 6)
    assert (env.single_observation_space[0].low, env.single_observation_space[0].high) == (0.0, 1.0)
    obs, info = env.reset()
    want = orc.reset()
    assert info == {} and all(np.array_equal(obs[i], want[:, i]) for i in range(2))
    rng = np.random.default_rng(0)
    finished = 0
    for _ in range(60):
        acts = rng.integers(0, 3, size=(2, P))
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
    frame = env.render()
    assert frame.shape == (1 + 2 * 41, 1 + 3 * 41, 3) and np.array_equal(frame, matrix_frame(orc.state()["last_action"][0], 3))
    env.close()


@pytest.mark.parametrize("table", [np.zeros((3, 3)), np.zeros((2,) * 5), np.zeros((8,) * 3), np.zeros((1,) * 32)], ids=["3x3", "2^5", "8^3", "1^32"])
def test_frames_match_the_numpy_restatement(table):
    cfg = _cfg("climbing-v0", 0, payoff_matrix=table)
    N, A, E = cfg.n_agents, cfg.n_actions, 37
    env = NativeMatrix(cfg, E, 1)
    env.reset()
    rng = np.random.default_rng(N)
    last = rng.integers(-1, A, size=(E, N)).astype(np.int8)
    env.set_state(torch.tensor(last), torch.zeros(E, dtype=torch.int32))
    assert env.frame_shape == (1 + N * 41, 1 + A * 41, 3)
    frames = env.render(0, E).cpu().numpy()
    for e in range(E):
        assert np.array_equal(frames[e], matrix_frame(last[e], A)), e
    one = env.render(5, 1).cpu().numpy()
    assert np.array_equal(one[0], frames[5])
    with pytest.raises(Exception, match="not a non-empty range"):
        env.render(E - 1, 2)


# ---- learner updates on a collected matrix-game batch -----------------------------------------------------------------------------------------
def _dqn_cfg(**kw):
    return types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200,
                                 standardise_returns=False, **kw)


def _collect_dqn(model, name, wrappers, E=256, T=25):
    from codebase_b200.dqn.train import Collector
    from codebase_b200.native_env import TrajStore
    from codebase_b200.utils.envs import make_env

    venv = make_env(3, name=name, time_limit=T, parallel_envs=E, wrappers=wrappers)
    rb = TrajStore(E, venv.n_agents, T, venv.cfg.obs_dim, venv.native.device)
    final_len, _ = Collector(venv, model, T).collect(rb, 0, 0.5)
    assert int(final_len.sum()) == E * T and int(rb.filled.sum()) == E * T
    return rb, {k: getattr(rb, k).cpu().numpy() for k in ("obs", "act", "rew", "done", "filled")}


@redraw_on_near_tie
def test_idqn_update_on_a_matrix_batch_matches_oracle():
    from codebase_b200.dqn.model import QNetwork

    N, D, A, B = 2, 6, 3, 64
    model = QNetwork([space(shape=(D,))] * N, [space(n=A)] * N, _dqn_cfg(), [128, 128], False, False, True, "cuda", max_batch=B, max_episode_length=25)
    rb, store = _collect_dqn(model, "matrixgames:climbing-v0", None)
    assert set(np.unique(store["rew"])) <= {11.0, -30.0, 0.0, 7.0, 6.0, 5.0}
    st = lr.DqnState(model.theta.cpu().clone(), model.theta_tgt.cpu().clone(), model.agent_net, D, A)
    idx = torch.arange(B, dtype=torch.int32, device="cuda") * 3
    batch = lr.batch_from_store(store, idx.cpu().numpy())
    hp = lr.DqnHP()
    check_margin(lr, st, batch, hp)
    st0 = copy.deepcopy(st)
    want = lr.dqn_update(st, batch, hp)
    got = float(model.update_from_store(rb, idx)[0].item())
    assert abs(got - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), (got, want["loss"])
    assert_grad_close(lr, st0, batch, hp, model.grad[: model.n_params].cpu().numpy() / float(batch["filled"].sum()), want["grad"].numpy(), tol=2e-5,
                      what="IDQN gradient")
    d = (model.theta.cpu() - st.theta).abs()
    assert float(d.quantile(0.999)) < 1e-5


@redraw_on_near_tie
def test_qmix_update_on_a_matrix_batch_matches_oracle():
    from codebase_b200.dqn import model as M
    from tests import qmix_options_ref as qo
    from tests.test_qmix_agents_gpu import Case, _check_update, _f64

    N, D, A, B, T = 2, 6, 3, 32, 25
    c = Case(N=N, D=D, T=T, B=B, tu=200.0)
    hp = lr.DqnHP(double_q=True, target_update_interval_or_tau=200.0)
    m = M.QMixNetwork([space(shape=(D,))] * N, [space(n=A)] * N, _dqn_cfg(), [128, 128], False, False, True,
                      dict(embed_dim=c.E, hypernet_layers=c.hl, hypernet_embed=c.He), "cuda", max_batch=B, max_episode_length=T)
    rb, store = _collect_dqn(m, "matrixgames:penalty-100-v0", ["CooperativeReward"])
    assert set(np.unique(store["rew"])) <= {-200.0, 0.0, 20.0, 4.0}   # N x payoff
    f = lambda t: t.detach().cpu().double().clone()   # noqa: E731
    st = qo.QmixOptState(f(m.theta), f(m.theta_tgt), f(m.mix), f(m.mix_tgt), list(range(N)), D, A, embed_dim=c.E, hypernet_embed=c.He,
                         hypernet_layers=c.hl, ret_ms=None)
    idx = torch.arange(B, dtype=torch.int32, device="cuda") * 5
    b64 = _f64(lr.batch_from_store(store, idx.cpu().numpy()))
    check_margin(lr, lr.DqnState(st.theta, st.theta_tgt, st.agent_net, D, A), b64, hp)
    st0 = copy.deepcopy(st)
    want = qo.qmix_update(st, b64, hp)
    met = m.update_from_store(rb, idx).cpu()
    _check_update(c, m, st, st0, b64, want, met, hp, "QMIX on penalty-100", per_block=False)


def test_ippo_update_on_a_matrix_batch_matches_oracle():
    from codebase_b200.ac.train import Collector
    from codebase_b200.utils.envs import make_env
    from tests.helpers import traj_store

    P, N, D, A, T = 64, 2, 6, 3, 25
    hp = lr.A2CHP(target_update_interval_or_tau=2)
    m = ac_model(hp, N, D, P, T, A=A, cls="PPONetwork", num_epochs=4)
    envs = make_env(3, name="climbing-v0", time_limit=T, parallel_envs=P)
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


# ---- drivers ---------------------------------------------------------------------------------------------------------------------------------
def _driver_args(alg, name, out, steps):
    args = [f"+algorithm={alg}", f"env.name={name}", "env.time_limit=25", "env.parallel_envs=64", "seed=0", f"algorithm.total_steps={steps}",
            f"algorithm.eval_interval={steps // 3}", f"algorithm.save_interval={steps // 3}", "algorithm.eval_episodes=32", f"run_dir={out}"]
    if alg in ("idqn", "vdn", "qmix"):
        args += ["algorithm.batch_size=64", "algorithm.buffer_size=1024", "algorithm.updates_per_iteration=8", "algorithm.training_start=1000"]
    return args


@pytest.mark.parametrize("alg", ["idqn", "vdn", "qmix", "ia2c", "ippo", "maa2c", "mappo"])
def test_drivers_write_finite_results_and_checkpoints_evaluate(tmp_path, monkeypatch, alg):
    import pandas as pd

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    run.main(_driver_args(alg, "matrixgames:climbing-v0", out, 9000))
    df = pd.read_csv(f"{out}/results.csv")
    for col in ("environment_steps", "mean_episode_returns", "mean_episode_length", "agent1/mean_episode_returns"):
        assert col in df.columns and np.isfinite(df[col]).all(), col
    assert len(df) >= 2 and (df["mean_episode_length"] == 25).all()
    assert df["mean_episode_returns"].between(-30 * 25, 11 * 25).all()
    monkeypatch.chdir(tmp_path)
    res = ev.main([f"path={out}", "episodes=16", "seed=3"])
    assert res["episodes"] == 16 and -30 * 25 <= res["mean_episode_returns"] <= 11 * 25


def test_video_interval_writes_an_mp4(tmp_path, monkeypatch):
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = tmp_path / "out"
    run.main(_driver_args("ippo", "matrixgames:penalty-100-nostate-v0", out, 8000) + ["algorithm.video_interval=4000", "algorithm.video_frames=30"])
    vids = sorted(os.listdir(out / "videos"))
    assert vids and all(v.startswith("step-") and v.endswith(".mp4") and os.path.getsize(out / "videos" / v) > 0 for v in vids)

