"""CPU: oracle/learner_ref.py (the torch-CPU restatement of the reference learners) pinned against golden vectors produced by the
reference classes (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests.helpers import STRIDE, golden_stride, load_params, reference_outputs, seeded_params

GOLD = os.path.join(os.path.dirname(__file__), "golden")
N, D, A, T = 2, 15, 6, 25
RT, AT = 1e-5, 1e-5


def _close(a, b, rtol=RT, atol=AT):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.allclose(a, b, rtol=rtol, atol=atol), float(np.abs(a - b).max())


def _close_scaled(a, b, tol=1e-5):
    """element-wise, relative to the tensor's own scale (Adam's second moment lives at 1e-6 .. 1e-10: a plain atol would hide it).  For
    v = (1 - beta2) g^2 pass tol=2e-5: a relative gradient error e shows up as 2e in v, so 2e-5 on v is the 1e-5 bar on g."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(float(np.abs(b).max()), 1e-30)
    assert np.abs(a - b).max() <= tol * scale, (float(np.abs(a - b).max()), scale)


def load_dqn_case(name):
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    hp = lr.DqnHP(lr=float(g["hp"][0]), gamma=float(g["hp"][1]), grad_clip=float(g["hp"][2]), double_q=bool(g["hp"][3]),
                  target_update_interval_or_tau=float(g["hp"][4]), mixer=int(g["mixer"]))
    return g, hp


@pytest.mark.parametrize("name", ["idqn_indep", "idqn_single_q_polyak_noclip", "idqn_shared", "vdn_indep"])
def test_dqn_update_matches_reference_golden(name):
    g, hp = load_dqn_case(name)
    theta = torch.tensor(g["theta0"])
    st = lr.DqnState(theta.clone(), theta.clone(), [int(x) for x in g["agent_net"]], D, A)
    S = golden_stride(g)
    for u in range(len(g["losses"])):
        store = {k: g[f"u{u}_{k}"] for k in ("obs", "act", "rew", "done", "filled")}
        out = lr.dqn_update(st, lr.batch_from_store(store, g[f"u{u}_idx"]), hp)
        _close(out["loss"], g["losses"][u])
        if u == 0:
            _close(out["grad"].numpy()[::S], g["grad0"])
            _close_scaled(out["grad_clipped"].numpy()[::S], g["grad0_clipped"])   # what Adam consumed (after clip_grad_norm_)
    _close_scaled(st.m.numpy()[::S], g["adam_m_final"])   # element-wise: the loose bound on theta below cannot hide a defect here
    _close_scaled(st.v.numpy()[::S], g["adam_v_final"], tol=2e-5)
    # Adam's first steps move every weight by ~lr regardless of |g|: elements whose gradient is rounding noise may
    # flip sign between two float32 summation orders, so compare the bulk tightly and bound the rest by 2*lr per step.
    d = np.abs(st.theta.numpy()[::S] - g["theta_final"])
    assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * len(g["losses"]) + 1e-6
    _close(np.quantile(np.abs(st.theta_tgt.numpy()[::S] - g["target_final"]), 0.999), 0, atol=1e-5)


@pytest.mark.parametrize("name", ["ia2c_indep", "ia2c_shared"])
def test_a2c_update_matches_reference_golden(name):
    g = np.load(os.path.join(GOLD, f"{name}.npz"))
    hp = lr.A2CHP(lr=float(g["hp"][0]), gamma=float(g["hp"][1]), grad_clip=float(g["hp"][2]), n_steps=int(g["hp"][3]), entropy_coef=float(g["hp"][4]),
                  value_loss_coef=float(g["hp"][5]), target_update_interval_or_tau=float(g["hp"][6]))
    nets = [int(x) for x in g["agent_net"]]
    st = lr.A2CState(torch.tensor(g["actor0"]), torch.tensor(g["critic0"]), torch.tensor(g["target0"]), nets, nets, D, A)
    S = golden_stride(g)
    for u, step in enumerate(g["steps"]):
        s = {k: torch.as_tensor(g[f"u{u}_{k}"]) for k in ("obs", "act", "rew", "done", "filled")}
        P = s["obs"].shape[0]
        batch = dict(obss=s["obs"].permute(2, 0, 1, 3).reshape(T + 1, P, N * D).float(), actions=s["act"].permute(2, 0, 1).long(),
                     rewards=s["rew"].permute(2, 0, 1).float(), dones=s["done"].permute(1, 0).float(), filled=s["filled"].permute(1, 0).float())
        out = lr.a2c_update(st, batch, hp, int(step))
        _close([out["loss"], out["actor_loss"], out["value_loss"], out["entropy"]], g["metrics"][u])
        if u == 0:
            _close(out["returns"].numpy(), g["returns0"])
            for k in ("actor", "critic"):
                _close_scaled(out["grad_clipped"][k].numpy()[::S], g[f"{k}_grad0_clipped"])
    for k in ("actor", "critic"):
        _close_scaled(st.m[k].numpy()[::S], g[f"{k}_adam_m_final"])
        _close_scaled(st.v[k].numpy()[::S], g[f"{k}_adam_v_final"], tol=2e-5)
    for mine, want in ((st.actor, "actor_final"), (st.critic, "critic_final"), (st.target, "target_final")):
        d = np.abs(mine.numpy()[::S] - g[want])
        assert np.quantile(d, 0.999) < 1e-5 and d.max() < 2 * hp.lr * len(g["steps"]) + 1e-6


def test_epsilon_schedule_and_nstep_returns_golden():
    g = np.load(os.path.join(GOLD, "misc.npz"))
    lin = lr.epsilon_schedule("linear", 0.5, 1.0, 0.05, 6.5, 100000)
    exp = lr.epsilon_schedule("exponential", 0.5, 1.0, 0.05, 6.5, 100000)
    assert np.array_equal(np.array([lin(int(s)) for s in g["steps"]]), g["eps_linear"])
    assert np.array_equal(np.array([exp(int(s)) for s in g["steps"]]), g["eps_exp"])
    for n in (1, 5, 30):
        got = lr.nstep_returns(torch.tensor(g["ns_rew"]), torch.tensor(g["ns_done"]), torch.tensor(g["ns_nv"]), n, 0.99)
        _close(got.numpy(), g[f"ns_ret_{n}"], rtol=1e-6, atol=1e-6)


def _replay_episodes(add):
    """twelve ragged episodes into a five-slot ring (slots are re-used: their stale tails must survive as in the reference)"""
    rng = np.random.default_rng(1)
    for ep in range(12):
        L = int(rng.integers(2, T + 1))
        add(None, [rng.standard_normal(D).astype(np.float32) for _ in range(N)])
        for t in range(L):
            o = [rng.standard_normal(D).astype(np.float32) for _ in range(N)]
            add((rng.integers(0, A, N), rng.random(N).astype(np.float32), t == L - 1), o)


def test_replay_ring_matches_live_reference_buffer():
    """ReplayRef (episode-major) == the reference's ReplayBuffer (time-major; recorded from the live class, stored transposed) incl. the stale tail of re-used slots."""
    g = reference_outputs("replay_reference")
    mine = lr.ReplayRef(5, N, T, D)
    _replay_episodes(lambda ard, o: mine.init_episode(o) if ard is None else mine.add(o, *ard))
    assert len(mine) == int(g["len"]) and mine.cur == int(g["cur_pos"])
    for k in ("obs", "act", "rew"):
        assert np.array_equal(g[k], mine.store[k]), k
    assert np.array_equal(g["done"], mine.store["done"].astype(bool)) and np.array_equal(g["filled"], mine.store["filled"].astype(bool))


def _fresh_batches():
    rng = np.random.default_rng(4)
    for _ in range(2):
        B = 16
        yield dict(obss=torch.tensor(rng.standard_normal((N, T + 1, B, D)), dtype=torch.float32), actions=torch.tensor(rng.integers(0, A, (N, T, B))),
                   rewards=torch.tensor(rng.random((N, T, B)), dtype=torch.float32), dones=torch.tensor(rng.random((T + 1, B)) < 0.05, dtype=torch.float32),
                   filled=torch.tensor(rng.random((T, B)) < 0.9, dtype=torch.float32))


def test_live_reference_update_on_fresh_seed():
    """Not only the trajectory-store fixtures: time-major batches drawn directly (standard-normal observations), two updates of the reference's
    QNetwork from the same seeded weights (recorded from the live class)."""
    g = reference_outputs("qnet_reference")
    theta = seeded_params(lr, N, D, A, 123)
    st = lr.DqnState(theta.clone(), theta.clone(), [0, 1], D, A)
    for u, b in enumerate(_fresh_batches()):
        _close(lr.dqn_update(st, b, lr.DqnHP())["loss"], g["losses"][u])
    assert np.quantile(np.abs(st.theta.numpy()[::STRIDE] - g["theta"]), 0.999) < 1e-5


def make_reference_outputs(ref, ref_shim):
    """tests/golden/replay_reference.npz and qnet_reference.npz: the reference's ReplayBuffer and QNetwork on the inputs of the two tests above."""
    spaces = [ref_shim.Space(shape=(D,)) for _ in range(N)]
    rb = ref.dqn_train.ReplayBuffer(5, N, spaces, [ref_shim.Space(n=A)] * N, T, "cpu")
    _replay_episodes(lambda ard, o: rb.init_episode(o) if ard is None else rb.add(o, *ard))
    np.savez_compressed(os.path.join(GOLD, "replay_reference.npz"), len=len(rb), cur_pos=rb.cur_pos,
                        obs=np.stack([rb.observations[i].transpose(1, 0, 2) for i in range(N)], 1), act=rb.actions.transpose(2, 0, 1),
                        rew=rb.rewards.transpose(2, 0, 1), done=rb.dones.T, filled=rb.filled.T)
    model = ref.dqn_model.QNetwork(spaces, [ref_shim.Space(n=A)] * N, ref_shim.dqn_cfg(), [128, 128], False, False, True, "cpu")
    load_params(model, lr, ("critic.independent", "target.independent"), seeded_params(lr, N, D, A, 123), N, D, A)
    losses = [model.update(ref.dqn_train.Batch(b["obss"], b["actions"], b["rewards"], b["dones"], b["filled"], None))["loss"] for b in _fresh_batches()]
    np.savez_compressed(os.path.join(GOLD, "qnet_reference.npz"), losses=np.array(losses, np.float64),
                        theta=lr.flat_from_state_dict(model.state_dict(), "critic.independent", N).numpy()[::STRIDE])


@pytest.mark.parametrize("alg", ["ia2c", "mappo"])
def test_cpu_actor_critic_loop_collects_the_reference_batch_layout(alg):
    """oracle/cpu_loop_ac.py (the CPU arm of tools/learning_curve_ac.py): one iteration fills a Batch as ac/train.py:24-119 does -- obs row 0 from
    reset, `filled` a prefix of ones per env, the done flag of the last filled step set, nothing written after an env finished -- and the update moves
    the parameters."""
    from oracle.cpu_loop_ac import CpuAC
    from oracle.lbf_ref import LBFConfig

    loop = CpuAC(alg, LBFConfig(time_limit=6), parallel_envs=5, seed=3)
    t, b, infos = loop.collect()
    assert 1 <= t <= 6 and len(infos) == 5 and all("episode_returns" in i for i in infos)
    filled = b["filled"].numpy()
    for i in range(5):
        L = int(filled[:, i].sum())
        assert L >= 1 and (filled[:L, i] == 1).all() and (filled[L:, i] == 0).all()
        assert b["dones"][L, i] == 1 and (b["dones"][:L, i] == 0).all()
        assert (b["obss"][L + 1:, i] == 0).all() and (b["rewards"][L:, i] == 0).all() and (b["actions"][L:, i] == 0).all()
        assert (b["obss"][: L + 1, i] != 0).any()
    before = loop.st.actor.clone()
    at, ret = loop.iteration()
    assert at == 0 and loop.step == loop.P * max(1, int(loop.step / loop.P)) and np.isfinite(ret) and not torch.equal(before, loop.st.actor)
