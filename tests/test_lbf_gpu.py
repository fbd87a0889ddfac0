"""GPU: the CUDA LBF transition (through the C ABI) must be BIT-EXACT against the CPU oracle: known answers,
random rollouts with autoreset, frozen (episode-synchronous) mode, fused epsilon-greedy / categorical selection
and trajectory writes."""
import numpy as np
import pytest
import torch

from oracle import lbf_c, policy_ref
from tests.lbf_kats import KATS, expected, materialise

pytestmark = pytest.mark.gpu


def _native(cfgkw, E, seed, gid0=0):
    from codebase_b200.lbf import LbfConfig, NativeLbf

    return NativeLbf(LbfConfig(**cfgkw), E, seed, gid0)


def _assert_state_equal(env, orc):
    st = {k: v.cpu().numpy() for k, v in env.get_state().items()}
    assert np.array_equal(st["field"], orc.field)
    assert np.array_equal(st["players"], orc.players)
    assert np.array_equal(st["step"], orc.step_count)
    assert np.array_equal(st["food_spawned"], orc.food_spawned)
    assert np.array_equal(st["ep_return"], orc.ep_return)
    assert np.array_equal(st["ep_len"], orc.ep_len)
    assert np.array_equal(st["episode_idx"].astype(np.uint32), orc.episode_idx)
    assert np.array_equal(st["active"], orc.active)


def test_known_answer_boards():
    for kat in KATS:
        cfgkw, field, players, step = materialise(kat)
        env = _native(cfgkw, 1, 0)
        env.set_state(torch.tensor(field[None]), torch.tensor(players[None]), torch.tensor([step], dtype=torch.int32))
        obs, rew, done, trunc = env.step(torch.tensor([kat["actions"]], dtype=torch.int32, device="cuda"))
        pa, want_rew, want_raw = expected(kat, cfgkw)
        st = {k: v.cpu().numpy() for k, v in env.get_state().items()}
        assert np.array_equal(st["players"][0], pa), kat["name"]
        want_field = field.copy().reshape(cfgkw["rows"], cfgkw["cols"])
        for r, c in kat["removed"]:
            want_field[r, c] = 0
        assert np.array_equal(st["field"][0], want_field.reshape(-1)), kat["name"]
        assert np.array_equal(rew.cpu().numpy()[0], want_rew), kat["name"]
        assert bool(done.cpu()[0]) == kat["done"] and bool(trunc.cpu()[0]) == kat["trunc"], kat["name"]
        if "obs_after" in kat:
            assert np.array_equal(obs.cpu().numpy()[0], np.array(kat["obs_after"], np.float32)), kat["name"]


CONFIGS = [
    (dict(), 4096),
    (dict(), 1000),  # ragged last CTA
    (dict(rows=15, cols=15, n_agents=4, max_num_food=5, sight=15, cooperative_reward=1), 2048),
    (dict(rows=10, cols=10, n_agents=3, max_num_food=4, sight=2, penalty=0.1, force_coop=1), 777),
    (dict(rows=5, cols=5, n_agents=5, max_num_food=2, sight=5, normalize_reward=0), 333),
    (dict(rows=9, cols=12, n_agents=1, max_num_food=1, sight=12, time_limit=7), 65),
    (dict(observe_id=1, standardise_rewards=1), 1500),                                                  # ObserveID + StandardiseReward wrappers
    (dict(rows=6, cols=6, n_agents=4, max_num_food=3, sight=6, upstream_reset=1), 900),                 # upstream's reset details (stale positions block, permutation draws)
    (dict(rows=10, cols=10, n_agents=3, max_num_food=4, sight=2, penalty=0.1, standardise_rewards=1, cooperative_reward=1, observe_id=1), 500),
]


@pytest.mark.parametrize("cfgkw,E", CONFIGS)
@pytest.mark.parametrize("autoreset", [True, False])
def test_random_rollouts_bit_exact(cfgkw, E, autoreset):
    rng = np.random.default_rng(11)
    seed, gid0 = 0xDEADBEEF12345, 1000
    env = _native(cfgkw, E, seed, gid0)
    orc = lbf_c.OracleVecEnv(lbf_c.make_cfg(**cfgkw), E, seed, gid0)
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())
    _assert_state_equal(env, orc)
    N = orc.N
    for t in range(40):
        acts = rng.integers(-1, 7, size=(E, N)).astype(np.int32)  # includes out-of-range actions -> NONE
        acts[rng.random(acts.shape) < 0.35] = 5
        o, r, d, tr = env.step(torch.tensor(acts, device="cuda"), autoreset=autoreset)
        oo, rr, dd, tt, fret, flen = orc.step(acts, autoreset=autoreset)
        assert np.array_equal(o.cpu().numpy(), oo), t
        assert np.array_equal(r.cpu().numpy(), rr), t
        assert np.array_equal(d.cpu().numpy(), dd) and np.array_equal(tr.cpu().numpy(), tt), t
        ended = flen > 0  # the oracle wrapper returns fresh zero arrays; only finished envs are written
        assert np.array_equal(env.final_len.cpu().numpy()[ended], flen[ended])
        assert np.array_equal(env.final_ret.cpu().numpy()[ended], fret[ended])
        if t % 5 == 0 or t == 39:
            _assert_state_equal(env, orc)
        if not autoreset and t == 30:  # partial reset of the finished envs only
            mask = (orc.active == 0).astype(np.uint8)
            assert np.array_equal(env.reset(torch.tensor(mask, device="cuda")).cpu().numpy(), orc.reset(mask))


def test_million_transitions_full_size():
    """BASELINE config-2 sized batch stepped against the oracle: 2^15 envs x 32 steps = 1.05 M transitions."""
    rng = np.random.default_rng(5)
    E = 1 << 15
    env = _native(dict(), E, 42)
    orc = lbf_c.OracleVecEnv(lbf_c.make_cfg(), E, 42)
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())
    for t in range(32):
        acts = rng.integers(0, 6, size=(E, 2)).astype(np.int32)
        o, r, d, tr = env.step(torch.tensor(acts, device="cuda"), autoreset=True)
        oo, rr, dd, tt, _, _ = orc.step(acts, autoreset=True)
        assert np.array_equal(o.cpu().numpy(), oo) and np.array_equal(r.cpu().numpy(), rr)
        assert np.array_equal(d.cpu().numpy(), dd) and np.array_equal(tr.cpu().numpy(), tt)
    _assert_state_equal(env, orc)


@pytest.mark.parametrize("cfgkw", [dict(), dict(rows=15, cols=15, n_agents=4, max_num_food=5, sight=15, cooperative_reward=1),
                                   dict(rows=6, cols=6, n_agents=6, max_num_food=2, sight=6)])
@pytest.mark.parametrize("proper", [False, True])
def test_fused_eps_greedy_rollout_and_replay_writes(cfgkw, proper):
    """marl_lbf_rollout_step == (oracle eps-greedy on the same Q-values) + oracle env step + ReplayBuffer.add semantics."""
    from codebase_b200.lbf import TrajStore

    rng = np.random.default_rng(3)
    E, seed, gid0, T = 512, 77, 64, 25
    env = _native(cfgkw, E, seed, gid0)
    orc = lbf_c.OracleVecEnv(lbf_c.make_cfg(**cfgkw), E, seed, gid0)
    N, D, A = orc.N, orc.D, 6
    cap, slot0 = E + 37, 300
    assert slot0 + E > cap  # the last envs' slots wrap to the front of the ring
    traj = TrajStore(cap, N, T, D, env.device)
    ref = dict(obs=np.zeros((cap, N, T + 1, D), np.float32), act=np.zeros((cap, N, T), np.int32), rew=np.zeros((cap, N, T), np.float32),
               done=np.zeros((cap, T + 1), np.uint8), filled=np.zeros((cap, T), np.uint8))
    slots = (slot0 + np.arange(E)) % cap
    for it in range(2):  # second iteration re-uses ring slots (stale tails stay, like the reference)
        o = env.reset(traj=traj, slot0=slot0).cpu().numpy()
        oo = orc.reset()
        assert np.array_equal(o, oo)
        ref["obs"][slots, :, 0] = oo
        gids = gid0 + np.arange(E)
        for t in range(T):
            q = rng.standard_normal((E, N, A)).astype(np.float32)
            q[rng.random((E, N)) < 0.2] = 0.0  # ties -> first argmax
            eps = 0.3
            ep_cur, step0, act0 = orc.episode_idx - 1, orc.step_count.copy(), orc.active.copy().astype(bool)
            want_a = policy_ref.eps_greedy(q, eps, seed, gids, ep_cur, step0)
            want_a = np.where(act0[:, None], want_a, 0)
            env.rollout_step(torch.tensor(q, device="cuda"), policy=1, epsilon=eps, traj=traj, slot0=slot0, use_proper_termination=proper)
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


def test_fused_categorical_rollout():
    rng = np.random.default_rng(9)
    E, seed = 2048, 5
    env = _native(dict(), E, seed)
    orc = lbf_c.OracleVecEnv(lbf_c.make_cfg(), E, seed)
    env.reset(); orc.reset()
    mismatch_allowed = 0
    for t in range(10):
        logits = (2.0 * rng.standard_normal((E, 2, 6))).astype(np.float32)
        want, margin = policy_ref.categorical(logits, seed, np.arange(E), orc.episode_idx - 1, orc.step_count)
        env.rollout_step(torch.tensor(logits, device="cuda"), policy=2)
        got = env.actions.cpu().numpy()
        bad = got != want
        # expf differs by an ulp between libm and CUDA: only samples whose threshold sits on a CDF edge may differ
        assert np.all(margin[bad] < 1e-5)
        mismatch_allowed += bad.sum()
        oo = orc.step(got, autoreset=False)[0]
        assert np.array_equal(env.obs.cpu().numpy(), oo)
    assert mismatch_allowed < 5
    # empirical frequencies follow softmax
    logits = np.tile(np.array([0.0, 1.0, 2.0, -1.0, 0.5, 0.0], np.float32), (E, 2, 1))
    env2 = _native(dict(), E, 123)
    env2.reset()
    env2.rollout_step(torch.tensor(logits, device="cuda"), policy=2)
    freq = np.bincount(env2.actions.cpu().numpy().reshape(-1), minlength=6) / (2 * E)
    p = np.exp(logits[0, 0]) / np.exp(logits[0, 0]).sum()
    assert np.abs(freq - p).max() < 0.03
