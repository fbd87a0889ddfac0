"""GPU: the LBF and RWARE env-step kernels from 9 to 32 agents (31 for RWARE) bit for bit against the CPU oracles (oracle/lbf_c.py,
tests/lbf_grid_ref.py, oracle/rware_ref.py): random rollouts with autoreset and in frozen mode with a masked reset, the fused epsilon-greedy and
categorical rollouts with their trajectory writes, frames, and the configurations create must refuse.

LBF gives each env a group of G = next_pow2(N) lanes, EPC = 4 * 32 / G envs per CTA; RWARE one warp per env (lane = agent, lane 31 is the
empty-cell sink of the move graph), 4 envs per CTA.  Every case's E leaves the last CTA ragged.

  case                    env                                         N   what it reaches
  lbf_n9_g16              10x10, 4 food, sight 3                      9   vector path at G = 16: 7 idle lanes per group, two envs per warp
  lbf_n16_crowded         8x8, 3 food, force_coop, penalty 0.1        16  a full G = 16 group; dense move collisions, loading with many adjacent agents
  lbf_n17_std_coop        12x12, 6 food, standardise + coop           17  G = 32 with 15 idle lanes; StandardiseReward state at 2N+1 floats
  lbf_n24_upstream        10x10, 4 food, upstream_reset               24  cell_empty over the stale positions of 24 players
  lbf_20x20_32p_10f       Foraging-20x20-32p-10f-v3                   32  full-warp masks (gbits = 0xFFFFFFFF), EPC = 4
  lbf_n32_obsid_32f       25x25, 32 food, sight 3, observe_id         32  D = 224: lbf_reset_kernel's observation buffer (reset, masked reset,
                                                                          the replay ring's first row); in-kernel autoreset
  lbf_grid_n32_std_coop   Foraging-grid-2s-12x12-32p-4f-v3 + wrappers 32  grid path at N = G = 32 with StandardiseReward and CooperativeReward
  rware_tiny_n31          tiny (11x10, 32 shelves)                    31  the densest board: chains and cycles through 31 lanes, sink lane 31
  rware_large_n31_s3      large, sensor_range 3, observe_id, std+coop 31  D = 382, the widest observation the validator admits (192,576 B per CTA);
                                                                          starts from the goal queue below, so the wrappers see deliveries
  rware_medium_n24_hard   medium, -hard queue (12 requests)           24  request redraws: every run starts with a queue of 16 loaded agents in the
                                                                          two goal columns

RWARE configs above the id parser's 19 agents are built as RwareConfig directly.  tests/test_env_agent_range.py checks, without a GPU, that each
case still sits on the edge it claims.
"""
import dataclasses

import numpy as np
import pytest
import torch

from codebase_b200.lbf import LbfConfig, parse_env_id
from codebase_b200.rware import RwareConfig, parse_rware_id
from oracle import lbf_c, policy_ref
from oracle import rware_ref as rw
from tests.lbf_grid_ref import GridOracleVecEnv

pytestmark = pytest.mark.gpu

SEED, GID0 = 0x5EED_32A6_E17, 321
STEPS, RESET_AT = 30, 12   # time limits of 8..12 steps: every frozen env has ended before the masked reset at RESET_AT


LBF = {   # name: (config, E)
    "lbf_n9_g16": (LbfConfig(rows=10, cols=10, n_agents=9, max_num_food=4, sight=3, time_limit=12), 203),
    "lbf_n16_crowded": (LbfConfig(rows=8, cols=8, n_agents=16, max_num_food=3, sight=2, force_coop=1, penalty=0.1, time_limit=10), 149),
    "lbf_n17_std_coop": (LbfConfig(rows=12, cols=12, n_agents=17, max_num_food=6, sight=4, standardise_rewards=1, cooperative_reward=1, time_limit=12), 103),
    "lbf_n24_upstream": (LbfConfig(rows=10, cols=10, n_agents=24, max_num_food=4, sight=10, upstream_reset=1, time_limit=8), 101),
    "lbf_20x20_32p_10f": (parse_env_id("Foraging-20x20-32p-10f-v3", 12), 67),
    "lbf_n32_obsid_32f": (LbfConfig(rows=25, cols=25, n_agents=32, max_num_food=32, sight=3, observe_id=1, time_limit=10), 63),
    "lbf_grid_n32_std_coop": (parse_env_id("Foraging-grid-2s-12x12-32p-4f-v3", 10, standardise_rewards=1, cooperative_reward=1), 67),
}
RWARE = {   # name: (config, E)
    "rware_tiny_n31": (RwareConfig(n_agents=31, request_queue_size=16, time_limit=12), 23),
    "rware_large_n31_s3": (RwareConfig(shelf_rows=3, shelf_columns=5, n_agents=31, request_queue_size=31, sensor_range=3, observe_id=1,
                                  standardise_rewards=1, cooperative_reward=1, time_limit=10), 11),
    "rware_medium_n24_hard": (dataclasses.replace(parse_rware_id("rware-medium-19ag-hard-v2", 12), n_agents=24, request_queue_size=12), 11),
}
QUEUED = ("rware_large_n31_s3", "rware_medium_n24_hard")   # cases that start from _queue_at_goals
# the vector tile of a 64x64 field with 2 agents: 64 envs per CTA x 4100 B of field alone, over the H100's 232,448 B opt-in limit
REFUSED_LBF = LbfConfig(rows=64, cols=64, n_agents=2, sight=2)
REFUSED_LBF_SMEM = 272_384   # step_smem_bytes of REFUSED_LBF, as the library's refusal states it


def _oracle_cfg(cfg):
    return lbf_c.make_cfg(**{k: v for k, v in dataclasses.asdict(cfg).items() if k != "grid_observation"})


def _lbf_pair(cfg, E, seed=SEED, gid0=GID0):
    from codebase_b200.lbf import NativeLbf

    orc = GridOracleVecEnv(dataclasses.asdict(cfg), E, seed, gid0) if cfg.grid_observation else lbf_c.OracleVecEnv(_oracle_cfg(cfg), E, seed, gid0)
    return NativeLbf(cfg, E, seed, gid0), orc


def _rware_pair(cfg, E, seed=SEED, gid0=GID0):
    from codebase_b200.rware import NativeRware

    return NativeRware(cfg, E, seed, gid0), rw.OracleVecRware(cfg, E, seed, gid0)


def _lbf_state_equal(env, orc, what):
    st = {k: v.cpu().numpy() for k, v in env.get_state().items()}
    want = dict(field=orc.field, players=orc.players, step=orc.step_count, food_spawned=orc.food_spawned, ep_return=orc.ep_return,
                ep_len=orc.ep_len, episode_idx=orc.episode_idx, active=orc.active)
    for k, v in want.items():
        got = st[k].astype(np.uint32) if k == "episode_idx" else st[k]
        assert np.array_equal(got, v), (what, k)


def _rware_state_equal(env, orc, what):
    st = {k: v.cpu().numpy() for k, v in env.get_state().items()}
    for k, v in orc.state().items():
        assert np.array_equal(st[k], v), (what, k)


def _queue_at_goals(env, orc, rng):
    """The 16 highest-numbered agents loaded and facing down in the two goal columns (highway cells), the two on the goals and the next ones
    carrying requested shelves, the others unloaded on the highway row y = column_height + 1: both goals deliver on the first step, to the
    last two lanes, and more loaded agents follow."""
    cfg, E, N = orc.cfg, orc.E, orc.N
    C = cfg.cols
    home = rw.home_shelves(cfg)
    (gx, gy), _ = rw.goals(cfg)
    st = orc.state()
    shelves, agents = np.tile(home, (E, 1)), np.zeros((E, N, 4), np.uint8)
    for e in range(E):
        bits = st["requested"][e].view(np.uint32)
        req = [k for k in range(1, rw.n_shelves(cfg) + 1) if (int(bits[k >> 5]) >> (k & 31)) & 1]
        free = [k for k in range(1, rw.n_shelves(cfg) + 1) if k not in req]
        carried = list(rng.permutation(req)[:16]) + list(rng.choice(free, max(0, 16 - len(req)), replace=False))
        for i in range(N):
            if i < 16:
                x, y, d, s = gx + i % 2, gy - i // 2, rw.DOWN, int(carried[i])
                shelves[e, np.nonzero(home == s)[0][0]] = 0
                shelves[e, y * C + x] = s
            else:
                x, y, d, s = i - 16, cfg.column_height + 1, int(rng.integers(0, 4)), 0
            agents[e, N - 1 - i] = (x, y, d, s)
    env.set_state(torch.from_numpy(shelves), torch.from_numpy(agents), torch.from_numpy(st["requested"]), torch.zeros(E, dtype=torch.int32),
                  torch.zeros(E, dtype=torch.int32))
    for e, w in enumerate(orc.envs):
        w.env.load(shelves[e], agents[e], st["requested"][e], 0, 0)
        w.episode_reward[:] = 0
        w.episode_length = 0
    orc.active[:] = 1


def _rollout(env, orc, acts, autoreset, state_equal, rng, after_reset=None):
    """STEPS steps of env and oracle on the same actions; frozen runs reset a random half of the envs at RESET_AT.  Returns (ended episodes,
    rewards summed over the run)."""
    E = orc.E
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())
    state_equal(env, orc, "reset")
    if after_reset:
        after_reset(env, orc, rng)
    ended, paid = 0, 0.0
    for t in range(STEPS):
        a = acts(rng)
        o, r, d, tr = env.step(torch.tensor(a, device="cuda"), autoreset=autoreset)
        oo, rew, dd, tt, fret, flen = orc.step(a, autoreset=autoreset)
        assert np.array_equal(o.cpu().numpy(), oo), t
        assert np.array_equal(r.cpu().numpy(), rew), t
        assert np.array_equal(d.cpu().numpy(), dd) and np.array_equal(tr.cpu().numpy(), tt), t
        fin = flen > 0   # the oracle returns fresh zero arrays; only finished envs are written
        assert np.array_equal(env.final_len.cpu().numpy()[fin], flen[fin]) and np.array_equal(env.final_ret.cpu().numpy()[fin], fret[fin]), t
        ended += int(fin.sum())
        paid += float(np.abs(rew).sum())
        if t % 5 == 4:
            state_equal(env, orc, t)
        if not autoreset and t == RESET_AT:
            assert not orc.active.any()
            mask = (rng.random(E) < 0.5).astype(np.uint8)
            assert np.array_equal(env.reset(torch.tensor(mask, device="cuda")).cpu().numpy(), orc.reset(mask))
            state_equal(env, orc, "masked reset")
    state_equal(env, orc, "end")
    return ended, paid


@pytest.mark.parametrize("autoreset", [True, False], ids=["autoreset", "frozen"])
@pytest.mark.parametrize("name", list(LBF))
def test_lbf_rollouts_bit_exact(name, autoreset):
    cfg, E = LBF[name]
    env, orc = _lbf_pair(cfg, E)
    N = cfg.n_agents

    def acts(rng):
        a = rng.integers(-1, 7, size=(E, N)).astype(np.int32)   # -1 and 6: out of range, NONE
        a[rng.random(a.shape) < 0.35] = 5
        return a

    ended, paid = _rollout(env, orc, acts, autoreset, _lbf_state_equal, np.random.default_rng(sum(map(ord, name))))
    assert ended >= (2 if autoreset else 1) * E and paid > 0


@pytest.mark.parametrize("autoreset", [True, False], ids=["autoreset", "frozen"])
@pytest.mark.parametrize("name", list(RWARE))
def test_rware_rollouts_bit_exact(name, autoreset):
    cfg, E = RWARE[name]
    env, orc = _rware_pair(cfg, E)
    N = cfg.n_agents

    def acts(rng):   # -1 and 5: out of range, NOOP
        return rng.choice(np.arange(-1, 6), size=(E, N), p=[0.03, 0.1, 0.45, 0.1, 0.1, 0.17, 0.05]).astype(np.int32)

    queue = _queue_at_goals if name in QUEUED else None
    ended, paid = _rollout(env, orc, acts, autoreset, _rware_state_equal, np.random.default_rng(sum(map(ord, name))), queue)
    assert ended >= (2 if autoreset else 1) * E
    if queue:
        assert paid >= 2 * E   # both goals deliver on the first step, and the request is redrawn each time


def test_lbf_fused_eps_greedy_rollout_and_replay_writes_at_32_agents():
    """marl_lbf_rollout_step at N = 32, D = 224 (Philox blocks 1..8 of epsilon-greedy) == policy_ref.eps_greedy + the oracle step +
    ReplayBuffer.add, over a wrapping ring whose first rows come from lbf_reset_kernel."""
    from codebase_b200.lbf import TrajStore

    cfg, E = LBF["lbf_n32_obsid_32f"]
    env, orc = _lbf_pair(cfg, E)
    N, D, A, T = orc.N, orc.D, 6, 12
    assert D == 224
    rng = np.random.default_rng(3)
    cap, slot0 = E + 37, 70
    assert slot0 + E > cap   # the last envs' slots wrap to the front of the ring
    traj = TrajStore(cap, N, T, D, env.device)
    ref = dict(obs=np.zeros((cap, N, T + 1, D), np.float32), act=np.zeros((cap, N, T), np.int32), rew=np.zeros((cap, N, T), np.float32),
               done=np.zeros((cap, T + 1), np.uint8), filled=np.zeros((cap, T), np.uint8))
    slots, gids = (slot0 + np.arange(E)) % cap, GID0 + np.arange(E)
    explored = 0
    for it in range(2):   # the second pass re-uses ring slots
        oo = orc.reset()
        assert np.array_equal(env.reset(traj=traj, slot0=slot0).cpu().numpy(), oo)
        ref["obs"][slots, :, 0] = oo
        for t in range(T):
            q = rng.standard_normal((E, N, A)).astype(np.float32)
            q[rng.random((E, N)) < 0.2] = 0.0   # ties -> first argmax
            ep_cur, step0, act0 = orc.episode_idx - 1, orc.step_count.copy(), orc.active.copy().astype(bool)
            want = np.where(act0[:, None], policy_ref.eps_greedy(q, 0.5, SEED, gids, ep_cur, step0), 0)
            explored += int((want != q.argmax(-1)).any(-1).sum())
            env.rollout_step(torch.tensor(q, device="cuda"), policy=1, epsilon=0.5, traj=traj, slot0=slot0)
            assert np.array_equal(env.actions.cpu().numpy(), want), (it, t)
            oo, rew, dd, tt, _, _ = orc.step(want, autoreset=False)
            assert np.array_equal(env.obs.cpu().numpy(), oo) and np.array_equal(env.rew.cpu().numpy(), rew), (it, t)
            s = slots[act0]
            ref["act"][s, :, step0[act0]] = want[act0]
            ref["rew"][s, :, step0[act0]] = rew[act0]
            ref["obs"][s, :, step0[act0] + 1] = oo[act0]
            ref["done"][s, step0[act0] + 1] = dd[act0] | tt[act0]
            ref["filled"][s, step0[act0]] = 1
        for k in ref:
            assert np.array_equal(getattr(traj, k).cpu().numpy(), ref[k]), (it, k)
    assert explored > 0 and 0 < ref["filled"].sum() < E * T   # episodes ended before T


def _categorical_with_batch_writes(env, orc, A, T, scale):
    """policy 2 with the on-policy batch writes: actions as policy_ref.categorical samples them (a threshold on a CDF edge may differ by the
    ulp of expf), everything after them bit for bit."""
    from codebase_b200.lbf import TrajStore

    E, N, D = orc.E, orc.N, orc.D
    rng = np.random.default_rng(9)
    traj = TrajStore(E, N, T, D, env.device)
    ref = dict(obs=np.zeros((E, N, T + 1, D), np.float32), act=np.zeros((E, N, T), np.int32), rew=np.zeros((E, N, T), np.float32),
               done=np.zeros((E, T + 1), np.uint8), filled=np.zeros((E, T), np.uint8))
    ref["obs"][:, :, 0] = orc.reset()
    assert np.array_equal(env.reset(traj=traj).cpu().numpy(), ref["obs"][:, :, 0])
    gids, loose = GID0 + np.arange(E), 0
    for t in range(T):
        logits = (scale * rng.standard_normal((E, N, A))).astype(np.float32)
        act0, step0 = orc.active.copy().astype(bool), orc.step_count.copy()
        want, margin = policy_ref.categorical(logits, SEED, gids, orc.episode_idx - 1, step0)
        env.rollout_step(torch.tensor(logits, device="cuda"), policy=2, traj=traj)
        got = env.actions.cpu().numpy()
        bad = (got != want) & act0[:, None]
        assert np.all(margin[bad] < 1e-5), t
        loose += int(bad.sum())
        got = np.where(act0[:, None], got, 0)
        oo, rew, dd, tt, _, _ = orc.step(got, autoreset=False)
        assert np.array_equal(env.obs.cpu().numpy(), oo) and np.array_equal(env.rew.cpu().numpy(), rew) and np.array_equal(env.done.cpu().numpy(), dd), t
        s = np.nonzero(act0)[0]
        ref["act"][s, :, step0[s]] = got[s]
        ref["rew"][s, :, step0[s]] = rew[s]
        ref["obs"][s, :, step0[s] + 1] = oo[s]
        ref["done"][s, step0[s] + 1] = dd[s] | tt[s]
        ref["filled"][s, step0[s]] = 1
    for k in ref:
        assert np.array_equal(getattr(traj, k).cpu().numpy(), ref[k]), k
    assert loose < 5 and 0 < ref["filled"].sum() < E * T


def test_lbf_fused_categorical_rollout_with_batch_writes_at_32_agents():
    """N = 32: Philox blocks 0..7 of the categorical stream."""
    cfg, E = LBF["lbf_20x20_32p_10f"]
    _categorical_with_batch_writes(*_lbf_pair(cfg, E), A=6, T=14, scale=2.0)


def test_rware_fused_categorical_rollout_with_batch_writes_at_31_agents():
    cfg, E = RWARE["rware_large_n31_s3"]
    _categorical_with_batch_writes(*_rware_pair(cfg, E), A=5, T=14, scale=1.5)


def test_frames_at_32_and_31_agents():
    from codebase_b200.lbf import NativeLbf
    from codebase_b200.rware import NativeRware
    from tests.test_render_gpu import random_lbf, random_rware

    for env, draw in ((NativeLbf(LBF["lbf_20x20_32p_10f"][0], 9, seed=0), random_lbf), (NativeRware(RWARE["rware_tiny_n31"][0], 9, seed=0), random_rware)):
        want = draw(env, np.random.default_rng(env.N))
        got = env.render(0, env.E).cpu().numpy()
        assert env.frame_shape == want[0].shape
        for e in range(env.E):
            assert np.array_equal(got[e], want[e]), (env.N, e, np.argwhere((got[e] != want[e]).any(-1))[:5])


def test_rware_refuses_32_agents():
    from codebase_b200 import _native as nat
    from codebase_b200.rware import NativeRware

    with pytest.raises(nat.NativeError, match=r"n_agents 32 out of range \(1\.\.31\)"):
        NativeRware(dataclasses.replace(RWARE["rware_tiny_n31"][0], n_agents=32), 4, 0)
    env, orc = _rware_pair(RWARE["rware_tiny_n31"][0], 5)
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())


def test_oversized_vector_tile_is_refused_with_its_limit():
    """The vector path names the shared-memory limit before any allocation, like the grid path, and leaves no CUDA error behind for the next
    launch (torch's own launch check or an env's) to report."""
    from codebase_b200 import _native as nat
    from codebase_b200.lbf import NativeLbf

    with pytest.raises(nat.NativeError, match=rf"vector observations of a 64x64 field with 2 agents need {REFUSED_LBF_SMEM} B of shared memory per CTA .*the device allows \d+ B"):
        NativeLbf(REFUSED_LBF, 4, 0)
    x = torch.arange(4096, device="cuda", dtype=torch.float32)
    assert float((2 * x).sum()) == 4096 * 4095
    cfg, E = LBF["lbf_n9_g16"]
    env, orc = _lbf_pair(cfg, E)
    assert np.array_equal(env.reset().cpu().numpy(), orc.reset())
    a = np.zeros((E, cfg.n_agents), np.int32)
    assert np.array_equal(env.step(torch.tensor(a, device="cuda"))[0].cpu().numpy(), orc.step(a)[0])
