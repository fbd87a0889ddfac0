// lbf_env.cu -- Level-Based Foraging transition for thousands of env instances per launch (sm_90a).
//
// Replaces the gym.make()'d third-party `lbforaging` ForagingEnv.reset/step plus marlbase's wrapper stack
// (TimeLimit -> RecordEpisodeStatistics -> [CooperativeReward]); reference call sites
// marlbase/utils/envs.py:27-63,90-111, marlbase/dqn/train.py:203,217, marlbase/ac/train.py:30,79-81,
// marlbase/utils/wrappers.py:13-45,106-108.  Fused on top: model.act's action selection
// (marlbase/dqn/model.py:105-115 epsilon-greedy, marlbase/ac/model.py:150-152 categorical sample) and the
// trajectory writes (marlbase/dqn/train.py:65-89, marlbase/ac/train.py:90-99).
//
// Layout / mapping (HBM-bound integer work, no tensor cores):
//   * state in HBM: int8 grid [E][pitch] (pitch = rows*cols rounded to 16 B so every env tile is moved with
//     128-bit coalesced loads), players as one 32-bit word (row, col, level, 0) per agent, int32 counters;
//   * one lane per (env, agent): G = next pow2 >= n_agents lanes form an env group, 32/G envs per warp,
//     4 warps per CTA; the CTA's grid tile is staged in shared memory, every neighbourhood read hits smem;
//   * collisions: __match_any_sync on (env, target cell); loading: __ballot_sync of the adjacent loading
//     lanes + shuffle reduction of their levels, food cells resolved in ascending agent order;
//   * observations are assembled in shared memory and written back as one contiguous coalesced run.
#include "common.cuh"
#include <string.h>

namespace marl {

struct LbfCfgDev {
  int R, C, N, NF, S, minp, maxp, minf, maxf, max_steps, time_limit, force_coop, normalize, coop_reward;
  double penalty;
  int RC, pitch, G, D;
  int obs_id, std_rew;   // ObserveID / StandardiseReward wrappers (marlbase/utils/wrappers.py:75-103, 111-141)
  int upstream_reset;    // marl_lbf_cfg.upstream_reset
};

struct LbfStateDev {
  int8_t* field; uint32_t* players; int32_t* step; int32_t* food_spawned; float* ep_return; int32_t* ep_len;
  uint32_t* episode_idx; uint8_t* active;
  float* stdr;       // StandardiseReward state per env: wmean[N] | t[N] | sumw (float32 like the wrapper's numpy arrays); survives resets
  int32_t* stdr_n;   // [E] number of rewards seen
};

struct TrajDev {
  float* obs; int32_t* act; float* rew; uint8_t* done; uint8_t* filled; int capacity, T; int enabled;
};

struct StepArgs {
  int E; uint64_t seed; uint32_t gid0;
  int policy;  // 0 explicit actions, 1 eps-greedy over values, 2 categorical over logits
  const int32_t* actions; const float* values; float epsilon; int n_actions;
  float* obs_out; float* rew_out; uint8_t* done_out; uint8_t* trunc_out; float* final_ret; int32_t* final_len;
  int32_t* actions_out;
  int autoreset, use_proper_termination, clear_stale, slot0;
};

constexpr int kThreads = 128;
constexpr int kMaxFood = 32;

__device__ __forceinline__ int imin(int a, int b) { return a < b ? a : b; }
__device__ __forceinline__ int imax(int a, int b) { return a > b ? a : b; }

// ---- spawning (ForagingEnv.spawn_players / spawn_food) ----------------------------------------------------
struct DrawStream {
  uint32_t k0, k1, gid, ep, n; u32x4 buf;
  __device__ DrawStream(uint64_t seed, uint32_t gid_, uint32_t ep_)
      : k0((uint32_t)seed), k1((uint32_t)(seed >> 32) ^ kTagReset), gid(gid_), ep(ep_), n(0), buf{0, 0, 0, 0} {}
  __device__ uint32_t next() {
    if ((n & 3u) == 0) buf = philox4x32_10(gid, ep, n >> 2, 0u, k0, k1);
    return pick(buf, (n++) & 3u);
  }
  __device__ int randint(int lo, int hi) { return lo + (int)bounded(next(), (uint32_t)(hi - lo)); }
};

// upstream _is_empty_location: no food on the cell and no player position equal to it.  Default: the players placed so far (positions were cleared);
// upstream_reset: every player that has a position -- level byte > 0 -- including the not yet re-placed ones of the previous episode.
__device__ bool cell_empty(const LbfCfgDev& c, const int8_t* f, const uint32_t* pl, int placed, int r, int cc) {
  if (f[r * c.C + cc] != 0) return false;
  const uint32_t want = (uint32_t)r | ((uint32_t)cc << 8);
  const int n = c.upstream_reset ? c.N : placed;
  for (int j = 0; j < n; ++j)
    if ((pl[j] & 0xFFFFu) == want && (!c.upstream_reset || ((pl[j] >> 16) & 0xFFu) != 0)) return false;
  return true;
}

// f: int8[pitch] (any address space), pl: one word per agent.  Returns food_spawned.
__device__ int reset_env(const LbfCfgDev& c, uint64_t seed, uint32_t gid, uint32_t episode, int8_t* f, uint32_t* pl) {
  DrawStream ds(seed, gid, episode);
  for (int p = 0; p < c.pitch; ++p) f[p] = 0;
  if (!c.upstream_reset) { for (int i = 0; i < c.N; ++i) pl[i] = 0; }
  else { for (int k = c.N - 1; k >= 1; --k) (void)ds.randint(0, k + 1); }   // spawn_players: np_random.permutation over the level bounds
  for (int i = 0; i < c.N; ++i) {
    bool placed = false;
    for (int attempts = 0; attempts < 1000 && !placed; ++attempts) {
      const int r = ds.randint(0, c.R), cc = ds.randint(0, c.C);
      if (cell_empty(c, f, pl, i, r, cc)) {
        const int lvl = ds.randint(c.minp, c.maxp + 1);
        pl[i] = (uint32_t)r | ((uint32_t)cc << 8) | ((uint32_t)lvl << 16);
        placed = true;
      }
    }
    for (int p = 0; p < c.RC && !placed; ++p)
      if (cell_empty(c, f, pl, i, p / c.C, p % c.C)) {
        pl[i] = (uint32_t)(p / c.C) | ((uint32_t)(p % c.C) << 8) | ((uint32_t)c.minp << 16);
        placed = true;
      }
  }
  int max_lvl = c.maxf;
  if (max_lvl <= 0) {  // sum of the three lowest player levels
    int a = 1 << 20, b = 1 << 20, d = 1 << 20;
    for (int i = 0; i < c.N; ++i) {
      int v = (int)((pl[i] >> 16) & 0xFF);
      if (v < a) { d = b; b = a; a = v; } else if (v < b) { d = b; b = v; } else if (v < d) { d = v; }
    }
    max_lvl = a + (c.N > 1 ? b : 0) + (c.N > 2 ? d : 0);
  }
  const int min_lvl = c.force_coop ? max_lvl : c.minf;
  if (c.upstream_reset) { for (int k = c.NF - 1; k >= 1; --k) (void)ds.randint(0, k + 1); }   // spawn_food: permutation over the food level bounds
  int count = 0, spawned = 0;
  for (int attempts = 0; count < c.NF && attempts < 1000; ++attempts) {
    const int r = ds.randint(1, c.R - 1), cc = ds.randint(1, c.C - 1);
    int box = 0, cross = 0;
    for (int rr = imax(r - 1, 0); rr < imin(r + 2, c.R); ++rr)
      for (int c2 = imax(cc - 1, 0); c2 < imin(cc + 2, c.C); ++c2) box += f[rr * c.C + c2];
    for (int rr = imax(r - 2, 0); rr < imin(r + 3, c.R); ++rr) cross += f[rr * c.C + cc];
    for (int c2 = imax(cc - 2, 0); c2 < imin(cc + 3, c.C); ++c2) cross += f[r * c.C + c2];
    if (box > 0 || cross > 0 || !cell_empty(c, f, pl, c.N, r, cc)) continue;
    const int lvl = (min_lvl == max_lvl) ? min_lvl : ds.randint(min_lvl, max_lvl + 1);
    f[r * c.C + cc] = (int8_t)lvl;
    spawned += lvl;
    ++count;
  }
  return spawned;
}

// ---- observation (ForagingEnv._make_gym_obs, non-grid) ----------------------------------------------------
// foods: packed (row | col<<8 | level<<16) in row-major order of the whole field.
__device__ int list_foods(const LbfCfgDev& c, const int8_t* f, uint32_t* foods, int cap) {
  int n = 0;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(f);
  for (int i = 0; i < c.pitch / 4; ++i) {
    const uint32_t v = w[i];
    if (v == 0) continue;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const uint32_t lv = (v >> (8 * b)) & 0xFF;
      const int cell = 4 * i + b;
      if (lv && n < cap) foods[n++] = (uint32_t)(cell / c.C) | ((uint32_t)(cell % c.C) << 8) | (lv << 16);
    }
  }
  return n;
}

__device__ void build_obs(const LbfCfgDev& c, const uint32_t* foods, int nf, const uint32_t* pl, int agent, float* out) {
  if (c.obs_id) {  // ObserveID.observation (wrappers.py:96-103): np.eye(n_agents) concatenated in front
    for (int j = 0; j < c.N; ++j) out[j] = j == agent ? 1.f : 0.f;
    out += c.N;
  }
  const int pr = (int)(pl[agent] & 0xFF), pc = (int)((pl[agent] >> 8) & 0xFF);
  const int r0 = imax(pr - c.S, 0), r1 = imin(pr + c.S + 1, c.R), c0 = imax(pc - c.S, 0), c1 = imin(pc + c.S + 1, c.C);
  int k = 0;
  for (int i = 0; i < nf; ++i) {
    const int fr = (int)(foods[i] & 0xFF), fc = (int)((foods[i] >> 8) & 0xFF), fl = (int)((foods[i] >> 16) & 0xFF);
    if (fr >= r0 && fr < r1 && fc >= c0 && fc < c1 && k < c.NF) {
      out[3 * k] = (float)(fr - r0); out[3 * k + 1] = (float)(fc - c0); out[3 * k + 2] = (float)fl; ++k;
    }
  }
  for (; k < c.NF; ++k) { out[3 * k] = -1.f; out[3 * k + 1] = -1.f; out[3 * k + 2] = 0.f; }
  float* po = out + 3 * c.NF;
  const int orow = pr - imin(c.S, pr), ocol = pc - imin(c.S, pc);
  int slot = 0;
  for (int pass = 0; pass < 2; ++pass)
    for (int j = 0; j < c.N; ++j) {
      if ((pass == 0) != (j == agent)) continue;
      const int y = (int)(pl[j] & 0xFF) - orow, x = (int)((pl[j] >> 8) & 0xFF) - ocol;
      if (imin(y, x) < 0 || imax(y, x) > 2 * c.S) continue;
      po[3 * slot] = (float)y; po[3 * slot + 1] = (float)x; po[3 * slot + 2] = (float)((pl[j] >> 16) & 0xFF); ++slot;
    }
  for (; slot < c.N; ++slot) { po[3 * slot] = -1.f; po[3 * slot + 1] = -1.f; po[3 * slot + 2] = 0.f; }
}

// upstream adjacent_food_location, `row > 1` / `col > 1` guards included
__device__ __forceinline__ bool food_location(const LbfCfgDev& c, const int8_t* f, int r, int cc, int& fr, int& fc) {
  if (r > 1 && f[(r - 1) * c.C + cc] > 0) { fr = r - 1; fc = cc; return true; }
  if (r < c.R - 1 && f[(r + 1) * c.C + cc] > 0) { fr = r + 1; fc = cc; return true; }
  if (cc > 1 && f[r * c.C + cc - 1] > 0) { fr = r; fc = cc - 1; return true; }
  if (cc < c.C - 1 && f[r * c.C + cc + 1] > 0) { fr = r; fc = cc + 1; return true; }
  return false;
}

// ---- reset kernel: one thread per env (rare: once per episode) ---------------------------------------------
__global__ void lbf_reset_kernel(LbfCfgDev c, LbfStateDev s, int E, uint64_t seed, uint32_t gid0, const uint8_t* mask,
                                 float* obs_out, TrajDev traj, int slot0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  int8_t* f = s.field + (size_t)e * c.pitch;
  uint32_t* pl = s.players + (size_t)e * c.N;
  const bool doit = (mask == nullptr) || mask[e];
  if (doit) {
    const uint32_t ep = s.episode_idx[e];
    s.food_spawned[e] = reset_env(c, seed, gid0 + (uint32_t)e, ep, f, pl);
    s.episode_idx[e] = ep + 1;
    s.step[e] = 0; s.ep_len[e] = 0; s.active[e] = 1;
    for (int i = 0; i < c.N; ++i) s.ep_return[(size_t)e * c.N + i] = 0.f;
  }
  if (obs_out == nullptr && !(traj.enabled && doit)) return;
  uint32_t foods[kMaxFood];
  const int nf = list_foods(c, f, foods, kMaxFood);
  float o[3 * (kMaxFood + MARL_MAX_AGENTS)];
  for (int i = 0; i < c.N; ++i) {
    build_obs(c, foods, nf, pl, i, o);
    if (obs_out) for (int d = 0; d < c.D; ++d) obs_out[((size_t)e * c.N + i) * c.D + d] = o[d];
    if (traj.enabled && doit) {  // ReplayBuffer.init_episode (dqn/train.py:65-71)
      const size_t slot = (size_t)((slot0 + e) % traj.capacity);
      float* dst = traj.obs + ((slot * c.N + i) * (size_t)(traj.T + 1)) * c.D;
      for (int d = 0; d < c.D; ++d) dst[d] = o[d];
    }
  }
}

__global__ void lbf_set_state_kernel(LbfCfgDev c, LbfStateDev s, int E, const int8_t* field, const uint32_t* players, const int32_t* step) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  int8_t* f = s.field + (size_t)e * c.pitch;
  int sum = 0;
  for (int p = 0; p < c.pitch; ++p) { const int8_t v = p < c.RC ? field[(size_t)e * c.RC + p] : (int8_t)0; f[p] = v; sum += v; }
  for (int i = 0; i < c.N; ++i) { s.players[(size_t)e * c.N + i] = players[(size_t)e * c.N + i] & 0x00FFFFFFu; s.ep_return[(size_t)e * c.N + i] = 0.f; }
  s.step[e] = step[e]; s.food_spawned[e] = sum; s.ep_len[e] = 0; s.active[e] = 1;
  if (s.episode_idx[e] == 0) s.episode_idx[e] = 1;
}

__global__ void lbf_get_state_kernel(LbfCfgDev c, LbfStateDev s, int E, int8_t* field, uint32_t* players, int32_t* step, int32_t* food_spawned,
                                     float* ep_return, int32_t* ep_len, uint32_t* episode_idx, uint8_t* active) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  if (field) for (int p = 0; p < c.RC; ++p) field[(size_t)e * c.RC + p] = s.field[(size_t)e * c.pitch + p];
  for (int i = 0; i < c.N; ++i) {
    if (players) players[(size_t)e * c.N + i] = s.players[(size_t)e * c.N + i];
    if (ep_return) ep_return[(size_t)e * c.N + i] = s.ep_return[(size_t)e * c.N + i];
  }
  if (step) step[e] = s.step[e];
  if (food_spawned) food_spawned[e] = s.food_spawned[e];
  if (ep_len) ep_len[e] = s.ep_len[e];
  if (episode_idx) episode_idx[e] = s.episode_idx[e];
  if (active) active[e] = s.active[e];
}

// ---- the transition kernel ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) lbf_step_kernel(LbfCfgDev c, LbfStateDev s, StepArgs a, TrajDev traj) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int G = c.G, EPW = 32 / G, EPC = (kThreads / 32) * EPW;
  // Shared-memory pitch of an env's grid = pitch + 4 bytes, i.e. an ODD number of words: the lanes of a warp work on different envs at the same cell
  // offset, and with the global pitch (64 B at 8x8: 16 words) every second env fell on the same bank.
  const int sp = c.pitch + 4, spw = sp >> 2, p16 = c.pitch >> 4;
  int8_t* field_s = reinterpret_cast<int8_t*>(smem_raw);                                   // [EPC][sp]
  uint32_t* pl_s = reinterpret_cast<uint32_t*>(field_s + (size_t)EPC * sp);                 // [EPC][G]
  uint32_t* foods_s = pl_s + EPC * G;                                                       // [EPC][NF]
  int* meta_s = reinterpret_cast<int*>(foods_s + EPC * c.NF);                               // [EPC][4]: nfood, traj slot (-1 = no write), t_next
  float* obs_s = reinterpret_cast<float*>(meta_s + EPC * 4);                                // [EPC][N][D]

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int le = warp * EPW + lane / G, sub = lane % G, gbase = (lane / G) * G;
  const int e0 = blockIdx.x * EPC, e = e0 + le;
  const int n_here = imin(EPC, a.E - e0);
  const uint32_t gbits = (G == 32) ? 0xFFFFFFFFu : ((1u << G) - 1u);
  constexpr uint32_t FULL = 0xFFFFFFFFu;

  {  // stage the CTA's grid tile: contiguous n_here*pitch bytes, 128-bit coalesced loads, word stores into the padded rows
    const uint4* src = reinterpret_cast<const uint4*>(s.field + (size_t)e0 * c.pitch);
    uint32_t* dst = reinterpret_cast<uint32_t*>(field_s);
    for (int i = threadIdx.x; i < n_here * p16; i += kThreads) {
      const int l = i / p16, q = i - l * p16;
      const uint4 v = src[i];
      uint32_t* d = dst + l * spw + 4 * q;
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
  }
  __syncthreads();

  const bool env_ok = e < a.E;
  int8_t* f = field_s + (size_t)le * sp;
  const int step0 = env_ok ? s.step[e] : 0;
  const bool active = env_ok && s.active[e];
  const bool alive = active && sub < c.N;
  const uint32_t gid = a.gid0 + (uint32_t)e;
  const uint32_t ep_cur = env_ok ? s.episode_idx[e] - 1u : 0u;
  const int spawned = env_ok ? s.food_spawned[e] : 1;
  uint32_t me = (env_ok && sub < c.N) ? s.players[(size_t)e * c.N + sub] : 0u;
  int r = (int)(me & 0xFF), cc = (int)((me >> 8) & 0xFF);
  const int lvl = (int)((me >> 16) & 0xFF);

  // ---- action selection -------------------------------------------------------------------------------
  int a_raw = 0;
  if (alive) {
    if (a.policy == 0) {
      a_raw = a.actions[(size_t)e * c.N + sub];
    } else if (a.policy == 1) {  // dqn/model.py:105-115: one uniform per step decides the joint exploration
      const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32) ^ kTagAct;
      const u32x4 b0 = philox4x32_10(gid, ep_cur, (uint32_t)step0, 0u, k0, k1);
      const float* q = a.values + ((size_t)e * c.N + sub) * a.n_actions;
      if (a.epsilon > u01(b0.x)) {
        const u32x4 bj = philox4x32_10(gid, ep_cur, (uint32_t)step0, 1u + (uint32_t)(sub >> 2), k0, k1);
        a_raw = (int)bounded(pick(bj, sub & 3), (uint32_t)a.n_actions);
      } else {
        float best = q[0];
        for (int k = 1; k < a.n_actions; ++k) { const float v = q[k]; if (v > best) { best = v; a_raw = k; } }
      }
    } else {  // ac/model.py:150-152: Categorical(logits).sample() by inverse CDF on a Philox uniform
      const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32) ^ kTagCat;
      const u32x4 bj = philox4x32_10(gid, ep_cur, (uint32_t)step0, (uint32_t)(sub >> 2), k0, k1);
      const float u = u01(pick(bj, sub & 3));
      const float* lg = a.values + ((size_t)e * c.N + sub) * a.n_actions;
      float m = lg[0];
      for (int k = 1; k < a.n_actions; ++k) m = fmaxf(m, lg[k]);
      float tot = 0.f;
      for (int k = 0; k < a.n_actions; ++k) tot += expf(lg[k] - m);
      const float thresh = u * tot;
      float cum = 0.f;
      a_raw = a.n_actions - 1;
      for (int k = 0; k < a.n_actions; ++k) { cum += expf(lg[k] - m); if (thresh < cum) { a_raw = k; break; } }
    }
  }
  if (a.actions_out && env_ok && sub < c.N) a.actions_out[(size_t)e * c.N + sub] = a_raw;

  // ---- validity (on the pre-step grid; other players are not checked) ---------------------------------------
  int act = 0;
  if (alive) {
    bool ok;
    switch (a_raw) {
      case 0: ok = true; break;
      case 1: ok = r > 0 && f[(r - 1) * c.C + cc] == 0; break;
      case 2: ok = r < c.R - 1 && f[(r + 1) * c.C + cc] == 0; break;
      case 3: ok = cc > 0 && f[r * c.C + cc - 1] == 0; break;
      case 4: ok = cc < c.C - 1 && f[r * c.C + cc + 1] == 0; break;
      case 5: ok = (f[imax(r - 1, 0) * c.C + cc] + f[imin(r + 1, c.R - 1) * c.C + cc] + f[r * c.C + imax(cc - 1, 0)] +
                    f[r * c.C + imin(cc + 1, c.C - 1)]) > 0; break;
      default: ok = false;
    }
    act = ok ? a_raw : 0;
  }
  // ---- moves: a cell proposed by more than one player is entered by nobody --------------------------------
  {
    const int tr = r + (act == 2) - (act == 1), tc = cc + (act == 4) - (act == 3);
    const uint32_t key = alive ? (((uint32_t)(lane / G) << 16) | (uint32_t)(tr * c.C + tc)) : (0x80000000u | (uint32_t)lane);
    const uint32_t same = __match_any_sync(FULL, key);
    if (alive && __popc(same) == 1) { r = tr; cc = tc; }
  }
  // ---- loading, ascending agent index --------------------------------------------------------------------
  double rew = 0.0;
  uint32_t pend = (__ballot_sync(FULL, alive && act == 5) >> gbase) & gbits;
  for (int i = 0; i < c.N; ++i) {
    const int ri = __shfl_sync(FULL, r, gbase + i), ci = __shfl_sync(FULL, cc, gbase + i);
    const bool proc = (pend >> i) & 1u;
    int fr = 0, fc = 0;
    const bool found = proc && food_location(c, f, ri, ci, fr, fc);
    const int food = found ? (int)f[fr * c.C + fc] : 0;
    const bool near = found && ((abs(r - fr) == 1 && cc == fc) || (abs(cc - fc) == 1 && r == fr));
    const bool inadj = alive && near && (((pend >> sub) & 1u) || sub == i);
    const uint32_t adjm = (__ballot_sync(FULL, inadj) >> gbase) & gbits;
    int lsum = inadj ? lvl : 0;
    for (int off = 1; off < G; off <<= 1) lsum += __shfl_xor_sync(FULL, lsum, off);
    if (proc) pend &= ~(adjm | (1u << i));
    const bool succ = found && lsum >= food;
    if (inadj) {
      if (succ) rew = c.normalize ? (double)(lvl * food) / (double)(lsum * spawned) : (double)(lvl * food);
      else rew -= c.penalty;
    }
    __syncwarp();
    if (succ && sub == i) f[fr * c.C + fc] = 0;
    __syncwarp();
  }
  // ---- termination + wrappers ------------------------------------------------------------------------------
  uint32_t nz = 0;
  if (env_ok) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(f);
    for (int i = sub; i < c.pitch / 4; i += G) nz |= w[i];
  }
  for (int off = 1; off < G; off <<= 1) nz |= __shfl_xor_sync(FULL, nz, off);
  const int step1 = step0 + 1;
  const bool done = active && ((nz == 0) || (c.max_steps <= step1));
  const bool trunc = active && (c.time_limit > 0 && step1 >= c.time_limit);
  const bool finished = done || trunc;

  // StandardiseReward.reward (wrappers.py:119-141), the wrapper's numpy arithmetic: float32 state arrays, float64 where the python-float reward list
  // enters (q, r, the standardised reward), float32 for the variance.  RecordEpisodeStatistics sits inside it and keeps the raw reward.
  double rew_w = rew;
  if (c.std_rew) {
    float wmean = 0.f, tt = 0.f, sumw = 0.f; int n = 0;
    float* st = s.stdr + (size_t)(env_ok ? e : 0) * (2 * c.N + 1);
    if (alive) { wmean = st[sub]; tt = st[c.N + sub]; sumw = st[2 * c.N]; n = s.stdr_n[e]; }
    __syncwarp();   // every agent lane has read sumw / n before lane 0 of the env writes them
    if (alive) {
      const double q = __dsub_rn(rew, (double)wmean);                                        // (no FMA contraction: numpy rounds every operation)
      const float temp_sumw = __fadd_rn(sumw, 1.0f);
      const double r = __ddiv_rn(q, (double)temp_sumw);
      wmean = (float)__dadd_rn((double)wmean, r);
      tt = (float)__dadd_rn((double)tt, __dmul_rn(__dmul_rn(q, r), (double)sumw));
      n += 1;
      st[sub] = wmean; st[c.N + sub] = tt;
      if (sub == 0) { st[2 * c.N] = temp_sumw; s.stdr_n[e] = n; }
      if (n > 1) {
        const float var = __fdiv_rn(__fmul_rn(tt, (float)n), __fmul_rn(temp_sumw, (float)(n - 1)));
        rew_w = __ddiv_rn(__dsub_rn(rew, (double)wmean), (double)__fadd_rn(__fsqrt_rn(var), 1e-6f));
      }
    }
  }
  double tot = 0.0;  // CooperativeReward: python sum() over agents in index order
  for (int i = 0; i < c.N; ++i) {
    const double ri = __shfl_sync(FULL, rew_w, gbase + i);
    tot += ri;
  }
  const float rew_f = (float)(c.coop_reward ? tot : rew_w);
  float ep_ret = 0.f;
  if (alive) {
    ep_ret = s.ep_return[(size_t)e * c.N + sub] + (float)rew;  // float32 accumulation, raw reward (wrappers.py:33)
    if (finished && a.final_ret) a.final_ret[(size_t)e * c.N + sub] = ep_ret;
  }
  if (env_ok && sub < c.N) a.rew_out[(size_t)e * c.N + sub] = alive ? rew_f : 0.f;

  // trajectory scalars (rb.add, dqn/train.py:73-89; batch_* writes, ac/train.py:90-99)
  int slot = -1;
  if (traj.enabled && env_ok) {
    const int sl = (a.slot0 + e) % traj.capacity;
    if (active && step0 < traj.T) {
      slot = sl;
      if (sub < c.N) {
        traj.act[((size_t)sl * c.N + sub) * traj.T + step0] = a_raw;
        traj.rew[((size_t)sl * c.N + sub) * traj.T + step0] = rew_f;
      }
      if (sub == 0) {
        traj.done[(size_t)sl * (traj.T + 1) + step1] = (uint8_t)(a.use_proper_termination ? done : finished);
        traj.filled[(size_t)sl * traj.T + step0] = 1;
      }
    } else if (!active && a.clear_stale && sub == 0 && step0 < traj.T) {
      // steps after the episode ended: the reference leaves a reused slot's old tail in place (SURVEY H6)
      for (int t = step0; t < traj.T; ++t) traj.filled[(size_t)sl * traj.T + t] = 0;
    }
  }

  // publish moved positions for the observation pass
  if (env_ok && sub < c.N) pl_s[le * G + sub] = (uint32_t)r | ((uint32_t)cc << 8) | ((uint32_t)lvl << 16);
  __syncwarp();

  if (env_ok && sub == 0) {
    if (active) {
      s.step[e] = step1;
      const int len1 = s.ep_len[e] + 1;
      s.ep_len[e] = len1;
      if (finished) {
        if (a.final_len) a.final_len[e] = len1;
        if (a.autoreset) {
          const uint32_t ep = s.episode_idx[e];
          s.food_spawned[e] = reset_env(c, a.seed, gid, ep, f, pl_s + le * G);
          s.episode_idx[e] = ep + 1;
          s.step[e] = 0; s.ep_len[e] = 0;
        } else {
          s.active[e] = 0;
        }
      }
    }
    a.done_out[e] = active ? (uint8_t)done : (uint8_t)1;
    a.trunc_out[e] = (uint8_t)trunc;
    meta_s[le * 4 + 0] = list_foods(c, f, foods_s + le * c.NF, c.NF);
    meta_s[le * 4 + 1] = slot;
    meta_s[le * 4 + 2] = step1;
  }
  __syncwarp();
  if (env_ok && sub < c.N) {
    if (alive) s.ep_return[(size_t)e * c.N + sub] = (finished && a.autoreset) ? 0.f : ep_ret;
    s.players[(size_t)e * c.N + sub] = pl_s[le * G + sub];
    build_obs(c, foods_s + le * c.NF, meta_s[le * 4 + 0], pl_s + le * G, sub, obs_s + ((size_t)le * c.N + sub) * c.D);
  }
  __syncthreads();

  // ---- coalesced write-back: grid tile, observation tile, trajectory observations ---------------------------
  {
    uint4* dst = reinterpret_cast<uint4*>(s.field + (size_t)e0 * c.pitch);
    const uint32_t* src = reinterpret_cast<const uint32_t*>(field_s);
    for (int i = threadIdx.x; i < n_here * p16; i += kThreads) {
      const int l = i / p16, q = i - l * p16;
      const uint32_t* w = src + l * spw + 4 * q;
      dst[i] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
  const int per_env = c.N * c.D;
  if (a.obs_out) {
    float* dst = a.obs_out + (size_t)e0 * per_env;
    for (int i = threadIdx.x; i < n_here * per_env; i += kThreads) dst[i] = obs_s[i];
  }
  if (traj.enabled) {
    for (int i = threadIdx.x; i < n_here * per_env; i += kThreads) {
      const int l = i / per_env, rem = i % per_env, ag = rem / c.D, d = rem % c.D;
      const int sl = meta_s[l * 4 + 1];
      if (sl >= 0) traj.obs[(((size_t)sl * c.N + ag) * (traj.T + 1) + meta_s[l * 4 + 2]) * c.D + d] = obs_s[i];
    }
  }
}

}  // namespace marl

// =============================================================================================================
// C ABI
// =============================================================================================================
using namespace marl;

struct marl_lbf {
  marl_lbf_cfg cfg;
  LbfCfgDev dev;
  LbfStateDev st;
  int E, device;
  uint64_t seed;
  uint32_t gid0;
  size_t step_smem;
};

static int validate_cfg(const marl_lbf_cfg* c) {
  MARL_REQUIRE(c != nullptr, "marl_lbf: cfg is NULL");
  MARL_REQUIRE(c->rows >= 3 && c->cols >= 3 && c->rows <= 127 && c->cols <= 127, "marl_lbf: field size %dx%d unsupported (3..127)", c->rows, c->cols);
  MARL_REQUIRE(c->rows * c->cols <= 4096, "marl_lbf: field too large for the shared-memory tile");
  MARL_REQUIRE(c->n_agents >= 1 && c->n_agents <= MARL_MAX_AGENTS, "marl_lbf: n_agents %d out of range (1..%d)", c->n_agents, MARL_MAX_AGENTS);
  MARL_REQUIRE(c->max_num_food >= 1 && c->max_num_food <= kMaxFood, "marl_lbf: max_num_food %d out of range (1..%d)", c->max_num_food, kMaxFood);
  MARL_REQUIRE(c->min_player_level >= 1 && c->max_player_level >= c->min_player_level && c->max_player_level <= 30, "marl_lbf: bad player levels");
  MARL_REQUIRE(c->sight >= 1, "marl_lbf: sight must be >= 1");
  MARL_REQUIRE(c->max_episode_steps >= 1, "marl_lbf: max_episode_steps must be >= 1");
  return MARL_OK;
}

static LbfCfgDev to_dev(const marl_lbf_cfg& c) {
  LbfCfgDev d;
  d.R = c.rows; d.C = c.cols; d.N = c.n_agents; d.NF = c.max_num_food; d.S = c.sight; d.minp = c.min_player_level;
  d.maxp = c.max_player_level; d.minf = c.min_food_level; d.maxf = c.max_food_level; d.max_steps = c.max_episode_steps;
  d.time_limit = c.time_limit; d.force_coop = c.force_coop; d.normalize = c.normalize_reward; d.coop_reward = c.cooperative_reward;
  d.penalty = c.penalty;
  d.RC = c.rows * c.cols; d.pitch = (d.RC + 15) & ~15;
  int g = 1; while (g < c.n_agents) g <<= 1;
  d.obs_id = c.observe_id ? 1 : 0; d.std_rew = c.standardise_rewards ? 1 : 0; d.upstream_reset = c.upstream_reset ? 1 : 0;
  d.G = g; d.D = 3 * c.max_num_food + 3 * c.n_agents + (d.obs_id ? c.n_agents : 0);
  return d;
}

static TrajDev to_traj(const marl_traj_view* t) {
  TrajDev d; memset(&d, 0, sizeof(d));
  if (t) { d.obs = t->obs; d.act = t->act; d.rew = t->rew; d.done = t->done; d.filled = t->filled; d.capacity = t->capacity; d.T = t->T; d.enabled = 1; }
  return d;
}

static int check_traj(const marl_lbf* env, const marl_traj_view* t) {
  if (!t) return MARL_OK;
  MARL_REQUIRE(t->obs && t->act && t->rew && t->done && t->filled, "traj view has NULL buffers");
  MARL_REQUIRE(t->n_agents == env->dev.N && t->obs_dim == env->dev.D, "traj view shape (N=%d, obs=%d) does not match env (N=%d, obs=%d)", t->n_agents, t->obs_dim, env->dev.N, env->dev.D);
  MARL_REQUIRE(t->capacity >= env->E && t->T >= 1, "traj capacity %d must hold one episode per env (%d)", t->capacity, env->E);
  return MARL_OK;
}

extern "C" {

int marl_lbf_obs_dim(const marl_lbf_cfg* cfg) { return cfg ? 3 * cfg->max_num_food + 3 * cfg->n_agents + (cfg->observe_id ? cfg->n_agents : 0) : MARL_EINVAL; }

int marl_lbf_create(const marl_lbf_cfg* cfg, int32_t n_envs, uint64_t seed, uint32_t env_gid0, int32_t device, marl_lbf** out) {
  MARL_REQUIRE(out != nullptr, "marl_lbf_create: out is NULL");
  *out = nullptr;
  if (int rc = validate_cfg(cfg)) return rc;
  MARL_REQUIRE(n_envs >= 1, "marl_lbf_create: n_envs must be >= 1");
  if (int rc = check_device(device)) return rc;
  marl_lbf* h = new marl_lbf();
  h->cfg = *cfg; h->dev = to_dev(*cfg); h->E = n_envs; h->device = device; h->seed = seed; h->gid0 = env_gid0;
  const LbfCfgDev& d = h->dev;
  const size_t E = (size_t)n_envs;
  memset(&h->st, 0, sizeof(h->st));
#define ALLOC0(ptr, bytes)                                                  \
  do {                                                                      \
    cudaError_t _e = cudaMalloc((void**)&(ptr), (bytes));                   \
    if (_e == cudaSuccess) _e = cudaMemset((ptr), 0, (bytes));              \
    if (_e != cudaSuccess) { set_error("marl_lbf_create: cudaMalloc(%zu) failed: %s", (size_t)(bytes), cudaGetErrorString(_e)); marl_lbf_destroy(h); return MARL_ENOMEM; } \
  } while (0)
  ALLOC0(h->st.field, E * d.pitch);
  ALLOC0(h->st.players, E * d.N * 4);
  ALLOC0(h->st.step, E * 4);
  ALLOC0(h->st.food_spawned, E * 4);
  ALLOC0(h->st.ep_return, E * d.N * 4);
  ALLOC0(h->st.ep_len, E * 4);
  ALLOC0(h->st.episode_idx, E * 4);
  ALLOC0(h->st.active, E);
  ALLOC0(h->st.stdr, E * (2 * d.N + 1) * 4);
  ALLOC0(h->st.stdr_n, E * 4);
#undef ALLOC0
  const int EPC = (kThreads / 32) * (32 / d.G);
  h->step_smem = (size_t)EPC * (d.pitch + 4) + (size_t)EPC * d.G * 4 + (size_t)EPC * d.NF * 4 + (size_t)EPC * 16 + (size_t)EPC * d.N * d.D * 4;
  // the attribute is a per-function, process-wide setting: only ever raise it (a second env with a smaller tile must not lower the limit of the first)
  static size_t step_smem_limit = 48 * 1024;
  if (h->step_smem > step_smem_limit) {
    cudaError_t e = cudaFuncSetAttribute(lbf_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->step_smem);
    if (e == cudaSuccess) step_smem_limit = h->step_smem;
    if (e != cudaSuccess) { set_error("marl_lbf_create: %zu B of shared memory per CTA not available: %s", h->step_smem, cudaGetErrorString(e)); marl_lbf_destroy(h); return MARL_EINVAL; }
  }
  *out = h;
  return MARL_OK;
}

int marl_lbf_destroy(marl_lbf* h) {
  if (!h) return MARL_OK;
  cudaSetDevice(h->device);
  cudaFree(h->st.field); cudaFree(h->st.players); cudaFree(h->st.step); cudaFree(h->st.food_spawned);
  cudaFree(h->st.ep_return); cudaFree(h->st.ep_len); cudaFree(h->st.episode_idx); cudaFree(h->st.active); cudaFree(h->st.stdr); cudaFree(h->st.stdr_n);
  delete h;
  return MARL_OK;
}

int marl_lbf_state_ptrs(marl_lbf* h, marl_lbf_state* out) {
  MARL_REQUIRE(h && out, "marl_lbf_state_ptrs: NULL argument");
  out->field = h->st.field; out->players = reinterpret_cast<int8_t*>(h->st.players); out->step = h->st.step;
  out->food_spawned = h->st.food_spawned; out->ep_return = h->st.ep_return; out->ep_len = h->st.ep_len;
  out->episode_idx = h->st.episode_idx; out->active = h->st.active; out->field_pitch = h->dev.pitch; out->n_envs = h->E;
  return MARL_OK;
}

int marl_lbf_set_state(marl_lbf* h, const int8_t* field, const int8_t* players, const int32_t* step, void* stream) {
  MARL_REQUIRE(h && field && players && step, "marl_lbf_set_state: NULL argument");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  lbf_set_state_kernel<<<(h->E + 127) / 128, 128, 0, (cudaStream_t)stream>>>(h->dev, h->st, h->E, field, reinterpret_cast<const uint32_t*>(players), step);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int marl_lbf_get_state(marl_lbf* h, int8_t* field, int8_t* players, int32_t* step, int32_t* food_spawned, float* ep_return, int32_t* ep_len,
                       uint32_t* episode_idx, uint8_t* active, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_lbf_get_state: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  lbf_get_state_kernel<<<(h->E + 127) / 128, 128, 0, (cudaStream_t)stream>>>(h->dev, h->st, h->E, field, reinterpret_cast<uint32_t*>(players), step, food_spawned,
                                                                             ep_return, ep_len, episode_idx, active);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int marl_lbf_reset(marl_lbf* h, const uint8_t* reset_mask, float* obs_out, const marl_traj_view* traj, int32_t slot0, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_lbf_reset: NULL handle");
  if (int rc = check_traj(h, traj)) return rc;
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  lbf_reset_kernel<<<(h->E + 127) / 128, 128, 0, (cudaStream_t)stream>>>(h->dev, h->st, h->E, h->seed, h->gid0, reset_mask, obs_out, to_traj(traj), slot0);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

static int launch_step(marl_lbf* h, const StepArgs& a, const marl_traj_view* traj, void* stream) {
  const int EPC = (kThreads / 32) * (32 / h->dev.G);
  const int grid = (h->E + EPC - 1) / EPC;
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  lbf_step_kernel<<<grid, kThreads, h->step_smem, (cudaStream_t)stream>>>(h->dev, h->st, a, to_traj(traj));
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int marl_lbf_step(marl_lbf* h, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out, uint8_t* trunc_out,
                  float* final_ret_out, int32_t* final_len_out, int32_t autoreset, void* stream) {
  MARL_REQUIRE(h && actions && rew_out && done_out && trunc_out, "marl_lbf_step: NULL argument");
  StepArgs a; memset(&a, 0, sizeof(a));
  a.E = h->E; a.seed = h->seed; a.gid0 = h->gid0; a.policy = 0; a.actions = actions; a.obs_out = obs_out; a.rew_out = rew_out;
  a.done_out = done_out; a.trunc_out = trunc_out; a.final_ret = final_ret_out; a.final_len = final_len_out; a.autoreset = autoreset;
  return launch_step(h, a, nullptr, stream);
}

int marl_lbf_rollout_step(marl_lbf* h, const float* values, const marl_rollout_args* ra, const marl_traj_view* traj, float* obs_inout,
                          float* rew_out, uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out,
                          int32_t* actions_out, void* stream) {
  MARL_REQUIRE(h && values && ra && rew_out && done_out && trunc_out, "marl_lbf_rollout_step: NULL argument");
  MARL_REQUIRE(ra->policy == 1 || ra->policy == 2, "marl_lbf_rollout_step: policy must be 1 (eps-greedy) or 2 (categorical)");
  MARL_REQUIRE(ra->n_actions >= 1 && ra->n_actions <= 64, "marl_lbf_rollout_step: n_actions out of range");
  if (int rc = check_traj(h, traj)) return rc;
  MARL_REQUIRE(!(traj && ra->autoreset), "marl_lbf_rollout_step: trajectory recording needs autoreset=0 (episode-synchronous collection)");
  StepArgs a; memset(&a, 0, sizeof(a));
  a.E = h->E; a.seed = h->seed; a.gid0 = h->gid0; a.policy = ra->policy; a.values = values; a.epsilon = ra->epsilon; a.n_actions = ra->n_actions;
  a.obs_out = obs_inout; a.rew_out = rew_out; a.done_out = done_out; a.trunc_out = trunc_out; a.final_ret = final_ret_out; a.final_len = final_len_out;
  a.actions_out = actions_out; a.autoreset = ra->autoreset; a.use_proper_termination = ra->use_proper_termination; a.clear_stale = ra->clear_stale; a.slot0 = ra->slot0;
  return launch_step(h, a, traj, stream);
}

}  // extern "C"
