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
#include "env_common.cuh"
#include "render.cuh"

namespace marl {

struct LbfCfgDev {
  int R, C, N, NF, S, minp, maxp, minf, maxf, max_steps, time_limit, force_coop, normalize, coop_reward;
  double penalty;
  int RC, pitch, G, D;
  int obs_id, std_rew;   // ObserveID / StandardiseReward wrappers (marlbase/utils/wrappers.py:75-103, 111-141)
  int upstream_reset;    // marl_lbf_cfg.upstream_reset
};

struct LbfStateDev {
  int8_t* field; uint32_t* players; int32_t* food_spawned;
  EpisodeStateDev ep;
};

constexpr int kThreads = 128;
constexpr int kMaxFood = 32;
constexpr int kMaxVecObs = 3 * kMaxFood + 4 * MARL_MAX_AGENTS;   // the widest vector observation validate_cfg admits: foods, players, ObserveID's one-hot
constexpr int kMaxGridSight = 127;   // the largest field side: a wider window only adds padding (and keeps N*D*E-per-CTA in int range)

__device__ __forceinline__ int imin(int a, int b) { return a < b ? a : b; }
__device__ __forceinline__ int imax(int a, int b) { return a > b ? a : b; }

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

// ---- grid observation (ForagingEnv._make_gym_obs with grid_observation=True; DESIGN.md Appendix A) --------
// Feature d of the agent whose player word is `me`: layer d / W^2 and window cell (wr, wc) = divmod(d % W^2, W), W = 2*sight + 1, which is
// field cell (row + wr - sight, col + wc - sight).  Layer 0: level of the player on the cell; 1: food level; 2 (access): 1 on a cell of the
// field that holds neither.  Every layer is 0 off the field (upstream pads by `sight`).  f, amap: one env's field tile and agent map.
__device__ __forceinline__ float grid_feature(const LbfCfgDev& c, const int8_t* f, const int8_t* amap, uint32_t me, int d) {
  const int W = 2 * c.S + 1, W2 = W * W;
  const int layer = d / W2, cell = d - layer * W2, wr = cell / W, wc = cell - wr * W;
  const int r = (int)(me & 0xFF) + wr - c.S, cc = (int)((me >> 8) & 0xFF) + wc - c.S;
  if (r < 0 || r >= c.R || cc < 0 || cc >= c.C) return 0.f;
  const int lv = amap[r * c.C + cc], fo = f[r * c.C + cc];
  return (float)(layer == 0 ? lv : layer == 1 ? fo : (lv == 0 && fo == 0));
}

// The CTA writes the grid observations of its envs (EPC per CTA, E in all), one thread per (env, agent, feature): every agent's D-run is
// contiguous in obs_out [E][N][D] and in the trajectory store, so the stores stay coalesced for any D.  Tiles: field_s / amap_s [EPC][sp],
// pl_s [EPC][G]; meta_s[l*4+1]: env l's trajectory slot (-1: no write), meta_s[l*4+2]: the observation row it fills.
__device__ __forceinline__ void write_grid_obs(const LbfCfgDev& c, int E, const int8_t* field_s, const int8_t* amap_s, const uint32_t* pl_s,
                                               const int* meta_s, float* obs_out, const TrajView& traj) {
  const int EPC = (kThreads / 32) * (32 / c.G), sp = c.pitch + 4, e0 = blockIdx.x * EPC, n_here = imin(EPC, E - e0);   // recomputed: nothing stays live
  const int per_env = c.N * c.D;
  for (int i = threadIdx.x; i < n_here * per_env; i += kThreads) {
    const int l = i / per_env, rem = i - l * per_env, ag = rem / c.D, d = rem - ag * c.D;
    const float v = grid_feature(c, field_s + (size_t)l * sp, amap_s + (size_t)l * sp, pl_s[l * c.G + ag], d);
    if (obs_out) obs_out[(size_t)e0 * per_env + i] = v;
    const int sl = meta_s[l * 4 + 1];
    if (sl >= 0) traj.obs_row(sl, ag, meta_s[l * 4 + 2])[d] = v;
  }
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
                                 float* obs_out, TrajView traj, int slot0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  int8_t* f = s.field + (size_t)e * c.pitch;
  uint32_t* pl = s.players + (size_t)e * c.N;
  const bool doit = (mask == nullptr) || mask[e];
  if (doit) s.food_spawned[e] = reset_env(c, seed, gid0 + (uint32_t)e, begin_episode(s.ep, e, c.N), f, pl);
  if (obs_out == nullptr && !(traj.obs && doit)) return;
  uint32_t foods[kMaxFood];
  const int nf = list_foods(c, f, foods, kMaxFood);
  float o[kMaxVecObs];
  for (int i = 0; i < c.N; ++i) {
    build_obs(c, foods, nf, pl, i, o);
    if (obs_out) for (int d = 0; d < c.D; ++d) obs_out[((size_t)e * c.N + i) * c.D + d] = o[d];
    if (traj.obs && doit) {  // ReplayBuffer.init_episode (dqn/train.py:65-71)
      float* dst = traj.obs_row((slot0 + e) % traj.capacity, i, 0);
      for (int d = 0; d < c.D; ++d) dst[d] = o[d];
    }
  }
}

// ---- grid observations after a reset: lbf_reset_kernel resets the state, this kernel writes obs_out and (for the masked envs)
// init_episode's row 0.  Same CTA shape and shared-memory layout as lbf_step_kernel<true>: field_s, pl_s, meta_s, amap_s.
__global__ void __launch_bounds__(kThreads) lbf_grid_obs_kernel(LbfCfgDev c, LbfStateDev s, int E, const uint8_t* mask, float* obs_out,
                                                               TrajView traj, int slot0) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int EPC = (kThreads / 32) * (32 / c.G), sp = c.pitch + 4;
  int8_t* field_s = reinterpret_cast<int8_t*>(smem_raw);
  uint32_t* pl_s = reinterpret_cast<uint32_t*>(field_s + (size_t)EPC * sp);
  int* meta_s = reinterpret_cast<int*>(pl_s + EPC * c.G);
  int8_t* amap_s = reinterpret_cast<int8_t*>(meta_s + EPC * 4);
  const int e0 = blockIdx.x * EPC, n_here = imin(EPC, E - e0);
  for (int i = threadIdx.x; i < n_here * sp; i += kThreads) {
    const int l = i / sp, p = i - l * sp;
    field_s[i] = p < c.pitch ? s.field[(size_t)(e0 + l) * c.pitch + p] : (int8_t)0;
    amap_s[i] = 0;
  }
  for (int l = threadIdx.x; l < n_here; l += kThreads) {
    const bool doit = (mask == nullptr) || mask[e0 + l];
    meta_s[l * 4 + 1] = (traj.obs && doit) ? (slot0 + e0 + l) % traj.capacity : -1;
    meta_s[l * 4 + 2] = 0;
  }
  __syncthreads();
  for (int l = threadIdx.x; l < n_here; l += kThreads)
    for (int ag = 0; ag < c.N; ++ag) {   // ascending agent order: on a shared cell the later player's level stays (see lbf_step_kernel)
      const uint32_t w = s.players[((size_t)e0 + l) * c.N + ag];
      pl_s[l * c.G + ag] = w;
      amap_s[(size_t)l * sp + (int)(w & 0xFF) * c.C + (int)((w >> 8) & 0xFF)] = (int8_t)((w >> 16) & 0xFF);
    }
  __syncthreads();
  write_grid_obs(c, E, field_s, amap_s, pl_s, meta_s, obs_out, traj);
}

__global__ void lbf_set_state_kernel(LbfCfgDev c, LbfStateDev s, int E, const int8_t* field, const uint32_t* players, const int32_t* step) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  int8_t* f = s.field + (size_t)e * c.pitch;
  int sum = 0;
  for (int p = 0; p < c.pitch; ++p) { const int8_t v = p < c.RC ? field[(size_t)e * c.RC + p] : (int8_t)0; f[p] = v; sum += v; }
  for (int i = 0; i < c.N; ++i) s.players[(size_t)e * c.N + i] = players[(size_t)e * c.N + i] & 0x00FFFFFFu;
  s.food_spawned[e] = sum;
  restart_episode(s.ep, e, c.N, step[e]);
}

__global__ void lbf_get_state_kernel(LbfCfgDev c, LbfStateDev s, int E, int8_t* field, uint32_t* players, int32_t* step, int32_t* food_spawned,
                                     float* ep_return, int32_t* ep_len, uint32_t* episode_idx, uint8_t* active) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  if (field) for (int p = 0; p < c.RC; ++p) field[(size_t)e * c.RC + p] = s.field[(size_t)e * c.pitch + p];
  if (players) for (int i = 0; i < c.N; ++i) players[(size_t)e * c.N + i] = s.players[(size_t)e * c.N + i];
  if (food_spawned) food_spawned[e] = s.food_spawned[e];
  copy_episode(s.ep, e, c.N, step, ep_return, ep_len, episode_idx, active);
}

// ---- the transition kernel ---------------------------------------------------------------------------------
// kGrid = false: the vector observation, staged [EPC][N][D] in shared memory.  kGrid = true: the grid observation, which does not fit that
// staging at grid widths (full sight on 8x8: 64 envs x 2 agents x 867 x 4 B = 444 KB); each env gets an int8 agent map beside its field tile
// instead, and write_grid_obs produces the observation from the two.
template <bool kGrid>
__global__ void __launch_bounds__(kThreads) lbf_step_kernel(LbfCfgDev c, LbfStateDev s, StepArgs a, TrajView traj) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int G = c.G, EPW = 32 / G, EPC = (kThreads / 32) * EPW;
  // Shared-memory pitch of an env's grid = pitch + 4 bytes, i.e. an ODD number of words: the lanes of a warp work on different envs at the same cell
  // offset, and with the global pitch (64 B at 8x8: 16 words) every second env fell on the same bank.
  const int sp = c.pitch + 4, spw = sp >> 2, p16 = c.pitch >> 4;
  int8_t* field_s = reinterpret_cast<int8_t*>(smem_raw);                                   // [EPC][sp]
  uint32_t* pl_s = reinterpret_cast<uint32_t*>(field_s + (size_t)EPC * sp);                 // [EPC][G]
  uint32_t* foods_s = pl_s + EPC * G;                                                       // [EPC][NF] (vector only)
  int* meta_s = reinterpret_cast<int*>(foods_s + (kGrid ? 0 : EPC * c.NF));                 // [EPC][4]: nfood, traj slot (-1 = no write), t_next
  float* obs_s = reinterpret_cast<float*>(meta_s + EPC * 4);                                // [EPC][N][D] (vector only)
  int8_t* amap_s = reinterpret_cast<int8_t*>(meta_s + EPC * 4);                             // [EPC][sp] (grid only): player level per cell

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
    if constexpr (kGrid) {
      uint32_t* am = reinterpret_cast<uint32_t*>(amap_s);
      for (int i = threadIdx.x; i < n_here * spw; i += kThreads) am[i] = 0u;
    }
  }
  __syncthreads();

  const bool env_ok = e < a.E;
  int8_t* f = field_s + (size_t)le * sp;
  const int step0 = env_ok ? s.ep.step[e] : 0;
  const bool active = env_ok && s.ep.active[e];
  const bool alive = active && sub < c.N;
  const uint32_t gid = a.gid0 + (uint32_t)e;
  const uint32_t ep_cur = env_ok ? episode_key(s.ep, e) : 0u;
  const int spawned = env_ok ? s.food_spawned[e] : 1;
  uint32_t me = (env_ok && sub < c.N) ? s.players[(size_t)e * c.N + sub] : 0u;
  int r = (int)(me & 0xFF), cc = (int)((me >> 8) & 0xFF);
  const int lvl = (int)((me >> 16) & 0xFF);

  // ---- action selection -------------------------------------------------------------------------------
  int a_raw = 0;
  if (alive) {
    if (a.policy == 0) {
      a_raw = a.actions[(size_t)e * c.N + sub];
    } else if (a.policy == 1) {
      a_raw = select_eps_greedy(a, gid, ep_cur, step0, e, c.N, sub);
    } else {
      a_raw = select_categorical(a, gid, ep_cur, step0, e, c.N, sub);
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
  const bool trunc = truncated(active, c.time_limit, step1);
  const bool finished = done || trunc;

  const float rew_f = wrap_reward(s.ep, a, e, env_ok, c.N, sub, gbase, alive, c.std_rew, c.coop_reward, rew);
  const float ep_ret = add_return(s.ep, a, e, c.N, sub, alive, finished, rew);

  int slot = -1;
  if (traj.obs && env_ok) slot = traj_write_scalars(traj, a, e, c.N, sub, active, step0, a_raw, rew_f, done, finished);

  // publish moved positions for the observation pass
  if (env_ok && sub < c.N) pl_s[le * G + sub] = (uint32_t)r | ((uint32_t)cc << 8) | ((uint32_t)lvl << 16);
  __syncwarp();

  if (env_ok && sub == 0) {
    end_step(s.ep, a, e, active, step1, done, trunc, [&](uint32_t ep) { s.food_spawned[e] = reset_env(c, a.seed, gid, ep, f, pl_s + le * G); });
    if constexpr (!kGrid) meta_s[le * 4 + 0] = list_foods(c, f, foods_s + le * c.NF, c.NF);
    if constexpr (kGrid) {
      // Two players can share a cell (one enters the cell of another whose own move collided), so the agent map is written in ascending
      // agent order: the later player's level stays, as in upstream's assignment loop.
      for (int i = 0; i < c.N; ++i) {
        const uint32_t w = pl_s[le * G + i];
        amap_s[(size_t)le * sp + (int)(w & 0xFF) * c.C + (int)((w >> 8) & 0xFF)] = (int8_t)((w >> 16) & 0xFF);
      }
    }
    meta_s[le * 4 + 1] = slot;
    meta_s[le * 4 + 2] = step1;
  }
  __syncwarp();
  if (env_ok && sub < c.N) {
    store_return(s.ep, a, e, c.N, sub, alive, finished, ep_ret);
    const uint32_t w = pl_s[le * G + sub];
    s.players[(size_t)e * c.N + sub] = w;
    if constexpr (!kGrid) build_obs(c, foods_s + le * c.NF, meta_s[le * 4 + 0], pl_s + le * G, sub, obs_s + ((size_t)le * c.N + sub) * c.D);
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
  if constexpr (kGrid) {
    write_grid_obs(c, a.E, field_s, amap_s, pl_s, meta_s, a.obs_out, traj);
    return;
  }
  const int per_env = c.N * c.D;
  if (a.obs_out) {
    float* dst = a.obs_out + (size_t)e0 * per_env;
    for (int i = threadIdx.x; i < n_here * per_env; i += kThreads) dst[i] = obs_s[i];
  }
  if (traj.obs) {
    for (int i = threadIdx.x; i < n_here * per_env; i += kThreads) {
      const int l = i / per_env, rem = i % per_env, ag = rem / c.D, d = rem % c.D;
      const int sl = meta_s[l * 4 + 1];
      if (sl >= 0) traj.obs_row(sl, ag, meta_s[l * 4 + 2])[d] = obs_s[i];
    }
  }
}

// ---- frames (DESIGN.md §4.8): one CTA per (env, band of pixel rows) --------------------------------------------------
// top: 1 + the index of the agent drawn last on each cell (0: none).  The cell's badge shows that agent's level, else the food's.
__device__ __forceinline__ render::Rgb lbf_pixel(const LbfCfgDev& c, const int8_t* field, const int8_t* top, const uint32_t* pl, int x, int y) {
  using namespace render;
  constexpr int P = kLbfCell + 1, M = kLbfCell / 2;
  if (x % P == 0 || y % P == 0) return kBlack;
  const int col = x / P, row = y / P, lx = x - col * P - 1, ly = y - row * P - 1;
  const int food = (uint8_t)field[row * c.C + col], who = top[row * c.C + col];
  if (food == 0 && who == 0) return kWhite;
  if (in_disc(lx, ly, kLbfBadgeC, kLbfBadgeC, kLbfBadgeR)) {
    const int level = who ? (int)((pl[who - 1] >> 16) & 0xFF) : food;
    const bool ink = in_number(lx, ly, level, kLbfBadgeC, kLbfBadgeC) || !in_disc(lx, ly, kLbfBadgeC, kLbfBadgeC, kLbfBadgeR - kLbfBadgeLine);
    return ink ? kBlack : kWhite;
  }
  if (who && in_disc(lx, ly, M, M, kLbfAgentR)) return kLbfAgent;
  if (food && in_disc(lx, ly, M, M, kLbfFoodR)) return kLbfFood;
  return kWhite;
}

// One kernel for vector and grid ids: they share the state.  frames: [n][H][W][3], frame l of env env_first + l.
__global__ void __launch_bounds__(render::kRenderThreads) lbf_render_kernel(LbfCfgDev c, LbfStateDev s, int env_first, uint8_t* frames, int H, int W) {
  __shared__ __align__(16) uint8_t band_s[render::kBandBytes + 16];
  __shared__ int8_t field_s[4096], top_s[4096];
  __shared__ uint32_t pl_s[MARL_MAX_AGENTS];
  const int l = blockIdx.x;
  const size_t e = (size_t)env_first + l;
  for (int i = threadIdx.x; i < c.RC; i += blockDim.x) { field_s[i] = s.field[e * c.pitch + i]; top_s[i] = 0; }
  for (int i = threadIdx.x; i < c.N; i += blockDim.x) pl_s[i] = s.players[e * c.N + i];
  __syncthreads();
  if (threadIdx.x == 0)   // ascending agent order: on a shared cell the higher index is drawn last, as in the observation
    for (int i = 0; i < c.N; ++i) {
      const int r = (int)(pl_s[i] & 0xFF), cc = (int)((pl_s[i] >> 8) & 0xFF);
      if (r < c.R && cc < c.C) top_s[r * c.C + cc] = (int8_t)(i + 1);
    }
  __syncthreads();
  const int rows = render::band_rows(W), y0 = blockIdx.y * rows, y1 = imin(H, y0 + rows);
  render::render_band(frames + (size_t)l * H * W * 3, W, y0, y1, band_s,
                      [&](int x, int y) { return lbf_pixel(c, field_s, top_s, pl_s, x, y); });
}

}  // namespace marl

// =============================================================================================================
// C ABI
// =============================================================================================================
using namespace marl;

struct marl_lbf : EnvHandle {
  marl_lbf_cfg cfg;
  LbfCfgDev dev;
  LbfStateDev st;
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
  if (c->grid_observation) {
    MARL_REQUIRE(!c->observe_id, "marl_lbf: grid observations cannot be combined with observe_id (ObserveID assumes a flattened observation space)");
    MARL_REQUIRE(c->sight <= kMaxGridSight, "marl_lbf: sight %d out of range for grid observations (1..%d)", c->sight, kMaxGridSight);
  } else {   // lbf_reset_kernel builds each observation in a float[kMaxVecObs]
    MARL_REQUIRE(marl_lbf_obs_dim(c) <= kMaxVecObs, "marl_lbf: vector observation width %d out of range (1..%d)", marl_lbf_obs_dim(c), kMaxVecObs);
  }
  return MARL_OK;
}

// Shared memory per CTA of lbf_step_kernel (both observation kinds) and lbf_grid_obs_kernel (grid)
static size_t step_smem_bytes(const LbfCfgDev& d, bool grid) {
  const size_t EPC = (size_t)(kThreads / 32) * (32 / d.G), sp = (size_t)d.pitch + 4;
  if (grid) return EPC * (2 * sp + (size_t)d.G * 4 + 16);
  return EPC * sp + EPC * d.G * 4 + EPC * d.NF * 4 + EPC * 16 + EPC * d.N * d.D * 4;
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
  d.G = g; d.D = marl_lbf_obs_dim(&c);
  return d;
}

extern "C" {

int marl_lbf_obs_dim(const marl_lbf_cfg* cfg) {
  if (!cfg) return MARL_EINVAL;
  if (cfg->grid_observation) {
    if (cfg->sight < 1 || cfg->sight > kMaxGridSight) return MARL_EINVAL;
    return 3 * (2 * cfg->sight + 1) * (2 * cfg->sight + 1);
  }
  return 3 * cfg->max_num_food + 3 * cfg->n_agents + (cfg->observe_id ? cfg->n_agents : 0);
}

int marl_lbf_create(const marl_lbf_cfg* cfg, int32_t n_envs, uint64_t seed, uint32_t env_gid0, int32_t device, marl_lbf** out) {
  MARL_REQUIRE(out != nullptr, "marl_lbf_create: out is NULL");
  *out = nullptr;
  if (int rc = validate_cfg(cfg)) return rc;
  MARL_REQUIRE(n_envs >= 1, "marl_lbf_create: n_envs must be >= 1");
  if (int rc = check_device(device)) return rc;
  const bool grid = cfg->grid_observation != 0;
  {   // every env of a CTA needs its tiles in shared memory: name the limit rather than fail in cudaFuncSetAttribute
    const LbfCfgDev d = to_dev(*cfg);
    const size_t need = step_smem_bytes(d, grid);
    const int epc = (kThreads / 32) * (32 / d.G);
    int optin = 0;
    MARL_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    if (grid)
      MARL_REQUIRE(need <= (size_t)optin, "marl_lbf_create: grid observations of a %dx%d field with %d agents need %zu B of shared memory per CTA "
                   "(%d envs x 2 tiles of %d B); the device allows %d B", cfg->rows, cfg->cols, cfg->n_agents, need, epc, d.pitch + 4, optin);
    else
      MARL_REQUIRE(need <= (size_t)optin, "marl_lbf_create: vector observations of a %dx%d field with %d agents need %zu B of shared memory per CTA "
                   "(%d envs x a %d B field tile and %d observations of %d floats); the device allows %d B", cfg->rows, cfg->cols, cfg->n_agents,
                   need, epc, d.pitch + 4, d.N, d.D, optin);
  }
  marl_lbf* h = new marl_lbf();
  h->cfg = *cfg; h->dev = to_dev(*cfg); h->E = n_envs; h->device = device; h->seed = seed; h->gid0 = env_gid0;
  const LbfCfgDev& d = h->dev;
  const size_t E = (size_t)n_envs;
  const int EPC = (kThreads / 32) * (32 / d.G);
  h->envs_per_cta = EPC; h->threads = kThreads;
  h->step_smem = step_smem_bytes(d, grid);
  static size_t step_smem_limit = 48 * 1024, grid_step_smem_limit = 48 * 1024, grid_obs_smem_limit = 48 * 1024;
  int rc = alloc_buffers(h, "marl_lbf_create", {{&h->st.field, E * d.pitch}, {&h->st.players, E * d.N * 4}, {&h->st.food_spawned, E * 4}});
  if (rc == MARL_OK) rc = alloc_episode_state(h, "marl_lbf_create", h->st.ep, E, d.N);
  if (rc == MARL_OK && !grid) rc = raise_smem_limit(lbf_step_kernel<false>, h->step_smem, step_smem_limit, "marl_lbf_create");
  if (rc == MARL_OK && grid) rc = raise_smem_limit(lbf_step_kernel<true>, h->step_smem, grid_step_smem_limit, "marl_lbf_create");
  if (rc == MARL_OK && grid) rc = raise_smem_limit(lbf_grid_obs_kernel, h->step_smem, grid_obs_smem_limit, "marl_lbf_create");
  if (rc != MARL_OK) { marl_lbf_destroy(h); return rc; }
  *out = h;
  return MARL_OK;
}

int marl_lbf_destroy(marl_lbf* h) { return destroy_handle(h); }

int marl_lbf_set_state(marl_lbf* h, const int8_t* field, const int8_t* players, const int32_t* step, void* stream) {
  MARL_REQUIRE(h && field && players && step, "marl_lbf_set_state: NULL argument");
  return launch_per_env(h, lbf_set_state_kernel, stream, field, reinterpret_cast<const uint32_t*>(players), step);
}

int marl_lbf_get_state(marl_lbf* h, int8_t* field, int8_t* players, int32_t* step, int32_t* food_spawned, float* ep_return, int32_t* ep_len,
                       uint32_t* episode_idx, uint8_t* active, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_lbf_get_state: NULL handle");
  return launch_per_env(h, lbf_get_state_kernel, stream, field, reinterpret_cast<uint32_t*>(players), step, food_spawned, ep_return, ep_len,
                        episode_idx, active);
}

int marl_lbf_reset(marl_lbf* h, const uint8_t* reset_mask, float* obs_out, const marl_traj_view* traj, int32_t slot0, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_lbf_reset: NULL handle");
  if (int rc = check_traj(h, traj)) return rc;
  if (!h->cfg.grid_observation) return launch_per_env(h, lbf_reset_kernel, stream, h->seed, h->gid0, reset_mask, obs_out, traj_view(traj), slot0);
  // the state here, the grid observations and init_episode's row 0 from the CTA-wide element loop of lbf_grid_obs_kernel
  if (int rc = launch_per_env(h, lbf_reset_kernel, stream, h->seed, h->gid0, reset_mask, nullptr, traj_view(nullptr), 0)) return rc;
  lbf_grid_obs_kernel<<<(h->E + h->envs_per_cta - 1) / h->envs_per_cta, kThreads, h->step_smem, (cudaStream_t)stream>>>(
      h->dev, h->st, h->E, reset_mask, obs_out, traj_view(traj), slot0);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int marl_lbf_step(marl_lbf* h, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out, uint8_t* trunc_out,
                  float* final_ret_out, int32_t* final_len_out, int32_t autoreset, void* stream) {
  MARL_REQUIRE(h && actions && rew_out && done_out && trunc_out, "marl_lbf_step: NULL argument");
  const StepArgs a = step_args(h, actions, obs_out, rew_out, done_out, trunc_out, final_ret_out, final_len_out, autoreset);
  return launch_step(h, h->cfg.grid_observation ? lbf_step_kernel<true> : lbf_step_kernel<false>, a, nullptr, stream);
}

int marl_lbf_rollout_step(marl_lbf* h, const float* values, const marl_rollout_args* ra, const marl_traj_view* traj, float* obs_inout,
                          float* rew_out, uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out,
                          int32_t* actions_out, void* stream) {
  MARL_REQUIRE(h && values && ra && rew_out && done_out && trunc_out, "marl_lbf_rollout_step: NULL argument");
  MARL_REQUIRE(ra->policy == 1 || ra->policy == 2, "marl_lbf_rollout_step: policy must be 1 (eps-greedy) or 2 (categorical)");
  StepArgs a;
  if (int rc = rollout_step_args(h, "marl_lbf_rollout_step", values, ra, traj, obs_inout, rew_out, done_out, trunc_out, final_ret_out, final_len_out,
                                 actions_out, a))
    return rc;
  return launch_step(h, h->cfg.grid_observation ? lbf_step_kernel<true> : lbf_step_kernel<false>, a, traj, stream);
}

int marl_lbf_frame_shape(const marl_lbf_cfg* cfg, int32_t* h, int32_t* w) {
  MARL_REQUIRE(cfg && h && w, "marl_lbf_frame_shape: NULL argument");
  if (int rc = validate_cfg(cfg)) return rc;
  *h = render::frame_side(cfg->rows, render::kLbfCell); *w = render::frame_side(cfg->cols, render::kLbfCell);
  return MARL_OK;
}

int marl_lbf_render(marl_lbf* h, int32_t env_first, int32_t n, uint8_t* frames, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_lbf_render: NULL handle");
  return render::launch_render(h, "marl_lbf_render", lbf_render_kernel, env_first, n, frames, render::frame_side(h->dev.R, render::kLbfCell),
                               render::frame_side(h->dev.C, render::kLbfCell), stream);
}

}  // extern "C"
