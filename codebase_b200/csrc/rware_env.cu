// rware_env.cu -- multi-robot warehouse (RWARE) transition for thousands of env instances per launch (sm_90a).
//
// Replaces the gym.make()'d third-party `rware` Warehouse.reset/step (2.x, gymnasium) under marlbase's wrapper stack (TimeLimit ->
// RecordEpisodeStatistics -> [ObserveID] -> [StandardiseReward] -> [CooperativeReward], marlbase/utils/envs.py:90-111), with the categorical
// action sampling of A2CNetwork.act and the on-policy batch writes fused in, as lbf_env.cu does for LBF.  Semantics: DESIGN.md Appendix B;
// oracle: oracle/rware_ref.py.
//
// Layout / mapping (integer work, no tensor cores):
//   * state in HBM: uint8 shelf-id grid [E][pitch] (pitch = rows*cols rounded to 16 B: 128-bit tile moves), agents as one 32-bit word
//     (x, y, dir, carried shelf id) per agent, the requested-shelf set as a 256-bit mask, int32 counters, float episode returns;
//   * one warp per env, lane = agent (N <= 31; lane 31 stands for "an empty cell" in the move graph); 4 envs per CTA, each warp works on its
//     own shared-memory tile and only synchronises itself;
//   * moves: the graph "agent -> agent standing on its target" is a functional graph; N rounds of pointer chasing with __shfl_sync give
//     every agent its cycle length, whether its chain ends on an empty cell, and the longest chain behind every agent (shared-memory
//     atomicMax); the winner of each merge is a max-reduction of (chain length, insertion rank) over the lanes with the same target;
//   * observations are assembled in shared memory and written back as one contiguous run per env.
#include "env_common.cuh"
#include "render.cuh"

namespace marl {

struct RwCfgDev {
  int R, C, RC, pitch, N, D, H, S, nshelf, qsize, max_steps, max_inact, time_limit, coop_reward, obs_id, std_rew;
  int goal0, goal1;   // goal cells (y * C + x)
};

struct RwStateDev {
  uint8_t* shelves; uint32_t* agents; uint32_t* req; int32_t* inactive;
  EpisodeStateDev ep;
};

constexpr int kRwThreads = 128, kRwEnvsPerCta = kRwThreads / 32, kReqWords = 8, kSink = 31;
constexpr int kNoop = 0, kForward = 1, kLeft = 2, kRight = 3, kToggle = 4;

__device__ __forceinline__ bool is_highway(const RwCfgDev& c, int x, int y) {
  return x % 3 == 0 || y % (c.H + 1) == 0 || y == c.R - 1 || (y > c.R - (c.H + 3) && (x == c.C / 2 - 1 || x == c.C / 2));
}
__device__ __forceinline__ bool requested(const uint32_t* req, int sid) { return (req[sid >> 5] >> (sid & 31)) & 1u; }
__device__ __forceinline__ uint32_t agent_word(int x, int y, int d, int s) { return (uint32_t)x | ((uint32_t)y << 8) | ((uint32_t)d << 16) | ((uint32_t)s << 24); }
// turning walks the cycle UP(0) -> RIGHT(3) -> DOWN(1) -> LEFT(2)
__device__ __forceinline__ int turn(int d, int step) {
  const int idx = (0x1320 >> (4 * d)) & 0xF;          // position of direction d in the cycle: UP 0, DOWN 2, LEFT 3, RIGHT 1
  return (0x2130 >> (4 * ((idx + step) & 3))) & 0xF;  // direction at a cycle position
}

// Warehouse.reset: N distinct cells, a direction per agent, qsize distinct requested shelves, every shelf at its home cell.
__device__ void reset_env(const RwCfgDev& c, uint64_t seed, uint32_t gid, uint32_t episode, uint8_t* sh, uint32_t* ag, uint32_t* req) {
  DrawStream ds(seed, gid, episode);
  for (int i = 0; i < c.N; ++i) {
    int p;
    bool taken;
    do {
      p = ds.randint(0, c.RC);
      taken = false;
      for (int j = 0; j < i; ++j) taken |= (int)((ag[j] & 0xFF) + ((ag[j] >> 8) & 0xFF) * c.C) == p;
    } while (taken);
    ag[i] = agent_word(p % c.C, p / c.C, 0, 0);
  }
  for (int i = 0; i < c.N; ++i) ag[i] |= (uint32_t)ds.randint(0, 4) << 16;
  for (int w = 0; w < kReqWords; ++w) req[w] = 0;
  for (int q = 0; q < c.qsize; ++q) {
    int s;
    do { s = 1 + ds.randint(0, c.nshelf); } while (requested(req, s));
    req[s >> 5] |= 1u << (s & 31);
  }
  int k = 0;
  for (int p = 0; p < c.pitch; ++p) sh[p] = (p < c.RC && !is_highway(c, p % c.C, p / c.C)) ? (uint8_t)(++k) : (uint8_t)0;
}

// Warehouse._make_obs (flattened), with ObserveID's one-hot id in front
__device__ void build_obs(const RwCfgDev& c, const uint8_t* sh, const uint32_t* ag, const uint32_t* req, int i, float* out) {
  if (c.obs_id) {
    for (int j = 0; j < c.N; ++j) out[j] = j == i ? 1.f : 0.f;
    out += c.N;
  }
  const uint32_t w = ag[i];
  const int x = (int)(w & 0xFF), y = (int)((w >> 8) & 0xFF), d = (int)((w >> 16) & 0xFF);
  out[0] = (float)x; out[1] = (float)y; out[2] = (w >> 24) ? 1.f : 0.f;
  for (int k = 0; k < 4; ++k) out[3 + k] = d == k ? 1.f : 0.f;
  out[7] = is_highway(c, x, y) ? 1.f : 0.f;
  float* o = out + 8;
  for (int yy = y - c.S; yy <= y + c.S; ++yy)
    for (int xx = x - c.S; xx <= x + c.S; ++xx, o += 7) {
      const bool inside = xx >= 0 && xx < c.C && yy >= 0 && yy < c.R;
      int who = -1;
      if (inside) {
        const uint32_t want = (uint32_t)xx | ((uint32_t)yy << 8);
        for (int j = 0; j < c.N; ++j) if ((ag[j] & 0xFFFFu) == want) who = j;
      }
      const int dw = who < 0 ? 0 : (int)((ag[who] >> 16) & 0xFF);   // an empty cell writes direction UP (recalled quirk)
      o[0] = who < 0 ? 0.f : 1.f;
      for (int k = 0; k < 4; ++k) o[1 + k] = dw == k ? 1.f : 0.f;
      const int sid = inside ? sh[yy * c.C + xx] : 0;
      o[5] = sid ? 1.f : 0.f;
      o[6] = (sid && requested(req, sid)) ? 1.f : 0.f;
    }
}

// ---- reset / state kernels: one thread per env (rare) ------------------------------------------------------------
__global__ void rware_reset_kernel(RwCfgDev c, RwStateDev s, int E, uint64_t seed, uint32_t gid0, const uint8_t* mask, float* obs_out, TrajView traj,
                                   int slot0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  uint8_t* sh = s.shelves + (size_t)e * c.pitch;
  uint32_t* ag = s.agents + (size_t)e * c.N;
  uint32_t* req = s.req + (size_t)e * kReqWords;
  const bool doit = (mask == nullptr) || mask[e];
  if (doit) {
    reset_env(c, seed, gid0 + (uint32_t)e, begin_episode(s.ep, e, c.N), sh, ag, req);
    s.inactive[e] = 0;
  }
  for (int i = 0; i < c.N; ++i) {
    if (obs_out) build_obs(c, sh, ag, req, i, obs_out + ((size_t)e * c.N + i) * c.D);
    if (traj.obs && doit) build_obs(c, sh, ag, req, i, traj.obs_row((slot0 + e) % traj.capacity, i, 0));
  }
}

__global__ void rware_set_state_kernel(RwCfgDev c, RwStateDev s, int E, const uint8_t* shelves, const uint32_t* agents, const uint32_t* req,
                                       const int32_t* step, const int32_t* inactive) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  for (int p = 0; p < c.pitch; ++p) s.shelves[(size_t)e * c.pitch + p] = p < c.RC ? shelves[(size_t)e * c.RC + p] : (uint8_t)0;
  for (int i = 0; i < c.N; ++i) s.agents[(size_t)e * c.N + i] = agents[(size_t)e * c.N + i];
  for (int w = 0; w < kReqWords; ++w) s.req[(size_t)e * kReqWords + w] = req[(size_t)e * kReqWords + w];
  s.inactive[e] = inactive[e];
  restart_episode(s.ep, e, c.N, step[e]);
}

__global__ void rware_get_state_kernel(RwCfgDev c, RwStateDev s, int E, uint8_t* shelves, uint32_t* agents, uint32_t* req, int32_t* step,
                                       int32_t* inactive, float* ep_return, int32_t* ep_len, uint32_t* episode_idx, uint8_t* active) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  if (shelves) for (int p = 0; p < c.RC; ++p) shelves[(size_t)e * c.RC + p] = s.shelves[(size_t)e * c.pitch + p];
  if (agents) for (int i = 0; i < c.N; ++i) agents[(size_t)e * c.N + i] = s.agents[(size_t)e * c.N + i];
  if (req) for (int w = 0; w < kReqWords; ++w) req[(size_t)e * kReqWords + w] = s.req[(size_t)e * kReqWords + w];
  if (inactive) inactive[e] = s.inactive[e];
  copy_episode(s.ep, e, c.N, step, ep_return, ep_len, episode_idx, active);
}

// Shared memory per warp (= per env): observations [N][D] floats | shelf grid [pitch] | agents [32] | requested [8] | chain lengths [32] | meta [4]
__host__ __device__ inline size_t rware_warp_smem(int N, int D, int pitch) {
  return (((size_t)N * D * 4 + 15) & ~(size_t)15) + (size_t)pitch + 32 * 4 + kReqWords * 4 + 32 * 4 + 16;
}

// ---- the transition kernel ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRwThreads) rware_step_kernel(RwCfgDev c, RwStateDev s, StepArgs a, TrajView traj) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr uint32_t FULL = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int e = blockIdx.x * kRwEnvsPerCta + w;
  if (e >= a.E) return;   // whole warps only: nothing below synchronises across warps
  unsigned char* base = smem_raw + (size_t)w * rware_warp_smem(c.N, c.D, c.pitch);
  float* obs_s = reinterpret_cast<float*>(base);
  uint8_t* sh_s = base + (((size_t)c.N * c.D * 4 + 15) & ~(size_t)15);
  uint32_t* ag_s = reinterpret_cast<uint32_t*>(sh_s + c.pitch);
  uint32_t* req_s = ag_s + 32;
  int* depth_s = reinterpret_cast<int*>(req_s + kReqWords);
  int* meta_s = depth_s + 32;

  {
    const uint4* src = reinterpret_cast<const uint4*>(s.shelves + (size_t)e * c.pitch);
    uint4* dst = reinterpret_cast<uint4*>(sh_s);
    for (int i = lane; i < (c.pitch >> 4); i += 32) dst[i] = src[i];
  }
  if (lane < kReqWords) req_s[lane] = s.req[(size_t)e * kReqWords + lane];
  depth_s[lane] = 0;
  const bool agent = lane < c.N;
  const uint32_t me = agent ? s.agents[(size_t)e * c.N + lane] : 0u;
  int x = (int)(me & 0xFF), y = (int)((me >> 8) & 0xFF), d = (int)((me >> 16) & 0xFF), sh = (int)(me >> 24);
  const int step0 = s.ep.step[e];
  const bool active = s.ep.active[e] != 0;   // warp-uniform
  const bool alive = active && agent;
  const uint32_t gid = a.gid0 + (uint32_t)e;
  const uint32_t ep_cur = episode_key(s.ep, e);
  __syncwarp();

  // ---- action selection --------------------------------------------------------------------------------------
  int a_raw = 0;
  if (alive) a_raw = a.policy == 0 ? a.actions[(size_t)e * c.N + lane] : select_categorical(a, gid, ep_cur, step0, e, c.N, lane);
  if (a.actions_out && agent) a.actions_out[(size_t)e * c.N + lane] = a_raw;
  int act = (alive && a_raw >= 0 && a_raw < 5) ? a_raw : kNoop;

  // ---- move resolution (DESIGN.md Appendix B; oracle/rware_ref.resolve_moves) ------------------------------------
  const int cell = agent ? y * c.C + x : -1 - lane;
  if (active) {
    int tc = cell;
    if (act == kForward) {
      int tx = x, ty = y;
      if (d == 0) ty = max(0, y - 1); else if (d == 1) ty = min(c.R - 1, y + 1); else if (d == 2) tx = max(0, x - 1); else tx = min(c.C - 1, x + 1);
      tc = ty * c.C + tx;
    }
    int occ = -1; bool occ_loaded = false;
    for (int j = 0; j < c.N; ++j) {
      const int cj = __shfl_sync(FULL, cell, j), sj = __shfl_sync(FULL, sh, j);
      if (cj == tc) { occ = j; occ_loaded = sj != 0; }
    }
    // a loaded agent cannot enter a cell holding a resting shelf
    const bool cancel = agent && act == kForward && sh && tc != cell && sh_s[agent ? tc : 0] && !occ_loaded;
    if (cancel) act = kNoop;
    const int t = cancel ? cell : tc;
    const int nxt = !agent ? kSink : (cancel ? lane : (occ >= 0 ? occ : kSink));
    int rank = 2 * lane;   // insertion position of the agent's cell as a node of upstream's graph
    for (int j = c.N - 1; j >= 0; --j) {
      const int tj = __shfl_sync(FULL, t, j);
      if (agent && j < lane && tj == cell) rank = 2 * j + 1;
    }
    int xw = lane, cyc = 0;
    bool sink = false;
    for (int k = 1; k <= c.N; ++k) {
      xw = __shfl_sync(FULL, nxt, xw);
      if (agent && !sink) {
        if (xw == kSink) sink = true;
        else { atomicMax(&depth_s[xw], k); if (xw == lane && cyc == 0) cyc = k; }
      }
    }
    __syncwarp();
    const int key = agent ? (depth_s[lane] << 8) | (255 - rank) : -1;
    int best = key;
    for (int j = 0; j < c.N; ++j) {
      const int kj = __shfl_sync(FULL, key, j), tj = __shfl_sync(FULL, t, j);
      if (agent && tj == t && kj > best) best = kj;
    }
    const uint32_t winmask = __ballot_sync(FULL, agent && best == key);
    bool ok = (winmask >> lane) & 1u;
    xw = lane;
    for (int k = 1; k <= c.N; ++k) {
      xw = __shfl_sync(FULL, nxt, xw);
      if (xw != kSink) ok = ok && ((winmask >> xw) & 1u);
    }
    const bool commit = cyc ? cyc != 2 : (sink && ok);
    if (act == kForward && !commit) act = kNoop;

    // ---- apply, in agent order (no two agents interact here: targets of committed moves are distinct) -------------
    const bool moving = act == kForward;
    if (moving && sh) sh_s[cell] = 0;
    __syncwarp();
    if (moving && sh) sh_s[t] = (uint8_t)sh;
    __syncwarp();
    if (moving) { x = t % c.C; y = t / c.C; }
    else if (act == kLeft) d = turn(d, 3);
    else if (act == kRight) d = turn(d, 1);
    else if (act == kToggle) {
      if (!sh) sh = sh_s[y * c.C + x];
      else if (!is_highway(c, x, y)) sh = 0;
    }
  }
  if (agent) ag_s[lane] = agent_word(x, y, d, sh);
  __syncwarp();

  // ---- deliveries, goals in order (lane 0) ---------------------------------------------------------------------
  const int step1 = step0 + 1;
  if (lane == 0) {
    uint32_t paid = 0;
    bool delivered = false;
    if (active) {
      for (int g = 0; g < 2; ++g) {
        const int gc = g ? c.goal1 : c.goal0;
        const int sid = sh_s[gc];
        if (!sid || !requested(req_s, sid)) continue;
        delivered = true;
        int nfree = 0;
        for (int k = 1; k <= c.nshelf; ++k) nfree += !requested(req_s, k);
        const u32x4 b = philox4x32_10(gid, ep_cur, (uint32_t)step1, (uint32_t)g, (uint32_t)a.seed, (uint32_t)(a.seed >> 32) ^ kTagRequest);
        int pickn = (int)bounded(b.x, (uint32_t)nfree), nw = 0;
        for (int k = 1; k <= c.nshelf; ++k)
          if (!requested(req_s, k) && pickn-- == 0) { nw = k; break; }
        req_s[sid >> 5] &= ~(1u << (sid & 31));
        req_s[nw >> 5] |= 1u << (nw & 31);
        const uint32_t want = (uint32_t)(gc % c.C) | ((uint32_t)(gc / c.C) << 8);
        for (int j = 0; j < c.N; ++j) if ((ag_s[j] & 0xFFFFu) == want) paid |= 1u << j;
      }
    }
    meta_s[0] = (int)paid; meta_s[1] = delivered;
  }
  __syncwarp();
  const double rew = (alive && ((meta_s[0] >> lane) & 1)) ? 1.0 : 0.0;
  const int inact1 = meta_s[1] ? 0 : s.inactive[e] + 1;

  // ---- termination + wrappers --------------------------------------------------------------------------------------
  const bool done = active && ((c.max_inact > 0 && inact1 >= c.max_inact) || (c.max_steps > 0 && step1 >= c.max_steps));
  const bool trunc = truncated(active, c.time_limit, step1);
  const bool finished = done || trunc;
  const float rew_f = wrap_reward(s.ep, a, e, true, c.N, lane, 0, alive, c.std_rew, c.coop_reward, rew);
  const float ep_ret = add_return(s.ep, a, e, c.N, lane, alive, finished, rew);
  const int slot = traj.obs ? traj_write_scalars(traj, a, e, c.N, lane, active, step0, a_raw, rew_f, done, finished) : -1;

  if (lane == 0) {
    if (active) s.inactive[e] = inact1;
    end_step(s.ep, a, e, active, step1, done, trunc, [&](uint32_t ep) {
      reset_env(c, a.seed, gid, ep, sh_s, ag_s, req_s);
      s.inactive[e] = 0;
    });
  }
  __syncwarp();
  if (agent) {
    store_return(s.ep, a, e, c.N, lane, alive, finished, ep_ret);
    s.agents[(size_t)e * c.N + lane] = ag_s[lane];
    build_obs(c, sh_s, ag_s, req_s, lane, obs_s + (size_t)lane * c.D);
  }
  __syncwarp();

  // ---- coalesced write-back: shelf grid, requests, observation run, trajectory observations ------------------------
  {
    uint4* dst = reinterpret_cast<uint4*>(s.shelves + (size_t)e * c.pitch);
    const uint4* src = reinterpret_cast<const uint4*>(sh_s);
    for (int i = lane; i < (c.pitch >> 4); i += 32) dst[i] = src[i];
  }
  if (lane < kReqWords) s.req[(size_t)e * kReqWords + lane] = req_s[lane];
  const int per_env = c.N * c.D;
  if (a.obs_out) {
    float* dst = a.obs_out + (size_t)e * per_env;
    for (int i = lane; i < per_env; i += 32) dst[i] = obs_s[i];
  }
  if (slot >= 0) {   // warp-uniform
    // the config's N and D, which check_traj requires the view's to equal: this kernel holds them already, and the view's own make ptxas spill
    TrajView tv = traj; tv.N = c.N; tv.D = c.D;
    for (int i = lane; i < per_env; i += 32) {
      const int ag = i / c.D, dd = i - ag * c.D;
      tv.obs_row(slot, ag, step1)[dd] = obs_s[i];
    }
  }
}

// ---- frames (DESIGN.md §4.8): one CTA per (env, band of pixel rows) --------------------------------------------------------
// Layers bottom to top: goal fill, shelf rectangle (its current cell, a carried one under its carrier), agent disc, direction line.
// top: 1 + the index of the agent drawn on each cell (0: none; agents stand on distinct cells, a later index would be drawn last).
__device__ __forceinline__ render::Rgb rware_pixel(const RwCfgDev& c, const uint8_t* sh, const int8_t* top, const uint32_t* ag, const uint32_t* req,
                                                   int x, int y) {
  using namespace render;
  constexpr int P = kRwCell + 1, M = kRwCell / 2;
  if (x % P == 0 || y % P == 0) return kBlack;
  const int col = x / P, row = y / P, lx = x - col * P - 1, ly = y - row * P - 1, cell = row * c.C + col;
  if (const int who = top[cell]) {
    const uint32_t w = ag[who - 1];
    const int d = (int)((w >> 16) & 0xFF);
    if (d < 4) {
      const int dx = d == 3 ? 1 : d == 2 ? -1 : 0, dy = d == 1 ? 1 : d == 0 ? -1 : 0;
      if (on_line(lx, ly, M, M, M + dx * kRwAgentR, M + dy * kRwAgentR, kRwDirLine)) return kRwDir;
    }
    if (in_disc(lx, ly, M, M, kRwAgentR)) return (w >> 24) ? kRwAgentLoaded : kRwAgent;
  }
  const int sid = sh[cell];
  if (sid && in_rect(lx, ly, kRwShelfPad, kRwShelfPad, kRwCell - kRwShelfPad, kRwCell - kRwShelfPad))
    return requested(req, sid) ? kRwShelfRequested : kRwShelf;
  if (cell == c.goal0 || cell == c.goal1) return kRwGoal;
  return kWhite;
}

// frames: [n][H][W][3], frame l of env env_first + l
__global__ void __launch_bounds__(render::kRenderThreads) rware_render_kernel(RwCfgDev c, RwStateDev s, int env_first, uint8_t* frames, int H, int W) {
  __shared__ __align__(16) uint8_t band_s[render::kBandBytes + 16];
  __shared__ uint8_t sh_s[4096];
  __shared__ int8_t top_s[4096];
  __shared__ uint32_t ag_s[32], req_s[kReqWords];
  const int l = blockIdx.x;
  const size_t e = (size_t)env_first + l;
  for (int i = threadIdx.x; i < c.RC; i += blockDim.x) { sh_s[i] = s.shelves[e * c.pitch + i]; top_s[i] = 0; }
  for (int i = threadIdx.x; i < c.N; i += blockDim.x) ag_s[i] = s.agents[e * c.N + i];
  if (threadIdx.x < kReqWords) req_s[threadIdx.x] = s.req[e * kReqWords + threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 0; i < c.N; ++i) {
      const int x = (int)(ag_s[i] & 0xFF), y = (int)((ag_s[i] >> 8) & 0xFF);
      if (x < c.C && y < c.R) top_s[y * c.C + x] = (int8_t)(i + 1);
    }
  __syncthreads();
  const int rows = render::band_rows(W), y0 = blockIdx.y * rows, y1 = min(H, y0 + rows);
  render::render_band(frames + (size_t)l * H * W * 3, W, y0, y1, band_s,
                      [&](int x, int y) { return rware_pixel(c, sh_s, top_s, ag_s, req_s, x, y); });
}

}  // namespace marl

// =============================================================================================================
// C ABI
// =============================================================================================================
using namespace marl;

struct marl_rware : EnvHandle {
  marl_rware_cfg cfg;
  RwCfgDev dev;
  RwStateDev st;
};

static int rware_count_shelves(const marl_rware_cfg& c) {
  const int R = (c.column_height + 1) * c.shelf_rows + 2, C = 3 * c.shelf_columns + 1;
  int n = 0;
  for (int y = 0; y < R; ++y)
    for (int x = 0; x < C; ++x)
      n += !(x % 3 == 0 || y % (c.column_height + 1) == 0 || y == R - 1 || (y > R - (c.column_height + 3) && (x == C / 2 - 1 || x == C / 2)));
  return n;
}

static int rware_validate(const marl_rware_cfg* c) {
  MARL_REQUIRE(c != nullptr, "marl_rware: cfg is NULL");
  MARL_REQUIRE(c->shelf_rows >= 1 && c->shelf_columns >= 1 && c->column_height >= 1, "marl_rware: shelf_rows, shelf_columns and column_height must be >= 1");
  const int R = (c->column_height + 1) * c->shelf_rows + 2, C = 3 * c->shelf_columns + 1;
  MARL_REQUIRE(R <= 255 && C <= 255 && R * C <= 4096, "marl_rware: a %dx%d grid is too large (at most 255 per side and 4096 cells)", R, C);
  MARL_REQUIRE(c->n_agents >= 1 && c->n_agents <= 31 && c->n_agents <= R * C, "marl_rware: n_agents %d out of range (1..31)", c->n_agents);
  const int ns = rware_count_shelves(*c);
  MARL_REQUIRE(ns >= 2 && ns <= 255, "marl_rware: %d shelves; the shelf-id grid is uint8 (2..255 shelves)", ns);
  MARL_REQUIRE(c->request_queue_size >= 1 && c->request_queue_size < ns, "marl_rware: request_queue_size %d out of range (1..%d: one shelf must stay unrequested)",
               c->request_queue_size, ns - 1);
  MARL_REQUIRE(c->sensor_range >= 0 && c->sensor_range <= 3, "marl_rware: sensor_range %d out of range (0..3)", c->sensor_range);
  MARL_REQUIRE(c->max_steps >= 0 && c->max_inactivity_steps >= 0 && c->time_limit >= 0, "marl_rware: negative step limit");
  return MARL_OK;
}

static RwCfgDev rware_to_dev(const marl_rware_cfg& c) {
  RwCfgDev d;
  d.R = (c.column_height + 1) * c.shelf_rows + 2; d.C = 3 * c.shelf_columns + 1; d.RC = d.R * d.C; d.pitch = (d.RC + 15) & ~15;
  d.N = c.n_agents; d.H = c.column_height; d.S = c.sensor_range; d.nshelf = rware_count_shelves(c); d.qsize = c.request_queue_size;
  d.max_steps = c.max_steps; d.max_inact = c.max_inactivity_steps; d.time_limit = c.time_limit;
  d.coop_reward = c.cooperative_reward ? 1 : 0; d.obs_id = c.observe_id ? 1 : 0; d.std_rew = c.standardise_rewards ? 1 : 0;
  d.D = marl_rware_obs_dim(&c);
  d.goal0 = (d.R - 1) * d.C + d.C / 2 - 1; d.goal1 = (d.R - 1) * d.C + d.C / 2;
  return d;
}

extern "C" {

int marl_rware_obs_dim(const marl_rware_cfg* cfg) {
  if (!cfg) return MARL_EINVAL;
  const int w = 2 * cfg->sensor_range + 1;
  return 8 + 7 * w * w + (cfg->observe_id ? cfg->n_agents : 0);
}

int marl_rware_create(const marl_rware_cfg* cfg, int32_t n_envs, uint64_t seed, uint32_t env_gid0, int32_t device, marl_rware** out) {
  MARL_REQUIRE(out != nullptr, "marl_rware_create: out is NULL");
  *out = nullptr;
  if (int rc = rware_validate(cfg)) return rc;
  MARL_REQUIRE(n_envs >= 1, "marl_rware_create: n_envs must be >= 1");
  if (int rc = check_device(device)) return rc;
  marl_rware* h = new marl_rware();
  h->cfg = *cfg; h->dev = rware_to_dev(*cfg); h->E = n_envs; h->device = device; h->seed = seed; h->gid0 = env_gid0;
  const RwCfgDev& d = h->dev;
  const size_t E = (size_t)n_envs;
  h->envs_per_cta = kRwEnvsPerCta; h->threads = kRwThreads;
  h->step_smem = kRwEnvsPerCta * rware_warp_smem(d.N, d.D, d.pitch);
  static size_t step_smem_limit = 48 * 1024;
  int rc = alloc_buffers(h, "marl_rware_create", {{&h->st.shelves, E * d.pitch}, {&h->st.agents, E * d.N * 4}, {&h->st.req, E * kReqWords * 4},
                                                  {&h->st.inactive, E * 4}});
  if (rc == MARL_OK) rc = alloc_episode_state(h, "marl_rware_create", h->st.ep, E, d.N);
  if (rc == MARL_OK) rc = raise_smem_limit(rware_step_kernel, h->step_smem, step_smem_limit, "marl_rware_create");
  if (rc != MARL_OK) { marl_rware_destroy(h); return rc; }
  *out = h;
  return MARL_OK;
}

int marl_rware_destroy(marl_rware* h) { return destroy_handle(h); }

int marl_rware_set_state(marl_rware* h, const uint8_t* shelves, const uint8_t* agents, const uint32_t* requested, const int32_t* step,
                         const int32_t* inactive, void* stream) {
  MARL_REQUIRE(h && shelves && agents && requested && step && inactive, "marl_rware_set_state: NULL argument");
  return launch_per_env(h, rware_set_state_kernel, stream, shelves, reinterpret_cast<const uint32_t*>(agents), requested, step, inactive);
}

int marl_rware_get_state(marl_rware* h, uint8_t* shelves, uint8_t* agents, uint32_t* requested, int32_t* step, int32_t* inactive, float* ep_return,
                         int32_t* ep_len, uint32_t* episode_idx, uint8_t* active, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_rware_get_state: NULL handle");
  return launch_per_env(h, rware_get_state_kernel, stream, shelves, reinterpret_cast<uint32_t*>(agents), requested, step, inactive, ep_return, ep_len,
                        episode_idx, active);
}

int marl_rware_reset(marl_rware* h, const uint8_t* reset_mask, float* obs_out, const marl_traj_view* traj, int32_t slot0, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_rware_reset: NULL handle");
  if (int rc = check_traj(h, traj)) return rc;
  return launch_per_env(h, rware_reset_kernel, stream, h->seed, h->gid0, reset_mask, obs_out, traj_view(traj), slot0);
}

int marl_rware_step(marl_rware* h, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out, uint8_t* trunc_out,
                    float* final_ret_out, int32_t* final_len_out, int32_t autoreset, void* stream) {
  MARL_REQUIRE(h && actions && rew_out && done_out && trunc_out, "marl_rware_step: NULL argument");
  const StepArgs a = step_args(h, actions, obs_out, rew_out, done_out, trunc_out, final_ret_out, final_len_out, autoreset);
  return launch_step(h, rware_step_kernel, a, nullptr, stream);
}

int marl_rware_rollout_step(marl_rware* h, const float* values, const marl_rollout_args* ra, const marl_traj_view* traj, float* obs_inout,
                            float* rew_out, uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out,
                            int32_t* actions_out, void* stream) {
  MARL_REQUIRE(h && values && ra && rew_out && done_out && trunc_out, "marl_rware_rollout_step: NULL argument");
  MARL_REQUIRE(ra->policy != 1, "marl_rware_rollout_step: policy 1 (epsilon-greedy) is not available on RWARE: no DQN-family learner takes its %d-feature "
               "observations (at most 32)", h->dev.D);
  MARL_REQUIRE(ra->policy == 2, "marl_rware_rollout_step: policy must be 2 (categorical)");
  StepArgs a;
  if (int rc = rollout_step_args(h, "marl_rware_rollout_step", values, ra, traj, obs_inout, rew_out, done_out, trunc_out, final_ret_out, final_len_out,
                                 actions_out, a))
    return rc;
  return launch_step(h, rware_step_kernel, a, traj, stream);
}

int marl_rware_frame_shape(const marl_rware_cfg* cfg, int32_t* h, int32_t* w) {
  MARL_REQUIRE(cfg && h && w, "marl_rware_frame_shape: NULL argument");
  if (int rc = rware_validate(cfg)) return rc;
  const RwCfgDev d = rware_to_dev(*cfg);
  *h = render::frame_side(d.R, render::kRwCell); *w = render::frame_side(d.C, render::kRwCell);
  return MARL_OK;
}

int marl_rware_render(marl_rware* h, int32_t env_first, int32_t n, uint8_t* frames, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_rware_render: NULL handle");
  return render::launch_render(h, "marl_rware_render", rware_render_kernel, env_first, n, frames, render::frame_side(h->dev.R, render::kRwCell),
                               render::frame_side(h->dev.C, render::kRwCell), stream);
}

}  // extern "C"
