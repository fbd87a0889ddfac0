// matrix_env.cu -- repeated matrix games (climbing, penalty-k) for hundreds of thousands of env instances per launch (sm_90a).
//
// Replaces the gym.make()'d `matrixgames` MatrixGame.reset/step under marlbase's wrapper stack (TimeLimit -> RecordEpisodeStatistics ->
// [ObserveID] -> [StandardiseReward] -> [CooperativeReward], marlbase/utils/envs.py:90-111), with the action selection of model.act and the
// trajectory writes fused in, as lbf_env.cu does for LBF.  Semantics: DESIGN.md Appendix C; oracle: oracle/matrix_ref.py.
//
// Layout / mapping (a table lookup; no tensor cores):
//   * state in HBM: int8 previous action per (env, player) (-1 after a reset), int32 counters, float episode returns; the payoff table is
//     double [A^N] in C order (at most 512 KB, read through the read-only path and L2-resident);
//   * one lane per (env, player): G = next pow2 >= N lanes form an env group, 32/G envs per warp, 4 warps per CTA;
//   * the joint action's table index is a shuffle-xor sum over the group of a_i * A^(N-1-i); every lane reads the same entry;
//   * observations are written by the whole CTA, one thread per (env, player, feature), from the CTA's previous-action tile in shared
//     memory: every env's N*D-run is contiguous in obs_out and each player's D-run in the trajectory store.
#include "env_common.cuh"
#include "render.cuh"

namespace marl {

struct MxCfgDev {
  const double* payoff;   // device copy of the table, A^N entries
  int N, A, G, D, ep_length, time_limit, state, obs_id, coop_reward, std_rew;
};

struct MxStateDev {
  int8_t* last_act;
  EpisodeStateDev ep;
};

constexpr int kMxThreads = 128;

// Feature d of player `agent`'s observation; last: the env's previous actions (-1: none).  ObserveID's one-hot id comes first, then the
// concatenated one-hot of every player's previous action (or the one constant 0 of the -nostate ids).
__device__ __forceinline__ float mx_obs(const MxCfgDev& c, const int* last, int agent, int d) {
  if (c.obs_id) {
    if (d < c.N) return d == agent ? 1.f : 0.f;
    d -= c.N;
  }
  if (!c.state) return 0.f;
  const int j = d / c.A;
  return last[j] == d - j * c.A ? 1.f : 0.f;
}

// ---- reset / state kernels: one thread per env (rare) ------------------------------------------------------------
__global__ void matrix_reset_kernel(MxCfgDev c, MxStateDev s, int E, const uint8_t* mask, float* obs_out, TrajView traj, int slot0) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const bool doit = (mask == nullptr) || mask[e];
  int last[MARL_MAX_AGENTS];
  if (doit) (void)begin_episode(s.ep, e, c.N);   // MatrixGame.reset draws nothing
  for (int i = 0; i < c.N; ++i) {
    if (doit) s.last_act[(size_t)e * c.N + i] = -1;
    last[i] = s.last_act[(size_t)e * c.N + i];
  }
  for (int i = 0; i < c.N; ++i)
    for (int d = 0; d < c.D; ++d) {
      const float v = mx_obs(c, last, i, d);
      if (obs_out) obs_out[((size_t)e * c.N + i) * c.D + d] = v;
      if (traj.obs && doit) traj.obs_row((slot0 + e) % traj.capacity, i, 0)[d] = v;
    }
}

__global__ void matrix_set_state_kernel(MxCfgDev c, MxStateDev s, int E, const int8_t* last_act, const int32_t* step) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  for (int i = 0; i < c.N; ++i) s.last_act[(size_t)e * c.N + i] = last_act[(size_t)e * c.N + i];
  restart_episode(s.ep, e, c.N, step[e]);
}

__global__ void matrix_get_state_kernel(MxCfgDev c, MxStateDev s, int E, int8_t* last_act, int32_t* step, float* ep_return, int32_t* ep_len,
                                        uint32_t* episode_idx, uint8_t* active) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  if (last_act) for (int i = 0; i < c.N; ++i) last_act[(size_t)e * c.N + i] = s.last_act[(size_t)e * c.N + i];
  copy_episode(s.ep, e, c.N, step, ep_return, ep_len, episode_idx, active);
}

// ---- the transition kernel ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMxThreads) matrix_step_kernel(MxCfgDev c, MxStateDev s, StepArgs a, TrajView traj) {
  // act_s[le * G + sub] == act_s[threadIdx.x]: player sub's previous action after this step; slot_s / row_s: env le's trajectory slot
  // (-1: no write) and the observation row it fills; flag_s[threadIdx.x]: the lane's active | done << 1 | finished << 2 across the reward
  // wrappers (their division slow paths are calls, and in a register ptxas spilled one of the flags around them)
  __shared__ int act_s[kMxThreads], slot_s[kMxThreads], row_s[kMxThreads], flag_s[kMxThreads];
  const int G = c.G, EPW = 32 / G, EPC = (kMxThreads / 32) * EPW;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int le = warp * EPW + lane / G, sub = lane % G, gbase = (lane / G) * G;
  const int e0 = blockIdx.x * EPC, e = e0 + le;
  const int n_here = min(EPC, a.E - e0);
  constexpr uint32_t FULL = 0xFFFFFFFFu;

  const bool env_ok = e < a.E;
  const bool agent = env_ok && sub < c.N;
  const int step0 = env_ok ? s.ep.step[e] : 0;
  const bool active = env_ok && s.ep.active[e];
  const bool alive = active && sub < c.N;
  const uint32_t gid = a.gid0 + (uint32_t)e;
  const uint32_t ep_cur = env_ok ? episode_key(s.ep, e) : 0u;
  const int last0 = agent ? (int)s.last_act[(size_t)e * c.N + sub] : -1;

  // ---- action selection -------------------------------------------------------------------------------
  int a_raw = 0;
  if (alive) {
    if (a.policy == 0) a_raw = a.actions[(size_t)e * c.N + sub];
    else if (a.policy == 1) a_raw = select_eps_greedy(a, gid, ep_cur, step0, e, c.N, sub);
    else a_raw = select_categorical(a, gid, ep_cur, step0, e, c.N, sub);
  }
  if (a.actions_out && agent) a.actions_out[(size_t)e * c.N + sub] = a_raw;
  const int act = (a_raw >= 0 && a_raw < c.A) ? a_raw : 0;

  // ---- payoff[a_0, ..., a_{N-1}]: C-order index summed over the group ----------------------------------------
  int stride = 1;
  for (int i = sub + 1; i < c.N; ++i) stride *= c.A;
  int idx = alive ? act * stride : 0;
  for (int off = 1; off < G; off <<= 1) idx += __shfl_xor_sync(FULL, idx, off);
  const double rew = alive ? __ldg(c.payoff + idx) : 0.0;

  // ---- termination, RecordEpisodeStatistics and the new state: the action just played, or none after an in-kernel reset; a frozen env
  // keeps its own.  (Nothing here depends on the wrapped reward: it is done before the wrappers, which leaves less live across them.) ------
  const int step1 = step0 + 1;
  const bool done = active && step1 >= c.ep_length;
  const bool trunc = truncated(active, c.time_limit, step1);
  const bool finished = done || trunc;
  const int last1 = !alive ? last0 : ((finished && a.autoreset) ? -1 : act);
  store_return(s.ep, a, e, c.N, sub, alive, finished, add_return(s.ep, a, e, c.N, sub, alive, finished, rew));
  if (alive) s.last_act[(size_t)e * c.N + sub] = (int8_t)last1;
  act_s[threadIdx.x] = last1;
  flag_s[threadIdx.x] = (int)active | (int)done << 1 | (int)finished << 2;
  if (env_ok && sub == 0) {   // every lane of the group read step / ep_len / episode_idx before the shuffles above
    end_step(s.ep, a, e, active, step1, done, trunc, [](uint32_t) {});   // the new episode's previous actions are the lanes' last1
    row_s[le] = step1;
  }

  // ---- reward wrappers, trajectory scalars ------------------------------------------------------------------------------------------
  const float rew_f = wrap_reward(s.ep, a, e, env_ok, c.N, sub, gbase, alive, c.std_rew, c.coop_reward, rew);
  const int fl = flag_s[threadIdx.x];
  const int slot = (traj.obs && env_ok) ? traj_write_scalars(traj, a, e, c.N, sub, fl & 1, step0, a_raw, rew_f, (fl >> 1) & 1, (fl >> 2) & 1) : -1;
  if (env_ok && sub == 0) slot_s[le] = slot;
  __syncthreads();

  // ---- observations: one thread per (env, player, feature) of the CTA's envs, contiguous stores ---------------------------------
  const int per_env = c.N * c.D;
  for (int i = threadIdx.x; i < n_here * per_env; i += kMxThreads) {
    const int l = i / per_env, rem = i - l * per_env, ag = rem / c.D, d = rem - ag * c.D;
    const float v = mx_obs(c, act_s + l * G, ag, d);
    if (a.obs_out) a.obs_out[(size_t)e0 * per_env + i] = v;
    const int sl = slot_s[l];
    if (sl >= 0) traj.obs_row(sl, ag, row_s[l])[d] = v;
  }
}

// ---- frames (DESIGN.md §4.8, §4.9): an N x A board, one CTA per (env, band of pixel rows) ------------------------------------------
// Row i is player i, column k action k; the cell of each player's previous action is filled.
__device__ __forceinline__ render::Rgb matrix_pixel(const int* last, int x, int y) {
  using namespace render;
  constexpr int P = kMxCell + 1;
  if (x % P == 0 || y % P == 0) return kBlack;
  return last[y / P] == x / P ? kMxChosen : kWhite;
}

// frames: [n][H][W][3], frame l of env env_first + l
__global__ void __launch_bounds__(render::kRenderThreads) matrix_render_kernel(MxCfgDev c, MxStateDev s, int env_first, uint8_t* frames, int H, int W) {
  __shared__ __align__(16) uint8_t band_s[render::kBandBytes + 16];
  __shared__ int last_s[MARL_MAX_AGENTS];
  const int l = blockIdx.x;
  const size_t e = (size_t)env_first + l;
  for (int i = threadIdx.x; i < c.N; i += blockDim.x) last_s[i] = s.last_act[e * c.N + i];
  __syncthreads();
  const int rows = render::band_rows(W), y0 = blockIdx.y * rows, y1 = min(H, y0 + rows);
  render::render_band(frames + (size_t)l * H * W * 3, W, y0, y1, band_s, [&](int x, int y) { return matrix_pixel(last_s, x, y); });
}

}  // namespace marl

// =============================================================================================================
// C ABI
// =============================================================================================================
using namespace marl;

struct marl_matrix : EnvHandle {
  marl_matrix_cfg cfg;   // cfg.payoff is the caller's pointer: read in create only
  MxCfgDev dev;
  MxStateDev st;
  double* payoff;
};

constexpr int kMxMaxActions = 8, kMxMaxEntries = 65536;

// A^N, or -1 above kMxMaxEntries
static long long matrix_entries(int N, int A) {
  long long n = 1;
  for (int i = 0; i < N && n <= kMxMaxEntries; ++i) n *= A;
  return n <= kMxMaxEntries ? n : -1;
}

static int matrix_validate(const marl_matrix_cfg* c) {
  MARL_REQUIRE(c != nullptr, "marl_matrix: cfg is NULL");
  MARL_REQUIRE(c->n_agents >= 1 && c->n_agents <= MARL_MAX_AGENTS, "marl_matrix: n_agents %d out of range (1..%d)", c->n_agents, MARL_MAX_AGENTS);
  MARL_REQUIRE(c->n_actions >= 1 && c->n_actions <= kMxMaxActions, "marl_matrix: n_actions %d out of range (1..%d)", c->n_actions, kMxMaxActions);
  MARL_REQUIRE(matrix_entries(c->n_agents, c->n_actions) > 0, "marl_matrix: %d players with %d actions exceed %d payoff entries", c->n_agents,
               c->n_actions, kMxMaxEntries);
  MARL_REQUIRE(c->payoff != nullptr, "marl_matrix: payoff is NULL");
  MARL_REQUIRE(c->ep_length >= 1, "marl_matrix: ep_length must be >= 1");
  MARL_REQUIRE(c->time_limit >= 0, "marl_matrix: negative time_limit");
  return MARL_OK;
}

extern "C" {

int marl_matrix_obs_dim(const marl_matrix_cfg* cfg) {
  if (!cfg) return MARL_EINVAL;
  return (cfg->last_action_state ? cfg->n_agents * cfg->n_actions : 1) + (cfg->observe_id ? cfg->n_agents : 0);
}

int marl_matrix_create(const marl_matrix_cfg* cfg, int32_t n_envs, uint64_t seed, uint32_t env_gid0, int32_t device, marl_matrix** out) {
  MARL_REQUIRE(out != nullptr, "marl_matrix_create: out is NULL");
  *out = nullptr;
  if (int rc = matrix_validate(cfg)) return rc;
  MARL_REQUIRE(n_envs >= 1, "marl_matrix_create: n_envs must be >= 1");
  if (int rc = check_device(device)) return rc;
  marl_matrix* h = new marl_matrix();
  h->cfg = *cfg; h->cfg.payoff = nullptr; h->E = n_envs; h->device = device; h->seed = seed; h->gid0 = env_gid0;
  MxCfgDev& d = h->dev;
  d.N = cfg->n_agents; d.A = cfg->n_actions; d.ep_length = cfg->ep_length; d.time_limit = cfg->time_limit; d.state = cfg->last_action_state ? 1 : 0;
  d.obs_id = cfg->observe_id ? 1 : 0; d.coop_reward = cfg->cooperative_reward ? 1 : 0; d.std_rew = cfg->standardise_rewards ? 1 : 0;
  d.D = marl_matrix_obs_dim(cfg);
  int g = 1; while (g < d.N) g <<= 1;
  d.G = g;
  const size_t E = (size_t)n_envs, n_entries = (size_t)matrix_entries(d.N, d.A);
  h->envs_per_cta = (kMxThreads / 32) * (32 / g); h->threads = kMxThreads; h->step_smem = 0;
  int rc = alloc_buffers(h, "marl_matrix_create", {{&h->payoff, n_entries * sizeof(double)}, {&h->st.last_act, E * d.N}});
  if (rc == MARL_OK) rc = alloc_episode_state(h, "marl_matrix_create", h->st.ep, E, d.N);
  if (rc == MARL_OK) {
    cudaError_t err = cudaMemcpy(h->payoff, cfg->payoff, n_entries * sizeof(double), cudaMemcpyHostToDevice);
    if (err == cudaSuccess) err = cudaMemset(h->st.last_act, 0xFF, E * d.N);   // -1: no previous action, as after a reset
    if (err != cudaSuccess) { set_error("marl_matrix_create: %s", cudaGetErrorString(err)); rc = MARL_ECUDA; }
  }
  if (rc != MARL_OK) { marl_matrix_destroy(h); return rc; }
  d.payoff = h->payoff;
  *out = h;
  return MARL_OK;
}

int marl_matrix_destroy(marl_matrix* h) { return destroy_handle(h); }

int marl_matrix_set_state(marl_matrix* h, const int8_t* last_action, const int32_t* step, void* stream) {
  MARL_REQUIRE(h && last_action && step, "marl_matrix_set_state: NULL argument");
  return launch_per_env(h, matrix_set_state_kernel, stream, last_action, step);
}

int marl_matrix_get_state(marl_matrix* h, int8_t* last_action, int32_t* step, float* ep_return, int32_t* ep_len, uint32_t* episode_idx,
                          uint8_t* active, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_matrix_get_state: NULL handle");
  return launch_per_env(h, matrix_get_state_kernel, stream, last_action, step, ep_return, ep_len, episode_idx, active);
}

int marl_matrix_reset(marl_matrix* h, const uint8_t* reset_mask, float* obs_out, const marl_traj_view* traj, int32_t slot0, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_matrix_reset: NULL handle");
  if (int rc = check_traj(h, traj)) return rc;
  return launch_per_env(h, matrix_reset_kernel, stream, reset_mask, obs_out, traj_view(traj), slot0);
}

int marl_matrix_step(marl_matrix* h, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out, uint8_t* trunc_out,
                     float* final_ret_out, int32_t* final_len_out, int32_t autoreset, void* stream) {
  MARL_REQUIRE(h && actions && rew_out && done_out && trunc_out, "marl_matrix_step: NULL argument");
  const StepArgs a = step_args(h, actions, obs_out, rew_out, done_out, trunc_out, final_ret_out, final_len_out, autoreset);
  return launch_step(h, matrix_step_kernel, a, nullptr, stream);
}

int marl_matrix_rollout_step(marl_matrix* h, const float* values, const marl_rollout_args* ra, const marl_traj_view* traj, float* obs_inout,
                             float* rew_out, uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out,
                             int32_t* actions_out, void* stream) {
  MARL_REQUIRE(h && values && ra && rew_out && done_out && trunc_out, "marl_matrix_rollout_step: NULL argument");
  MARL_REQUIRE(ra->policy == 1 || ra->policy == 2, "marl_matrix_rollout_step: policy must be 1 (eps-greedy) or 2 (categorical)");
  MARL_REQUIRE(ra->n_actions == h->dev.A, "marl_matrix_rollout_step: n_actions %d does not match the game's %d actions", ra->n_actions, h->dev.A);
  StepArgs a;
  if (int rc = rollout_step_args(h, "marl_matrix_rollout_step", values, ra, traj, obs_inout, rew_out, done_out, trunc_out, final_ret_out,
                                 final_len_out, actions_out, a))
    return rc;
  return launch_step(h, matrix_step_kernel, a, traj, stream);
}

int marl_matrix_frame_shape(const marl_matrix_cfg* cfg, int32_t* h, int32_t* w) {
  MARL_REQUIRE(cfg && h && w, "marl_matrix_frame_shape: NULL argument");
  if (int rc = matrix_validate(cfg)) return rc;
  *h = render::frame_side(cfg->n_agents, render::kMxCell); *w = render::frame_side(cfg->n_actions, render::kMxCell);
  return MARL_OK;
}

int marl_matrix_render(marl_matrix* h, int32_t env_first, int32_t n, uint8_t* frames, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_matrix_render: NULL handle");
  return render::launch_render(h, "marl_matrix_render", matrix_render_kernel, env_first, n, frames, render::frame_side(h->dev.N, render::kMxCell),
                               render::frame_side(h->dev.A, render::kMxCell), stream);
}

}  // extern "C"
