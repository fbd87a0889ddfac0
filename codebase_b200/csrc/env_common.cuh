// env_common.cuh -- the parts of an env-step kernel that do not depend on the environment (sm_90a): the episode record with its reset,
// step and autoreset rules (TimeLimit, RecordEpisodeStatistics), the fused action selection (epsilon-greedy, categorical), marlbase's
// StandardiseReward and CooperativeReward wrappers and the trajectory-store writes; and on the host, the handle, trajectory checks and the
// launches of the env C ABIs.
// Included by lbf_env.cu, rware_env.cu and matrix_env.cu.  Lanes of one env form a group of G consecutive lanes starting at `gbase`; `sub` is
// the agent.
#pragma once
#include <string.h>
#include "traj.cuh"

namespace marl {

// The episode record of every env kind, one array per field: step[E] (TimeLimit's elapsed steps), ep_return[E][N] and ep_len[E]
// (RecordEpisodeStatistics), episode_idx[E] (resets performed so far: the running episode is episode_idx - 1, the key of its Philox streams),
// active[E] (0 once an episode ended without autoreset), and the StandardiseReward state, which survives resets.
struct EpisodeStateDev {
  int32_t* step; float* ep_return; int32_t* ep_len; uint32_t* episode_idx; uint8_t* active;
  float* stdr;       // per env: wmean[N] | t[N] | sumw (float32 like the wrapper's numpy arrays)
  int32_t* stdr_n;   // [E] number of rewards seen
};

struct StepArgs {
  int E; uint64_t seed; uint32_t gid0;
  int policy;  // 0 explicit actions, 1 eps-greedy over values, 2 categorical over logits
  const int32_t* actions; const float* values; float epsilon; int n_actions;
  float* obs_out; float* rew_out; uint8_t* done_out; uint8_t* trunc_out; float* final_ret; int32_t* final_len;
  int32_t* actions_out;
  int autoreset, use_proper_termination, clear_stale, slot0;
};

// Sequential 32-bit draws of one (seed, env, episode) reset: draw i = word i % 4 of Philox block (env_gid, episode, i / 4, 0)
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

// dqn/model.py:105-115: one uniform per step decides the joint exploration
__device__ __forceinline__ int select_eps_greedy(const StepArgs& a, uint32_t gid, uint32_t ep_cur, int step0, int e, int N, int sub) {
  const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32) ^ kTagAct;
  const u32x4 b0 = philox4x32_10(gid, ep_cur, (uint32_t)step0, 0u, k0, k1);
  const float* q = a.values + ((size_t)e * N + sub) * a.n_actions;
  int a_raw = 0;
  if (a.epsilon > u01(b0.x)) {
    const u32x4 bj = philox4x32_10(gid, ep_cur, (uint32_t)step0, 1u + (uint32_t)(sub >> 2), k0, k1);
    a_raw = (int)bounded(pick(bj, sub & 3), (uint32_t)a.n_actions);
  } else {
    float best = q[0];
    for (int k = 1; k < a.n_actions; ++k) { const float v = q[k]; if (v > best) { best = v; a_raw = k; } }
  }
  return a_raw;
}

// ac/model.py:150-152: Categorical(logits).sample() by inverse CDF on a Philox uniform
__device__ __forceinline__ int select_categorical(const StepArgs& a, uint32_t gid, uint32_t ep_cur, int step0, int e, int N, int sub) {
  const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32) ^ kTagCat;
  const u32x4 bj = philox4x32_10(gid, ep_cur, (uint32_t)step0, (uint32_t)(sub >> 2), k0, k1);
  const float u = u01(pick(bj, sub & 3));
  const float* lg = a.values + ((size_t)e * N + sub) * a.n_actions;
  float m = lg[0];
  for (int k = 1; k < a.n_actions; ++k) m = fmaxf(m, lg[k]);
  float tot = 0.f;
  for (int k = 0; k < a.n_actions; ++k) tot += expf(lg[k] - m);
  const float thresh = u * tot;
  float cum = 0.f;
  int a_raw = a.n_actions - 1;
  for (int k = 0; k < a.n_actions; ++k) { cum += expf(lg[k] - m); if (thresh < cum) { a_raw = k; break; } }
  return a_raw;
}

// StandardiseReward.reward (wrappers.py:119-141), the wrapper's numpy arithmetic: float32 state arrays, float64 where the python-float reward list
// enters (q, r, the standardised reward), float32 for the variance.  RecordEpisodeStatistics sits inside it and keeps the raw reward.
// st: the env's state wmean[N] | t[N] | sumw; n: its reward count.  Every lane of the warp calls it (it has a __syncwarp).
__device__ __forceinline__ double standardise_reward(float* st, int32_t* n_ptr, int N, int sub, bool alive, double rew) {
  double rew_w = rew;
  float wmean = 0.f, tt = 0.f, sumw = 0.f; int n = 0;
  if (alive) { wmean = st[sub]; tt = st[N + sub]; sumw = st[2 * N]; n = *n_ptr; }
  __syncwarp();   // every agent lane has read sumw / n before lane 0 of the env writes them
  if (alive) {
    const double q = __dsub_rn(rew, (double)wmean);                                        // (no FMA contraction: numpy rounds every operation)
    const float temp_sumw = __fadd_rn(sumw, 1.0f);
    const double r = __ddiv_rn(q, (double)temp_sumw);
    wmean = (float)__dadd_rn((double)wmean, r);
    tt = (float)__dadd_rn((double)tt, __dmul_rn(__dmul_rn(q, r), (double)sumw));
    n += 1;
    st[sub] = wmean; st[N + sub] = tt;
    if (sub == 0) { st[2 * N] = temp_sumw; *n_ptr = n; }
    if (n > 1) {
      const float var = __fdiv_rn(__fmul_rn(tt, (float)n), __fmul_rn(temp_sumw, (float)(n - 1)));
      rew_w = __ddiv_rn(__dsub_rn(rew, (double)wmean), (double)__fadd_rn(__fsqrt_rn(var), 1e-6f));
    }
  }
  return rew_w;
}

// CooperativeReward: python sum() over agents in index order
__device__ __forceinline__ double cooperative_sum(double rew_w, int gbase, int N) {
  double tot = 0.0;
  for (int i = 0; i < N; ++i) {
    const double ri = __shfl_sync(0xFFFFFFFFu, rew_w, gbase + i);
    tot += ri;
  }
  return tot;
}

// ---- the episode record: every env kernel changes it through these -----------------------------------------------------------------------
// Reset of env e (one thread per env): returns the index of the new episode, the key of the env's reset draws, and starts the record on it.
__device__ __forceinline__ uint32_t begin_episode(const EpisodeStateDev& s, int e, int N) {
  const uint32_t ep = s.episode_idx[e];
  s.episode_idx[e] = ep + 1;
  s.step[e] = 0; s.ep_len[e] = 0; s.active[e] = 1;
  for (int i = 0; i < N; ++i) s.ep_return[(size_t)e * N + i] = 0.f;
  return ep;
}

// set_state of env e: an episode continued from an injected state at `step`, keyed as the first episode when no reset has happened yet
__device__ __forceinline__ void restart_episode(const EpisodeStateDev& s, int e, int N, int32_t step) {
  s.step[e] = step; s.ep_len[e] = 0; s.active[e] = 1;
  for (int i = 0; i < N; ++i) s.ep_return[(size_t)e * N + i] = 0.f;
  if (s.episode_idx[e] == 0) s.episode_idx[e] = 1;
}

// get_state of env e: the record's fields into the outputs that are not NULL
__device__ __forceinline__ void copy_episode(const EpisodeStateDev& s, int e, int N, int32_t* step, float* ep_return, int32_t* ep_len,
                                             uint32_t* episode_idx, uint8_t* active) {
  if (step) step[e] = s.step[e];
  if (ep_return) for (int i = 0; i < N; ++i) ep_return[(size_t)e * N + i] = s.ep_return[(size_t)e * N + i];
  if (ep_len) ep_len[e] = s.ep_len[e];
  if (episode_idx) episode_idx[e] = s.episode_idx[e];
  if (active) active[e] = s.active[e];
}

// The running episode of env e: the key of its action and transition draws
__device__ __forceinline__ uint32_t episode_key(const EpisodeStateDev& s, int e) { return s.episode_idx[e] - 1u; }

// TimeLimit (envs.py:95-96): an active episode is truncated once it has run `time_limit` steps (0: no limit)
__device__ __forceinline__ bool truncated(bool active, int time_limit, int step1) { return active && (time_limit > 0 && step1 >= time_limit); }

// RecordEpisodeStatistics of agent `sub` of env e (alive: the env is active and the lane is an agent), in two calls so that a kernel stores
// the return where its registers allow (right after the accumulation, lbf_step_kernel<true> spills 16 B more).  add_return: the float32
// accumulation of the raw reward (wrappers.py:33), and final_ret when the episode ended.  store_return: the running return, which an
// autoreset restarts at 0.
__device__ __forceinline__ float add_return(const EpisodeStateDev& s, const StepArgs& a, int e, int N, int sub, bool alive, bool finished, double rew) {
  if (!alive) return 0.f;
  const float ep_ret = s.ep_return[(size_t)e * N + sub] + (float)rew;
  if (finished && a.final_ret) a.final_ret[(size_t)e * N + sub] = ep_ret;
  return ep_ret;
}

__device__ __forceinline__ void store_return(const EpisodeStateDev& s, const StepArgs& a, int e, int N, int sub, bool alive, bool finished,
                                             float ep_ret) {
  if (alive) s.ep_return[(size_t)e * N + sub] = (finished && a.autoreset) ? 0.f : ep_ret;
}

// The reward wrappers over RecordEpisodeStatistics: StandardiseReward (std_rew), then CooperativeReward (coop: every agent gets the sum over
// the env), then rew_out (0 for the agents of a frozen env).  Returns the reward as written.  Every lane of the warp calls it (see
// standardise_reward and cooperative_sum); env_ok: the lane's env exists.
__device__ __forceinline__ float wrap_reward(const EpisodeStateDev& s, const StepArgs& a, int e, bool env_ok, int N, int sub, int gbase, bool alive,
                                             int std_rew, int coop, double rew) {
  double rew_w = rew;
  if (std_rew) rew_w = standardise_reward(s.stdr + (size_t)(env_ok ? e : 0) * (2 * N + 1), s.stdr_n + (env_ok ? e : 0), N, sub, alive, rew);
  const double tot = cooperative_sum(rew_w, gbase, N);
  const float rew_f = (float)(coop ? tot : rew_w);
  if (env_ok && sub < N) a.rew_out[(size_t)e * N + sub] = alive ? rew_f : 0.f;
  return rew_f;
}

// End of the step of env e, on one lane of the env: step and ep_len, final_len when the episode ended, then either the autoreset --
// new_episode(ep) resets the env's own state for episode ep -- or a frozen env; then done_out (1 for a frozen env) and trunc_out.
template <typename NewEpisode>
__device__ __forceinline__ void end_step(const EpisodeStateDev& s, const StepArgs& a, int e, bool active, int step1, bool done, bool trunc,
                                         const NewEpisode& new_episode) {
  if (active) {
    s.step[e] = step1;
    const int len1 = s.ep_len[e] + 1;
    s.ep_len[e] = len1;
    if (done || trunc) {
      if (a.final_len) a.final_len[e] = len1;
      if (a.autoreset) {
        const uint32_t ep = s.episode_idx[e];
        new_episode(ep);
        s.episode_idx[e] = ep + 1;
        s.step[e] = 0; s.ep_len[e] = 0;
      } else {
        s.active[e] = 0;
      }
    }
  }
  a.done_out[e] = active ? (uint8_t)done : (uint8_t)1;
  a.trunc_out[e] = (uint8_t)trunc;
}

// trajectory scalars (rb.add, dqn/train.py:73-89; batch_* writes, ac/train.py:90-99) of env e.  Returns the slot whose observation row
// step1 this step fills, -1 for none.
__device__ __forceinline__ int traj_write_scalars(const TrajView& traj, const StepArgs& a, int e, int N, int sub, bool active, int step0, int a_raw,
                                                  float rew_f, bool done, bool finished) {
  int slot = -1;
  const int step1 = step0 + 1;
  const int sl = (a.slot0 + e) % traj.capacity;
  if (active && step0 < traj.T) {
    slot = sl;
    if (sub < N) {
      traj.act[traj.step_at(sl, sub, step0)] = a_raw;
      traj.rew[traj.step_at(sl, sub, step0)] = rew_f;
    }
    if (sub == 0) {
      traj.done[traj.done_at(sl, step1)] = (uint8_t)(a.use_proper_termination ? done : finished);
      traj.filled[traj.filled_at(sl, step0)] = 1;
    }
  } else if (!active && a.clear_stale && sub == 0 && step0 < traj.T) {
    // steps after the episode ended: the reference leaves a reused slot's old tail in place (SURVEY H6)
    for (int t = step0; t < traj.T; ++t) traj.filled[traj.filled_at(sl, t)] = 0;
  }
  return slot;
}

// ---- host side: the handle layer of the env C ABIs ----------------------------------------------------------------------------------------
// A handle (marl_lbf, marl_rware, marl_matrix) derives from EnvHandle and adds its config `cfg`, device config `dev` (with N and D) and state
// pointers `st`, whose episode record is `st.ep`.  Its device buffers come from alloc_buffers and are released by destroy_handle.
struct EnvHandle : BufferOwner {
  int E, device;
  uint64_t seed;
  uint32_t gid0;
  int envs_per_cta, threads;   // step kernel launch shape
  size_t step_smem;
};

// The zero-filled episode record of E envs of N agents
inline int alloc_episode_state(BufferOwner* h, const char* who, EpisodeStateDev& s, size_t E, int N) {
  return alloc_buffers(h, who, {{&s.step, E * 4}, {&s.ep_return, E * N * 4}, {&s.ep_len, E * 4}, {&s.episode_idx, E * 4}, {&s.active, E},
                                {&s.stdr, E * (2 * N + 1) * 4}, {&s.stdr_n, E * 4}});
}

// The attribute is a per-function, process-wide setting: only ever raise it (a second env with a smaller tile must not lower the limit of the
// first).  `limit` is the kernel's current limit, kept by the caller.  A refused size is reported through set_error only: nothing is left
// in the runtime's last error for a later, unrelated cudaGetLastError (another launch's check, torch's) to report.  Defensive: no config
// reaches the refusal today (marl_lbf_create checks its tile against the opt-in limit first, and RWARE's widest tile is about 207 KB).
template <typename K>
int raise_smem_limit(K* kernel, size_t bytes, size_t& limit, const char* who) {
  if (bytes <= limit) return MARL_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("%s: %zu B of shared memory per CTA not available: %s", who, bytes, cudaGetErrorString(e));
    return MARL_EINVAL;
  }
  limit = bytes;
  return MARL_OK;
}

template <typename H>
int check_traj(const H* env, const marl_traj_view* t) {
  if (!t) return MARL_OK;
  MARL_REQUIRE(t->obs && t->act && t->rew && t->done && t->filled, "traj view has NULL buffers");
  MARL_REQUIRE(t->n_agents == env->dev.N && t->obs_dim == env->dev.D, "traj view shape (N=%d, obs=%d) does not match env (N=%d, obs=%d)", t->n_agents, t->obs_dim, env->dev.N, env->dev.D);
  MARL_REQUIRE(t->capacity >= env->E && t->T >= 1, "traj capacity %d must hold one episode per env (%d)", t->capacity, env->E);
  return MARL_OK;
}

// StepArgs of a step on explicit actions (policy 0)
inline StepArgs step_args(const EnvHandle* h, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out, uint8_t* trunc_out,
                          float* final_ret_out, int32_t* final_len_out, int32_t autoreset) {
  StepArgs a; memset(&a, 0, sizeof(a));
  a.E = h->E; a.seed = h->seed; a.gid0 = h->gid0; a.policy = 0; a.actions = actions; a.obs_out = obs_out; a.rew_out = rew_out;
  a.done_out = done_out; a.trunc_out = trunc_out; a.final_ret = final_ret_out; a.final_len = final_len_out; a.autoreset = autoreset;
  return a;
}

// StepArgs of a rollout step, after the checks every env shares.  The caller has checked its pointers and the policy.
template <typename H>
int rollout_step_args(const H* h, const char* who, const float* values, const marl_rollout_args* ra, const marl_traj_view* traj, float* obs_inout,
                      float* rew_out, uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out, int32_t* actions_out,
                      StepArgs& a) {
  MARL_REQUIRE(ra->n_actions >= 1 && ra->n_actions <= 64, "%s: n_actions out of range", who);
  if (int rc = check_traj(h, traj)) return rc;
  MARL_REQUIRE(!(traj && ra->autoreset), "%s: trajectory recording needs autoreset=0 (episode-synchronous collection)", who);
  a = step_args(h, nullptr, obs_inout, rew_out, done_out, trunc_out, final_ret_out, final_len_out, ra->autoreset);
  a.policy = ra->policy; a.values = values; a.epsilon = ra->epsilon; a.n_actions = ra->n_actions; a.actions_out = actions_out;
  a.use_proper_termination = ra->use_proper_termination; a.clear_stale = ra->clear_stale; a.slot0 = ra->slot0;
  return MARL_OK;
}

template <typename H, typename Dev, typename St>
int launch_step(const H* h, void (*kernel)(Dev, St, StepArgs, TrajView), const StepArgs& a, const marl_traj_view* traj, void* stream) {
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  kernel<<<(h->E + h->envs_per_cta - 1) / h->envs_per_cta, h->threads, h->step_smem, (cudaStream_t)stream>>>(h->dev, h->st, a, traj_view(traj));
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

// The reset, set_state and get_state kernels: one thread per env, kernel(h->dev, h->st, h->E, args...)
template <typename H, typename... KArgs, typename... Args>
int launch_per_env(const H* h, void (*kernel)(KArgs...), void* stream, Args... args) {
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  kernel<<<(h->E + 127) / 128, 128, 0, (cudaStream_t)stream>>>(h->dev, h->st, h->E, args...);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

}  // namespace marl
