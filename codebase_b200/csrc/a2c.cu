// a2c.cu -- C ABI of the independent actor-critic learner (marl_a2c_*), host-side orchestration of the fused kernels.
//
// Replaces marlbase/ac/model.py A2CNetwork (22-246): act's actor forward (147-153), get_value (155-163),
// update (189-246: target-critic pass, compute_nstep_returns utils/utils.py:38-63, evaluate_actions 165-182,
// policy-gradient + entropy + value losses, Adam, target sync), for independent or shared per-agent networks with a
// decentralised critic (critic.centralised: False, configs/algorithm/ia2c.yaml:18).
//
// Recurrent parts (marl_a2c_create_rnn; actor.use_rnn / critic.use_rnn, utils/models.py:51-116): every pass runs each env's episode from h = 0
// (ac/model.py:189-246, 265-352 call the networks with hiddens=None) through gru_forward; a trained part then runs the sequence loss head and the
// BPTT backward (gru_kernels.cu) into the same per-CTA partials and reduce + Adam tail as the MLP parts.
#include "gru.cuh"
#include "retms.cuh"
#include <math.h>

namespace marl {

constexpr int kMaxNStep = 64;

struct NStepParams {
  const float* vt;     // [N][P][T+1] target-critic values
  TrajView traj; const int32_t* idx; int N, P, n_steps;
  float gpow[kMaxNStep + 1];  // float32(gamma ** k), the Python-float powers of utils/utils.py:57-60
  float* ret;          // [N][P][T]
  const float* ret_ms; // standardise_returns (ac/model.py:195-196): [mean[N] | var[N]] of the running return statistics, or NULL
};

// compute_nstep_returns (utils/utils.py:38-63): G_t = sum_{k<n} g^k r_{t+k}(1-d_{t+k}) + g^n V(o_{t+n})(1-d_{t+n}), cut (no
// bootstrap) where t+k reaches the end of the stored episode; d_t = dones[t] is the terminal flag of observation t.
__global__ void nstep_returns_kernel(NStepParams p) {
  const int T = p.traj.T, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.N * p.P * T) return;
  const int a = i / (p.P * T), rem = i - a * p.P * T, b = rem / T, t = rem - b * T;
  const size_t ep = (size_t)p.idx[b];
  float acc = 0.f;
  for (int k = 0; k <= p.n_steps; ++k) {
    const int tt = t + k;
    if (tt >= T) break;
    const float d = (float)p.traj.done[p.traj.done_at(ep, tt)];
    float src;
    if (k == p.n_steps) {
      src = p.vt[row_index(a, b, tt, p.P, T + 1)];
      if (p.ret_ms) src = unstandardise(src, p.ret_ms[a], p.ret_ms[p.N + a]);
    } else {
      src = p.traj.rew[p.traj.step_at(ep, a, tt)];
    }
    acc += (p.gpow[k] * src) * (1.f - d);
  }
  p.ret[i] = acc;
}

// λ-returns (algorithm.gae_lambda): the mixture (1 - λ) Σ_{n>=1} λ^(n-1) G_t^(n) of the n-step returns above, by the backward recursion
//   R_t = a_t + b R_{t+1},  a_t = m_t r_t + γ(1 - λ) m_{t+1} V_{t+1},  b = γλ,  m_t = 1 - d_t,  R_T = 0 and m_T V_T taken as 0.
// One warp per (agent, env) sequence, right to left over windows of 32 x kLamChunk steps: the warp stages a_t coalesced into shared memory, each
// lane folds its kLamChunk-step chunk into the affine map R_in -> c + g R_in, a fixed-order suffix scan over the lanes composes the maps, each
// lane replays its chunk from the return after it, and the warp writes the returns coalesced.  The window's first return carries into the next.
constexpr int kLamChunk = 8, kLamWindow = 32 * kLamChunk, kLamWarps = 8;

struct LambdaParams {
  const float* vt;     // [N][P][T+1] target-critic values
  TrajView traj; const int32_t* idx; int N, P;
  float coef_v, coef_r;   // float32(γ(1 - λ)), float32(γλ)
  float* ret;          // [N][P][T]
  const float* ret_ms; // [mean[N] | var[N]] of the running return statistics, or NULL
};

__device__ __forceinline__ int lam_slot(int s) { return (s / kLamChunk) * (kLamChunk + 1) + s % kLamChunk; }   // lane chunks padded: no bank conflicts

__global__ void lambda_returns_kernel(LambdaParams p) {
  __shared__ float buf[kLamWarps][32 * (kLamChunk + 1)];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, seq = blockIdx.x * kLamWarps + w;
  if (seq >= p.N * p.P) return;
  const int T = p.traj.T, a = seq / p.P, b = seq - a * p.P;
  const size_t ep = (size_t)p.idx[b];
  const float* vt = p.vt + row_index(a, b, 0, p.P, T + 1);
  const float* rew = p.traj.rew + p.traj.step_at(ep, a, 0);
  const uint8_t* done = p.traj.done + p.traj.done_at(ep, 0);
  float* ret = p.ret + row_index(a, b, 0, p.P, T);
  const float mean = p.ret_ms ? p.ret_ms[a] : 0.f, var = p.ret_ms ? p.ret_ms[p.N + a] : 1.f;
  float* s = buf[w];
  float carry = 0.f;   // R at the step after the window
  for (int w0 = ((T - 1) / kLamWindow) * kLamWindow; w0 >= 0; w0 -= kLamWindow) {
    const int len = min(kLamWindow, T - w0);
    for (int j = lane; j < len; j += 32) {
      const int t = w0 + j;
      float av = 0.f;
      if (t + 1 < T) {
        float v = vt[t + 1];
        if (p.ret_ms) v = unstandardise(v, mean, var);
        av = (p.coef_v * v) * (1.f - (float)done[t + 1]);
      }
      s[lam_slot(j)] = rew[t] * (1.f - (float)done[t]) + av;
    }
    __syncwarp();
    const int lo = lane * kLamChunk, hi = min(lo + kLamChunk, len);
    float c = 0.f, g = 1.f;   // this lane's chunk: R_lo = c + g R_hi
    for (int j = hi - 1; j >= lo; --j) { c = s[lam_slot(j)] + p.coef_r * c; g *= p.coef_r; }
    // suffix scan: lane l ends with the composition of the maps of lanes l .. 31
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const float c2 = __shfl_down_sync(0xffffffffu, c, off), g2 = __shfl_down_sync(0xffffffffu, g, off);
      if (lane + off < 32) { c = c + g * c2; g *= g2; }
    }
    float r = __shfl_down_sync(0xffffffffu, c + g * carry, 1);   // R at the step after this lane's chunk
    if (lane == 31) r = carry;
    for (int j = hi - 1; j >= lo; --j) { r = s[lam_slot(j)] + p.coef_r * r; s[lam_slot(j)] = r; }
    carry = __shfl_sync(0xffffffffu, r, 0);   // R_{w0}, as written
    __syncwarp();
    for (int j = lane; j < len; j += 32) ret[w0 + j] = s[lam_slot(j)];
    __syncwarp();
  }
}

// log-probabilities of the taken actions under the collecting policy (ac/model.py:281-292), from the actor outputs of every gathered row:
// old_logp[a][b][t] = log_softmax(logits[a][b][t][:])[act[a][b][t]] -- the formulas of head_a2c_actor (learner_kernels.cu)
struct OldLogpParams { const float* logits; TrajView traj; const int32_t* idx; int N, P, A; float* out; };
__global__ void old_logp_kernel(OldLogpParams p) {
  const int T = p.traj.T, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.N * p.P * T) return;
  const int a = i / (p.P * T), rem = i - a * p.P * T, b = rem / T, t = rem - b * T;
  const float* q = p.logits + row_index(a, b, t, p.P, T + 1) * p.A;
  const int act = p.traj.act[p.traj.step_at(p.idx[b], a, t)];
  float m = q[0];
  for (int o = 1; o < p.A; ++o) m = fmaxf(m, q[o]);
  float s = 0.f;
  for (int o = 0; o < p.A; ++o) s += expf(q[o] - m);
  p.out[i] = q[act] - (m + logf(s));
}

// mean over the epochs of the six device metrics (ac/model.py:352)
__global__ void mean_metrics_kernel(const float* per_epoch, int n_epochs, float* out) {
  const int k = threadIdx.x;
  if (k >= 6) return;
  float s = 0.f;
  for (int e = 0; e < n_epochs; ++e) s += per_epoch[6 * e + k];
  out[k] = k == 4 ? per_epoch[4] : s / (float)n_epochs;   // [4] = filled count (the same every epoch)
}

// centralised critic (ac/model.py:62-65,156-157): the joint observation of every (env, step) = the agents' observations side by side
struct JointParams { TrajView traj; const int32_t* idx; int P; float* out; };   // out: [P][T+1][N * D]
__global__ void joint_obs_kernel(JointParams p) {
  const int T1 = p.traj.T + 1, ND = p.traj.N * p.traj.D;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)p.P * T1 * ND) return;
  const int c = (int)(i % ND), t = (int)((i / ND) % T1), b = (int)(i / ((size_t)ND * T1));
  const int j = c / p.traj.D, d = c - j * p.traj.D;
  p.out[i] = p.traj.obs_row(p.idx[b], j, t)[d];
}

__global__ void iota_kernel(int32_t* x, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = i;
}

}  // namespace marl

using namespace marl;

struct A2cPass { RowSource src, csrc; RowPlan cplan, aplan; int n_envs; };   // csrc: the critic's rows (== src unless the critic is centralised)

struct marl_a2c : LearnerHandle {
  NetSet actor, critic;
  marl_a2c_hp hp;
  int max_envs = 0, max_T = 0;
  int64_t n_actor = 0, n_critic = 0;
  float *vt = nullptr, *ret = nullptr, *adv = nullptr, *metrics = nullptr;
  int64_t opt_steps = 0;
  float *logits_all = nullptr, *old_logp = nullptr, *epoch_metrics = nullptr;   // PPO (allocated on first use)
  A2cPass ppo_pass = {}; bool ppo_prepared = false;   // PPO split into epochs: the batch's rows and plans from marl_ppo_prepare
  int centralised = 0; float* joint = nullptr;   // critic.centralised: joint observations of the batch [P][T+1][N * D]
  // recurrent parts: GRU layouts, the sequence outputs of the part being trained and their gradient [N][P][T+1][out], the online pass's saved rows
  // [N][P][T+1][kGruSaveRow] (one buffer: the critic pass ends before the actor pass starts)
  int actor_rnn = 0, critic_rnn = 0; GruLayout agl = {}, cgl = {};
  float *rnn_q = nullptr, *rnn_dq = nullptr, *gru_save = nullptr;
  int gae = 0; float gae_lambda = 0.f;   // algorithm.gae_lambda: λ-returns (lambda_returns_kernel) in place of the n-step returns
};
constexpr int kMaxPpoEpochs = 64;

extern "C" {

int marl_a2c_destroy(marl_a2c* h) { return destroy_handle(h); }

static int a2c_create(const marl_mlp_cfg* actor, const marl_mlp_cfg* critic, const marl_a2c_hp* hp, bool actor_rnn, bool critic_rnn, int32_t max_envs, int32_t max_T,
                      int32_t device, marl_a2c** out) {
  MARL_REQUIRE(hp && out, "marl_a2c_create: NULL argument");
  *out = nullptr;
  if (int rc = check_mlp_cfg(actor, "marl_a2c_create(actor)", kMaxInDim)) return rc;
  if (int rc = check_mlp_cfg(critic, "marl_a2c_create(critic)", kMaxInDim)) return rc;
  MARL_REQUIRE(actor->n_agents == critic->n_agents && (actor->in_dim == critic->in_dim || critic->in_dim == actor->n_agents * actor->in_dim),
               "marl_a2c_create: the critic's input width must be the actor's (%d) or, for a centralised critic, n_agents x it (%d)", actor->in_dim, actor->n_agents * actor->in_dim);
  MARL_REQUIRE(critic->out_dim == 1, "marl_a2c_create: the critic outputs one state value per agent");
  MARL_REQUIRE(max_envs >= 1 && max_T >= 1, "marl_a2c_create: max_envs/max_T must be >= 1");
  MARL_REQUIRE(hp->n_steps >= 1 && hp->n_steps <= kMaxNStep, "marl_a2c_create: n_steps %d out of range (1..%d)", hp->n_steps, kMaxNStep);
  marl_a2c* h = nullptr;
  if (int rc = open_learner(device, *hp, &h)) return rc;
  h->actor = to_netset(actor); h->critic = to_netset(critic);
  h->max_envs = max_envs; h->max_T = max_T;
  h->centralised = critic->in_dim != actor->in_dim ? 1 : 0;
  h->actor_rnn = actor_rnn ? 1 : 0; h->critic_rnn = critic_rnn ? 1 : 0;
  h->agl = GruLayout::make(actor->in_dim, actor->out_dim, actor->hidden); h->cgl = GruLayout::make(critic->in_dim, critic->out_dim, critic->hidden);
  const int pa = actor_rnn ? h->agl.P : h->actor.lay.P, pc = critic_rnn ? h->cgl.P : h->critic.lay.P;
  h->n_actor = (int64_t)actor->n_nets * pa; h->n_critic = (int64_t)critic->n_nets * pc; h->n_params = h->n_actor + h->n_critic;
  const int pmax = pa > pc ? pa : pc;
  h->scratch_pitch = (pmax + 3) & ~3;
  const size_t rows = (size_t)actor->n_agents * max_envs * (max_T + 1), F = sizeof(float);
  const bool rnn = actor_rnn || critic_rnn;
  // the loss statistics: one part per training CTA of an MLP part, one per head block of a recurrent part
  const size_t loss_parts = (size_t)h->n_sm + (rnn ? (size_t)gru_head_blocks(actor->n_agents, max_envs, max_T) : 0);
  const char* who = "marl_a2c_create";
  int rc = alloc_buffers(h, who, {{&h->theta, h->n_params * F}, {&h->theta_tgt, h->n_critic * F}, {&h->m, h->n_params * F}, {&h->v, h->n_params * F},
                                  {&h->grad, (h->n_params + 4) * F}, {&h->scratch, (size_t)h->n_sm * h->scratch_pitch * F}, {&h->loss_part, 4 * loss_parts * F},
                                  {&h->vt, rows * F}, {&h->ret, rows * F}, {&h->adv, rows * F}, {&h->metrics, 8 * F}, {&h->idx, max_envs * F}});
  if (!rc && actor->hidden == kHidden && critic->hidden == kHidden)   // the tensor-core images exist for 128-wide networks only (no image: the FP32 kernels)
    rc = alloc_buffers(h, who, {{&h->image, ((size_t)(actor->n_nets > critic->n_nets ? actor->n_nets : critic->n_nets) * tc_image_bytes() / 4 + 4) * F}});
  if (!rc && rnn) {
    const int out_max = actor_rnn ? actor->out_dim : 1;
    rc = alloc_buffers(h, who, {{&h->rnn_q, rows * out_max * F}, {&h->rnn_dq, rows * out_max * F}, {&h->gru_save, rows * kGruSaveRow * F}});
  }
  if (rc) { marl_a2c_destroy(h); return rc; }
  iota_kernel<<<(max_envs + 255) / 256, 256>>>(h->idx, max_envs);
  if (h->centralised) {
    if (int rc2 = alloc_buffers(h, who, {{&h->joint, (size_t)max_envs * (max_T + 1) * critic->in_dim * F}})) { marl_a2c_destroy(h); return rc2; }
  }
  if (int rc2 = learner_kernels_init(actor->in_dim, kMaxInDim)) { marl_a2c_destroy(h); return rc2; }
  if (int rc2 = learner_kernels_init(critic->in_dim, kMaxInDim)) { marl_a2c_destroy(h); return rc2; }
  if (int rc2 = tc_forward_init()) { marl_a2c_destroy(h); return rc2; }
  if (rnn) {
    if (int rc2 = gru_kernels_init()) { marl_a2c_destroy(h); return rc2; }
  }
  if (cudaDeviceSynchronize() != cudaSuccess) { set_error("marl_a2c_create: device error during setup"); marl_a2c_destroy(h); return MARL_ECUDA; }
  *out = h;
  return MARL_OK;
}

int marl_a2c_create(const marl_mlp_cfg* actor, const marl_mlp_cfg* critic, const marl_a2c_hp* hp, int32_t max_envs, int32_t max_T, int32_t device, marl_a2c** out) {
  return a2c_create(actor, critic, hp, false, false, max_envs, max_T, device, out);
}

int marl_a2c_create_rnn(const marl_mlp_cfg* actor, const marl_mlp_cfg* critic, const marl_a2c_hp* hp, int32_t actor_rnn, int32_t critic_rnn, int32_t max_envs,
                        int32_t max_T, int32_t device, marl_a2c** out) {
  return a2c_create(actor, critic, hp, actor_rnn != 0, critic_rnn != 0, max_envs, max_T, device, out);
}

/* theta = [actor nets | critic nets] (flat, reference state_dict order per net), theta_tgt = target critic. */
int marl_a2c_param_ptrs(marl_a2c* h, float** theta, float** theta_tgt, float** adam_m, float** adam_v, float** grad, int64_t* n_actor, int64_t* n_critic) {
  MARL_REQUIRE(h != nullptr, "marl_a2c_param_ptrs: NULL handle");
  if (theta) *theta = h->theta; if (theta_tgt) *theta_tgt = h->theta_tgt; if (adam_m) *adam_m = h->m; if (adam_v) *adam_v = h->v;
  if (grad) *grad = h->grad; if (n_actor) *n_actor = h->n_actor; if (n_critic) *n_critic = h->n_critic;
  return MARL_OK;
}

int marl_a2c_scratch_ptrs(marl_a2c* h, float** target_values, float** returns, float** advantages) {
  MARL_REQUIRE(h != nullptr, "marl_a2c_scratch_ptrs: NULL handle");
  if (target_values) *target_values = h->vt; if (returns) *returns = h->ret; if (advantages) *advantages = h->adv;
  return MARL_OK;
}

int marl_a2c_sync_target(marl_a2c* h, void* stream) {  // soft_update(1.0), ac/model.py:101
  MARL_REQUIRE(h != nullptr, "marl_a2c_sync_target: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  MARL_CUDA_TRY(cudaMemcpyAsync(h->theta_tgt, h->theta + h->n_actor, h->n_critic * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return MARL_OK;
}

static int a2c_dense_forward(marl_a2c* h, const NetSet& ns, const float* theta, const float* obs, int n_envs, float* out, void* stream) {
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  const RowPlan plan = make_plan(ns, n_envs, 1, h->n_sm, 32);
  const RowSource src = dense_rows(obs, n_envs, ns.n_agents, ns.in, ns.in != h->actor.in);   // (a centralised critic reads joint rows)
  return forward_any(ns, plan, src, theta, h->image, out, (cudaStream_t)stream);
}

/* actor forward of A2CNetwork.act (ac/model.py:148-150): obs float[E][N][in] -> logits float[E][N][n_actions] */
int marl_a2c_forward_actor(marl_a2c* h, const float* obs, int32_t n_envs, float* logits_out, void* stream) {
  MARL_REQUIRE(h && obs && logits_out && n_envs >= 1, "marl_a2c_forward_actor: bad argument");
  MARL_REQUIRE(!h->actor_rnn, "marl_a2c_forward_actor: the actor is recurrent: use marl_a2c_forward_rnn, which carries the hidden state");
  return a2c_dense_forward(h, h->actor, h->theta, obs, n_envs, logits_out, stream);
}

/* get_value (ac/model.py:155-163): values float[E][N][1] from the critic or the target critic */
int marl_a2c_forward_critic(marl_a2c* h, const float* obs, int32_t n_envs, int32_t use_target, float* values_out, void* stream) {
  MARL_REQUIRE(h && obs && values_out && n_envs >= 1, "marl_a2c_forward_critic: bad argument");
  MARL_REQUIRE(!h->critic_rnn, "marl_a2c_forward_critic: the critic is recurrent: use marl_a2c_forward_rnn, which carries the hidden state");
  return a2c_dense_forward(h, h->critic, use_target ? h->theta_tgt : h->theta + h->n_actor, obs, n_envs, values_out, stream);
}

/* one step of a recurrent part (ac/model.py:147-153 act, 155-163 get_value) carrying the hidden state; which: 0 actor, 1 critic, 2 target critic */
int marl_a2c_forward_rnn(marl_a2c* h, int32_t which, const float* obs, int32_t n_envs, const float* h_in, float* h_out, float* out, void* stream) {
  MARL_REQUIRE(h && obs && out && n_envs >= 1 && which >= 0 && which <= 2, "marl_a2c_forward_rnn: bad argument");
  const bool actor = which == 0;
  MARL_REQUIRE(actor ? h->actor_rnn : h->critic_rnn, "marl_a2c_forward_rnn: the %s is not recurrent: use marl_a2c_forward_%s", actor ? "actor" : "critic",
               actor ? "actor" : "critic");
  MARL_REQUIRE(h_in == nullptr || h_in != h_out, "marl_a2c_forward_rnn: h_in and h_out must not alias");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  const NetSet& ns = actor ? h->actor : h->critic;
  GruFwdParams fp; memset(&fp, 0, sizeof(fp));
  fp.plan = make_plan(ns, n_envs, 1, 1, 1);
  fp.src = dense_rows(obs, n_envs, ns.n_agents, ns.in, !actor && h->centralised);
  fp.theta = which == 0 ? h->theta : (which == 1 ? h->theta + h->n_actor : h->theta_tgt);
  fp.lay = actor ? h->agl : h->cgl;
  fp.h_in = h_in; fp.h_out = h_out; fp.q_out = out;
  return launch_gru_forward(fp, (cudaStream_t)stream);
}

// sequence forward of a recurrent part over every env's T + 1 steps from h = 0: outputs [N][P][T+1][out], saved rows for BPTT when `save`
static int a2c_gru_forward(const NetSet& ns, const GruLayout& gl, const RowSource& src, const float* theta, int n_envs, float* q_out, float* save, cudaStream_t st) {
  GruFwdParams fp; memset(&fp, 0, sizeof(fp));
  fp.plan = make_plan(ns, n_envs, src.traj.T + 1, 1, 1); fp.src = src;
  fp.theta = theta; fp.lay = gl; fp.q_out = q_out; fp.save = save;
  return launch_gru_forward(fp, st);
}

// target-critic pass + n-step returns (ac/model.py:190-201): everything of an update that does not depend on the trainable parameters
static int a2c_prepare(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, cudaStream_t st, A2cPass& ps) {
  MARL_REQUIRE(h && batch, "marl_a2c_update: NULL argument");
  MARL_REQUIRE(n_envs >= 1 && n_envs <= h->max_envs && n_envs <= batch->capacity, "marl_a2c_update: n_envs %d out of range", n_envs);
  MARL_REQUIRE(batch->T >= 1 && batch->T <= h->max_T, "marl_a2c_update: T %d exceeds max_T %d", batch->T, h->max_T);
  MARL_REQUIRE(batch->n_agents == h->actor.n_agents && batch->obs_dim == h->actor.in, "marl_a2c_update: batch shape mismatch");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  const int T = batch->T, N = h->actor.n_agents;
  ps.n_envs = n_envs;
  ps.src = episode_rows(batch, h->idx, N, h->actor.in);
  ps.cplan = episode_plan(h->critic, n_envs, T, h->n_sm);
  ps.aplan = episode_plan(h->actor, n_envs, T, h->n_sm);
  ps.csrc = ps.src;
  if (h->centralised) {   // get_value (ac/model.py:156-157): every agent's critic reads the concatenated observations
    JointParams jp; jp.traj = ps.src.traj; jp.idx = h->idx; jp.P = n_envs; jp.out = h->joint;
    const size_t n = (size_t)n_envs * (T + 1) * h->critic.in;
    joint_obs_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(jp);
    MARL_CUDA_TRY(cudaGetLastError());
    ps.csrc.mode = kRowsEpisodeJoint; ps.csrc.joint = h->joint; ps.csrc.D = h->critic.in;
  }
  // 1. target critic on all T+1 observations (ac/model.py:190-193)
  if (h->critic_rnn) {
    if (int rc = a2c_gru_forward(h->critic, h->cgl, ps.csrc, h->theta_tgt, n_envs, h->vt, nullptr, st)) return rc;
  } else {
    if (int rc = forward_any(h->critic, ps.cplan, ps.csrc, h->theta_tgt, h->image, h->vt, st)) return rc;
  }
  // 2. n-step returns (ac/model.py:198-201), or the λ-returns of algorithm.gae_lambda
  if (h->gae) {
    LambdaParams lp; lp.vt = h->vt; lp.traj = ps.src.traj; lp.idx = h->idx; lp.N = N; lp.P = n_envs; lp.ret = h->ret;
    lp.ret_ms = h->standardise ? h->ret_ms : nullptr;
    lp.coef_v = (float)((double)h->hp.gamma * (1.0 - (double)h->gae_lambda)); lp.coef_r = (float)((double)h->hp.gamma * (double)h->gae_lambda);
    lambda_returns_kernel<<<(N * n_envs + kLamWarps - 1) / kLamWarps, 32 * kLamWarps, 0, st>>>(lp);
  } else {
    NStepParams np; np.vt = h->vt; np.traj = ps.src.traj; np.idx = h->idx; np.N = N; np.P = n_envs; np.n_steps = h->hp.n_steps; np.ret = h->ret;
    np.ret_ms = h->standardise ? h->ret_ms : nullptr;
    for (int k = 0; k <= h->hp.n_steps; ++k) np.gpow[k] = (float)pow((double)h->hp.gamma, (double)k);
    nstep_returns_kernel<<<(N * n_envs * T + 255) / 256, 256, 0, st>>>(np);
  }
  MARL_CUDA_TRY(cudaGetLastError());
  if (h->standardise) {  // ac/model.py:202-204
    RetMsParams rp; rp.ret = h->ret; rp.N = N; rp.P = n_envs; rp.T = T; rp.part = h->ret_part; rp.ret_ms = h->ret_ms; rp.count = h->ret_count;
    MARL_CUDA_TRY(ret_ms_step(rp, st));
  }
  return MARL_OK;
}

/* cfg.standardise_returns (ac/model.py:112-114): switches the RunningMeanStd over the n-step returns on (mean 0, var 1, count 1e-4) or off. */
int marl_a2c_standardise_returns(marl_a2c* h, int32_t enable) {
  MARL_REQUIRE(h != nullptr, "marl_a2c_standardise_returns: NULL handle");
  MARL_REQUIRE(h->actor.n_agents <= 32, "marl_a2c_standardise_returns: at most 32 agents");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  if (enable)
    if (int rc = enable_ret_stats(h, h->actor.n_agents, "marl_a2c_standardise_returns")) return rc;
  h->standardise = enable ? 1 : 0;
  return MARL_OK;
}
/* algorithm.gae_lambda: enable != 0 replaces the n-step returns of every later update (A2C and PPO) by the λ-returns of `lambda` in [0, 1];
 * enable == 0 restores them.  n_steps is not read while λ-returns are on. */
int marl_a2c_set_gae_lambda(marl_a2c* h, int32_t enable, float lambda) {
  MARL_REQUIRE(h != nullptr, "marl_a2c_set_gae_lambda: NULL handle");
  MARL_REQUIRE(!enable || (lambda >= 0.f && lambda <= 1.f), "marl_a2c_set_gae_lambda: lambda %g is outside [0, 1]", (double)lambda);
  h->gae = enable ? 1 : 0;
  h->gae_lambda = enable ? lambda : 0.f;
  return MARL_OK;
}
/* the running statistics as device pointers: ret_ms float[2 n_agents] = mean | var, count double[1] (NULL before the first enable) */
int marl_a2c_ret_ms_ptrs(marl_a2c* h, float** ret_ms, double** count) {
  MARL_REQUIRE(h != nullptr, "marl_a2c_ret_ms_ptrs: NULL handle");
  if (ret_ms) *ret_ms = h->ret_ms; if (count) *count = h->ret_count;
  return MARL_OK;
}

// critic and actor training passes -> grad[] (un-normalised sums) + loss statistics; old_logp != NULL: PPO's clipped surrogate
// A recurrent part's training pass: sequence forward from h = 0 saving what BPTT needs (outputs of row T are not used: the GRU is causal, so this
// equals the reference's pass over the first T observations), the loss head on rows t < T, BPTT from the dense dL/dout -> per-CTA gradient
// partials in scratch and per-block loss statistics in loss_part.  Sets the reduction's plan, P and loss-part count in rp.
static int a2c_rnn_part(marl_a2c* h, const NetSet& ns, const GruLayout& gl, const RowSource& src, const TrainParams& tp, int head, int n_envs, cudaStream_t st,
                        ReduceParams& rp) {
  const int T = src.traj.T;
  if (int rc = a2c_gru_forward(ns, gl, src, tp.theta, n_envs, h->rnn_q, h->gru_save, st)) return rc;
  GruHeadParams hp; hp.tp = tp; hp.traj = src.traj; hp.idx = h->idx; hp.N = ns.n_agents; hp.P = n_envs; hp.A = ns.out;
  hp.q = h->rnn_q; hp.dq = h->rnn_dq; hp.loss_part = h->loss_part;
  if (int rc = launch_gru_ac_head(hp, head, st)) return rc;
  GruBwdParams bp; memset(&bp, 0, sizeof(bp));
  bp.plan = make_plan(ns, n_envs, 1, h->n_sm, kGruSeqs); bp.traj = src.traj; bp.idx = h->idx; bp.B = n_envs; bp.theta = tp.theta; bp.lay = gl;
  bp.save = h->gru_save; bp.src = src; bp.dout = h->rnn_dq; bp.scratch = h->scratch; bp.scratch_pitch = h->scratch_pitch;
  if (int rc = launch_gru_backward(bp, st)) return rc;
  memcpy(rp.cta_begin, bp.plan.cta_begin, sizeof(rp.cta_begin));
  rp.P = gl.P; rp.n_loss_parts = gru_head_blocks(ns.n_agents, n_envs, T);
  return MARL_OK;
}

static int a2c_gradients(marl_a2c* h, const A2cPass& ps, cudaStream_t st, const float* old_logp, float ppo_clip) {
  // 3. critic: forward, value loss, backward; leaves advantage = returns - V for the actor pass
  TrainParams tp; memset(&tp, 0, sizeof(tp));
  tp.plan = ps.cplan; tp.src = ps.csrc; tp.theta = h->theta + h->n_actor; tp.lay = h->critic.lay; tp.scratch = h->scratch; tp.scratch_pitch = h->scratch_pitch;
  tp.loss_part = h->loss_part; tp.returns = h->ret; tp.adv_out = h->adv; tp.value_coef = h->hp.value_loss_coef;
  ReduceParams rp; memset(&rp, 0, sizeof(rp));  // (sumsq_part stays NULL: two passes write different gradient slices)
  rp.scratch = h->scratch; rp.loss_part = h->loss_part; rp.n_nets = h->critic.n_nets; rp.scratch_pitch = h->scratch_pitch;
  if (h->critic_rnn) {
    if (int rc = a2c_rnn_part(h, h->critic, h->cgl, ps.csrc, tp, kHeadA2cCritic, ps.n_envs, st, rp)) return rc;
  } else {
    if (int rc = launch_train(tp, kHeadA2cCritic, st)) return rc;
    rp.P = h->critic.lay.P; memcpy(rp.cta_begin, ps.cplan.cta_begin, sizeof(rp.cta_begin)); rp.n_loss_parts = ps.cplan.cta_begin[ps.cplan.n_nets];
  }
  rp.grad = h->grad + h->n_actor; rp.stats = h->grad + h->n_params; rp.stats_accumulate = 0;
  if (int rc = launch_grad_reduce(rp, st)) return rc;
  // 4. actor: forward, log-softmax, policy-gradient (or clipped surrogate) + entropy loss, backward
  tp.plan = ps.aplan; tp.src = ps.src; tp.theta = h->theta; tp.lay = h->actor.lay; tp.adv = h->adv; tp.entropy_coef = h->hp.entropy_coef;
  tp.old_logp = old_logp; tp.ppo_clip = ppo_clip;
  rp.n_nets = h->actor.n_nets;
  if (h->actor_rnn) {
    if (int rc = a2c_rnn_part(h, h->actor, h->agl, ps.src, tp, kHeadA2cActor, ps.n_envs, st, rp)) return rc;
  } else {
    if (int rc = launch_train(tp, kHeadA2cActor, st)) return rc;
    rp.P = h->actor.lay.P; memcpy(rp.cta_begin, ps.aplan.cta_begin, sizeof(rp.cta_begin)); rp.n_loss_parts = ps.aplan.cta_begin[ps.aplan.n_nets];
  }
  rp.grad = h->grad; rp.stats_accumulate = 1;
  return launch_grad_reduce(rp, st);
}

int marl_a2c_update_grads(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, void* stream) {
  A2cPass ps;
  if (int rc = a2c_prepare(h, batch, n_envs, (cudaStream_t)stream, ps)) return rc;
  return a2c_gradients(h, ps, (cudaStream_t)stream, nullptr, 0.f);
}

/* metrics_out device float[6] = (policy-gradient term, grad norm, entropy, value_loss, filled count, 0):
 * actor_loss = m[0] - entropy_coef*m[2]; loss = actor_loss + value_loss_coef*m[3]  (ac/model.py:216-226,241-246) */
static int a2c_apply(marl_a2c* h, int64_t step, float* metrics_out, void* stream, bool target_update) {
  MARL_REQUIRE(h != nullptr, "marl_a2c_update_apply: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  h->opt_steps += 1;
  h->opt_stepped = true;
  AdamParams ap; memset(&ap, 0, sizeof(ap));
  ap.theta = h->theta; ap.theta_tgt = h->theta_tgt; ap.m = h->m; ap.v = h->v; ap.grad = h->grad; ap.n = (int)h->n_params;
  ap.tgt_begin = (int)h->n_actor; ap.tgt_n = (int)h->n_critic;
  ap.grad_clip = h->hp.grad_clip;
  set_step_consts(ap, h->opt, h->hp.lr, h->opt_steps);
  const float tu = h->hp.target_update_interval_or_tau;  // ac/model.py:233-239: `step` counts environment steps
  ap.tau = tu;
  if (target_update && tu > 1.0f && fmod((double)step, (double)tu) == 0.0) ap.target_mode = 1;
  else if (target_update && tu < 1.0f) ap.target_mode = 2;
  ap.loss_out = metrics_out ? metrics_out : h->metrics;
  return launch_adam(ap, h->opt.kind, (cudaStream_t)stream);
}

int marl_a2c_update_apply(marl_a2c* h, int64_t step, float* metrics_out, void* stream) { return a2c_apply(h, step, metrics_out, stream, true); }

/* PPONetwork.update (ac/model.py:265-352) on the same handle: returns and the collecting policy's log-probabilities once, then `num_epochs`
 * optimisation steps on the same batch with the clipped surrogate (-min(r adv, clip(r, 1 -+ ppo_clip) adv) - entropy_coef H + value_loss_coef
 * value loss; clip_grad_norm_ over all parameters when hp.grad_clip > 0), the target critic synchronised after the last epoch.
 * metrics_out: device float[6] as marl_a2c_update, averaged over the epochs ([0] = the surrogate term).
 * = marl_ppo_prepare, then num_epochs x (marl_ppo_epoch_grads + marl_ppo_epoch_apply) with nothing in between. */
static int ppo_prepare(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, cudaStream_t st) {
  h->ppo_prepared = false;
  A2cPass& ps = h->ppo_pass;
  if (int rc = a2c_prepare(h, batch, n_envs, st, ps)) return rc;
  if (!h->logits_all) {
    const size_t rows = (size_t)h->actor.n_agents * h->max_envs * (h->max_T + 1), F = sizeof(float);
    if (int rc = alloc_buffers(h, "marl_ppo_update", {{&h->logits_all, rows * h->actor.out * F}, {&h->old_logp, rows * F}, {&h->epoch_metrics, 6 * kMaxPpoEpochs * F}}))
      return rc;
  }
  // log-probabilities of the taken actions under the collecting policy = the current actor (ac/model.py:281-292)
  if (h->actor_rnn) {
    if (int rc = a2c_gru_forward(h->actor, h->agl, ps.src, h->theta, n_envs, h->logits_all, nullptr, st)) return rc;
  } else {
    if (int rc = forward_any(h->actor, ps.aplan, ps.src, h->theta, h->image, h->logits_all, st)) return rc;
  }
  OldLogpParams op; op.logits = h->logits_all; op.traj = ps.src.traj; op.idx = h->idx; op.N = h->actor.n_agents; op.P = n_envs; op.A = h->actor.out; op.out = h->old_logp;
  old_logp_kernel<<<(op.N * n_envs * batch->T + 255) / 256, 256, 0, st>>>(op);
  MARL_CUDA_TRY(cudaGetLastError());
  h->ppo_prepared = true;
  return MARL_OK;
}

// one epoch's optimiser step; the last epoch (epoch == num_epochs - 1) also updates the target critic and writes the epochs' mean metrics
static int ppo_epoch_apply(marl_a2c* h, int64_t step, int epoch, int num_epochs, float* metrics_out, cudaStream_t st) {
  const bool last = epoch == num_epochs - 1;
  if (int rc = a2c_apply(h, step, h->epoch_metrics + 6 * epoch, st, last)) return rc;
  if (!last) return MARL_OK;
  mean_metrics_kernel<<<1, 32, 0, st>>>(h->epoch_metrics, num_epochs, metrics_out ? metrics_out : h->metrics);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int marl_ppo_update(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, int64_t step, int32_t num_epochs, float ppo_clip, float* metrics_out, void* stream) {
  MARL_REQUIRE(h != nullptr && num_epochs >= 1 && num_epochs <= kMaxPpoEpochs, "marl_ppo_update: num_epochs %d out of range (1..%d)", (int)num_epochs, kMaxPpoEpochs);
  MARL_REQUIRE(ppo_clip > 0.f, "marl_ppo_update: ppo_clip must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = ppo_prepare(h, batch, n_envs, st)) return rc;
  for (int e = 0; e < num_epochs; ++e) {
    if (int rc = a2c_gradients(h, h->ppo_pass, st, h->old_logp, ppo_clip)) return rc;
    if (int rc = ppo_epoch_apply(h, step, e, num_epochs, metrics_out, st)) return rc;
  }
  return MARL_OK;
}

int marl_ppo_prepare(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_ppo_prepare: NULL handle");
  return ppo_prepare(h, batch, n_envs, (cudaStream_t)stream);
}

int marl_ppo_epoch_grads(marl_a2c* h, float ppo_clip, void* stream) {
  MARL_REQUIRE(h != nullptr && h->ppo_prepared, "marl_ppo_epoch_grads: call marl_ppo_prepare first");
  MARL_REQUIRE(ppo_clip > 0.f, "marl_ppo_epoch_grads: ppo_clip must be positive");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  return a2c_gradients(h, h->ppo_pass, (cudaStream_t)stream, h->old_logp, ppo_clip);
}

int marl_ppo_epoch_apply(marl_a2c* h, int64_t step, int32_t epoch, int32_t num_epochs, float* metrics_out, void* stream) {
  MARL_REQUIRE(h != nullptr && h->ppo_prepared, "marl_ppo_epoch_apply: call marl_ppo_prepare first");
  MARL_REQUIRE(num_epochs >= 1 && num_epochs <= kMaxPpoEpochs && epoch >= 0 && epoch < num_epochs,
               "marl_ppo_epoch_apply: epoch %d / num_epochs %d out of range (1..%d epochs)", (int)epoch, (int)num_epochs, kMaxPpoEpochs);
  return ppo_epoch_apply(h, step, epoch, num_epochs, metrics_out, (cudaStream_t)stream);
}

/* The optimiser of actor + critic: before the first step only; zeroes the optimiser state. */
int marl_a2c_set_optimizer(marl_a2c* h, const marl_optimizer* opt) {
  if (int rc = check_set_optimizer(h, opt, "marl_a2c_set_optimizer")) return rc;
  return reset_optimizer(h, *opt);
}

int marl_a2c_update(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, int64_t step, float* metrics_out, void* stream) {
  if (int rc = marl_a2c_update_grads(h, batch, n_envs, stream)) return rc;
  return marl_a2c_update_apply(h, step, metrics_out, stream);
}

}  // extern "C"
