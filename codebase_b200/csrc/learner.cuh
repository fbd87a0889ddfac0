// learner.cuh -- kernels shared by the DQN-family and actor-critic learners: gathered MLP forward, fused
// forward+loss-head+backward training pass, deterministic gradient reduction, clip + Adam + target update.
#pragma once
#include "mlp.cuh"
#include "traj.cuh"
#include <string.h>

namespace marl {

constexpr int kMaxObsDim = 32;   // tensor-core paths and the DQN family: KP = 16 or 32 float input tiles
constexpr int kMaxInDim = 128;   // FP32 MLP kernels (actor-critic learners: KP = 64 / 128 tiles above 32) and the GRU kernels

// Which rows a launch covers and how CTAs split them.  A "unit" is an indivisible run of rows that must stay inside
// one CTA: one sampled episode (T+1 rows) for training passes, one row for plain inference.
struct RowPlan {
  int n_nets;
  int cta_begin[MARL_MAX_AGENTS + 1];   // CTAs [cta_begin[k], cta_begin[k+1]) work on net k
  int slot_begin[MARL_MAX_AGENTS + 1];  // agents of net k = slot_agent[slot_begin[k] .. slot_begin[k+1])
  int slot_agent[MARL_MAX_AGENTS];
  int unit_rows;                        // rows per unit
  int units_per_agent;                  // B (episodes) or E (envs)
};

// Where a launch's observation rows come from.  The JOINT modes are observation rows shared by all agents (centralised critic,
// ac/model.py:62-65,156-157: every agent's critic sees the concatenation of all agents' observations; D = their total width).
enum RowMode {
  kRowsDense = 0,         // dense obs float[E][N][D]: one row per (unit = env, agent); outputs [E][N]
  kRowsEpisode = 1,       // the trajectory store's episodes idx[unit]; outputs and loss scalars per row (row_index)
  kRowsEpisodeJoint = 2,  // joint rows float[units][T+1][D], outputs like kRowsEpisode, loss scalars from the trajectory store
  kRowsDenseJoint = 3     // joint rows float[E][D]: the dense obs array read as [E][N * D_agent]; outputs like kRowsDense
};
struct RowSource {
  int mode;   // RowMode
  const float* dense; int E, N, D;
  TrajView traj; const int32_t* idx;  // idx[B] ring slots (device)
  const float* joint;
};
__host__ __device__ __forceinline__ bool src_dense_out(int mode) { return mode == kRowsDense || mode == kRowsDenseJoint; }

// The learner's per-row buffers (target outputs, Q-values, values, logits, GRU saved rows, tensor-core activations and records) are laid out
// [agent][units_per_agent][unit_rows]: the index of row `off` of unit `unit` of `agent`
__host__ __device__ __forceinline__ size_t row_index(int agent, int unit, int off, int units_per_agent, int unit_rows) {
  return ((size_t)agent * units_per_agent + unit) * unit_rows + off;
}

__device__ __forceinline__ void cta_rows(const RowPlan& p, int& net, int& row_begin, int& row_end) {
  net = 0;
  while (net + 1 < p.n_nets && (int)blockIdx.x >= p.cta_begin[net + 1]) ++net;
  const int ncta = p.cta_begin[net + 1] - p.cta_begin[net], c = (int)blockIdx.x - p.cta_begin[net];
  const long long units = (long long)(p.slot_begin[net + 1] - p.slot_begin[net]) * p.units_per_agent;
  row_begin = (int)(units * c / ncta) * p.unit_rows;
  row_end = (int)(units * (c + 1) / ncta) * p.unit_rows;
}

// virtual row of net -> (agent, unit index within agent, offset within unit)
__device__ __forceinline__ void decode_row(const RowPlan& p, int net, int vr, int& agent, int& unit, int& off) {
  const int rpa = p.units_per_agent * p.unit_rows;
  const int slot = vr / rpa, rem = vr - slot * rpa;
  agent = p.slot_agent[p.slot_begin[net] + slot];
  unit = rem / p.unit_rows;
  off = rem - unit * p.unit_rows;
}

// Observation row of (agent, unit, row off of the unit).  Independent of the plan: an episode's rows are its T + 1 steps, a dense unit has one
// row (off == 0).
__device__ __forceinline__ const float* src_row(const RowSource& s, int agent, int unit, int off) {
  if (s.mode == kRowsDense) return s.dense + ((size_t)unit * s.N + agent) * s.D;
  if (s.mode != kRowsEpisode) return s.joint + ((size_t)unit * (s.mode == kRowsEpisodeJoint ? s.traj.T + 1 : 1) + off) * s.D;
  return s.traj.obs_row(s.idx[unit], agent, off);
}

// Where the outputs of a row go: [unit][N] for the dense sources, the per-row layout (row_index) otherwise
__device__ __forceinline__ size_t out_row(const RowSource& s, int agent, int unit, int off, int units_per_agent, int unit_rows) {
  return src_dense_out(s.mode) ? (size_t)unit * s.N + agent : row_index(agent, unit, off, units_per_agent, unit_rows);
}

// Per-tile row metadata staged in shared memory by the first 128 threads (one row each): the source pointer of the
// row's observation and, for training passes, the scalars the loss head needs.  Two dependent global latencies per tile
// (episode index, then its fields) instead of a dependent chain per element / per head.
struct RowMeta {
  const float* src[kTileRows];
  int act[kTileRows];
  float rew[kTileRows];
  int flags[kTileRows];  // bit 0: filled[t], bit 1: done[t+1]
  static constexpr int kBytes = kTileRows * (8 + 4 + 4 + 4);
};

template <bool kWithScalars>
__device__ __forceinline__ void setup_rows(RowMeta* m, const RowPlan& p, const RowSource& s, int net, int vr0, int nrows) {
  const int r = threadIdx.x;
  if (r >= kTileRows) return;
  const float* src = nullptr; int act = 0, flags = 0; float rew = 0.f;
  if (r < nrows) {
    int agent, unit, off;
    decode_row(p, net, vr0 + r, agent, unit, off);
    src = src_row(s, agent, unit, off);
    const TrajView& tv = s.traj;
    if (kWithScalars && !src_dense_out(s.mode) && off < tv.T) {
      const size_t ep = (size_t)s.idx[unit];
      act = tv.act[tv.step_at(ep, agent, off)];
      rew = tv.rew[tv.step_at(ep, agent, off)];
      flags = (int)tv.filled[tv.filled_at(ep, off)] | ((int)tv.done[tv.done_at(ep, off + 1)] << 1);
    }
  }
  m->src[r] = src; m->act[r] = act; m->rew[r] = rew; m->flags[r] = flags;
}

// Fill the [128][KP] input tile from the staged row pointers (asynchronous copies; zero padding in both directions).
// Caller: cp_async_wait_all() + __syncthreads() before the tile is read.
template <int KP>
__device__ __forceinline__ void gather_tile_async(float* X, const RowMeta* m, int D) {
#pragma unroll 4
  for (int i = threadIdx.x; i < kTileRows * KP; i += kMlpThreads) {
    const int r = i / KP, k = i - r * KP;
    const float* src = m->src[r];
    if (src != nullptr && k < D) cp_async4(&at1<KP>(X, r, k), src + k);
    else at1<KP>(X, r, k) = 0.f;
  }
}

struct FwdParams {
  RowPlan plan; RowSource src;
  const float* theta;   // [n_nets][P]
  NetLayout lay;
  float* out;           // dense sources: [E][N][out]; the others: [N][B][T+1][out] (out_row)
};

// Loss heads of the fused training kernel (what happens between the forward and the backward of a tile).
enum TrainHead { kHeadDqn = 0, kHeadA2cCritic = 1, kHeadA2cActor = 2 };

struct TrainParams {
  RowPlan plan; RowSource src;
  const float* theta; NetLayout lay;
  float* scratch;         // [gridDim][pitch] per-CTA gradient sums (un-normalised); pitch = P rounded up to 4 floats
  int scratch_pitch;
  float* loss_part;       // [gridDim][4] per-CTA loss statistics, meaning depends on the head (see below)
  // kHeadDqn: parts = (sum delta^2*filled, sum filled on agent 0, 0, 0)
  const float* tq;        // target-net Q-values of every gathered row, [N][B][T+1][out] (from the forward kernel)
  const float* td_ext;    // precomputed 2*delta*filled (VDN: per (b, t), [B][T]; standardise_returns: per (agent, b, t) with td_agent_stride = B*T); NULL: the head computes it
  int td_agent_stride;
  float gamma; int double_q;
  float huber;            // algorithm.huber_delta (> 0: the Huber TD loss of dqn_heads.cuh; <= 0: the squared error)
  // kHeadA2cCritic: parts = (0, sum filled on agent 0, 0, sum adv^2*filled); writes adv = returns - V
  const float* returns;   // [N][B][T] n-step returns
  float* adv_out;         // [N][B][T]
  float value_coef;
  // kHeadA2cActor: parts = (sum -logp*adv*filled, 0, sum entropy*filled, 0)
  const float* adv;       // [N][B][T]
  float entropy_coef;
  // PPO (ac/model.py:305-321): old_logp != NULL switches the actor head to the clipped surrogate -min(ratio adv, clip(ratio, 1 -+ ppo_clip) adv),
  // ratio = exp(logp - old_logp); parts[0] = sum of that term * filled
  const float* old_logp;  // [N][B][T] log-probabilities of the taken actions under the policy the batch was collected with
  float ppo_clip;
};

struct ReduceParams {
  const float* scratch; const float* loss_part; int n_nets; int cta_begin[MARL_MAX_AGENTS + 1]; int P; int scratch_pitch;
  int n_loss_parts;
  float* grad;       // [n_nets*P] gradient sums of this network set
  float* stats;      // [4] sums of the loss parts (NULL: skip)
  int stats_accumulate;  // add to stats instead of overwriting (second pass of an actor-critic update)
  float* sumsq_part;     // [ceil(n_nets*P / 64)] per-block sum of squares of the reduced gradients (NULL: skip)
};

// The optimiser of a step (marl_optimizer.kind): a template parameter of the two step kernels, so each one compiles to its own code
enum OptKind { kOptAdam = MARL_OPT_ADAM, kOptAdamW = MARL_OPT_ADAMW, kOptRmsprop = MARL_OPT_RMSPROP, kOptAdagrad = MARL_OPT_ADAGRAD, kOptSgd = MARL_OPT_SGD,
               kNumOpt };

// The optimiser state lives in m / v: Adam, AdamW exp_avg / exp_avg_sq; RMSprop square_avg in v; Adagrad sum in v; SGD none.
struct AdamParams {
  float* theta; float* theta_tgt; float* m; float* v;
  const float* grad;   // [n] gradient sums followed by 4 statistics: (loss numerator, filled count, aux0, aux1)
  int n;               // trainable floats
  int tgt_begin, tgt_n;  // theta[tgt_begin .. tgt_begin+tgt_n) is mirrored by theta_tgt[0 .. tgt_n)
  float lr, beta1, beta2, eps, bc1, bc2_sqrt, grad_clip;  // grad_clip <= 0: off; RMSprop: beta2 = alpha, beta1 = 1 - alpha (rounded from double)
  int target_mode;  // 0 none, 1 hard copy, 2 polyak
  float tau;
  float* loss_out;  // [6]: stats[0]/filled, grad norm, stats[2]/filled, stats[3]/filled, filled, 0
  const float* sumsq_part; int n_sumsq;  // optional per-block sums of squares of grad[0..n) (local gradients only: single GPU)
  float decay;      // AdamW: theta *= decay (= 1 - lr * weight_decay) before the Adam step.  In the slot before `image`: no other field moves
  // optional packed tensor-core images of theta[0 .. img_nets * img_lay.P), kept current parameter by parameter (NULL: none)
  uint8_t* image; uint8_t* bwd_image; NetLayout img_lay; int img_nets; size_t image_bytes, bwd_image_bytes;
};

// host-side launchers (defined next to the kernels in learner_kernels.cu); return MARL_* codes
int learner_kernels_init(int in_dim, int max_in);           // opt in to > 48 KB dynamic shared memory; max_in: kMaxObsDim or kMaxInDim
int launch_mlp_forward(const FwdParams& p, cudaStream_t st);
int launch_train(const TrainParams& p, int head, cudaStream_t st);
int launch_grad_reduce(const ReduceParams& p, cudaStream_t st);
// Gradient exchange over NVLink peer memory (reduce_adam_kernel<true>): every rank owns an exchange buffer
// [2 parities][world source ranks][slot_floats] floats + [world] 64-bit flags, opened by the other ranks through CUDA IPC.
constexpr int kMaxRanks = 8;
struct XchgParams {
  int world, rank, slot_floats;
  unsigned long long epoch;                        // number of exchanges so far, this one included
  float* peers[kMaxRanks];                         // every rank's buffer (own included)
  unsigned long long* peer_flags[kMaxRanks];       // every rank's flag array (own included): flag[source rank]
  const unsigned long long* own_flags;             // = peer_flags[rank]
  int* timed_out;                                  // device flag (sticky): a peer's epoch flag did not arrive within the spin bound
  // a second buffer summed in the same exchange (QMIX: the mixer's gradient sums, already reduced): slot = [n grads | n_extra | 4 statistics].
  // extra[0 .. n_extra) is pushed, then overwritten with the all-rank sum, and extra[n_extra .. n_extra + 4) with the all-rank statistics
  float* extra; int n_extra;
};
// replay indices for the next update, drawn by the fused tail kernel (idx == NULL: none); same stream as replay_sample_kernel
struct SampleParams { uint64_t seed, update_idx; int batch, n_valid; int32_t* idx; };
// opt: the OptKind of the step
int launch_reduce_adam(const ReduceParams& rp, const AdamParams& ap, int opt, XchgParams* xp, const SampleParams& sp, unsigned long long* barrier,
                       unsigned long long* epoch, int n_sm, cudaStream_t st);
int launch_adam(const AdamParams& p, int opt, cudaStream_t st);
// can the fused tail with optimiser `opt` cover n parameters with one co-resident wave on n_sm SMs?  (pb, ns: the block shape it would use)
int reduce_adam_shape(int n, int n_sm, bool xchg, int opt, int* pb, int* ns);
// the step constants of `o` for the next step (step = 1, 2, ...): lr, betas, eps, bias corrections, AdamW's decay.  The handle has checked o.
// Adam / AdamW: the betas as float32 (the hp fields' values: a handle's Adam steps stay what they were before marl_optimizer existed).
// RMSprop / AdamW: torch's Python-scalar arithmetic in double, rounded once to float32 as torch's CPU kernels round a scalar argument.
inline void set_step_consts(AdamParams& ap, const marl_optimizer& o, float lr, int64_t step) {
  ap.lr = lr; ap.eps = (float)o.eps; ap.bc1 = 1.f; ap.bc2_sqrt = 1.f; ap.decay = 1.f;
  if (o.kind == MARL_OPT_ADAM || o.kind == MARL_OPT_ADAMW) {
    const float b1 = (float)o.beta1, b2 = (float)o.beta2;
    ap.beta1 = b1; ap.beta2 = b2;
    ap.bc1 = (float)(1.0 - pow((double)b1, (double)step));
    ap.bc2_sqrt = (float)sqrt(1.0 - pow((double)b2, (double)step));
    if (o.kind == MARL_OPT_ADAMW) ap.decay = (float)(1.0 - (double)lr * o.weight_decay);   // param.mul_(1 - lr * weight_decay)
  } else if (o.kind == MARL_OPT_RMSPROP) {
    ap.beta2 = (float)o.alpha;                // square_avg.mul_(alpha)
    ap.beta1 = (float)(1.0 - o.alpha);        // addcmul_(grad, grad, value=1 - alpha)
  }
}
// marl_*_set_optimizer's argument check
inline int check_optimizer(const marl_optimizer* o, const char* who) {
  MARL_REQUIRE(o != nullptr, "%s: NULL optimizer", who);
  MARL_REQUIRE(o->kind >= 0 && o->kind < kNumOpt, "%s: optimizer kind %d unknown (Adam 0, AdamW 1, RMSprop 2, Adagrad 3, SGD 4)", who, o->kind);
  MARL_REQUIRE(o->eps >= 0.0 && o->weight_decay >= 0.0 && o->beta1 >= 0.0 && o->beta1 < 1.0 && o->beta2 >= 0.0 && o->beta2 < 1.0 && o->alpha >= 0.0 && o->alpha <= 1.0,
               "%s: optimizer constants out of range", who);
  return MARL_OK;
}

template <int KP>
constexpr size_t forward_smem_bytes() { return sizeof(float) * (WeightSmem<KP>::kFloats + 2 * kTileRows * kPitchH + kTileRows * kOutPad + 48) + RowMeta::kBytes; }
template <int KP>
constexpr size_t train_smem_bytes() { return forward_smem_bytes<KP>(); }

// ---- host-side planning -----------------------------------------------------------------------------------------
struct NetSet {
  int n_agents = 0, n_nets = 0, in = 0, out = 0;
  int agent_net[MARL_MAX_AGENTS];
  NetLayout lay;
};

// Split `n_cta_max` CTAs over the networks in proportion to their row counts; every CTA gets >= min_units units.
inline RowPlan make_plan(const NetSet& ns, int units_per_agent, int unit_rows, int n_cta_max, int min_units) {
  RowPlan p; memset(&p, 0, sizeof(p));
  p.n_nets = ns.n_nets; p.unit_rows = unit_rows; p.units_per_agent = units_per_agent;
  int s = 0;
  for (int k = 0; k < ns.n_nets; ++k) {
    p.slot_begin[k] = s;
    for (int a = 0; a < ns.n_agents; ++a) if (ns.agent_net[a] == k) p.slot_agent[s++] = a;
  }
  p.slot_begin[ns.n_nets] = s;
  long long total = (long long)ns.n_agents * units_per_agent;
  int c = 0;
  for (int k = 0; k < ns.n_nets; ++k) {
    const long long units = (long long)(p.slot_begin[k + 1] - p.slot_begin[k]) * units_per_agent;
    long long want = (long long)n_cta_max * units / (total > 0 ? total : 1);
    const long long cap = (units + min_units - 1) / min_units;
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    p.cta_begin[k] = c;
    c += (int)want;
  }
  p.cta_begin[ns.n_nets] = c;
  return p;
}

// A training pass over sampled episodes: one unit per episode (T + 1 rows), at least 64 rows per CTA
inline RowPlan episode_plan(const NetSet& ns, int episodes, int T, int n_cta_max) {
  const int min_units = (64 + T) / (T + 1) > 0 ? (64 + T) / (T + 1) : 1;
  return make_plan(ns, episodes, T + 1, n_cta_max, min_units);
}

// Dense rows obs float[E][N][D].  joint: a centralised critic's rows, obs float[E][N][D_agent] read as float[E][D = N * D_agent].
inline RowSource dense_rows(const float* obs, int E, int N, int D, bool joint = false) {
  RowSource s; memset(&s, 0, sizeof(s));
  s.mode = joint ? kRowsDenseJoint : kRowsDense; s.dense = obs; s.E = E; s.N = N; s.D = D;
  if (joint) s.joint = obs;
  return s;
}

// Rows of the episodes idx[] of a trajectory store
inline RowSource episode_rows(const marl_traj_view* t, const int32_t* idx, int N, int D) {
  RowSource s; memset(&s, 0, sizeof(s));
  s.mode = kRowsEpisode; s.traj = traj_view(t); s.idx = idx; s.N = N; s.D = D;
  return s;
}

inline int launch_forward(const NetSet& ns, const RowPlan& plan, const RowSource& src, const float* theta, float* out, cudaStream_t st) {
  FwdParams fp; fp.plan = plan; fp.src = src; fp.theta = theta; fp.lay = ns.lay; fp.out = out;
  return launch_mlp_forward(fp, st);
}

// ---- tensor-core forward path (tc_forward.cu) -----------------------------------------------------------------------------
size_t tc_image_bytes();
int tc_forward_init();
size_t tc_bwd_image_bytes();
int launch_pack_weights(const float* theta, const NetLayout& lay, int n_nets, uint8_t* image, cudaStream_t st, uint8_t* bwd_image = nullptr);
int launch_tc_forward(const FwdParams& p, const uint8_t* images, cudaStream_t st);
// ---- tensor-core training pipeline (tc_train.cu) ----------------------------------------------------------------------------
struct TcBuffers {
  uint8_t* image; uint8_t* bwd_image;       // packed online-network images (forward K-major, backward K-major W2^T)
  float* h2;                                // H2 activations in fragment order: [h2_tiles][16][128] float4, a slab of 64-row tiles per CTA
  size_t h2_tiles;                          // allocated 64-row tiles of h2 (ceil(rows / 64) + grid hold any row split: tc_train.cu, h2_slab)
  float* rec;                               // [rows][kRowRec] row records (tc_train.cu)
  float* x;                                 // [rows][8 ceil(in / 8)] gathered observation rows
};
int tc_train_init();
// the training forward (tc_dqn_fwd_kernel): the online network, and with tgt_images the target network on the same rows into tq_out; q_out (optional):
// the online outputs for an external TD head
int launch_tc_dqn_forward(const TrainParams& tp, const TcBuffers& buf, const uint8_t* tgt_images, float* tq_out, float* q_out, cudaStream_t st);
// the backward kernels (tc_dh1_kernel, tc_dw_kernel) behind it; after_dh1 (optional) is recorded between them
int launch_tc_dqn_backward(const TrainParams& tp, const TcBuffers& buf, cudaStream_t st, cudaEvent_t after_dh1 = nullptr);
// tc_forward_enabled(): process-wide switch (marl_set_option("tensor_core_forward", 0|1)), declared in common.cuh

// Forward pass through whichever implementation is selected.  `image` is scratch for the packed weights (n_nets images);
// it is rebuilt from `theta` on every call (3 us) so that it can never go stale against direct parameter writes.
// The tensor-core forward's W1 image is kMaxObsDim wide and its hidden layers 128 wide: wider inputs and narrower networks always run
// the FP32 kernel (their handles allocate no image).
inline int forward_any(const NetSet& ns, const RowPlan& plan, const RowSource& src, const float* theta, uint8_t* image, float* out, cudaStream_t st,
                       bool image_is_current = false) {
  if (tc_forward_enabled() && image != nullptr && ns.in <= kMaxObsDim && ns.lay.H == kHidden) {
    if (!image_is_current)
      if (int rc = launch_pack_weights(theta, ns.lay, ns.n_nets, image, st)) return rc;
    FwdParams fp; fp.plan = plan; fp.src = src; fp.theta = theta; fp.lay = ns.lay; fp.out = out;
    return launch_tc_forward(fp, image, st);
  }
  return launch_forward(ns, plan, src, theta, out, st);
}

// max_in: the widest input the caller's kernels take (kMaxObsDim or kMaxInDim)
inline int check_mlp_cfg(const marl_mlp_cfg* cfg, const char* who, int max_in) {
  MARL_REQUIRE(cfg != nullptr, "%s: NULL network config", who);
  MARL_REQUIRE(cfg->n_agents >= 1 && cfg->n_agents <= MARL_MAX_AGENTS, "%s: n_agents out of range", who);
  MARL_REQUIRE(cfg->n_nets >= 1 && cfg->n_nets <= cfg->n_agents, "%s: n_nets out of range", who);
  MARL_REQUIRE(cfg->hidden >= 1 && cfg->hidden <= kHidden, "%s: hidden width %d not supported (layers = [H, H], 1 <= H <= %d)", who, cfg->hidden, kHidden);
  MARL_REQUIRE(cfg->in_dim >= 1 && cfg->in_dim <= max_in, "%s: obs dim %d not supported (1..%d)", who, cfg->in_dim, max_in);
  MARL_REQUIRE(cfg->out_dim >= 1 && cfg->out_dim <= kOutPad, "%s: output width %d not supported (1..%d)", who, cfg->out_dim, kOutPad);
  for (int a = 0; a < cfg->n_agents; ++a) MARL_REQUIRE(cfg->agent_net[a] >= 0 && cfg->agent_net[a] < cfg->n_nets, "%s: agent_net[%d] out of range", who, a);
  return MARL_OK;
}

inline NetSet to_netset(const marl_mlp_cfg* cfg) {
  NetSet ns; ns.n_agents = cfg->n_agents; ns.n_nets = cfg->n_nets; ns.in = cfg->in_dim; ns.out = cfg->out_dim;
  memcpy(ns.agent_net, cfg->agent_net, sizeof(int) * MARL_MAX_AGENTS);
  ns.lay = NetLayout::make(cfg->in_dim, cfg->out_dim, cfg->hidden);
  return ns;
}

// ---- host side: the handle layer of the learner C ABIs ---------------------------------------------------------------------------------------
// A learner handle (marl_dqn, marl_a2c) derives from LearnerHandle and adds its networks and hyper-parameters `hp`.  Every device buffer it
// allocates comes from alloc_buffers and is released by destroy_handle.
struct LearnerHandle : BufferOwner {
  int device = 0, n_sm = 148;
  int64_t n_params = 0;          // trainable floats of theta, m and v (grad: + 4 loss statistics)
  int scratch_pitch = 0;         // floats per CTA of `scratch`: the largest network's P rounded up to 4
  float *theta = nullptr, *theta_tgt = nullptr, *m = nullptr, *v = nullptr, *grad = nullptr, *scratch = nullptr, *loss_part = nullptr;
  int32_t* idx = nullptr;
  uint8_t* image = nullptr;      // packed weight images for the tensor-core forward path (NULL: hidden width below 128)
  marl_optimizer opt = {};       // the optimiser (marl_*_set_optimizer; Adam with hp's constants by default)
  bool opt_stepped = false;      // an optimiser step has been launched: the state in m / v belongs to `opt`
  // standardise_returns: RunningMeanStd of n_stat columns -- mean[n_stat] | var[n_stat] (float32), count (a Python float in the reference),
  // per-block partial sums (retms.cuh)
  int standardise = 0, n_stat = 0; float* ret_ms = nullptr; double *ret_count = nullptr, *ret_part = nullptr;
};

// create's prologue: the device, its SM count and the default optimiser, Adam with hp's constants
template <typename H, typename HP>
int open_learner(int device, const HP& hp, H** out) {
  if (int rc = check_device(device)) return rc;
  H* h = new H();
  h->hp = hp; h->device = device;
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, device); h->n_sm = prop.multiProcessorCount;
  h->opt.kind = MARL_OPT_ADAM; h->opt.beta1 = hp.beta1; h->opt.beta2 = hp.beta2; h->opt.eps = hp.eps;
  *out = h;
  return MARL_OK;
}

// marl_*_set_optimizer up to the learner's own checks: the handle, the argument, no step taken yet
inline int check_set_optimizer(const LearnerHandle* h, const marl_optimizer* o, const char* who) {
  MARL_REQUIRE(h != nullptr, "%s: NULL handle", who);
  if (int rc = check_optimizer(o, who)) return rc;
  MARL_REQUIRE(!h->opt_stepped, "%s: the learner has already taken an optimiser step; choose the optimiser right after creation", who);
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  return MARL_OK;
}

// ... and after them: zero the optimiser state and switch to `o`
inline int reset_optimizer(LearnerHandle* h, const marl_optimizer& o) {
  MARL_CUDA_TRY(cudaMemset(h->m, 0, h->n_params * sizeof(float)));
  MARL_CUDA_TRY(cudaMemset(h->v, 0, h->n_params * sizeof(float)));
  h->opt = o;
  return MARL_OK;
}

}  // namespace marl
