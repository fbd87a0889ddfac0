// dqn.cu -- C ABI of the IDQN / VDN learner (marl_dqn_*), host-side orchestration of the fused kernels.
//
// Replaces marlbase/dqn/model.py: QNetwork (14-196) and VDNetwork (199-269) -- act's forward pass, _compute_loss,
// update (zero_grad/backward/clip/Adam), update_target/hard_update/soft_update -- and ReplayBuffer.sample's index
// draw + gather (marlbase/dqn/train.py:94-124).
#include "learner.cuh"
#include "dqn_heads.cuh"
#include "retms.cuh"
#include "qmix.cuh"
#include "gru.cuh"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace marl {

// ---- replay sampling: np.random.randint(0, len(rb), batch) with replacement (dqn/train.py:95) ------------------
__global__ void replay_sample_kernel(uint64_t seed, uint64_t update_idx, int batch, int n_valid, int32_t* idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  pdl_wait();
  pdl_launch_dependents();
  if (i >= batch) return;
  const u32x4 b = philox4x32_10((uint32_t)update_idx, (uint32_t)(update_idx >> 32), (uint32_t)(i >> 2), 0u, (uint32_t)seed, (uint32_t)(seed >> 32) ^ kTagSample);
  idx[i] = (int32_t)bounded(pick(b, i & 3), (uint32_t)n_valid);
}

// ---- TD error over C columns of G agents (marlbase/dqn/model.py:138-163, VDN 224-269) -----------------------------
// Column c sums the Q-values and bootstrap values of agents [c G, c G + G) and takes agent c G's reward.  VDN: C = 1, G = N; independent learners
// (the recurrent pass, whose backward has no TD head of its own; standardise_returns): C = N, G = 1.  One thread per (c, b, t).
//   STAGE 0: td[c][b][t] = dLoss/dQ filled (2 delta; Huber: clamp(delta, -huber, huber)) and the loss statistics.
//   STAGE 1 (standardise_returns, dqn/model.py:147-158, VDN 256-264: the TD target needs statistics of the whole batch's returns before any loss):
//            ret = r + gamma (next * sqrt(var) + mean) (1 - done[t + 1]) and chosen = Q(o_t)[a_t], for every (b, t), filled or not, as the
//            reference.  Columns of the statistics: one per agent (IDQN); the reference's VDN reshapes its (E, B) returns with reshape(-1, B), i.e.
//            one column per batch entry -- stat_per_b selects that.  ret_ms_step (retms.cuh) then absorbs and standardises ret in place.
//   STAGE 2: td from chosen and the standardised returns, and the loss statistics.
//   STAGE 3 (algorithm.td_lambda): the bootstrap value boot[c][b][t] = v_{t+1} (unstandardised with the statistics so far when ret_ms is set; no
//            reward or done applied) and chosen, for every (b, t); td_lambda_kernel then turns them into the λ-returns in ret, which STAGE 2 reads.
struct ColTdParams {
  const float* q; const float* tq;  // [N][B][T+1][A]
  TrajView traj; const int32_t* idx; int B, A; float gamma; int double_q;
  int C, G;
  float huber;       // STAGES 0, 2: algorithm.huber_delta (> 0: the Huber TD loss; <= 0: the squared error)
  const float* ret_ms; int n_stat, stat_per_b;   // STAGE 1 (STAGE 3: or NULL): mean[n_stat] | var[n_stat]
  float* ret; float* chosen;                     // STAGES 1, 2, 3: [C][B][T]
  float* boot;       // STAGE 3: [C][B][T]
  float* td;         // [C][B][T] = td_dloss(delta) * filled
  float* loss_part;  // [gridDim][4]
};

// loss_part[block] = (sum of loss, sum of fill, 0, 0) over the block's 256 threads, in a fixed tree order
__device__ __forceinline__ void block_loss_part(float loss, float fill, float* loss_part) {
  __shared__ float red[512];
  red[threadIdx.x] = loss; red[256 + threadIdx.x] = fill;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) { red[threadIdx.x] += red[threadIdx.x + s]; red[256 + threadIdx.x] += red[256 + threadIdx.x + s]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { loss_part[4 * blockIdx.x] = red[0]; loss_part[4 * blockIdx.x + 1] = red[256]; loss_part[4 * blockIdx.x + 2] = 0.f; loss_part[4 * blockIdx.x + 3] = 0.f; }
}

template <int STAGE>
__global__ void __launch_bounds__(256) col_td_kernel(ColTdParams p) {
  const int T = p.traj.T, i = blockIdx.x * 256 + threadIdx.x;
  float loss = 0.f, fill = 0.f;
  if (i < p.C * p.B * T) {
    const int c = i / (p.B * T), rem = i - c * p.B * T, b = rem / T, t = rem - b * T;
    const size_t ep = (size_t)p.idx[b];
    if constexpr (STAGE == 2) {
      p.td[i] = td_error(p.chosen[i], p.ret[i], (float)p.traj.filled[p.traj.filled_at(ep, t)], c == 0, loss, fill, p.huber);
    } else {
      float chosen = 0.f, next = 0.f;
      for (int a = c * p.G; a < (c + 1) * p.G; ++a) {
        const size_t row = row_index(a, b, t, p.B, T + 1);
        const float* q0 = p.q + row * p.A;
        chosen += q0[p.traj.act[p.traj.step_at(ep, a, t)]];
        next += next_value(q0 + p.A, p.tq + (row + 1) * p.A, p.A, p.double_q);
      }
      const float rew = p.traj.rew[p.traj.step_at(ep, c * p.G, t)], done1 = (float)p.traj.done[p.traj.done_at(ep, t + 1)];
      if constexpr (STAGE == 0) {
        p.td[i] = td_error(chosen, td_target(rew, p.gamma, next, done1), (float)p.traj.filled[p.traj.filled_at(ep, t)], c == 0, loss, fill, p.huber);
      } else if constexpr (STAGE == 1) {
        const int col = p.stat_per_b ? b : c;
        p.ret[i] = td_target_rn(rew, p.gamma, unstandardise(next, p.ret_ms[col], p.ret_ms[p.n_stat + col]), done1);
        p.chosen[i] = chosen;
      } else {
        const int col = p.stat_per_b ? b : c;
        p.boot[i] = p.ret_ms ? unstandardise(next, p.ret_ms[col], p.ret_ms[p.n_stat + col]) : next;
        p.chosen[i] = chosen;
      }
    }
  }
  if constexpr (STAGE == 0 || STAGE == 2) block_loss_part(loss, fill, p.loss_part);
}

// TD(λ) targets (algorithm.td_lambda) of C columns over the sampled episodes, from the bootstrap values boot[c][b][t] = v_{t+1}:
//   G_t = b_t + a_t G_{t+1},  a_t = γλ (1 - d_{t+1}) f_{t+1},  b_t = r_t + γ (1 - d_{t+1}) (1 - λ f_{t+1}) v_{t+1},  f_T := 0,
// for every t in [0, T), filled or not; r_t is agent c G's reward.  The chain stops at the first unfilled row after t: a stale tail never reaches a
// filled row's target.  One warp per (column, episode) sequence, right to left over windows of 32 x kTdlChunk steps: the warp stages (a_t, b_t)
// coalesced in shared memory, each lane folds its chunk into the affine map G_in -> c + g G_in, a fixed-order suffix scan over the lanes composes the
// maps, each lane replays its chunk from the return after it, and the warp writes the returns coalesced.  The window's first return carries into the next.
constexpr int kTdlChunk = 8, kTdlWindow = 32 * kTdlChunk, kTdlWarps = 8;

struct TdLambdaParams {
  const float* boot;   // [C][B][T]
  TrajView traj; const int32_t* idx; int C, G, B;
  float gamma, lambda, gl;   // gl = float32(γλ)
  float* ret;          // [C][B][T]
};

__device__ __forceinline__ int tdl_slot(int s) { return (s / kTdlChunk) * (kTdlChunk + 1) + s % kTdlChunk; }   // lane chunks padded: no bank conflicts

__global__ void __launch_bounds__(32 * kTdlWarps) td_lambda_kernel(TdLambdaParams p) {
  __shared__ float sa[kTdlWarps][32 * (kTdlChunk + 1)], sb[kTdlWarps][32 * (kTdlChunk + 1)];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, seq = blockIdx.x * kTdlWarps + w;
  if (seq >= p.C * p.B) return;
  const int T = p.traj.T, c = seq / p.B, b = seq - c * p.B;
  const size_t ep = (size_t)p.idx[b];
  const float* boot = p.boot + (size_t)seq * T;
  const float* rew = p.traj.rew + p.traj.step_at(ep, c * p.G, 0);
  const uint8_t* done = p.traj.done + p.traj.done_at(ep, 0);
  const uint8_t* filled = p.traj.filled + p.traj.filled_at(ep, 0);
  float* ret = p.ret + (size_t)seq * T;
  float* a_s = sa[w];
  float* b_s = sb[w];
  float carry = 0.f;   // G at the step after the window
  for (int w0 = ((T - 1) / kTdlWindow) * kTdlWindow; w0 >= 0; w0 -= kTdlWindow) {
    const int len = min(kTdlWindow, T - w0);
    for (int j = lane; j < len; j += 32) {
      const int t = w0 + j;
      const float live1 = 1.f - (float)done[t + 1], f1 = t + 1 < T ? (float)filled[t + 1] : 0.f;
      a_s[tdl_slot(j)] = p.gl * live1 * f1;
      b_s[tdl_slot(j)] = rew[t] + (p.gamma * live1) * ((1.f - p.lambda * f1) * boot[t]);
    }
    __syncwarp();
    const int lo = lane * kTdlChunk, hi = min(lo + kTdlChunk, len);
    float cc = 0.f, g = 1.f;   // this lane's chunk: G_lo = cc + g G_hi
    for (int j = hi - 1; j >= lo; --j) { cc = b_s[tdl_slot(j)] + a_s[tdl_slot(j)] * cc; g *= a_s[tdl_slot(j)]; }
    // suffix scan: lane l ends with the composition of the maps of lanes l .. 31
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const float c2 = __shfl_down_sync(0xffffffffu, cc, off), g2 = __shfl_down_sync(0xffffffffu, g, off);
      if (lane + off < 32) { cc = cc + g * c2; g *= g2; }
    }
    float r = __shfl_down_sync(0xffffffffu, cc + g * carry, 1);   // G at the step after this lane's chunk
    if (lane == 31) r = carry;
    for (int j = hi - 1; j >= lo; --j) { r = b_s[tdl_slot(j)] + a_s[tdl_slot(j)] * r; b_s[tdl_slot(j)] = r; }
    carry = __shfl_sync(0xffffffffu, r, 0);   // G_{w0}, as written
    __syncwarp();
    for (int j = lane; j < len; j += 32) ret[w0 + j] = b_s[tdl_slot(j)];
    __syncwarp();
  }
}

static cudaError_t launch_td_lambda(const TdLambdaParams& p, cudaStream_t st) {
  td_lambda_kernel<<<(p.C * p.B + kTdlWarps - 1) / kTdlWarps, 32 * kTdlWarps, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace marl

using namespace marl;

struct marl_dqn : LearnerHandle {
  NetSet ns;
  marl_dqn_hp hp;
  int max_batch = 0, max_T = 0;
  size_t loss_part_n = 0;   // 4-float blocks of loss statistics that loss_part holds
  float *tq = nullptr, *q_all = nullptr, *td = nullptr, *loss_dev = nullptr, *sumsq = nullptr;
  bool grads_are_local = false;  // set by update_grads, cleared when the caller may have all-reduced grad
  uint8_t* image_tgt = nullptr;  // image of theta_tgt, rebuilt only when the target network changed
  uint8_t* image_bwd = nullptr;  // MN-major image of W2 (online net) for the tensor-core backward
  float *tc_h2 = nullptr, *tc_rec = nullptr, *tc_x = nullptr;
  bool tgt_image_current = false;
  unsigned long long* grid_barrier = nullptr; unsigned long long grid_epoch = 0;   // arrival counter of the fused reduce + Adam kernel
  // gradient exchange over peer memory (several ranks, one process per GPU): own buffer + the peers' buffers opened through CUDA IPC
  XchgParams xchg = {}; float* xbuf = nullptr; void* peer_base[kMaxRanks] = {};
  // online images: valid = a full pack happened and every later change of theta came from adam_kernel (which updates them in place)
  bool image_current = false, bwd_image_current = false;
  int64_t updates = 0, last_target_update = 0;
  RowPlan train_plan; int n_loss_parts = 0;
  // optional CUDA-event timing of the training kernel (bench.py's roofline leg)
  // measurement hook: 4 events per timed update (before the training pass, after each of its kernels; the FP32 path uses 0 and 3)
  bool timing = false; std::vector<cudaEvent_t> ev; int ev_used = 0; bool ev_split = false;
  // cfg.standardise_returns, algorithm.td_lambda: returns / chosen-Q scratch next to the statistics
  float *ret = nullptr, *chosen = nullptr;
  // algorithm.td_lambda (marl_dqn_set_td_lambda): λ-returns in place of the one-step target; boot: the bootstrap values v_{t+1} per (column, b, t)
  bool td_lambda_on = false; float td_lambda = 0.f; float* boot = nullptr;
  // algorithm.huber_delta (marl_dqn_set_huber_delta): the Huber TD loss's delta; 0: the reference's squared error
  float huber = 0.f;
  // QMIX (hp.mixer == 2): the mixing network's parameters / Adam state / gradient (+ 4 statistics), per-sample records, chunked partial sums, tile list
  QmixLayout ql = {}; float *mix = nullptr, *mix_tgt = nullptr, *mix_m = nullptr, *mix_v = nullptr, *mix_grad = nullptr, *mix_rec = nullptr, *mix_part = nullptr, *mix_img = nullptr, *mix_img_tgt = nullptr;
  QmixTile* mix_tiles = nullptr; int mix_n_tiles = 0; QmixMicro* mix_micro = nullptr; int mix_n_micro = 0; bool mix_wgrad_tiles = false;
  // recurrent agent networks (marl_dqn_create_rnn): GRU parameter layout and the online pass's saved rows [N][B][T+1][kGruSaveRow]
  bool rnn = false; GruLayout gl = {}; float* gru_save = nullptr;
  int P() const { return rnn ? gl.P : ns.lay.P; }
};
static const int kTimingPairs = 1024;

// loss_part only ever grows: standardise_returns and the QMIX mixer each need room for their own statistics blocks, in either call order
static int dqn_grow_loss_part(marl_dqn* h, size_t blocks, const char* who) {
  if (blocks <= h->loss_part_n) return MARL_OK;
  free_buffer(h, &h->loss_part); h->loss_part_n = 0;
  if (int rc = alloc_buffers(h, who, {{&h->loss_part, 4 * blocks * sizeof(float)}})) return rc;
  h->loss_part_n = blocks;
  return MARL_OK;
}

extern "C" {

static int dqn_create(const marl_mlp_cfg* cfg, const marl_dqn_hp* hp, int32_t max_batch, int32_t max_T, int32_t device, bool rnn, marl_dqn** out) {
  MARL_REQUIRE(cfg && hp && out, "marl_dqn_create: NULL argument");
  *out = nullptr;
  // the recurrent kernels take kMaxObsDim inputs; the MLP kernels' limit (learner_kernels_init) depends on the path that runs
  const char* who = rnn ? "marl_dqn_create_rnn" : "marl_dqn_create";
  if (int rc = check_mlp_cfg(cfg, who, rnn ? kMaxObsDim : kMaxInDim)) return rc;
  MARL_REQUIRE(max_batch >= 1 && max_T >= 1, "marl_dqn_create: max_batch/max_T must be >= 1");
  MARL_REQUIRE(hp->mixer >= 0 && hp->mixer <= 2, "marl_dqn_create: mixer must be 0 (independent), 1 (VDN) or 2 (QMIX)");
  marl_dqn* h = nullptr;
  if (int rc = open_learner(device, *hp, &h)) return rc;
  h->ns = to_netset(cfg);
  h->max_batch = max_batch; h->max_T = max_T;
  h->rnn = rnn; h->gl = GruLayout::make(cfg->in_dim, cfg->out_dim, cfg->hidden);
  h->n_params = (int64_t)cfg->n_nets * h->P();
  h->scratch_pitch = (h->P() + 3) & ~3;
  const size_t rows = (size_t)cfg->n_agents * max_batch * (max_T + 1), F = sizeof(float);
  int rc = alloc_buffers(h, who, {{&h->theta, h->n_params * F}, {&h->theta_tgt, h->n_params * F}, {&h->m, h->n_params * F}, {&h->v, h->n_params * F},
                                  {&h->grad, (h->n_params + 4) * F}, {&h->scratch, (size_t)h->n_sm * h->scratch_pitch * F}});
  if (!rc) rc = dqn_grow_loss_part(h, (size_t)h->n_sm + (size_t)(rnn ? cfg->n_agents : 1) * max_batch * max_T / 256 + 2, who);
  if (!rc)
    rc = alloc_buffers(h, who, {{&h->tq, rows * cfg->out_dim * F}, {&h->loss_dev, 8 * F}, {&h->sumsq, ((size_t)(h->n_params + 63) / 64 + 1) * F},
                                {&h->grid_barrier, sizeof(unsigned long long)}});   // the grid barrier's zero-initialised 64-bit arrival counter
  // online Q-values of every row for the external TD heads (VDN, QMIX; the recurrent pass always hands the TD error to its backward) and the TD
  // error: VDN one entry per (b, t), QMIX and the recurrent pass one per (agent, b, t)
  if (!rc && (hp->mixer != 0 || rnn))
    rc = alloc_buffers(h, who, {{&h->q_all, rows * cfg->out_dim * F}, {&h->td, (size_t)(hp->mixer == 1 ? 1 : cfg->n_agents) * max_batch * max_T * F}});
  if (!rc) rc = alloc_buffers(h, who, {{&h->idx, max_batch * F}});
  if (!rc && rnn) {
    rc = alloc_buffers(h, who, {{&h->gru_save, rows * kGruSaveRow * F}});
  } else if (!rc && cfg->hidden == kHidden) {   // the tensor-core images exist for 128-wide networks only: narrower ones run the FP32 kernels
    const size_t image_bytes = ((size_t)cfg->n_nets * tc_image_bytes() / 4 + 4) * F;
    rc = alloc_buffers(h, who, {{&h->image, image_bytes}, {&h->image_tgt, image_bytes}});
  }
  if (rc) { marl_dqn_destroy(h); return rc; }
  if (rnn) {
    if (int rc2 = gru_kernels_init()) { marl_dqn_destroy(h); return rc2; }
  } else {
    if (int rc2 = learner_kernels_init(cfg->in_dim, kMaxObsDim)) { marl_dqn_destroy(h); return rc2; }
    if (int rc2 = tc_forward_init()) { marl_dqn_destroy(h); return rc2; }
    if (int rc2 = tc_train_init()) { marl_dqn_destroy(h); return rc2; }
  }
  *out = h;
  return MARL_OK;
}

int marl_dqn_create(const marl_mlp_cfg* cfg, const marl_dqn_hp* hp, int32_t max_batch, int32_t max_T, int32_t device, marl_dqn** out) {
  return dqn_create(cfg, hp, max_batch, max_T, device, false, out);
}

int marl_dqn_create_rnn(const marl_mlp_cfg* cfg, const marl_dqn_hp* hp, int32_t max_batch, int32_t max_T, int32_t device, marl_dqn** out) {
  return dqn_create(cfg, hp, max_batch, max_T, device, true, out);
}

int marl_dqn_destroy(marl_dqn* h) {
  if (!h) return MARL_OK;
  cudaSetDevice(h->device);
  for (int r = 0; r < kMaxRanks; ++r) if (h->peer_base[r] != nullptr && r != h->xchg.rank) cudaIpcCloseMemHandle(h->peer_base[r]);
  for (auto& e : h->ev) cudaEventDestroy(e);
  return destroy_handle(h);
}

// (column, b, t) entries of the external TD head at max_batch and max_T: one column per agent (IDQN), one of all agents (VDN, QMIX)
static size_t dqn_head_entries(const marl_dqn* h) { return (size_t)(h->hp.mixer != 0 ? 1 : h->ns.n_agents) * h->max_batch * h->max_T; }

// The external TD head's buffers (standardise_returns, algorithm.td_lambda), each allocated where missing: returns and chosen Q-values per entry,
// the online Q-values of every row, the TD error (IDQN's MLP path has none yet; every other learner's was sized at create: QMIX's and the recurrent
// pass's per agent) and room for the head's loss statistics, one block per 256 entries (QMIX: per tile, sized by marl_dqn_qmix_init).
static int dqn_external_buffers(marl_dqn* h, const char* who) {
  const size_t rows = (size_t)h->ns.n_agents * h->max_batch * (h->max_T + 1), cbt = dqn_head_entries(h), F = sizeof(float);
  if (!h->ret)
    if (int rc = alloc_buffers(h, who, {{&h->ret, cbt * F}, {&h->chosen, cbt * F}})) return rc;
  if (!h->q_all)
    if (int rc = alloc_buffers(h, who, {{&h->q_all, rows * h->ns.out * F}})) return rc;
  if (!h->td)
    if (int rc = alloc_buffers(h, who, {{&h->td, cbt * F}})) return rc;
  return dqn_grow_loss_part(h, (size_t)h->n_sm + cbt / 256 + 2, who);
}

/* cfg.standardise_returns (dqn/model.py:82-84, 221-222, 357-358): RunningMeanStd over the TD targets, one column per agent (VDN and QMIX: per
 * batch entry, see the kernels above and qmix.cuh); mean 0, var 1, count 1e-4 on first enable. */
int marl_dqn_standardise_returns(marl_dqn* h, int32_t enable) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_standardise_returns: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  if (enable && !h->ret_ms) {
    const char* who = "marl_dqn_standardise_returns";
    if (int rc = dqn_external_buffers(h, who)) return rc;
    if (int rc = enable_ret_stats(h, h->hp.mixer != 0 ? h->max_batch : h->ns.n_agents, who)) return rc;
  }
  h->standardise = enable ? 1 : 0;
  return MARL_OK;
}
/* algorithm.td_lambda: enable != 0 replaces the one-step TD target of every later update (marl_dqn_update*, update_n, the fused tail) by the λ-return
 * of `lambda` in [0, 1] over the sampled episode (DESIGN.md §4.4d); enable == 0 restores the one-step target.  The first enable allocates the
 * bootstrap values and the rest of the external TD head's buffers, which IDQN then takes on every path. */
int marl_dqn_set_td_lambda(marl_dqn* h, int32_t enable, float lambda) {
  MARL_REQUIRE(!enable || (lambda >= 0.f && lambda <= 1.f), "marl_dqn_set_td_lambda: lambda %g is outside [0, 1]", (double)lambda);
  MARL_REQUIRE(h != nullptr, "marl_dqn_set_td_lambda: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  if (enable && !h->boot) {
    const char* who = "marl_dqn_set_td_lambda";
    if (int rc = dqn_external_buffers(h, who)) return rc;
    if (int rc = alloc_buffers(h, who, {{&h->boot, dqn_head_entries(h) * sizeof(float)}})) return rc;
  }
  h->td_lambda_on = enable != 0;
  h->td_lambda = enable ? lambda : 0.f;
  return MARL_OK;
}

/* algorithm.huber_delta: enable != 0 replaces the squared TD error of every later update (marl_dqn_update*, update_n, the fused tail) by
 * torch.nn.functional.huber_loss with delta = `delta` > 0 (DESIGN.md §4.4e); enable == 0 restores the squared error.  Every TD head takes delta
 * as a run-time argument, so nothing is allocated and every path stays the one it was. */
int marl_dqn_set_huber_delta(marl_dqn* h, int32_t enable, float delta) {
  MARL_REQUIRE(!enable || (delta > 0.f && isfinite(delta)), "marl_dqn_set_huber_delta: delta %g must be a finite number > 0", (double)delta);
  MARL_REQUIRE(h != nullptr, "marl_dqn_set_huber_delta: NULL handle");
  h->huber = enable ? delta : 0.f;
  return MARL_OK;
}

int marl_dqn_ret_ms_ptrs(marl_dqn* h, float** ret_ms, double** count, int32_t* n_stat) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_ret_ms_ptrs: NULL handle");
  if (ret_ms) *ret_ms = h->ret_ms; if (count) *count = h->ret_count; if (n_stat) *n_stat = h->n_stat;
  return MARL_OK;
}

int marl_dqn_scratch_ptrs(marl_dqn* h, float** boot, float** ret, float** chosen, float** td) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_scratch_ptrs: NULL handle");
  if (boot) *boot = h->boot; if (ret) *ret = h->ret; if (chosen) *chosen = h->chosen; if (td) *td = h->td;
  return MARL_OK;
}

/* QMixNetwork.__init__ (dqn/model.py:365-379): the mixing network over the concatenated observations (state_dim = N * in_dim).  Parameters are
 * initialised by the caller through marl_dqn_qmix_ptrs (nn.Linear defaults), then marl_dqn_sync_target copies them to the target mixer. */
typedef void (*QmixMixFn)(QmixParams, const float*, const float*);
static QmixMixFn qmix_mix_fn(int hl, int mode) {
  static const QmixMixFn fns[2][4] = {{qmix_mix_kernel<1, 0>, qmix_mix_kernel<1, 1>, qmix_mix_kernel<1, 2>, qmix_mix_kernel<1, 3>},
                                      {qmix_mix_kernel<2, 0>, qmix_mix_kernel<2, 1>, qmix_mix_kernel<2, 2>, qmix_mix_kernel<2, 3>}};
  return fns[hl - 1][mode];
}

int marl_dqn_qmix_init(marl_dqn* h, int32_t embed_dim, int32_t hypernet_layers, int32_t hypernet_embed) {
  MARL_REQUIRE(h != nullptr && h->hp.mixer == 2, "marl_dqn_qmix_init: the learner was not created with mixer = 2");
  MARL_REQUIRE(h->mix == nullptr, "marl_dqn_qmix_init: already initialised");
  MARL_REQUIRE(hypernet_layers == 1 || hypernet_layers == 2, "marl_dqn_qmix_init: hypernet_layers = %d: the reference's QMixer has 1 or 2 hypernetwork layers", hypernet_layers);
  MARL_REQUIRE(embed_dim >= 4 && embed_dim <= kQmixEmbedMax && embed_dim % 4 == 0, "marl_dqn_qmix_init: embed_dim %d not supported (multiple of 4, <= %d)", embed_dim, kQmixEmbedMax);
  MARL_REQUIRE(hypernet_layers == 1 || (hypernet_embed >= 4 && hypernet_embed <= kQmixHypMax && hypernet_embed % 4 == 0),
               "marl_dqn_qmix_init: hypernet_embed %d not supported (multiple of 4, <= %d)", hypernet_embed, kQmixHypMax);
  const int N = h->ns.n_agents, S = N * h->ns.in;
  MARL_REQUIRE(S <= kQmixStateMax && N <= kQmixAgentsMax, "marl_dqn_qmix_init: state_dim %d (<= %d) or n_agents %d (<= %d) too large", S, kQmixStateMax, N, kQmixAgentsMax);
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  h->ql = qmix_layout(N, S, embed_dim, hypernet_embed, hypernet_layers);
  const size_t n = (size_t)h->ql.n, samples = (size_t)h->max_batch * h->max_T;
  MARL_REQUIRE(qm_smem_bytes(h->ql) <= 227 * 1024, "marl_dqn_qmix_init: the mixer's %zu resident parameters + a 32-sample tile (%zu bytes) do not fit shared memory",
               n - (size_t)h->ql.res0, qm_smem_bytes(h->ql));
  std::vector<QmixTile> tiles(kQmixMaxTiles);
  const int nt = qmix_tiles(h->ql, tiles.data());
  MARL_REQUIRE(nt > 0, "marl_dqn_qmix_init: too many weight-gradient tiles");
  const char* who = "marl_dqn_qmix_init";
  const size_t F = sizeof(float), n_img = (n + 3) & ~(size_t)3;
  if (int rc = alloc_buffers(h, who, {{&h->mix, n * F}, {&h->mix_tgt, n * F}, {&h->mix_m, n * F}, {&h->mix_v, n * F}, {&h->mix_grad, (n + 4) * F},
                                      {&h->mix_rec, (size_t)h->ql.R * samples * F}, {&h->mix_part, (size_t)(2 * h->n_sm > kQmixChunks ? 2 * h->n_sm : kQmixChunks) * n * F},
                                      {&h->mix_tiles, (size_t)nt * sizeof(QmixTile)}, {&h->mix_img, n_img * F}, {&h->mix_img_tgt, n_img * F}}))
    return rc;
  if (int rc = dqn_grow_loss_part(h, (size_t)h->n_sm + samples / kQmTS + 2, who)) return rc;   // one block of statistics per tile of kQmTS samples
  MARL_CUDA_TRY(cudaMemcpy(h->mix_tiles, tiles.data(), (size_t)nt * sizeof(QmixTile), cudaMemcpyHostToDevice));
  h->mix_n_tiles = nt;
  std::vector<QmixMicro> micro(1 << 14);
  const int nm = qmix_micro_tiles(h->ql, micro.data(), (int)micro.size());
  MARL_REQUIRE(nm > 0, "marl_dqn_qmix_init: too many weight-gradient micro-tiles");
  if (int rc = alloc_buffers(h, who, {{&h->mix_micro, (size_t)nm * sizeof(QmixMicro)}})) return rc;
  MARL_CUDA_TRY(cudaMemcpy(h->mix_micro, micro.data(), (size_t)nm * sizeof(QmixMicro), cudaMemcpyHostToDevice));
  h->mix_n_micro = nm;
  // the attribute is per function, process-wide: only ever raise it (a second learner with a smaller mixer must not lower the first one's limit).
  // Every instantiation of qmix_mix_kernel is a function of its own; standardise_returns and td_lambda may be switched on after this call, so all
  // four modes.
  static size_t mix_limits[64][2][4] = {}, wg_limits[64] = {};   // per device (one process normally drives one GPU)
  size_t& wg_smem_limit = wg_limits[h->device & 63];
  const size_t wg_smem = (size_t)(h->ql.R + 2) * kQmP * sizeof(float);
  const char* ev = getenv("MARL_QMIX_WGRAD_TILES");
  h->mix_wgrad_tiles = (ev != nullptr && ev[0] == '1') || wg_smem > 110 * 1024;   // the single-read form needs all record fields of 32 samples in shared memory
  if (!h->mix_wgrad_tiles && wg_smem > wg_smem_limit) {
    MARL_CUDA_TRY(cudaFuncSetAttribute(qmix_wgrad2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wg_smem));
    wg_smem_limit = wg_smem;
  }
  for (int mode = 0; mode < 4; ++mode) {
    size_t& mix_smem_limit = mix_limits[h->device & 63][hypernet_layers - 1][mode];
    if (qm_smem_bytes(h->ql) > mix_smem_limit) {
      MARL_CUDA_TRY(cudaFuncSetAttribute(qmix_mix_fn(hypernet_layers, mode), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)qm_smem_bytes(h->ql)));
      mix_smem_limit = qm_smem_bytes(h->ql);
    }
  }
  return MARL_OK;
}
/* Host-only self-check of the QMIX weight-gradient decompositions (no device needed): counts[0 .. n) = how many micro-tile entries of the single-read
 * kernel write parameter j, counts[n .. 2n) = the same for the 32 x 32 tile form; both must be 1 everywhere.  Returns n through n_params. */
int marl_debug_qmix_coverage_layers(int32_t n_agents, int32_t state_dim, int32_t embed_dim, int32_t hypernet_layers, int32_t hypernet_embed, int32_t* counts,
                                    int64_t cap, int64_t* n_params) {
  MARL_REQUIRE(n_agents >= 1 && state_dim >= 1 && embed_dim >= 4 && n_params != nullptr, "marl_debug_qmix_coverage: bad argument");
  MARL_REQUIRE(hypernet_layers == 1 || (hypernet_layers == 2 && hypernet_embed >= 4), "marl_debug_qmix_coverage: hypernet_layers = %d (1 or 2) / hypernet_embed = %d",
               hypernet_layers, hypernet_embed);
  const QmixLayout L = qmix_layout(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers);
  *n_params = L.n;
  if (counts == nullptr) return MARL_OK;
  MARL_REQUIRE(cap >= 2 * (int64_t)L.n, "marl_debug_qmix_coverage: counts needs 2 x %d entries", L.n);
  for (int j = 0; j < 2 * L.n; ++j) counts[j] = 0;
  std::vector<QmixMicro> micro(1 << 16);
  const int nm = qmix_micro_tiles(L, micro.data(), (int)micro.size());
  MARL_REQUIRE(nm > 0, "marl_debug_qmix_coverage: too many micro-tiles");
  for (int m = 0; m < nm; ++m) {
    const QmixMicro& mt = micro[m];
    for (int oo = 0; oo < mt.n_o; ++oo)
      for (int ii = 0; ii < 8; ++ii) {
        const int o = mt.o0 + oo, i = mt.i0 + ii;
        if (i < mt.I) counts[mt.woff + o * mt.I + i] += 1;
        else if (i == mt.I) counts[mt.boff + o] += 1;
      }
  }
  std::vector<QmixTile> tiles(kQmixMaxTiles);
  const int nt = qmix_tiles(L, tiles.data());
  MARL_REQUIRE(nt > 0, "marl_debug_qmix_coverage: too many tiles");
  for (int t = 0; t < nt; ++t) {
    const QmixTile& tl = tiles[t];
    for (int oo = 0; oo < 32; ++oo)
      for (int ii = 0; ii < 32; ++ii) {
        const int o = tl.o0 + oo, i = tl.i0 + ii;
        if (o >= tl.O) continue;
        if (i < tl.I) counts[L.n + tl.woff + o * tl.I + i] += 1;
        else if (i == tl.I) counts[L.n + tl.boff + o] += 1;
      }
  }
  return MARL_OK;
}

int marl_debug_qmix_coverage(int32_t n_agents, int32_t state_dim, int32_t embed_dim, int32_t hypernet_embed, int32_t* counts, int64_t cap, int64_t* n_params) {
  return marl_debug_qmix_coverage_layers(n_agents, state_dim, embed_dim, 2, hypernet_embed, counts, cap, n_params);
}

int marl_dqn_qmix_ptrs(marl_dqn* h, float** mix, float** mix_tgt, float** adam_m, float** adam_v, float** grad, int64_t* n_params) {
  MARL_REQUIRE(h != nullptr && h->mix != nullptr, "marl_dqn_qmix_ptrs: no mixer (marl_dqn_qmix_init)");
  if (mix) *mix = h->mix; if (mix_tgt) *mix_tgt = h->mix_tgt; if (adam_m) *adam_m = h->mix_m; if (adam_v) *adam_v = h->mix_v;
  if (grad) *grad = h->mix_grad; if (n_params) *n_params = h->ql.n;
  return MARL_OK;
}

int marl_dqn_param_ptrs(marl_dqn* h, float** theta, float** theta_tgt, float** adam_m, float** adam_v, float** grad, int64_t* n_params) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_param_ptrs: NULL handle");
  if (theta) *theta = h->theta; if (theta_tgt) *theta_tgt = h->theta_tgt; if (adam_m) *adam_m = h->m; if (adam_v) *adam_v = h->v;
  if (grad) *grad = h->grad; if (n_params) *n_params = h->n_params;
  return MARL_OK;
}

int marl_dqn_sync_target(marl_dqn* h, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_sync_target: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  MARL_CUDA_TRY(cudaMemcpyAsync(h->theta_tgt, h->theta, h->n_params * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  if (h->mix) MARL_CUDA_TRY(cudaMemcpyAsync(h->mix_tgt, h->mix, (size_t)h->ql.n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));   // dqn/model.py:438-443
  h->tgt_image_current = false;
  return MARL_OK;
}

static GruFwdParams gru_fwd_params(const marl_dqn* h, const RowSource& src, int units, int steps, bool target) {
  GruFwdParams fp; memset(&fp, 0, sizeof(fp));
  fp.plan = make_plan(h->ns, units, steps, 1, 1); fp.src = src;
  fp.theta = target ? h->theta_tgt : h->theta; fp.lay = h->gl;
  return fp;
}

// The online or target agent networks on the rows of src -> q_out: the GRU forward (training rows: whole episodes of the plan's units; save:
// what the backward needs, NULL: nothing), else the tensor-core or the FP32 forward (forward_any), after which the packed image of the weights
// it read is current exactly when the tensor-core forward is on.
static int dqn_forward(marl_dqn* h, const RowPlan& plan, const RowSource& src, bool target, float* q_out, float* save, cudaStream_t st) {
  if (h->rnn) {
    GruFwdParams fp = gru_fwd_params(h, src, plan.units_per_agent, src.traj.T + 1, target);
    fp.q_out = q_out; fp.save = save;
    return launch_gru_forward(fp, st);
  }
  bool& current = target ? h->tgt_image_current : h->image_current;
  if (int rc = forward_any(h->ns, plan, src, target ? h->theta_tgt : h->theta, target ? h->image_tgt : h->image, q_out, st, current)) return rc;
  current = tc_forward_enabled() != 0;
  return MARL_OK;
}

int marl_dqn_forward(marl_dqn* h, const float* obs, int32_t n_envs, int32_t use_target, float* q_out, void* stream) {
  MARL_REQUIRE(h && obs && q_out && n_envs >= 1, "marl_dqn_forward: bad argument");
  MARL_REQUIRE(!h->rnn, "marl_dqn_forward: the learner has recurrent agent networks: use marl_dqn_forward_rnn, which carries the hidden state");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  const RowPlan plan = make_plan(h->ns, n_envs, 1, h->n_sm, 32);
  return dqn_forward(h, plan, dense_rows(obs, n_envs, h->ns.n_agents, h->ns.in), use_target != 0, q_out, nullptr, (cudaStream_t)stream);
}

int marl_dqn_forward_rnn(marl_dqn* h, const float* obs, int32_t n_envs, int32_t use_target, const float* h_in, float* h_out, float* q_out, void* stream) {
  MARL_REQUIRE(h && obs && q_out && n_envs >= 1, "marl_dqn_forward_rnn: bad argument");
  MARL_REQUIRE(h->rnn, "marl_dqn_forward_rnn: the learner was not created with marl_dqn_create_rnn");
  MARL_REQUIRE(h_in == nullptr || h_in != h_out, "marl_dqn_forward_rnn: h_in and h_out must not alias");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  GruFwdParams fp = gru_fwd_params(h, dense_rows(obs, n_envs, h->ns.n_agents, h->ns.in), n_envs, 1, use_target != 0);
  fp.h_in = h_in; fp.h_out = h_out; fp.q_out = q_out;
  return launch_gru_forward(fp, (cudaStream_t)stream);
}

int marl_replay_sample(uint64_t seed, uint64_t update_idx, int32_t batch, int32_t n_valid, int32_t* idx_out, void* stream) {
  MARL_REQUIRE(idx_out && batch >= 1 && n_valid >= 1, "marl_replay_sample: bad argument");
  MARL_CUDA_TRY(launch_pdl(replay_sample_kernel, dim3((batch + 255) / 256), dim3(256), 0, (cudaStream_t)stream, seed, update_idx, (int)batch, (int)n_valid, idx_out));
  return MARL_OK;
}

static bool dqn_external_head(const marl_dqn* h) { return h->hp.mixer != 0 || h->rnn || h->standardise || h->td_lambda_on; }

// The external TD head, for the cases the training pass's own head does not cover (QMIX, standardise_returns, td_lambda, VDN, the recurrent pass):
// the online forward on every row (forward = false: the fused training forward has already written q_all), then dL/dQ of the taken actions into td,
// which becomes tp.td_ext (per agent at tp.td_agent_stride; VDN: per (b, t), stride 0), and the head's loss statistics into loss_part blocks
// [n_loss_parts, ...), which n_loss_parts is advanced past.  The TD error comes from col_td_kernel over C columns of G agents (VDN: one column of all
// agents; independent learners: one column per agent) or, for QMIX, from the mixer (qmix.cuh: one column of all agents, agent 0's reward), which
// hands dL/dq_a back per agent.  Both run the same stage sequence.
static int dqn_td_head(marl_dqn* h, const RowPlan& plan, const RowSource& src, int batch, TrainParams& tp, int& n_loss_parts, bool forward, cudaStream_t st) {
  if (!dqn_external_head(h)) return MARL_OK;
  if (forward)
    if (int rc = dqn_forward(h, plan, src, false, h->q_all, h->gru_save, st)) return rc;
  const int T = src.traj.T;
  const bool qmix = h->hp.mixer == 2, per_b = h->hp.mixer != 0;   // per_b: the return statistics keep one column per batch entry
  const int C = per_b ? 1 : h->ns.n_agents, G = h->ns.n_agents / C;
  const float* ret_ms = h->standardise ? h->ret_ms : nullptr;   // stage 1 needs it; stage 3 de-standardises its bootstrap values exactly when it is set
  const int n_stat = h->standardise ? h->n_stat : 0;
  float* loss_part = h->loss_part + 4 * (size_t)n_loss_parts;
  QmixParams qp; memset(&qp, 0, sizeof(qp));
  ColTdParams cp; memset(&cp, 0, sizeof(cp));
  int blocks = 0;
  if (qmix) {
    qp.L = h->ql; qp.q = h->q_all; qp.tq = h->tq; qp.traj = src.traj; qp.idx = src.idx; qp.B = batch; qp.A = h->ns.out; qp.D = h->ns.in;
    qp.gamma = h->hp.gamma; qp.double_q = h->hp.double_q; qp.huber = h->huber; qp.mix = h->mix; qp.mix_tgt = h->mix_tgt; qp.rec = h->mix_rec; qp.td = h->td;
    qp.loss_part = loss_part; qp.ret_ms = ret_ms; qp.n_stat = n_stat; qp.ret = h->ret; qp.boot = h->boot;
    blocks = (batch * T + kQmTS - 1) / kQmTS;
    qmix_pack_kernel<<<dim3((h->ql.n + 255) / 256, 2), 256, 0, st>>>(h->ql, h->mix, h->mix_tgt, h->mix_img, h->mix_img_tgt);
  } else {
    cp.q = h->q_all; cp.tq = h->tq; cp.traj = src.traj; cp.idx = src.idx; cp.B = batch; cp.A = h->ns.out;
    cp.gamma = h->hp.gamma; cp.double_q = h->hp.double_q; cp.huber = h->huber; cp.C = C; cp.G = G;
    cp.ret_ms = ret_ms; cp.n_stat = n_stat; cp.stat_per_b = per_b; cp.ret = h->ret; cp.chosen = h->chosen; cp.boot = h->boot;
    cp.td = h->td; cp.loss_part = loss_part;
    blocks = (C * batch * T + 255) / 256;
  }
  static void (*const col_td_fns[4])(ColTdParams) = {col_td_kernel<0>, col_td_kernel<1>, col_td_kernel<2>, col_td_kernel<3>};
  const auto stage = [&](int S) {
    if (qmix) qmix_mix_fn(h->ql.hl, S)<<<blocks, kQmWarps * 32, qm_smem_bytes(h->ql), st>>>(qp, h->mix_img, h->mix_img_tgt);
    else col_td_fns[S]<<<blocks, 256, 0, st>>>(cp);
  };
  if (h->td_lambda_on || h->standardise) {
    // λ: bootstrap values (+ chosen Q), the λ-return scan; else the one-step returns (+ chosen Q).  Then [RunningMeanStd step], TD error on the returns
    stage(h->td_lambda_on ? 3 : 1);
    if (h->td_lambda_on) {
      TdLambdaParams lp; lp.boot = h->boot; lp.traj = src.traj; lp.idx = src.idx; lp.C = C; lp.G = G; lp.B = batch; lp.ret = h->ret;
      lp.gamma = h->hp.gamma; lp.lambda = h->td_lambda; lp.gl = (float)((double)h->hp.gamma * (double)h->td_lambda);
      MARL_CUDA_TRY(launch_td_lambda(lp, st));
    }
    if (h->standardise) {
      RetMsParams rp; rp.ret = h->ret; rp.part = h->ret_part; rp.ret_ms = h->ret_ms; rp.count = h->ret_count; rp.T = T;
      rp.N = per_b ? batch : C; rp.P = per_b ? 1 : batch;
      MARL_CUDA_TRY(ret_ms_step(rp, st));
    }
    stage(2);
  } else {
    stage(0);
  }
  if (qmix) {   // the mixer's weight gradient: per-chunk partial sums, then their reduction (with the head's loss statistics)
    const int Sn = batch * T, n = h->ql.n, want = h->mix_wgrad_tiles ? kQmixChunks : 2 * h->n_sm;
    const int chunk_len = (((Sn + want - 1) / want) + 31) & ~31, chunks = (Sn + chunk_len - 1) / chunk_len;
    if (h->mix_wgrad_tiles) {
      qmix_wgrad_kernel<<<dim3(h->mix_n_tiles, chunks), 256, 0, st>>>(h->mix_rec, Sn, h->mix_tiles, chunk_len, h->mix_part, n);
    } else {
      for (int round = 0; round * kQmMicroPerRound < h->mix_n_micro; ++round)
        qmix_wgrad2_kernel<<<chunks, 256, (size_t)(h->ql.R + 2) * kQmP * sizeof(float), st>>>(h->mix_rec, Sn, h->ql.R, h->mix_micro, h->mix_n_micro, round, chunk_len, h->mix_part, n);
    }
    qmix_reduce_kernel<<<(n + 255) / 256, 256, 0, st>>>(h->mix_part, chunks, n, h->mix_grad, loss_part, blocks);
  }
  MARL_CUDA_TRY(cudaGetLastError());
  n_loss_parts += blocks;
  tp.td_ext = h->td;
  tp.td_agent_stride = h->hp.mixer == 1 ? 0 : batch * T;
  return MARL_OK;
}

// Does the tensor-core training pipeline run (else GRU BPTT or the fused FP32 kernel)?  (No image: hidden width below 128.)
static bool dqn_tc_train(const marl_dqn* h) { return !h->rnn && tc_backward_enabled() && h->ns.in < kMaxObsDim && h->image != nullptr; }

// The tensor-core pipeline's buffers (allocated on first use) and current online images
static int dqn_tc_prepare(marl_dqn* h, TcBuffers& tb, cudaStream_t st) {
  // H2 slabs of every row split of up to `rows` rows over at most n_sm CTAs (the per-CTA gradient scratch has n_sm rows): tc_train.cu, h2_slab
  const size_t rows = (size_t)h->ns.n_agents * h->max_batch * (h->max_T + 1), h2_tiles = (rows + 63) / 64 + (size_t)h->n_sm;
  if (!h->tc_h2) {  // intermediates of the tensor-core pipeline, allocated on first use (observation rows at pitch 8 ceil(in / 8))
    const size_t F = sizeof(float);
    if (int rc = alloc_buffers(h, "marl_dqn_update", {{&h->tc_h2, h2_tiles * 64 * kHidden * F},
                                                      {&h->tc_rec, rows * 32 /* kRowRec */ * F}, {&h->tc_x, rows * ((h->ns.in + 7) / 8 * 8) * F},
                                                      {&h->image_bwd, ((size_t)h->ns.n_nets * tc_bwd_image_bytes() / 4 + 4) * F}}))
      return rc;
  }
  if (!h->image_current || !h->bwd_image_current) {
    if (int rc = launch_pack_weights(h->theta, h->ns.lay, h->ns.n_nets, h->image, st, h->image_bwd)) return rc;
    h->image_current = h->bwd_image_current = true;
  }
  tb.image = h->image; tb.bwd_image = h->image_bwd; tb.h2 = h->tc_h2; tb.h2_tiles = h2_tiles; tb.rec = h->tc_rec; tb.x = h->tc_x;
  return MARL_OK;
}

// The training pass from tp.td_ext, or from the agents' own TD head: GRU BPTT, the tensor-core pipeline (between: two timing events recorded
// between its kernels, NULL: none; tc is set when it runs) or the fused FP32 kernel.
static int dqn_train_pass(marl_dqn* h, const TrainParams& tp, cudaEvent_t* between, bool& tc, cudaStream_t st) {
  tc = false;
  if (h->rnn) {
    GruBwdParams bp; memset(&bp, 0, sizeof(bp));
    bp.plan = tp.plan; bp.traj = tp.src.traj; bp.idx = tp.src.idx; bp.B = tp.plan.units_per_agent; bp.theta = h->theta; bp.lay = h->gl; bp.save = h->gru_save;
    bp.td = tp.td_ext; bp.td_agent_stride = tp.td_agent_stride; bp.src = tp.src; bp.scratch = h->scratch; bp.scratch_pitch = h->scratch_pitch;
    return launch_gru_backward(bp, st);
  }
  if (!dqn_tc_train(h)) return launch_train(tp, kHeadDqn, st);
  TcBuffers tb;
  if (int rc = dqn_tc_prepare(h, tb, st)) return rc;
  tc = true;
  if (int rc = launch_tc_dqn_forward(tp, tb, nullptr, nullptr, nullptr, st)) return rc;
  if (between) MARL_CUDA_TRY(cudaEventRecord(between[0], st));
  return launch_tc_dqn_backward(tp, tb, st, between ? between[1] : nullptr);
}

// The tensor-core training pass with the target network in its forward kernel: pack the stale images, then one forward kernel for both networks
// (q_all too when an external TD head runs), the external head, the two backward kernels.  ev (NULL: none): 4 timing events, before the forward,
// after it, after the dH1 kernel (the external head runs between the last two) and at the end.
static int dqn_fused_pass(marl_dqn* h, const RowPlan& plan, const RowSource& src, int batch, TrainParams& tp, int& n_loss_parts, cudaEvent_t* ev,
                          cudaStream_t st) {
  TcBuffers tb;
  if (int rc = dqn_tc_prepare(h, tb, st)) return rc;
  if (!h->tgt_image_current) {
    if (int rc = launch_pack_weights(h->theta_tgt, h->ns.lay, h->ns.n_nets, h->image_tgt, st)) return rc;
    h->tgt_image_current = true;
  }
  if (ev) MARL_CUDA_TRY(cudaEventRecord(ev[0], st));
  if (int rc = launch_tc_dqn_forward(tp, tb, h->image_tgt, h->tq, dqn_external_head(h) ? h->q_all : nullptr, st)) return rc;
  if (ev) MARL_CUDA_TRY(cudaEventRecord(ev[1], st));
  if (int rc = dqn_td_head(h, plan, src, batch, tp, n_loss_parts, false, st)) return rc;
  if (int rc = launch_tc_dqn_backward(tp, tb, st, ev ? ev[2] : nullptr)) return rc;
  if (ev) { MARL_CUDA_TRY(cudaEventRecord(ev[3], st)); h->ev_used += 1; h->ev_split = true; }
  return MARL_OK;
}

// Gradient half of an update.  rp_out == NULL: the per-CTA partials are reduced into grad[] (grad_reduce_kernel); otherwise the
// reduction is left to the caller (fused reduce + Adam tail) and its parameters are returned.
static int dqn_grads(marl_dqn* h, const marl_traj_view* traj, const int32_t* episode_idx, int32_t batch, void* stream, ReduceParams* rp_out) {
  MARL_REQUIRE(h && traj && episode_idx, "marl_dqn_update_grads: NULL argument");
  MARL_REQUIRE(batch >= 1 && batch <= h->max_batch, "marl_dqn_update_grads: batch %d exceeds max_batch %d", batch, h->max_batch);
  MARL_REQUIRE(traj->T >= 1 && traj->T <= h->max_T, "marl_dqn_update_grads: T %d exceeds max_T %d", traj->T, h->max_T);
  MARL_REQUIRE(traj->n_agents == h->ns.n_agents && traj->obs_dim == h->ns.in, "marl_dqn_update_grads: trajectory shape mismatch");
  MARL_REQUIRE(h->hp.mixer != 2 || h->mix != nullptr, "marl_dqn_update: QMIX needs marl_dqn_qmix_init first");
  MARL_REQUIRE(h->hp.mixer == 0 || !h->standardise || batch == h->n_stat, "marl_dqn_update: %s's standardise_returns keeps one statistic per batch entry (the "
               "reference's reshape(-1, B)): batch %d must stay at max_batch %d", h->hp.mixer == 2 ? "QMIX" : "VDN", batch, h->n_stat);
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  const RowPlan plan = h->rnn ? make_plan(h->ns, batch, 1, h->n_sm, kGruSeqs) : episode_plan(h->ns, batch, traj->T, h->n_sm);
  const RowSource src = episode_rows(traj, episode_idx, h->ns.n_agents, h->ns.in);
  // timing (bench.py's roofline leg): 4 events per timed update, around the training pass and between the tensor-core kernels; the recurrent
  // path's window opens before its online forward
  cudaEvent_t* ev = h->timing && h->ev_used < kTimingPairs ? &h->ev[4 * h->ev_used] : nullptr;
  TrainParams tp; memset(&tp, 0, sizeof(tp));
  tp.plan = plan; tp.src = src; tp.theta = h->theta; tp.lay = h->ns.lay; tp.tq = h->tq;
  tp.gamma = h->hp.gamma; tp.double_q = h->hp.double_q; tp.huber = h->huber; tp.scratch = h->scratch; tp.scratch_pitch = h->scratch_pitch; tp.loss_part = h->loss_part;
  int n_loss_parts = h->rnn ? 0 : plan.cta_begin[plan.n_nets];
  // The target network on every gathered row (dqn/model.py:132-134) runs inside the tensor-core training forward when that pipeline runs with the
  // tensor-core forward on (an FP32 target forward gives other bits).  Otherwise it is a forward of its own.
  if (dqn_tc_train(h) && tc_forward_enabled()) {
    if (int rc = dqn_fused_pass(h, plan, src, batch, tp, n_loss_parts, ev, st)) return rc;
  } else {
    if (int rc = dqn_forward(h, plan, src, true, h->tq, nullptr, st)) return rc;
    if (ev && h->rnn) cudaEventRecord(ev[0], st);
    if (int rc = dqn_td_head(h, plan, src, batch, tp, n_loss_parts, true, st)) return rc;
    if (ev && !h->rnn) cudaEventRecord(ev[0], st);
    bool tc = false;
    if (int rc = dqn_train_pass(h, tp, ev ? ev + 1 : nullptr, tc, st)) return rc;
    if (ev) { cudaEventRecord(ev[3], st); h->ev_used += 1; h->ev_split |= tc; }
  }
  ReduceParams rp; rp.scratch = h->scratch; rp.loss_part = h->loss_part; rp.n_nets = h->ns.n_nets; rp.P = h->P(); rp.scratch_pitch = h->scratch_pitch;
  memcpy(rp.cta_begin, plan.cta_begin, sizeof(rp.cta_begin));
  rp.n_loss_parts = n_loss_parts; rp.grad = h->grad; rp.stats = h->grad + h->n_params; rp.stats_accumulate = 0; rp.sumsq_part = h->sumsq;
  if (rp_out != nullptr) { *rp_out = rp; return MARL_OK; }
  return launch_grad_reduce(rp, st);
}

int marl_dqn_update_grads(marl_dqn* h, const marl_traj_view* traj, const int32_t* episode_idx, int32_t batch, void* stream) {
  return dqn_grads(h, traj, episode_idx, batch, stream, nullptr);
}

// Optimiser-step parameters of the next update (advances the update counters)
static void dqn_adam_params(marl_dqn* h, float* loss_out, AdamParams& ap) {
  h->updates += 1;
  h->opt_stepped = true;
  memset(&ap, 0, sizeof(ap)); ap.theta = h->theta; ap.theta_tgt = h->theta_tgt; ap.m = h->m; ap.v = h->v; ap.grad = h->grad; ap.n = (int)h->n_params;
  ap.grad_clip = h->hp.grad_clip;
  set_step_consts(ap, h->opt, h->hp.lr, h->updates);
  // update_target (dqn/model.py:176-185)
  const float tu = h->hp.target_update_interval_or_tau;
  ap.target_mode = 0; ap.tau = tu; ap.tgt_begin = 0; ap.tgt_n = (int)h->n_params;
  if (tu > 1.0f && (float)(h->updates - h->last_target_update) >= tu) { ap.target_mode = 1; h->last_target_update = h->updates; }
  else if (tu < 1.0f) ap.target_mode = 2;
  if (ap.target_mode != 0) h->tgt_image_current = false;  // theta_tgt changes in this launch
  ap.loss_out = loss_out ? loss_out : h->loss_dev;
  ap.sumsq_part = h->grads_are_local ? h->sumsq : nullptr; ap.n_sumsq = (int)((h->n_params + 63) / 64);
  h->grads_are_local = false;
  if (h->image != nullptr && tc_forward_enabled()) {  // valid images stay valid: adam_kernel rewrites the entries of every parameter it steps
    ap.image = h->image; ap.bwd_image = h->image_bwd; ap.img_lay = h->ns.lay; ap.img_nets = h->ns.n_nets;
    ap.image_bytes = tc_image_bytes(); ap.bwd_image_bytes = tc_bwd_image_bytes();
    if (h->image_bwd == nullptr) h->bwd_image_current = false;
  } else {
    h->image_current = h->bwd_image_current = false;
  }
}

// QMIX: the mixer's share of the single optimiser step (same optimiser, step count, learning rate and target update as the agents' networks; no clipping:
// clip_grad_norm_ covers self.critic.parameters() only, dqn/model.py:169-170)
static int qmix_adam(marl_dqn* h, const AdamParams& main, cudaStream_t st) {
  if (h->hp.mixer != 2) return MARL_OK;
  AdamParams ap = main;
  ap.theta = h->mix; ap.theta_tgt = h->mix_tgt; ap.m = h->mix_m; ap.v = h->mix_v; ap.grad = h->mix_grad; ap.n = h->ql.n; ap.tgt_begin = 0; ap.tgt_n = h->ql.n;
  ap.grad_clip = 0.f; ap.loss_out = nullptr; ap.sumsq_part = nullptr; ap.n_sumsq = 0; ap.image = nullptr; ap.bwd_image = nullptr; ap.img_nets = 0;
  return launch_adam(ap, h->opt.kind, st);
}

int marl_dqn_update_apply(marl_dqn* h, float* loss_out, void* stream) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_update_apply: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  AdamParams ap;
  dqn_adam_params(h, loss_out, ap);
  if (int rc = launch_adam(ap, h->opt.kind, (cudaStream_t)stream)) return rc;
  return qmix_adam(h, ap, (cudaStream_t)stream);
}

// one update; `next` (optional): replay indices of the following update, drawn inside the fused tail kernel; *fused_out says whether it was
static int dqn_update(marl_dqn* h, const marl_traj_view* traj, const int32_t* episode_idx, int32_t batch, float* loss_out, void* stream, const SampleParams* next,
                      bool* fused_out) {
  if (fused_out) *fused_out = false;
  ReduceParams rp;
  if (int rc = dqn_grads(h, traj, episode_idx, batch, stream, &rp)) return rc;
  h->grads_are_local = true;  // nobody touches grad between the two halves: the clip can use the per-block sums of squares
  AdamParams ap;
  dqn_adam_params(h, loss_out, ap);
  // one kernel for reduce + clip + Adam when its grid fits the GPU in one wave, else the two kernels
  SampleParams sp; memset(&sp, 0, sizeof(sp));
  if (next != nullptr) sp = *next;
  if (launch_reduce_adam(rp, ap, h->opt.kind, &h->xchg, sp, h->grid_barrier, &h->grid_epoch, h->n_sm, (cudaStream_t)stream) == MARL_OK) {
    if (fused_out) *fused_out = true;
    return qmix_adam(h, ap, (cudaStream_t)stream);
  }
  MARL_REQUIRE(h->xchg.world <= 1, "marl_dqn_update: the peer-memory exchange needs the fused tail kernel (parameter count too large for one wave)");
  if (int rc = launch_grad_reduce(rp, (cudaStream_t)stream)) return rc;
  if (int rc = launch_adam(ap, h->opt.kind, (cudaStream_t)stream)) return rc;
  return qmix_adam(h, ap, (cudaStream_t)stream);
}

int marl_dqn_update(marl_dqn* h, const marl_traj_view* traj, const int32_t* episode_idx, int32_t batch, float* loss_out, void* stream) {
  return dqn_update(h, traj, episode_idx, batch, loss_out, stream, nullptr, nullptr);
}

/* n_updates back-to-back updates with on-device replay sampling: the `rb.sample(); model.update()` pair of
 * marlbase/dqn/train.py:308-311 repeated, without returning to Python in between. */
int marl_dqn_update_n(marl_dqn* h, const marl_traj_view* traj, int32_t batch, int32_t n_valid, uint64_t seed, uint64_t first_update_idx,
                      int32_t n_updates, float* loss_out, void* stream) {
  MARL_REQUIRE(h && traj && n_updates >= 0, "marl_dqn_update_n: bad argument");
  MARL_REQUIRE(n_valid >= 1 && n_valid <= traj->capacity, "marl_dqn_update_n: n_valid %d out of range", n_valid);
  bool have_idx = false;   // the previous update's tail kernel already drew this update's indices
  for (int u = 0; u < n_updates; ++u) {
    if (!have_idx)
      if (int rc = marl_replay_sample(seed, first_update_idx + (uint64_t)u, batch, n_valid, h->idx, stream)) return rc;
    SampleParams next; next.seed = seed; next.update_idx = first_update_idx + (uint64_t)u + 1; next.batch = batch; next.n_valid = n_valid; next.idx = h->idx;
    bool fused = false;
    if (int rc = dqn_update(h, traj, h->idx, batch, loss_out, stream, u + 1 < n_updates ? &next : nullptr, &fused)) return rc;
    have_idx = fused && u + 1 < n_updates;
  }
  return MARL_OK;
}

/* CUDA-event timing of dqn_train_kernel launches: enable=1 starts recording (first 1024 launches), enable=0 stops, synchronises
 * the recorded events and returns their summed duration and count. */
int marl_dqn_timing(marl_dqn* h, int32_t enable, float* total_ms, int32_t* count) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_timing: NULL handle");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  if (enable) {
    if (h->ev.empty()) { h->ev.resize(4 * kTimingPairs); for (auto& e : h->ev) MARL_CUDA_TRY(cudaEventCreate(&e)); }
    h->ev_used = 0; h->timing = true; h->ev_split = false;
    return MARL_OK;
  }
  h->timing = false;
  float tot = 0.f;
  for (int i = 0; i < h->ev_used; ++i) {
    MARL_CUDA_TRY(cudaEventSynchronize(h->ev[4 * i + 3]));
    float ms = 0.f; MARL_CUDA_TRY(cudaEventElapsedTime(&ms, h->ev[4 * i], h->ev[4 * i + 3]));
    tot += ms;
  }
  if (total_ms) *total_ms = tot;
  if (count) *count = h->ev_used;
  return MARL_OK;
}

/* Tell the library that the caller wrote to the parameter buffers returned by marl_dqn_param_ptrs (cached derived data --
 * the packed tensor-core images of the online and target networks -- is rebuilt on next use). */
int marl_dqn_params_changed(marl_dqn* h) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_params_changed: NULL handle");
  h->tgt_image_current = false; h->image_current = false; h->bwd_image_current = false;
  return MARL_OK;
}

/* Per-kernel split of the launches timed by the last marl_dqn_timing(1) .. marl_dqn_timing(0) window: summed CUDA-event durations of
 * the three kernels of the tensor-core training pass (training forward, dH1 + TD head, weight gradients).  With the tensor-core forward on,
 * slot 0 is the forward of both the online and the target network, and for VDN, QMIX and standardise_returns slot 1 includes the external TD
 * head that runs between the forward and the dH1 kernel.  *count = 0 when the window ran the single fused FP32 kernel instead. */
int marl_dqn_timing_kernels(marl_dqn* h, float* ms3, int32_t* count) {
  MARL_REQUIRE(h != nullptr && ms3 != nullptr, "marl_dqn_timing_kernels: NULL argument");
  MARL_REQUIRE(!h->timing, "marl_dqn_timing_kernels: call marl_dqn_timing(q, 0, ...) first");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  ms3[0] = ms3[1] = ms3[2] = 0.f;
  if (count) *count = h->ev_split ? h->ev_used : 0;
  if (!h->ev_split) return MARL_OK;
  for (int i = 0; i < h->ev_used; ++i) {
    MARL_CUDA_TRY(cudaEventSynchronize(h->ev[4 * i + 3]));
    for (int k = 0; k < 3; ++k) {
      float ms = 0.f; MARL_CUDA_TRY(cudaEventElapsedTime(&ms, h->ev[4 * i + k], h->ev[4 * i + k + 1]));
      ms3[k] += ms;
    }
  }
  return MARL_OK;
}

/* ---- gradient exchange over NVLink peer memory (one process per GPU) ---------------------------------------------------------------
 * marl_dqn_peer_handle: allocates this rank's exchange buffer (2 slots of [n_params + 4] floats + a flag) and writes its 64-byte
 * cudaIpcMemHandle_t to handle_out; the caller gathers the handles of all ranks (any transport) and passes them, rank-ordered, to
 * marl_dqn_peer_attach.  From then on marl_dqn_update / marl_dqn_update_n perform the all-rank gradient sum inside the fused
 * reduce + Adam kernel (every rank must make the same sequence of update calls); the two-call form with an external all-reduce
 * between marl_dqn_update_grads and marl_dqn_update_apply keeps working. */
static size_t xbuf_data_bytes(const marl_dqn* h) { return (size_t)2 * kMaxRanks * h->xchg.slot_floats * sizeof(float); }

int marl_dqn_peer_handle(marl_dqn* h, void* handle_out) {
  MARL_REQUIRE(h != nullptr && handle_out != nullptr, "marl_dqn_peer_handle: NULL argument");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  MARL_REQUIRE(h->hp.mixer != 2 || h->mix != nullptr, "marl_dqn_peer_handle: QMIX needs marl_dqn_qmix_init first (the mixer's gradient is part of the exchange)");
  if (h->xbuf == nullptr) {   // sized for the largest world: [2 parities][kMaxRanks sources][slot] floats + kMaxRanks flags
    // slot = [agents' gradient sums | QMIX: the mixer's gradient sums | 4 statistics]
    const int64_t n_extra = h->hp.mixer == 2 ? h->ql.n : 0;
    h->xchg.slot_floats = (int)((h->n_params + n_extra + 4 + 63) / 64 * 64);
    if (int rc = alloc_buffers(h, "marl_dqn_peer_handle", {{&h->xbuf, xbuf_data_bytes(h) + 256}})) return rc;
  }
  cudaIpcMemHandle_t mh;
  MARL_CUDA_TRY(cudaIpcGetMemHandle(&mh, h->xbuf));
  memcpy(handle_out, &mh, sizeof(mh));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size is part of the ABI");
  return MARL_OK;
}

int marl_dqn_peer_attach(marl_dqn* h, int32_t rank, int32_t world, const void* handles) {
  MARL_REQUIRE(h != nullptr && handles != nullptr, "marl_dqn_peer_attach: NULL argument");
  MARL_REQUIRE(world >= 2 && world <= kMaxRanks && rank >= 0 && rank < world, "marl_dqn_peer_attach: rank %d / world %d out of range (2..%d ranks)", rank, world, kMaxRanks);
  MARL_REQUIRE(h->xbuf != nullptr && h->xchg.world <= 1, "marl_dqn_peer_attach: call marl_dqn_peer_handle first, attach once");
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  {  // the exchange lives inside the fused reduce + Adam kernel: refuse here, before any update mutates counters, when that kernel cannot
     // cover this parameter count with one co-resident wave (a later fallback to the two-kernel tail would dead-lock the peers' polls)
    int pb = 0, ns = 0;
    MARL_REQUIRE(reduce_adam_shape((int)h->n_params, h->n_sm, true, h->opt.kind, &pb, &ns) == MARL_OK,
                 "marl_dqn_peer_attach: %lld parameters do not fit the fused reduce + Adam kernel on %d SMs; use the all-reduce between marl_dqn_update_grads and _apply",
                 (long long)h->n_params, h->n_sm);
  }
  for (int r = 0; r < world; ++r) {
    void* base = h->xbuf;
    if (r != rank) {
      cudaIpcMemHandle_t mh;
      memcpy(&mh, static_cast<const char*>(handles) + 64 * (size_t)r, sizeof(mh));
      MARL_CUDA_TRY(cudaIpcOpenMemHandle(&base, mh, cudaIpcMemLazyEnablePeerAccess));
    }
    h->peer_base[r] = base;
    h->xchg.peers[r] = static_cast<float*>(base);
    h->xchg.peer_flags[r] = reinterpret_cast<unsigned long long*>(static_cast<char*>(base) + xbuf_data_bytes(h));
  }
  h->xchg.own_flags = h->xchg.peer_flags[rank];
  h->xchg.timed_out = reinterpret_cast<int*>(static_cast<char*>(h->peer_base[rank]) + xbuf_data_bytes(h) + 128);   // behind the 8 flags, zeroed with the buffer
  h->xchg.rank = rank; h->xchg.world = world; h->xchg.epoch = 0;
  if (h->hp.mixer == 2) { h->xchg.extra = h->mix_grad; h->xchg.n_extra = h->ql.n; }   // the mixer's step then reads the all-rank sum
  return MARL_OK;
}

/* 0 = healthy.  1 = some update's exchange gave up waiting for a peer's flag (a rank died, skipped an update or fell out of step): every
 * result since is invalid.  Synchronises the device. */
int marl_dqn_peer_status(marl_dqn* h, int32_t* timed_out) {
  MARL_REQUIRE(h != nullptr && timed_out != nullptr, "marl_dqn_peer_status: NULL argument");
  *timed_out = 0;
  if (h->xchg.world <= 1) return MARL_OK;
  MARL_CUDA_TRY(cudaSetDevice(h->device));
  int v = 0;
  MARL_CUDA_TRY(cudaMemcpy(&v, h->xchg.timed_out, sizeof(int), cudaMemcpyDeviceToHost));
  *timed_out = v;
  return MARL_OK;
}

int marl_dqn_counters(marl_dqn* h, int64_t* updates, int64_t* last_target_update) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_counters: NULL handle");
  if (updates) *updates = h->updates;
  if (last_target_update) *last_target_update = h->last_target_update;
  return MARL_OK;
}

/* The optimiser of the agents' networks (and of the mixer): before the first step only; zeroes the optimiser state. */
int marl_dqn_set_optimizer(marl_dqn* h, const marl_optimizer* opt) {
  if (int rc = check_set_optimizer(h, opt, "marl_dqn_set_optimizer")) return rc;
  if (h->xchg.world > 1) {   // the peer exchange lives in the fused tail: the new optimiser's instantiation must fit one wave as well
    int pb = 0, ns = 0;
    MARL_REQUIRE(reduce_adam_shape((int)h->n_params, h->n_sm, true, opt->kind, &pb, &ns) == MARL_OK,
                 "marl_dqn_set_optimizer: %lld parameters do not fit the fused tail of optimizer kind %d on %d SMs", (long long)h->n_params, opt->kind, h->n_sm);
  }
  if (h->mix) {
    MARL_CUDA_TRY(cudaMemset(h->mix_m, 0, (size_t)h->ql.n * sizeof(float)));
    MARL_CUDA_TRY(cudaMemset(h->mix_v, 0, (size_t)h->ql.n * sizeof(float)));
  }
  return reset_optimizer(h, *opt);
}

int marl_dqn_set_counters(marl_dqn* h, int64_t updates, int64_t last_target_update) {
  MARL_REQUIRE(h != nullptr, "marl_dqn_set_counters: NULL handle");
  h->updates = updates; h->last_target_update = last_target_update;
  return MARL_OK;
}

}  // extern "C"
