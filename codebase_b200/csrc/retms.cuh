// retms.cuh -- RunningMeanStd (marlbase/utils/standardise_stream.py:6-43) over a batch of returns, on the device: shared by the actor-critic
// learners (a2c.cu: one column per agent) and the DQN family (dqn.cu: one column per agent, VDN: one column per batch entry -- the reference's
// reshape(-1, arr.size(-1)) of its (E, B) returns); and on the host, the handle's statistics buffers.
#pragma once
#include "learner.cuh"

namespace marl {

// standardise_returns (ac/model.py:202-204, utils/standardise_stream.py:6-43): RunningMeanStd over ALL T x P returns per agent (unmasked, as the
// reference), parallel-variance update, then returns <- (returns - mean) / sqrt(var).  Batch moments are accumulated in FP64 in a fixed order
// (per-block partials, then one block): the reference's float32 torch.mean / torch.var differ from them by rounding only.
constexpr int kRetBlocks = 64;
struct RetMsParams { float* ret; int N, P, T; double* part; float* ret_ms; double* count; };   // part: [kRetBlocks][N][2]
static __global__ void __launch_bounds__(256) ret_moments_kernel(RetMsParams p) {
  __shared__ double sh[256][2];
  const int n_per = p.P * p.T;
  for (int a = 0; a < p.N; ++a) {
    double s1 = 0.0, s2 = 0.0;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n_per; i += kRetBlocks * 256) { const double x = (double)p.ret[(size_t)a * n_per + i]; s1 += x; s2 += x * x; }
    sh[threadIdx.x][0] = s1; sh[threadIdx.x][1] = s2;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
      if ((int)threadIdx.x < s) { sh[threadIdx.x][0] += sh[threadIdx.x + s][0]; sh[threadIdx.x][1] += sh[threadIdx.x + s][1]; }
      __syncthreads();
    }
    if (threadIdx.x == 0) { p.part[((size_t)blockIdx.x * p.N + a) * 2] = sh[0][0]; p.part[((size_t)blockIdx.x * p.N + a) * 2 + 1] = sh[0][1]; }
    __syncthreads();
  }
}
// one thread per agent: batch mean / unbiased variance, RunningMeanStd.update_from_moments in the reference's float32 operation order
static __global__ void ret_ms_update_kernel(RetMsParams p) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= p.N) return;
  double s1 = 0.0, s2 = 0.0;
  for (int b = 0; b < kRetBlocks; ++b) { s1 += p.part[((size_t)b * p.N + a) * 2]; s2 += p.part[((size_t)b * p.N + a) * 2 + 1]; }
  const double n = (double)p.P * p.T;
  const double bm = s1 / n, bv = n > 1.0 ? (s2 - n * bm * bm) / (n - 1.0) : 0.0;
  const float batch_mean = (float)bm, batch_var = (float)bv, batch_count = (float)n;
  const double count = *p.count;
  const float mean = p.ret_ms[a], var = p.ret_ms[p.N + a], cnt = (float)count, tot = (float)(count + n);
  const float delta = __fsub_rn(batch_mean, mean);
  const float new_mean = __fadd_rn(mean, __fdiv_rn(__fmul_rn(delta, batch_count), tot));
  const float m_a = __fmul_rn(var, cnt), m_b = __fmul_rn(batch_var, batch_count);
  const float m_2 = __fadd_rn(__fadd_rn(m_a, m_b), __fdiv_rn(__fmul_rn(__fmul_rn(__fmul_rn(delta, delta), cnt), batch_count), tot));
  p.ret_ms[a] = new_mean; p.ret_ms[p.N + a] = __fdiv_rn(m_2, tot);
}
// (the count moves in its own launch: every thread of the update reads the old value)
static __global__ void ret_count_kernel(RetMsParams p) { *p.count += (double)p.P * p.T; }
static __global__ void ret_standardise_kernel(RetMsParams p) {
  const int n_per = p.P * p.T, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.N * n_per) return;
  const int a = i / n_per;
  p.ret[i] = __fdiv_rn(__fsub_rn(p.ret[i], p.ret_ms[a]), sqrtf(p.ret_ms[p.N + a]));
}
// a value in standardised units back in return units, x * sqrt(var) + mean, without FMA contraction as the reference's separate torch ops
__device__ __forceinline__ float unstandardise(float x, float mean, float var) { return __fadd_rn(__fmul_rn(x, sqrtf(var)), mean); }
// many short columns (VDN: one per batch entry, T values each): one thread per column, the other blocks' partials read as zero
static __global__ void ret_moments_cols_kernel(RetMsParams p) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x, n_per = p.P * p.T;
  if (a >= p.N) return;
  double s1 = 0.0, s2 = 0.0;
  for (int i = 0; i < n_per; ++i) { const double x = (double)p.ret[(size_t)a * n_per + i]; s1 += x; s2 += x * x; }
  p.part[(size_t)a * 2] = s1; p.part[(size_t)a * 2 + 1] = s2;
  for (int b = 1; b < kRetBlocks; ++b) { p.part[((size_t)b * p.N + a) * 2] = 0.0; p.part[((size_t)b * p.N + a) * 2 + 1] = 0.0; }
}
// the whole step on a stream: moments -> statistics -> standardised returns
static inline cudaError_t ret_ms_step(const RetMsParams& rp, cudaStream_t st) {
  if (rp.N > 64 && rp.P * rp.T <= 1024) ret_moments_cols_kernel<<<(rp.N + 127) / 128, 128, 0, st>>>(rp);
  else ret_moments_kernel<<<kRetBlocks, 256, 0, st>>>(rp);
  ret_ms_update_kernel<<<(rp.N + 127) / 128, 128, 0, st>>>(rp);
  ret_count_kernel<<<1, 1, 0, st>>>(rp);
  ret_standardise_kernel<<<(rp.N * rp.P * rp.T + 255) / 256, 256, 0, st>>>(rp);
  return cudaGetLastError();
}

// The handle's statistics of n columns, allocated on first enable: mean 0, var 1, count 1e-4 (RunningMeanStd.__init__).  The device is current.
inline int enable_ret_stats(LearnerHandle* h, int n, const char* who) {
  if (h->ret_ms) return MARL_OK;
  if (int rc = alloc_buffers(h, who, {{&h->ret_ms, 2 * n * sizeof(float)}, {&h->ret_count, sizeof(double)},
                                      {&h->ret_part, (size_t)kRetBlocks * n * 2 * sizeof(double)}}))
    return rc;
  std::vector<float> init(2 * n, 0.f);
  for (int a = 0; a < n; ++a) init[n + a] = 1.f;
  const double c0 = 1e-4;
  MARL_CUDA_TRY(cudaMemcpy(h->ret_ms, init.data(), 2 * n * sizeof(float), cudaMemcpyHostToDevice));
  MARL_CUDA_TRY(cudaMemcpy(h->ret_count, &c0, sizeof(double), cudaMemcpyHostToDevice));
  h->n_stat = n;
  return MARL_OK;
}

}  // namespace marl
