// common.cuh -- shared helpers of libmarlb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/marl_b200.h"

namespace marl {

void set_error(const char* fmt, ...);

#define MARL_CUDA_TRY(expr)                                                                     \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      ::marl::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return MARL_ECUDA;                                                                        \
    }                                                                                           \
  } while (0)

#define MARL_REQUIRE(cond, ...)          \
  do {                                   \
    if (!(cond)) {                       \
      ::marl::set_error(__VA_ARGS__);    \
      return MARL_EINVAL;                \
    }                                    \
  } while (0)

// Stream tags (second key word is seed_hi ^ tag).  The reset tag value is shared by specification with the
// CPU oracle; the product never includes anything from oracle/.
constexpr uint32_t kTagReset = 0x52455345u;   // env spawns: ctr = (env_gid, episode, block, 0)
constexpr uint32_t kTagAct = 0x41435430u;     // epsilon-greedy: ctr = (env_gid, episode, t, block)
constexpr uint32_t kTagCat = 0x43415430u;     // categorical:    ctr = (env_gid, episode, t, block)
constexpr uint32_t kTagSample = 0x53414d50u;  // replay sampling: ctr = (update_lo, update_hi, block, 0)

struct u32x4 { uint32_t x, y, z, w; };

// Philox4x32-10 (Random123).
__host__ __device__ __forceinline__ u32x4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                         uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
#ifdef __CUDA_ARCH__
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
#else
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t h0 = (uint32_t)(p0 >> 32), l0 = (uint32_t)p0, h1 = (uint32_t)(p1 >> 32), l1 = (uint32_t)p1;
#endif
    const uint32_t n0 = h1 ^ c1 ^ k0, n2 = h0 ^ c3 ^ k1;
    c0 = n0; c1 = l1; c2 = n2; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return u32x4{c0, c1, c2, c3};
}

__host__ __device__ __forceinline__ uint32_t pick(const u32x4& v, int i) {
  return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w;
}

// integer in [0, n) by multiply-shift
__host__ __device__ __forceinline__ uint32_t bounded(uint32_t u, uint32_t n) {
#ifdef __CUDA_ARCH__
  return __umulhi(u, n);
#else
  return (uint32_t)(((uint64_t)u * n) >> 32);
#endif
}

// uniform float in [0, 1) with 24 random bits
__host__ __device__ __forceinline__ float u01(uint32_t u) { return (float)(u >> 8) * (1.0f / 16777216.0f); }

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------------------------
// The per-update kernels form one dependency chain on one stream; each is launched with programmatic stream serialization so that
// its CTAs are scheduled (and run their data-independent setup: barrier init) while the previous kernel drains.
// Contract of every kernel launched through launch_pdl: no global memory access before pdl_wait(); pdl_launch_dependents() right
// after it (when kernel K starts, K-1 has passed its wait, hence K-2 and everything before it has completed).
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}
#endif

int check_device(int device);
int tc_forward_enabled();
int tc_backward_enabled();
int tc_split_exchange_enabled();

}  // namespace marl
