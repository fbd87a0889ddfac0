// core.cu -- error reporting and device checks shared by every entry point of libmarlb200.
#include "tc_common.cuh"
#include <string.h>

namespace marl {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// No CPU fallback: a missing / non-Hopper device is an error, never a silent slow path (sm_90a code loads on compute capability 9.0 only).
int check_device(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("libmarlb200: no CUDA device available (%s); this library has no CPU fallback", e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    return MARL_ECUDA;
  }
  if (device < 0 || device >= n) { set_error("libmarlb200: device %d out of range (0..%d)", device, n - 1); return MARL_EINVAL; }
  cudaDeviceProp p;
  MARL_CUDA_TRY(cudaGetDeviceProperties(&p, device));
  if (p.major != 9 || p.minor != 0) {
    set_error("libmarlb200: device %d is sm_%d%d; this build targets sm_90a (H100) only", device, p.major, p.minor);
    return MARL_ECUDA;
  }
  MARL_CUDA_TRY(cudaSetDevice(device));
  return MARL_OK;
}

static int g_tc_forward = 1, g_tc_backward = 1;
int tc_forward_enabled() { return g_tc_forward; }
int tc_backward_enabled() { return g_tc_backward; }

}  // namespace marl

extern "C" {
/* Process-wide options.  "tensor_core_forward": 1 = forward-only passes (act, target networks) run on the tensor cores (wgmma) with the
 * 3xTF32 split (default), 0 = FP32 FFMA kernels.  "tensor_core_backward": 1 = the DQN-family training pass runs as the three-kernel
 * tensor-core pipeline (tc_train.cu, default), 0 = fused FP32 kernel. */
int marl_set_option(const char* name, int32_t value) {
  if (name && strcmp(name, "tensor_core_forward") == 0) { marl::g_tc_forward = value ? 1 : 0; return MARL_OK; }
  if (name && strcmp(name, "tensor_core_backward") == 0) { marl::g_tc_backward = value ? 1 : 0; return MARL_OK; }
  marl::set_error("marl_set_option: unknown option '%s'", name ? name : "(null)");
  return MARL_EINVAL;
}
/* Profiling builds only (MARL_NVCC_DEFINES=-DMARL_TC_TIMESTAMPS, tools/ts_timeline.py): the timeline probes of kernel `which` (0 forward, 1 training
 * forward, 2 TD head + dH1, 3 weight gradients, 4 reduce + Adam) as [160 CTAs][32 slots][globaltimer ns, clock64] -> host memory;
 * product builds return MARL_EINVAL. */
int marl_debug_timestamps(int32_t which, uint64_t* out) {
  int rc = -1;
  unsigned long long* o = reinterpret_cast<unsigned long long*>(out);
  switch (which) {
    case 0: rc = marl::tsg_forward(o); break; case 1: rc = marl::tsg_fwd(o); break; case 2: rc = marl::tsg_dh1(o); break;
    case 3: rc = marl::tsg_dw(o); break; case 4: rc = marl::tsg_adam(o); break;
    default: break;
  }
  if (rc != 0) { marl::set_error("marl_debug_timestamps: kernel %d has no probes in this build (build with -DMARL_TC_TIMESTAMPS)", (int)which); return MARL_EINVAL; }
  return MARL_OK;
}
int marl_version(void) { return MARL_ABI_VERSION; }
const char* marl_last_error(void) { return marl::g_err; }
}
