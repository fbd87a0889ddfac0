// tc_forward.cu -- warpgroup-MMA (wgmma) implementation of the forward-only MLP pass (sm_90a).
//
// Same contract as mlp_forward_kernel (model.act's network pass, the target-network / target-critic pass of the
// learners; marlbase/dqn/model.py:99,132-134, marlbase/ac/model.py:148-149,190-193) but the two hidden layers of each 64-row
// warpgroup tile run on the tensor cores:
//   * activations never touch shared memory: the accumulator of one layer (registers) becomes, after bias + ReLU, the register A operand
//     of the next (the images' permuted K order, kperm, makes the accumulator layout the A fragment layout);
//   * weights are the B operand, resident in shared memory as a pre-packed image (K-major, 128-byte swizzle, one 16-KB panel per 32 input
//     features) built by pack_weights_kernel and kept current by the optimiser step (pack_param), loaded with TMA bulk copies;
//   * FP32 parity (<= 1e-5, SURVEY H3) is kept with the error-compensated 3xTF32 split: every operand is stored as hi = tf32(x) and
//     lo = x - hi, and each product is accumulated as lo*hi + hi*lo + hi*hi in FP32;
//   * the head (out <= 8 columns) runs on the CUDA cores against the FP32 copy of W3.
#include "tc_common.cuh"

namespace marl {

size_t tc_image_bytes() { return kImageBytes; }
size_t tc_bwd_image_bytes() { return kBwdImageBytes; }

// Whole images from the flat parameters: the padding (observation columns >= in, head rows >= out) is zeroed, everything else goes
// through pack_param (tc_common.cuh).
__global__ void pack_weights_kernel(const float* __restrict__ theta, NetLayout lay, int n_nets, uint8_t* __restrict__ image, uint8_t* __restrict__ bwd_image) {
  const int net = blockIdx.y;
  if (net >= n_nets) return;
  const float* th = theta + (size_t)net * lay.P;
  uint8_t* img = image + (size_t)net * kImageBytes;
  uint8_t* bwd = bwd_image ? bwd_image + (size_t)net * kBwdImageBytes : nullptr;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kHidden * 32 && (i & 31) >= lay.in) {  // W1 [128][32]: zero columns beyond in
    const int o = panel_offset(i >> 5, kperm(i & 31), kPanelBytes);
    *reinterpret_cast<float*>(img + kOffW1Hi + o) = 0.f; *reinterpret_cast<float*>(img + kOffW1Lo + o) = 0.f;
  }
  if (i < kOutPad * kHidden && (i >> 7) >= lay.out) reinterpret_cast<float*>(img + kOffW3F)[i] = 0.f;   // W3 [8][128]: zero rows beyond out
  if (i < kOutPad && i >= lay.out) reinterpret_cast<float*>(img + kOffB3)[i] = 0.f;
  if (i < lay.P) pack_param(lay, i, th[i], img, bwd);
}

// observation row of a virtual row and where its outputs go
__device__ __forceinline__ const float* fwd_src_row(const FwdParams& p, int net, int vr, size_t& dst) {
  int agent, unit, off;
  decode_row(p.plan, net, vr, agent, unit, off);
  dst = out_row(p.src, agent, unit, off, p.plan.units_per_agent, p.plan.unit_rows);
  return src_row(p.src, agent, unit, off);
}

TSG_DEFINE(g_ts_forward)
TSG_GETTER(tsg_forward, g_ts_forward)
// Two warpgroups, each running its own 64-row tiles through layer 1 -> layer 2 -> head with nothing shared but the weight image, so that the
// CUDA-core epilogue of one overlaps the MMAs of the other.
template <int K1>
__global__ void __launch_bounds__(kTcThreads, 1) tc_forward_kernel(FwdParams p, const uint8_t* __restrict__ images) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);  // swizzle atoms need 1024-byte alignment
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kImageBytes);   // [0] W1 + biases + FP32 W3, [1] W2
  const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31, g = lane >> 2, tq = lane & 3;
  int net, row_begin, row_end;
  cta_rows(p.plan, net, row_begin, row_end);
  if (row_begin >= row_end) { pdl_wait(); return; }
  TSG(g_ts_forward, 0);
  if (t == 0) { mbar_init(bar, 1); mbar_init(bar + 1, 1); fence_mbar_init(); }
  __syncthreads();
  pdl_wait();   // nothing above touches global memory (PDL contract, common.cuh)
  pdl_launch_dependents();
  const uint32_t sb = smem_u32(smem);
  if (t == 0) tma_forward_image(sb, images + (size_t)net * kImageBytes, bar);
  const float* b1 = reinterpret_cast<const float*>(smem + kOffB1);
  const float* b2 = reinterpret_cast<const float*>(smem + kOffB2);
  const float* b3 = reinterpret_cast<const float*>(smem + kOffB3);
  const float* w3f = reinterpret_cast<const float*>(smem + kOffW3F);
  const int D = p.src.D, out = p.lay.out;
  bool first = true;
  for (int vr0 = row_begin + kWgRows * wg; vr0 < row_end; vr0 += kTileRows) {
    const int r0 = vr0 + 16 * wq + g, r1 = r0 + 8;
    size_t d0 = 0, d1 = 0;
    const float* s0 = r0 < row_end ? fwd_src_row(p, net, r0, d0) : nullptr;
    const float* s1 = r1 < row_end ? fwd_src_row(p, net, r1, d1) : nullptr;
    float acc[64];
    {
      float x[kMaxObsDim / 8][4];
      load_x_frag(s0, s1, D, tq, x);
      if (first) mbar_wait(bar, 0);
      layer1_tile<K1>(acc, x, sb + kOffW1Hi, b1, tq);
    }
    {
      uint32_t hi[16][4], lo[16][4];
      frag_to_a(acc, hi, lo);
      if (first) { mbar_wait(bar + 1, 0); first = false; }
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      layer_rs<16>(acc, hi, lo, sb + kOffW2Hi, sb + kOffW2Lo, 16);
    }
    float q0[kOutPad], q1[kOutPad];
    head_quad(acc, b2, w3f, out, tq, q0, q1);
    if (tq < 2 && (tq == 0 ? s0 : s1) != nullptr) {
      float* o = p.out + (tq == 0 ? d0 : d1) * out;
#pragma unroll
      for (int a = 0; a < kOutPad; ++a)
        if (a < out) o[a] = (tq == 0 ? q0[a] : q1[a]) + b3[a];
    }
  }
  TSG(g_ts_forward, 31);
}

// ---- launchers ----------------------------------------------------------------------------------------------------------
constexpr int kFwdSmem = kImageBytes + 64 + 1024;   // + mbarriers, + slack for the 1024-byte alignment

int tc_forward_init() {
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_forward_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_forward_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_forward_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_forward_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdSmem));
  return MARL_OK;
}

int launch_pack_weights(const float* theta, const NetLayout& lay, int n_nets, uint8_t* image, cudaStream_t st, uint8_t* bwd_image) {
  dim3 grid((lay.P + 255) / 256, n_nets);   // P > 128 * 128 >= every padded extent
  pack_weights_kernel<<<grid, 256, 0, st>>>(theta, lay, n_nets, image, bwd_image);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int launch_tc_forward(const FwdParams& p, const uint8_t* images, cudaStream_t st) {
  return with_k1(p.src.D, [&](auto k1) {
    MARL_CUDA_TRY(launch_pdl(tc_forward_kernel<decltype(k1)::value>, dim3(p.plan.cta_begin[p.plan.n_nets]), dim3(kTcThreads), kFwdSmem, st, p, images));
    return MARL_OK;
  });
}

}  // namespace marl
