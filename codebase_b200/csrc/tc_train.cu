// tc_train.cu -- tensor-core (wgmma, 3xTF32) training pass of the DQN-family learner as a three-kernel pipeline (sm_90a).
//
// Same arithmetic as train_kernel<KP, kHeadDqn> (QNetwork._compute_loss + backward, marlbase/dqn/model.py:118-168), split where a
// weight gradient needs the rows of many tiles as its K dimension (tf32 wgmma reads both shared-memory operands K-major only):
//   tc_dqn_fwd_kernel   online forward (A operand in registers, weights = K-major image), head on the CUDA cores; stores H1, H2 (FP32,
//                        feature-major), the gathered observation row, the row's outputs and the ReLU masks of H1 / H2 (row record)
//   tc_dh1_kernel       TD head (needs the next row's outputs, hence after the forward) -> dLoss/dq[act] and the loss statistics;
//                        dH1 = (dH2 x W2) * relu'(H1) with dH2[r][j] = g_r W3[act_r][j] relu'(H2[r][j]) built in registers (the TD loss touches
//                        one output per row); B = K-major image of W2^T
//   tc_dw_kernel        dW2 | db2, dW1 | db1, dW3: row-streaming TN GEMMs over 32-row chunks staged transposed (K = rows) into shared
//                        memory, accumulators in registers across all the CTA's rows; db3 on the CUDA cores
// The partials feed the same grad_reduce_kernel / adam_kernel as the FP32 path.
#include "tc_common.cuh"

namespace marl {

// observation row of a virtual row of the training batch and the row's index in the [agent][unit][T + 1] layout of every per-row buffer
__device__ __forceinline__ const float* train_row(const TcTrainParams& p, int net, int vr, size_t& d, int& agent, int& unit, int& off, int& ep) {
  decode_row(p.plan, net, vr, agent, unit, off);
  d = ((size_t)agent * p.plan.units_per_agent + unit) * p.plan.unit_rows + off;
  const TrajView& tv = p.src.traj;
  ep = p.src.idx[unit];
  return tv.obs + (((size_t)ep * tv.N + agent) * (size_t)(tv.T + 1) + off) * p.src.D;
}

// =====================================================================================================================
// 1. online forward: H1, H2, X, outputs
// =====================================================================================================================
TSG_DEFINE(g_ts_fwd)
TSG_GETTER(tsg_fwd, g_ts_fwd)
TSG_DEFINE(g_ts_dh1)
TSG_GETTER(tsg_dh1, g_ts_dh1)
TSG_DEFINE(g_ts_dw)
TSG_GETTER(tsg_dw, g_ts_dw)

__device__ __forceinline__ void load_x_frag_t(const float* s0, const float* s1, int D, int quad_lane, float (&x)[kMaxObsDim / 8][4]) {
#pragma unroll
  for (int ks = 0; ks < kMaxObsDim / 8; ++ks) {
    const int c = 8 * ks + 2 * quad_lane;
    x[ks][0] = (s0 && c < D) ? s0[c] : 0.f; x[ks][1] = (s1 && c < D) ? s1[c] : 0.f;
    x[ks][2] = (s0 && c + 1 < D) ? s0[c + 1] : 0.f; x[ks][3] = (s1 && c + 1 < D) ? s1[c + 1] : 0.f;
  }
}

// store a 64 x 128 fragment feature-major (dst[j * rows + row]) and its ReLU mask words (rec field `mask`); rows of a missing source (d < 0)
// are skipped
__device__ __forceinline__ void store_frag_fm(float* dst, size_t rows, const float (&v)[64], long long d0, long long d1, int quad_lane, float* rec, int mask) {
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const long long d = (i & 2) ? d1 : d0;
    if (d >= 0) dst[(size_t)frag_col(i, quad_lane) * rows + (size_t)d] = v[i];
  }
  uint32_t m0, m1;
  frag_masks(v, m0, m1);
  if (d0 >= 0) rec[(size_t)d0 * kRowRec + mask + quad_lane] = __uint_as_float(m0);
  if (d1 >= 0) rec[(size_t)d1 * kRowRec + mask + quad_lane] = __uint_as_float(m1);
}

__global__ void __launch_bounds__(kTcThreads, 1) tc_dqn_fwd_kernel(TcTrainParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kImageBytes);   // [0] W1 + biases + FP32 W3, [1] W2
  const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31, g = lane >> 2, tq = lane & 3;
  int net, row_begin, row_end;
  cta_rows(p.plan, net, row_begin, row_end);
  if (row_begin >= row_end) { pdl_wait(); return; }
  TSG(g_ts_fwd, 0);
  if (t == 0) { mbar_init(bar, 1); mbar_init(bar + 1, 1); fence_mbar_init(); }
  __syncthreads();
  pdl_wait();   // nothing above touches global memory
  pdl_launch_dependents();
  const uint32_t sb = smem_u32(smem);
  if (t == 0) tma_forward_image(sb, p.images + (size_t)net * kImageBytes, bar);
  const float* b1 = reinterpret_cast<const float*>(smem + kOffB1);
  const float* b2 = reinterpret_cast<const float*>(smem + kOffB2);
  const float* b3 = reinterpret_cast<const float*>(smem + kOffB3);
  const float* w3f = reinterpret_cast<const float*>(smem + kOffW3F);
  const int D = p.src.D, A = p.lay.out, k1steps = (D + 7) >> 3;
  bool first = true;
  for (int vr0 = row_begin + kWgRows * wg; vr0 < row_end; vr0 += kTileRows) {
    const int r0 = vr0 + 16 * wq + g, r1 = r0 + 8;
    size_t d0u = 0, d1u = 0;
    int agent, unit, off, ep;
    const float* s0 = r0 < row_end ? train_row(p, net, r0, d0u, agent, unit, off, ep) : nullptr;
    const float* s1 = r1 < row_end ? train_row(p, net, r1, d1u, agent, unit, off, ep) : nullptr;
    const long long d0 = s0 ? (long long)d0u : -1, d1 = s1 ? (long long)d1u : -1;
    float acc[64];
    {
      float x[kMaxObsDim / 8][4];
      uint32_t xhi[kMaxObsDim / 8][4], xlo[kMaxObsDim / 8][4];
      load_x_frag_t(s0, s1, D, tq, x);
#pragma unroll
      for (int ks = 0; ks < kMaxObsDim / 8; ++ks) {   // the gathered row for the weight-gradient kernel
        const int c = 8 * ks + 2 * tq;
        if (ks < k1steps) {
          if (d0 >= 0) *reinterpret_cast<float2*>(p.xg + (size_t)d0 * kMaxObsDim + c) = make_float2(x[ks][0], x[ks][2]);
          if (d1 >= 0) *reinterpret_cast<float2*>(p.xg + (size_t)d1 * kMaxObsDim + c) = make_float2(x[ks][1], x[ks][3]);
        }
        tf32_split_u(x[ks][0], xhi[ks][0], xlo[ks][0]); tf32_split_u(x[ks][1], xhi[ks][1], xlo[ks][1]);
        tf32_split_u(x[ks][2], xhi[ks][2], xlo[ks][2]); tf32_split_u(x[ks][3], xhi[ks][3], xlo[ks][3]);
      }
      if (first) mbar_wait(bar, 0);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      layer_rs<kMaxObsDim / 8>(acc, xhi, xlo, sb + kOffW1Hi, sb + kOffW1Lo, k1steps);
    }
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const float2 bb = *reinterpret_cast<const float2*>(b1 + frag_col(i, tq));
      acc[i] = fmaxf(acc[i] + bb.x, 0.f); acc[i + 1] = fmaxf(acc[i + 1] + bb.y, 0.f);
    }
    store_frag_fm(p.h1g, p.rows, acc, d0, d1, tq, p.rec, kRecMask1);
    {
      uint32_t hi[16][4], lo[16][4];
      frag_to_a(acc, hi, lo);
      if (first) { mbar_wait(bar + 1, 0); first = false; }
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      layer_rs<16>(acc, hi, lo, sb + kOffW2Hi, sb + kOffW2Lo, 16);
    }
    float q0[kOutPad], q1[kOutPad];
    head_quad(acc, b2, w3f, A, tq, q0, q1);   // acc = H2 from here
    store_frag_fm(p.h2g, p.rows, acc, d0, d1, tq, p.rec, kRecMask2);
    if (tq < 2 && (tq == 0 ? d0 : d1) >= 0) {
      float* o = p.rec + (size_t)(tq == 0 ? d0 : d1) * kRowRec;
#pragma unroll
      for (int a = 0; a < kOutPad; ++a) o[a] = a < A ? (tq == 0 ? q0[a] : q1[a]) + b3[a] : 0.f;
    }
  }
  TSG(g_ts_fwd, 31);
}

// =====================================================================================================================
// 2. TD head + dH1 = (dH2 x W2) * relu'(H1)
// =====================================================================================================================
constexpr int kDh1W3 = kBwdImageBytes;                        // FP32 copy of W3 [8][128] behind the W2^T image
constexpr int kDh1Bar = kDh1W3 + kOutPad * kHidden * 4;
constexpr int kDh1Red = kDh1Bar + 64;                         // [2][kTcThreads] loss statistics
constexpr int kDh1Smem = kDh1Red + 2 * kTcThreads * 4 + 1024;

// dLoss/dq[act] of one row (0 at t == T) and its loss statistics (delta^2 filled, filled on agent 0)
__device__ __forceinline__ float td_grad(const TcTrainParams& p, size_t d, int agent, int b, int tt, int ep, int& act, float& s0, float& s1) {
  const TrajView& tv = p.src.traj;
  const int T = tv.T, A = p.lay.out;
  act = 0;
  if (tt >= T) return 0.f;
  act = tv.act[((size_t)ep * tv.N + agent) * T + tt];
  if (p.td_ext) return p.td_ext[(size_t)agent * p.td_agent_stride + (size_t)b * T + tt];
  const float rew = tv.rew[((size_t)ep * tv.N + agent) * T + tt];
  const float filled = (float)tv.filled[(size_t)ep * T + tt], done1 = (float)tv.done[(size_t)ep * (T + 1) + tt + 1];
  const float* q = p.rec + d * kRowRec;
  const float* qn = q + kRowRec;                 // the next row of the same episode
  const float* tq = p.tq + (d + 1) * A;          // target outputs share the [agent][unit][T + 1] row layout
  float tsel;
  if (p.double_q) {
    int best = 0; float bv = qn[0];
    for (int o = 1; o < A; ++o) if (qn[o] > bv) { bv = qn[o]; best = o; }
    tsel = tq[best];
  } else {
    tsel = tq[0];
    for (int o = 1; o < A; ++o) tsel = fmaxf(tsel, tq[o]);
  }
  const float y = rew + p.gamma * tsel * (1.f - done1);
  const float delta = q[act] - y;
  s0 += delta * delta * filled;
  if (agent == 0) s1 += filled;
  return 2.f * delta * filled;
}

__global__ void __launch_bounds__(kTcThreads, 1) tc_dh1_kernel(TcTrainParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kDh1Bar);
  const float* w3f = reinterpret_cast<const float*>(smem + kDh1W3);
  float* red = reinterpret_cast<float*>(smem + kDh1Red);
  const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31, g = lane >> 2, tq = lane & 3;
  int net, row_begin, row_end;
  cta_rows(p.plan, net, row_begin, row_end);
  if (row_begin >= row_end) {
    pdl_wait();
    if (t < 4) p.loss_part[4 * blockIdx.x + t] = 0.f;
    return;
  }
  TSG(g_ts_dh1, 0);
  if (t == 0) { mbar_init(bar, 1); fence_mbar_init(); }
  __syncthreads();
  pdl_wait();   // nothing above touches global memory
  pdl_launch_dependents();
  const uint32_t sb = smem_u32(smem);
  if (t == 0) {  // W2^T image + FP32 W3: TMA bulk copies onto one mbarrier
    mbar_expect_tx(bar, (uint32_t)(kBwdImageBytes + kOutPad * kHidden * 4));
    tma_image_range(sb, p.bwd_images + (size_t)net * kBwdImageBytes, 0, kBwdImageBytes, bar);
    tma_bulk_g2s(sb + kDh1W3, p.images + (size_t)net * kImageBytes + kOffW3F, kOutPad * kHidden * 4, bar);
  }
  float st0 = 0.f, st1 = 0.f;
  bool first = true;
  for (int vr0 = row_begin + kWgRows * wg; vr0 < row_end; vr0 += kTileRows) {
    long long d[2];
    float gr[2];
    int act[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int vr = vr0 + 16 * wq + g + 8 * k;
      d[k] = -1; gr[k] = 0.f; act[k] = 0;
      if (vr < row_end) {
        size_t du; int agent, unit, off, ep;
        train_row(p, net, vr, du, agent, unit, off, ep);
        d[k] = (long long)du;
        float a0 = 0.f, a1 = 0.f;   // the four threads of a quad share the row: only the first counts its statistics
        gr[k] = td_grad(p, du, agent, unit, off, ep, act[k], a0, a1);
        if (tq == 0) { st0 += a0; st1 += a1; }
      }
    }
    if (first) { mbar_wait(bar, 0); first = false; }
    // dH2 = g W3[act][j] relu'(H2) and relu'(H1), from the mask words the forward stored for this thread's columns (rows without a source: 0)
    uint32_t mh1[2] = {0u, 0u}, mh2[2] = {0u, 0u};
#pragma unroll
    for (int k = 0; k < 2; ++k)
      if (d[k] >= 0) {
        const float* rp = p.rec + (size_t)d[k] * kRowRec;
        mh1[k] = __float_as_uint(rp[kRecMask1 + tq]); mh2[k] = __float_as_uint(rp[kRecMask2 + tq]);
      }
    float v[64];
    uint64_t m1 = 0;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int k = (i >> 1) & 1, bit = ((i >> 2) << 1) | (i & 1);
      v[i] = ((mh2[k] >> bit) & 1u) ? gr[k] * w3f[act[k] * kHidden + frag_col(i, tq)] : 0.f;
      m1 |= (uint64_t)((mh1[k] >> bit) & 1u) << i;
    }
    float acc[64];
    {
      uint32_t hi[16][4], lo[16][4];
      frag_to_a(v, hi, lo);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      // D[r][j1] = sum_{j2} dH2[r][j2] W2[j2][j1]: B = K-major image of W2^T (rows j1, K = j2)
      layer_rs<16>(acc, hi, lo, sb, sb + 4 * kPanelBytes, 16);
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int k = (i >> 1) & 1;
      if (d[k] >= 0) p.dh1g[(size_t)frag_col(i, tq) * p.rows + (size_t)d[k]] = ((m1 >> i) & 1) ? acc[i] : 0.f;
    }
    const long long dr = tq == 0 ? d[0] : d[1];
    if (tq < 2 && dr >= 0) {
      float* rp = p.rec + (size_t)dr * kRowRec;
      rp[kRecG] = tq == 0 ? gr[0] : gr[1]; rp[kRecAct] = __int_as_float(tq == 0 ? act[0] : act[1]);
    }
  }
  // ---- per-CTA loss statistics, summed in a fixed order ----------------------------------------------------------------
  red[t] = st0; red[kTcThreads + t] = st1;
  __syncthreads();
  for (int s = kTcThreads / 2; s > 0; s >>= 1) {
    if (t < s) { red[t] += red[t + s]; red[kTcThreads + t] += red[kTcThreads + t + s]; }
    __syncthreads();
  }
  if (t < 4) p.loss_part[4 * blockIdx.x + t] = t < 2 ? red[t * kTcThreads] : 0.f;
  TSG(g_ts_dh1, 31);
}

// =====================================================================================================================
// 3. weight gradients: row-streaming TN GEMMs over 32-row chunks, accumulators in registers
// =====================================================================================================================
// Every operand is staged K-major (one 128-byte swizzled line of 32 rows per feature), hi | lo:
//   dW2 | db2 [j2][j1 | 1] += dH2^T x [H1 | 1]^T   (A: 128 lines, B: 136 lines, line 128 = ones)
//   dW1 | db1 [j1][i | 1]  += dH1^T x [X | 1]^T    (B: 32 lines, line D = ones)
//   dW3^T [j][a]           += H2^T x dq^T          (B: 8 lines, dq[r][a] = g_r at a = act_r)
// Warpgroup w accumulates the M rows [64 w, 64 w + 64) of all three.
constexpr int kChunk = 32;
constexpr int kLine = 128;                                              // one feature's 32 rows
constexpr int kSA2 = 0, kSB2 = kSA2 + 2 * 128 * kLine, kSA1 = kSB2 + 2 * 136 * kLine, kSB1 = kSA1 + 2 * 128 * kLine;
constexpr int kSA3 = kSB1 + 2 * 32 * kLine, kSB3 = kSA3 + 2 * 128 * kLine, kSW3 = kSB3 + 2 * 8 * kLine;
constexpr int kDwSmem = kSW3 + kOutPad * kHidden * 4 + 1024;
static_assert(kSB2 % 1024 == 0 && kSA1 % 1024 == 0 && kSB1 % 1024 == 0 && kSA3 % 1024 == 0 && kSB3 % 1024 == 0 && kDwSmem <= 227 * 1024,
              "weight-gradient staging: 1024-byte aligned operands within the shared memory of one SM");

// byte offset of (line f, row r) in a K-major SWIZZLE_128B operand of 32 rows
__device__ __forceinline__ int line_off(int f, int r) { return f * kLine + ((((r >> 2) ^ (f & 7)) & 7) << 4) + ((r & 3) << 2); }
__device__ __forceinline__ void stage_hl(uint8_t* base, int lines, int f, int r, float x) {
  float hi, lo;
  tf32_split(x, hi, lo);
  *reinterpret_cast<float*>(base + line_off(f, r)) = hi;
  *reinterpret_cast<float*>(base + lines * kLine + line_off(f, r)) = lo;
}

__global__ void __launch_bounds__(kTcThreads, 1) tc_dw_kernel(TcTrainParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  const float* w3f = reinterpret_cast<const float*>(smem + kSW3);
  const int t = threadIdx.x, warp = t >> 5, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31, g = lane >> 2, tq = lane & 3;
  int net, row_begin, row_end;
  cta_rows(p.plan, net, row_begin, row_end);
  float* gs = p.scratch + (size_t)blockIdx.x * p.scratch_pitch;
  pdl_wait();
  pdl_launch_dependents();
  if (row_begin >= row_end) {
    for (int i = t; i < p.lay.P; i += kTcThreads) gs[i] = 0.f;
    return;
  }
  TSG(g_ts_dw, 0);
  const int D = p.src.D, A = p.lay.out;
  // constant lines: the ones line (hi 1, lo 0) of [H1 | 1] and [X | 1] and the zero lines behind them; W3 copy
  for (int i = t; i < 8 * kChunk; i += kTcThreads) {
    const int f = 128 + i / kChunk, r = i % kChunk;
    stage_hl(smem + kSB2, 136, f, r, f == 128 ? 1.f : 0.f);
  }
  for (int i = t; i < 32 * kChunk; i += kTcThreads) {
    const int f = i / kChunk, r = i % kChunk;
    if (f >= D) stage_hl(smem + kSB1, 32, f, r, f == D ? 1.f : 0.f);
  }
  {
    const float4* w3src = reinterpret_cast<const float4*>(p.images + (size_t)net * kImageBytes + kOffW3F);
    for (int i = t; i < kOutPad * kHidden / 4; i += kTcThreads) reinterpret_cast<float4*>(smem + kSW3)[i] = w3src[i];
  }
  __syncthreads();
  const uint32_t sb = smem_u32(smem);
  float acc2[68], acc1[16], acc3[4];
#pragma unroll
  for (int i = 0; i < 68; ++i) acc2[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) acc1[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) acc3[i] = 0.f;
  float db3 = 0.f;   // warp a, lane 0: sum of dq[.][a]
  const int n_chunks = (row_end - row_begin + kChunk - 1) / kChunk;
  for (int c = 0; c < n_chunks; ++c) {
    // ---- this thread's row (lane) and features (warp + 8 i) of the chunk -> registers; their loads overlap the previous chunk's MMAs
    const int vr = row_begin + c * kChunk + lane;
    float h1v[16], dh1v[16], h2v[16], xv[kMaxObsDim / 8], gr = 0.f;
    int act = 0;
    {
      long long d = -1;
      if (vr < row_end) {
        int agent, unit, off;
        decode_row(p.plan, net, vr, agent, unit, off);
        d = ((long long)agent * p.plan.units_per_agent + unit) * p.plan.unit_rows + off;
        const float* rp = p.rec + (size_t)d * kRowRec;
        gr = rp[kRecG]; act = __float_as_int(rp[kRecAct]);
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const size_t o = (size_t)(warp + 8 * i) * p.rows + (size_t)d;
        h1v[i] = d >= 0 ? p.h1g[o] : 0.f; dh1v[i] = d >= 0 ? p.dh1g[o] : 0.f; h2v[i] = d >= 0 ? p.h2g[o] : 0.f;
      }
#pragma unroll
      for (int m = 0; m < kMaxObsDim / 8; ++m) {
        const int f = warp + 8 * m;
        xv[m] = (d >= 0 && f < D) ? p.xg[(size_t)d * kMaxObsDim + f] : 0.f;
      }
    }
    wg_wait<0>();
    fence_regs(acc2); fence_regs(acc1); fence_regs(acc3);
    __syncthreads();   // both warpgroups are done reading the previous chunk
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int j = warp + 8 * i;
      const float dh2 = h2v[i] > 0.f ? gr * w3f[act * kHidden + j] : 0.f;
      stage_hl(smem + kSA2, 128, j, lane, dh2);
      stage_hl(smem + kSB2, 136, j, lane, h1v[i]);
      stage_hl(smem + kSA1, 128, j, lane, dh1v[i]);
      stage_hl(smem + kSA3, 128, j, lane, h2v[i]);
    }
#pragma unroll
    for (int m = 0; m < kMaxObsDim / 8; ++m)
      if (warp + 8 * m < D) stage_hl(smem + kSB1, 32, warp + 8 * m, lane, xv[m]);
    {
      const float dq = act == warp ? gr : 0.f;   // warp = output a
      stage_hl(smem + kSB3, 8, warp, lane, dq);
      float s = dq;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
      db3 += s;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes, read by wgmma through the async proxy
    __syncthreads();
    wg_fence();
    const uint32_t m_off = (uint32_t)(wg * kWgRows * kLine);
#pragma unroll
    for (int term = 0; term < 3; ++term) {
      const uint32_t ah = term == 0 ? 1u : 0u, bh = term == 1 ? 1u : 0u;   // lo*hi, hi*lo, hi*hi
#pragma unroll
      for (int ks = 0; ks < kChunk / 8; ++ks) {
        const uint32_t ko = (uint32_t)(ks * 32);
        wgmma_ss_n136(acc2, sw128_desc(sb + kSA2 + ah * 128 * kLine + m_off + ko), sw128_desc(sb + kSB2 + bh * 136 * kLine + ko), 1u);
        wgmma_ss_n32(acc1, sw128_desc(sb + kSA1 + ah * 128 * kLine + m_off + ko), sw128_desc(sb + kSB1 + bh * 32 * kLine + ko), 1u);
        wgmma_ss_n8(acc3, sw128_desc(sb + kSA3 + ah * 128 * kLine + m_off + ko), sw128_desc(sb + kSB3 + bh * 8 * kLine + ko), 1u);
      }
    }
    wg_commit();
  }
  wg_wait<0>();
  fence_regs(acc2); fence_regs(acc1); fence_regs(acc3);
  TSG(g_ts_dw, 30);
  // ---- accumulators -> this CTA's gradient sums ------------------------------------------------------------------------------------
  const NetLayout& L = p.lay;
#pragma unroll
  for (int i = 0; i < 68; ++i) {
    const int m = wg * kWgRows + 16 * wq + g + ((i & 2) ? 8 : 0), n = frag_col(i, tq);
    if (n < kHidden) gs[L.w2 + m * kHidden + n] = acc2[i];
    else if (n == kHidden) gs[L.b2 + m] = acc2[i];
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int m = wg * kWgRows + 16 * wq + g + ((i & 2) ? 8 : 0), n = frag_col(i, tq);
    if (n < D) gs[L.w1 + m * D + n] = acc1[i];
    else if (n == D) gs[L.b1 + m] = acc1[i];
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = wg * kWgRows + 16 * wq + g + ((i & 2) ? 8 : 0), n = frag_col(i, tq);
    if (n < A) gs[L.w3 + n * kHidden + m] = acc3[i];
  }
  if (lane == 0 && warp < A) gs[L.b3 + warp] = db3;
  TSG(g_ts_dw, 31);
}

// =====================================================================================================================
// launchers
// =====================================================================================================================
constexpr int kFwdTrainSmem = kImageBytes + 64 + 1024;

int tc_train_init() {
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_dqn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdTrainSmem));
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_dh1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDh1Smem));
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDwSmem));
  return MARL_OK;
}

// all three kernels walk the same episode-aligned row split, so the per-CTA partials line up with ReduceParams::cta_begin
int launch_tc_dqn_train(const TrainParams& tp, const TcBuffers& buf, cudaStream_t st, cudaEvent_t* between) {
  MARL_REQUIRE(tp.lay.in < kMaxObsDim, "tensor-core backward: observation width %d needs a spare column for the bias trick (max %d)", tp.lay.in, kMaxObsDim - 1);
  MARL_REQUIRE(tp.src.mode == 1, "tensor-core backward: rows must be gathered from the trajectory store (mode %d)", tp.src.mode);
  TcTrainParams p; memset(&p, 0, sizeof(p));
  p.plan = tp.plan; p.src = tp.src; p.lay = tp.lay; p.images = buf.image; p.bwd_images = buf.bwd_image;
  p.h1g = buf.h1; p.h2g = buf.h2; p.dh1g = buf.dh1; p.rec = buf.rec; p.xg = buf.x; p.rows = buf.rows;
  p.tq = tp.tq; p.td_ext = tp.td_ext; p.td_agent_stride = tp.td_agent_stride; p.gamma = tp.gamma; p.double_q = tp.double_q;
  p.scratch = tp.scratch; p.scratch_pitch = tp.scratch_pitch; p.loss_part = tp.loss_part;
  const int grid = tp.plan.cta_begin[tp.plan.n_nets];
  MARL_CUDA_TRY(launch_pdl(tc_dqn_fwd_kernel, dim3(grid), dim3(kTcThreads), kFwdTrainSmem, st, p));
  if (between) MARL_CUDA_TRY(cudaEventRecord(between[0], st));
  MARL_CUDA_TRY(launch_pdl(tc_dh1_kernel, dim3(grid), dim3(kTcThreads), kDh1Smem, st, p));
  if (between) MARL_CUDA_TRY(cudaEventRecord(between[1], st));
  MARL_CUDA_TRY(launch_pdl(tc_dw_kernel, dim3(grid), dim3(kTcThreads), kDwSmem, st, p));
  return MARL_OK;
}

}  // namespace marl
