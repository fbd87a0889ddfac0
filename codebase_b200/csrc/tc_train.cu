// tc_train.cu -- tensor-core (wgmma, 3xTF32) training pass of the DQN-family learner as a three-kernel pipeline (sm_90a).
//
// Same arithmetic as train_kernel<KP, kHeadDqn> (QNetwork._compute_loss + backward, marlbase/dqn/model.py:118-168), split where a
// weight gradient needs the rows of many tiles as its K dimension (tf32 wgmma reads both shared-memory operands K-major only):
//   tc_dqn_fwd_kernel   online forward (A operand in registers, weights = K-major image), head on the CUDA cores; stores H2 (FP32, in
//                        accumulator-fragment order: h2_slab), the gathered observation row, the row's outputs and the ReLU masks of H1 / H2
//                        (row record);
//                        then, on the same rows, the target network's forward (the TD target's bootstrap values)
//   tc_dh1_kernel       TD head (needs the next row's outputs, hence after the forward) -> dLoss/dq[act] and the loss statistics;
//                        dH1 = (dH2 x W2) * relu'(H1) with dH2[r][j] = g_r W3[act_r][j] relu'(H2[r][j]) built in registers (the TD loss touches
//                        one output per row); B = K-major image of W2^T; then dW1 | db1 = dH1^T x [X | 1] from dH1 staged transposed
//                        (K = rows) into shared memory, so dH1 never leaves the SM
//   tc_dw_kernel        dW2 | db2, dW3: row-streaming TN GEMMs over 32-row chunks staged transposed (K = rows) into shared memory,
//                        accumulators in registers across all the CTA's rows; db3 on the CUDA cores.  H1 is rebuilt from the gathered
//                        observation rows with the forward's own layer-1 sequence (layer1_tile) instead of round-tripping through HBM
// The partials feed the same grad_reduce_kernel / adam_kernel as the FP32 path.
#include "tc_common.cuh"
#include "dqn_heads.cuh"

namespace marl {

// observation row of a virtual row of the training batch (episode rows only: launch_tc_dqn_forward) and the row's index in every per-row buffer
__device__ __forceinline__ const float* train_row(const TcTrainParams& p, int net, int vr, size_t& d, int& agent, int& unit, int& off, int& ep) {
  decode_row(p.plan, net, vr, agent, unit, off);
  d = row_index(agent, unit, off, p.plan.units_per_agent, p.plan.unit_rows);
  ep = p.src.idx[unit];
  return p.src.traj.obs_row(ep, agent, off);
}

// The weight gradients contract over rows, so both operands of each are staged K-major (one 128-byte swizzled line of 32 rows per feature),
// hi | lo, in 32-row chunks: chunk c of a CTA is rows [row_begin + 32 c, + 32), i.e. tile c / 4, warpgroup (c / 2) % 2, half c % 2.
constexpr int kChunk = 32;
constexpr int kLine = 128;                                              // one feature's 32 rows

// byte offset of (line f, row r) in a K-major SWIZZLE_128B operand of 32 rows
__device__ __forceinline__ int line_off(int f, int r) { return f * kLine + ((((r >> 2) ^ (f & 7)) & 7) << 4) + ((r & 3) << 2); }
__device__ __forceinline__ void stage_hl(uint8_t* base, int lines, int f, int r, float x) {
  float hi, lo;
  tf32_split(x, hi, lo);
  *reinterpret_cast<float*>(base + line_off(f, r)) = hi;
  *reinterpret_cast<float*>(base + lines * kLine + line_off(f, r)) = lo;
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

// the ReLU mask words of a 64 x 128 fragment (rec field `mask`); rows of a missing source (d < 0) are skipped
__device__ __forceinline__ void store_frag_masks(const float (&v)[64], long long d0, long long d1, int quad_lane, float* rec, int mask) {
  uint32_t m0, m1;
  frag_masks(v, m0, m1);
  if (d0 >= 0) rec[(size_t)d0 * kRowRec + mask + quad_lane] = __uint_as_float(m0);
  if (d1 >= 0) rec[(size_t)d1 * kRowRec + mask + quad_lane] = __uint_as_float(m1);
}
// H2 in the forward's accumulator-fragment order.  CTA b owns a slab of 64-row tiles starting at tile h2_slab(b); its tile k (rows
// row_begin + 64 k, + 64) holds element group n (0..15: elements 4 n .. 4 n + 3, i.e. columns 8 n + 2 q, + 1 of rows 16 w + g and + 8) of thread
// u (0..127) of the warpgroup that ran it as the float4 ((h2_slab(b) + k) * 16 + n) * 128 + u.  A warp's store is then 512 contiguous bytes, and
// the weight-gradient kernel's chunk c (tile c / 2, threads [64 (c % 2), + 64)) is 16 KB in one piece.  The slab starts at the CTA's first row
// over all networks, in tiles, plus its index: every CTA of n rows has at least ceil(n / 64) tiles before the next CTA's slab, whatever the
// plan, so ceil(rows / 64) + grid tiles hold any split of `rows` rows (TcBuffers::h2_tiles).  Rows past row_end are written, never staged.
__device__ __forceinline__ size_t h2_slab(const RowPlan& p, int net, int row_begin) {
  return (size_t)(((long long)p.slot_begin[net] * p.units_per_agent * p.unit_rows + row_begin) / kWgRows) + blockIdx.x;
}
constexpr int kH2TileF4 = 16 * 128;   // float4 per 64-row tile

// Shared memory of the training forward: the online image at 0, then the target network's W1 hi | lo (1024-byte aligned, as the swizzled panels
// need) and its b1 | b2 | b3 | FP32 W3, then the mbarriers.  The target's W2 has no room of its own: it is loaded over the online W2 once every
// phase-A layer 2 has run.
constexpr int kTgtW1 = (kImageBytes + 1023) / 1024 * 1024;
constexpr int kTgtB1 = kTgtW1 + (kOffW2Hi - kOffW1Hi);
constexpr int kFwdBar = kTgtB1 + (kImageBytes - kOffB1);
constexpr int kFwdTrainSmem = kFwdBar + 4 * 8 + 1024;
static_assert(kOffW1Hi == 0 && kTgtW1 % 1024 == 0 && kFwdBar % 16 == 0 && kFwdTrainSmem <= 227 * 1024,
              "training forward: 1024-byte aligned target W1 panels, online image and target operands within the shared memory of one SM");

// Phase A runs the online network on the CTA's rows (warpgroup w: its 64-row tiles k = w, w + 2, ...) and stores what the backward needs.
// Phase B (p.tgt_images != NULL) runs the target network on the same rows and writes p.tq_out.  Each thread of phase B re-reads the observation
// values it stored in xg in phase A (same rows, same fragment mapping) instead of gathering them from the trajectory store again.  Tile split of
// phase B: every warpgroup takes its own phase-A tiles again, except that with an odd tile count the last tile moves from warpgroup 0 (which had
// one tile more in phase A) to the end of warpgroup 1's list, so both run the same number of tiles over the two phases.  Warpgroup 1 reads that
// tile's rows after the target W2 wait, which thread 0 releases only after warpgroup 0 has passed the named barrier behind its stores.
// Barriers: [0] online W1 + biases + FP32 W3, [1] online W2, [2] target W1 + biases + FP32 W3 (both at kernel start), [3] target W2 (issued
// by thread 0 once both warpgroups are past their last phase-A layer 2: named barrier 1).
template <int K1>
__global__ void __launch_bounds__(kTcThreads, 1) tc_dqn_fwd_kernel(TcTrainParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kFwdBar);
  const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, lane = t & 31, g = lane >> 2, tq = lane & 3;
  int net, row_begin, row_end;
  cta_rows(p.plan, net, row_begin, row_end);
  if (row_begin >= row_end) { pdl_wait(); return; }
  TSG(g_ts_fwd, 0);
  const bool tgt = p.tgt_images != nullptr;
  if (t == 0) { for (int i = 0; i < 4; ++i) mbar_init(bar + i, 1); fence_mbar_init(); }
  __syncthreads();
  pdl_wait();   // nothing above touches global memory
  pdl_launch_dependents();
  const uint32_t sb = smem_u32(smem);
  if (t == 0) {
    tma_forward_image(sb, p.images + (size_t)net * kImageBytes, bar);
    if (tgt) {
      const uint8_t* timg = p.tgt_images + (size_t)net * kImageBytes;
      mbar_expect_tx(bar + 2, (uint32_t)((kOffW2Hi - kOffW1Hi) + (kImageBytes - kOffB1)));
      tma_image_range(sb + kTgtW1, timg, kOffW1Hi, kOffW2Hi, bar + 2);
      tma_image_range(sb + kTgtB1 - kOffB1, timg, kOffB1, kImageBytes, bar + 2);
    }
  }
  const float* b1 = reinterpret_cast<const float*>(smem + kOffB1);
  const float* b2 = reinterpret_cast<const float*>(smem + kOffB2);
  const float* b3 = reinterpret_cast<const float*>(smem + kOffB3);
  const float* w3f = reinterpret_cast<const float*>(smem + kOffW3F);
  const int D = p.src.D, A = p.lay.out;
  // both warpgroups are done with the online W2: warpgroup 0 (the last to finish phase A: it has as many tiles as warpgroup 1 or one more)
  // waits for warpgroup 1's arrival, then thread 0 loads the target's W2 over it
  auto online_w2_done = [&]() {
    if (wg == 0) {
      named_bar_sync(1, kTcThreads);
      if (t == 0) {
        mbar_expect_tx(bar + 3, (uint32_t)(kOffB1 - kOffW2Hi));
        tma_image_range(sb, p.tgt_images + (size_t)net * kImageBytes, kOffW2Hi, kOffB1, bar + 3);
      }
    } else {
      named_bar_arrive(1, kTcThreads);
    }
  };
  bool first = true;
  float4* const h2s = p.h2s + h2_slab(p.plan, net, row_begin) * kH2TileF4 + (t & 127);
  int it = 0;   // this warpgroup's phase-A tile count so far (probe slots 1 + 3 it .. 3 + 3 it of warpgroup 0's first five tiles)
  for (int vr0 = row_begin + kWgRows * wg; vr0 < row_end; vr0 += kTileRows, ++it) {
    if (it < 5) TSG(g_ts_fwd, 1 + 3 * it);
    const int r0 = vr0 + 16 * wq + g, r1 = r0 + 8;
    size_t d0u = 0, d1u = 0;
    int agent, unit, off, ep;
    const float* s0 = r0 < row_end ? train_row(p, net, r0, d0u, agent, unit, off, ep) : nullptr;
    const float* s1 = r1 < row_end ? train_row(p, net, r1, d1u, agent, unit, off, ep) : nullptr;
    const long long d0 = s0 ? (long long)d0u : -1, d1 = s1 ? (long long)d1u : -1;
    float acc[64];
    {
      float x[kMaxObsDim / 8][4];
      load_x_frag(s0, s1, D, tq, x);
#pragma unroll
      for (int ks = 0; ks < kMaxObsDim / 8; ++ks) {   // the gathered row for the dH1 and weight-gradient kernels (and phase B)
        const int c = 8 * ks + 2 * tq;
        if (ks < K1) {
          if (d0 >= 0) *reinterpret_cast<float2*>(p.xg + (size_t)d0 * p.x_pitch + c) = make_float2(x[ks][0], x[ks][2]);
          if (d1 >= 0) *reinterpret_cast<float2*>(p.xg + (size_t)d1 * p.x_pitch + c) = make_float2(x[ks][1], x[ks][3]);
        }
      }
      if (first) mbar_wait(bar, 0);
      layer1_tile<K1>(acc, x, sb + kOffW1Hi, b1, tq);
    }
    store_frag_masks(acc, d0, d1, tq, p.rec, kRecMask1);   // H1 itself is rebuilt by the weight-gradient kernel
    {
      uint32_t hi[16][4], lo[16][4];
      frag_to_a(acc, hi, lo);
      if (first) { mbar_wait(bar + 1, 0); first = false; }
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      layer_rs<16>(acc, hi, lo, sb + kOffW2Hi, sb + kOffW2Lo, 16);
    }
    if (it < 5) TSG(g_ts_fwd, 2 + 3 * it);
    if (tgt && vr0 + kTileRows >= row_end) online_w2_done();   // this warpgroup's last phase-A tile
    float q0[kOutPad], q1[kOutPad];
    head_quad(acc, b2, w3f, A, tq, q0, q1);   // acc = H2 from here
    {
      float4* h2 = h2s + (size_t)((vr0 - row_begin) / kWgRows) * kH2TileF4;
#pragma unroll
      for (int n = 0; n < 16; ++n) h2[n * 128] = make_float4(acc[4 * n], acc[4 * n + 1], acc[4 * n + 2], acc[4 * n + 3]);
    }
    store_frag_masks(acc, d0, d1, tq, p.rec, kRecMask2);
    const long long d = tq == 0 ? d0 : d1;
    if (tq < 2 && d >= 0) {
      float* o = p.rec + (size_t)d * kRowRec;
#pragma unroll
      for (int a = 0; a < kOutPad; ++a) {
        const float v = a < A ? (tq == 0 ? q0[a] : q1[a]) + b3[a] : 0.f;
        o[a] = v;
        if (p.q_out != nullptr && a < A) p.q_out[(size_t)d * A + a] = v;
      }
    }
    if (it < 5) TSG(g_ts_fwd, 3 + 3 * it);
  }
  if (!tgt) { TSG(g_ts_fwd, 31); return; }
  if (row_begin + kWgRows * wg >= row_end) online_w2_done();   // no phase-A tile (warpgroup 1 of a CTA of at most 64 rows)
  TSG(g_ts_fwd, 16);
  // ---- phase B: the target network on the same rows -> tq_out
  const float* tb1 = reinterpret_cast<const float*>(smem + kTgtB1);
  const float* tb2 = reinterpret_cast<const float*>(smem + kTgtB1 + (kOffB2 - kOffB1));
  const float* tb3 = reinterpret_cast<const float*>(smem + kTgtB1 + (kOffB3 - kOffB1));
  const float* tw3f = reinterpret_cast<const float*>(smem + kTgtB1 + (kOffW3F - kOffB1));
  const int n_tiles = (row_end - row_begin + kWgRows - 1) / kWgRows, n_mine = wg == 0 ? n_tiles / 2 : (n_tiles + 1) / 2;
  first = true;
  for (int i = 0; i < n_mine; ++i) {
    const bool moved = wg + 2 * i >= n_tiles;   // warpgroup 1's extra tile (odd n_tiles): the last one, stored by warpgroup 0
    const int vr0 = row_begin + kWgRows * (moved ? n_tiles - 1 : wg + 2 * i);
    if (moved && first) mbar_wait(bar + 3, 0);   // its only tile (n_tiles == 1): read warpgroup 0's stores only after the barrier as well
    const int r0 = vr0 + 16 * wq + g, r1 = r0 + 8;
    long long d0 = -1, d1 = -1;
    {
      int agent, unit, off;
      if (r0 < row_end) { decode_row(p.plan, net, r0, agent, unit, off); d0 = (long long)row_index(agent, unit, off, p.plan.units_per_agent, p.plan.unit_rows); }
      if (r1 < row_end) { decode_row(p.plan, net, r1, agent, unit, off); d1 = (long long)row_index(agent, unit, off, p.plan.units_per_agent, p.plan.unit_rows); }
    }
    float acc[64];
    {
      float x[kMaxObsDim / 8][4];
#pragma unroll
      for (int ks = 0; ks < kMaxObsDim / 8; ++ks) {   // what phase A stored: zero beyond D, and for rows past the CTA's end
        const int c = 8 * ks + 2 * tq;
        float2 v0 = make_float2(0.f, 0.f), v1 = make_float2(0.f, 0.f);
        if (ks < K1) {
          if (d0 >= 0) v0 = *reinterpret_cast<const float2*>(p.xg + (size_t)d0 * p.x_pitch + c);
          if (d1 >= 0) v1 = *reinterpret_cast<const float2*>(p.xg + (size_t)d1 * p.x_pitch + c);
        }
        x[ks][0] = v0.x; x[ks][1] = v1.x; x[ks][2] = v0.y; x[ks][3] = v1.y;
      }
      if (first) mbar_wait(bar + 2, 0);
      layer1_tile<K1>(acc, x, sb + kTgtW1, tb1, tq);
    }
    {
      uint32_t hi[16][4], lo[16][4];
      frag_to_a(acc, hi, lo);
      if (first) { mbar_wait(bar + 3, 0); first = false; }
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      layer_rs<16>(acc, hi, lo, sb + kOffW2Hi, sb + kOffW2Lo, 16);
    }
    float q0[kOutPad], q1[kOutPad];
    head_quad(acc, tb2, tw3f, A, tq, q0, q1);
    const long long d = tq == 0 ? d0 : d1;
    if (tq < 2 && d >= 0) {
      float* o = p.tq_out + (size_t)d * A;
#pragma unroll
      for (int a = 0; a < kOutPad; ++a)
        if (a < A) o[a] = (tq == 0 ? q0[a] : q1[a]) + tb3[a];
    }
  }
  TSG(g_ts_fwd, 31);
}

// =====================================================================================================================
// 2. TD head + dH1 = (dH2 x W2) * relu'(H1) + dW1 | db1 [j1][i | 1] += dH1^T x [X | 1]^T
// =====================================================================================================================
// Two staging buffers, one chunk each: A = dH1 (128 lines), B = [X | 1] (32 lines, line D = ones, the lines behind it zero)
constexpr int kDh1SA = kBwdImageBytes;                        // behind the W2^T image: [2][hi | lo][128 lines]
constexpr int kDh1SB = kDh1SA + 2 * 2 * 128 * kLine;          // [2][hi | lo][32 lines]
constexpr int kDh1W3 = kDh1SB + 2 * 2 * 32 * kLine;           // FP32 copy of W3 [8][128]
constexpr int kDh1Bar = kDh1W3 + kOutPad * kHidden * 4;
constexpr int kDh1Red = kDh1Bar + 64;                         // [2][kTcThreads] loss statistics
constexpr int kDh1Smem = kDh1Red + 2 * kTcThreads * 4 + 1024;
static_assert(kDh1SA % 1024 == 0 && kDh1SB % 1024 == 0 && kDh1Smem <= 227 * 1024,
              "dH1 kernel: 1024-byte aligned operands within the shared memory of one SM");

// dLoss/dq[act] of one row (0 at t == T) and its loss statistics (delta^2 filled, filled on agent 0)
__device__ __forceinline__ float td_grad(const TcTrainParams& p, size_t d, int agent, int b, int tt, int ep, int& act, float& s0, float& s1) {
  const TrajView& tv = p.src.traj;
  const int T = tv.T, A = p.lay.out;
  act = 0;
  if (tt >= T) return 0.f;
  act = tv.act[tv.step_at(ep, agent, tt)];
  if (p.td_ext) return p.td_ext[(size_t)agent * p.td_agent_stride + (size_t)b * T + tt];
  const float rew = tv.rew[tv.step_at(ep, agent, tt)];
  const float filled = (float)tv.filled[tv.filled_at(ep, tt)], done1 = (float)tv.done[tv.done_at(ep, tt + 1)];
  const float* q = p.rec + d * kRowRec;
  const float* qn = q + kRowRec;                 // the next row of the same episode
  const float* tq = p.tq + (d + 1) * A;          // target outputs share the [agent][unit][T + 1] row layout
  return td_error(q[act], td_target(rew, p.gamma, next_value(qn, tq, A, p.double_q), done1), filled, agent == 0, s0, s1, p.huber);
}

// One staging phase of the dW1 product: warpgroup `owner` stages its two chunks of a tile, c and c + 1 (its 64 rows of dH1 from the accumulator
// fragments `h` masked by relu'(H1) `m1`, and of [X | 1] from `xv`), one per buffer; then both warpgroups issue the MMAs of those that hold rows
// (warpgroup w: output rows j1 in [64 w, 64 w + 64); term order lo*hi, hi*lo, hi*hi per k-step).  Block-wide; the caller skips a phase with
// no rows (c past the CTA's rows) on every thread.
__device__ __forceinline__ void dw1_phase(int owner, int c, int row_begin, int row_end, int D, uint8_t* smem, uint32_t sb, const float (&h)[64],
                                          uint64_t m1, const float (&xv)[2][kMaxObsDim / 4], float (&acc1)[16]) {
  const int t = threadIdx.x, wg = t >> 7, wq = (t >> 5) & 3, g = (t & 31) >> 2, tq = t & 3;
  const int half = wq >> 1, cr = 16 * (wq & 1) + g;   // this warp's rows are the warpgroup's chunk `half`, rows cr and cr + 8 of it
  wg_wait<0>();
  fence_regs(acc1);
  __syncthreads();   // both warpgroups are done reading the buffers
  if (wg == owner && row_begin + (c + half) * kChunk < row_end) {
    uint8_t* sa = smem + kDh1SA + half * 2 * 128 * kLine;
    uint8_t* sbx = smem + kDh1SB + half * 2 * 32 * kLine;
#pragma unroll
    for (int i = 0; i < 64; ++i) stage_hl(sa, 128, frag_col(i, tq), cr + ((i & 2) ? 8 : 0), ((m1 >> i) & 1) ? h[i] : 0.f);
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int m = 0; m < kMaxObsDim / 4; ++m)
        if (tq + 4 * m < D) stage_hl(sbx, 32, tq + 4 * m, cr + 8 * k, xv[k][m]);
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes, read by wgmma through the async proxy
  __syncthreads();
  wg_fence();
  const uint32_t m_off = (uint32_t)(wg * kWgRows * kLine);
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    if (row_begin + (c + b) * kChunk >= row_end) continue;
    const uint32_t a_base = sb + kDh1SA + b * 2 * 128 * kLine + m_off, b_base = sb + kDh1SB + b * 2 * 32 * kLine;
#pragma unroll
    for (int term = 0; term < 3; ++term) {
      const uint32_t ah = term == 0 ? 1u : 0u, bh = term == 1 ? 1u : 0u;   // lo*hi, hi*lo, hi*hi
#pragma unroll
      for (int ks = 0; ks < kChunk / 8; ++ks) {
        const uint32_t ko = (uint32_t)(ks * 32);
        wgmma_ss_n32(acc1, sw128_desc(a_base + ah * 128 * kLine + ko), sw128_desc(b_base + bh * 32 * kLine + ko), 1u);
      }
    }
  }
  wg_commit();
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
  const int D = p.src.D;
  for (int i = t; i < 2 * 32 * kChunk; i += kTcThreads) {   // constant lines of both B buffers: the ones line (hi 1, lo 0) and the zero lines behind it
    const int b = i / (32 * kChunk), f = (i / kChunk) % 32, r = i % kChunk;
    if (f >= D) stage_hl(smem + kDh1SB + b * 2 * 32 * kLine, 32, f, r, f == D ? 1.f : 0.f);
  }
  float acc1[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc1[i] = 0.f;
  // dH1 fragments, relu'(H1) and observation rows of the tile before: warpgroup 1 stages them after this tile's loads have been issued
  float acc[64], xv[2][kMaxObsDim / 4];
  uint64_t m1 = 0;
  float st0 = 0.f, st1 = 0.f;
  bool first = true;
  // both warpgroups walk every tile (the staging barriers are block-wide); a warpgroup whose rows all lie past row_end skips its product
  for (int t0 = row_begin; t0 < row_end; t0 += kTileRows) {
    const int vr0 = t0 + kWgRows * wg, c0 = (t0 - row_begin) / kChunk;
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
    // the previous tile's chunks 2 and 3 (warpgroup 1), behind this tile's gathers and mask loads: the MMAs on the buffers are long done by now
    if (t0 > row_begin && row_begin + (c0 - 2) * kChunk < row_end) dw1_phase(1, c0 - 2, row_begin, row_end, D, smem, sb, acc, m1, xv, acc1);
    float v[64];
    m1 = 0;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int k = (i >> 1) & 1, bit = ((i >> 2) << 1) | (i & 1);
      v[i] = ((mh2[k] >> bit) & 1u) ? gr[k] * w3f[act[k] * kHidden + frag_col(i, tq)] : 0.f;
      m1 |= (uint64_t)((mh1[k] >> bit) & 1u) << i;
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    if (vr0 < row_end) {
      uint32_t hi[16][4], lo[16][4];
      frag_to_a(v, hi, lo);
      // D[r][j1] = sum_{j2} dH2[r][j2] W2[j2][j1]: B = K-major image of W2^T (rows j1, K = j2)
      layer_rs<16>(acc, hi, lo, sb, sb + 4 * kPanelBytes, 16);
    }
    // the observation rows of this thread's two rows, features tq + 4 m (a quad covers a row; 0 for rows without a source)
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int m = 0; m < kMaxObsDim / 4; ++m) {
        const int f = tq + 4 * m;
        xv[k][m] = (d[k] >= 0 && f < D) ? p.xg[(size_t)d[k] * p.x_pitch + f] : 0.f;
      }
    const long long dr = tq == 0 ? d[0] : d[1];
    if (tq < 2 && dr >= 0) {
      float* rp = p.rec + (size_t)dr * kRowRec;
      rp[kRecG] = tq == 0 ? gr[0] : gr[1]; rp[kRecAct] = __int_as_float(tq == 0 ? act[0] : act[1]);
    }
    // ---- dW1 | db1 over the tile's four chunks in row order: warpgroup 0 stages chunks 0 and 1 now, warpgroup 1 chunks 2 and 3 at the top of
    // the next tile (or after the last one)
    dw1_phase(0, c0, row_begin, row_end, D, smem, sb, acc, m1, xv, acc1);
  }
  {
    const int c_last = (row_end - 1 - row_begin) / kTileRows * (kTileRows / kChunk);
    if (row_begin + (c_last + 2) * kChunk < row_end) dw1_phase(1, c_last + 2, row_begin, row_end, D, smem, sb, acc, m1, xv, acc1);
  }
  wg_wait<0>();
  fence_regs(acc1);
  TSG(g_ts_dh1, 30);
  // ---- dW1 | db1 -> this CTA's gradient sums (the weight-gradient kernel writes the other parameters) ---------------------------------
  {
    const NetLayout& L = p.lay;
    float* gs = p.scratch + (size_t)blockIdx.x * p.scratch_pitch;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int m = wg * kWgRows + 16 * wq + g + ((i & 2) ? 8 : 0), n = frag_col(i, tq);
      if (n < D) gs[L.w1 + m * D + n] = acc1[i];
      else if (n == D) gs[L.b1 + m] = acc1[i];
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
//   dW2 | db2 [j2][j1 | 1] += dH2^T x [H1 | 1]^T   (A: 128 lines, B: 136 lines, line 128 = ones)
//   dW3^T [j][a]           += H2^T x dq^T          (B: 8 lines, dq[r][a] = g_r at a = act_r)
// Warpgroup w accumulates the M rows [64 w, 64 w + 64) of both.  A2 and A3 are staged per chunk by all eight warps from the forward's fragment
// order of H2 (h2_slab): thread t loads element groups n = 4 (t / 64) + m (m < 4) of forward thread u = 64 (c % 2) + t % 64, four 16-byte loads
// of rows cr and cr + 8 (cr = 16 (warp % 2) + lane / 4), columns 8 n + 2 (lane % 4) and + 1; under line_off the 32 lanes of a staging store hit
// 32 distinct banks.  B3 and db3 are staged lane = row, and the fragment rows take g and act from those lanes by shuffle.  H1 is rebuilt per 64
// rows (two chunks) by the warpgroup that ran those rows in the forward (layer1_tile on the W1 panels of the forward image) and staged from its
// accumulator fragments into two B2 buffers, one per chunk.
// The FP32 copy of W3 has rows of kW3Pitch = 136 floats, read as float2 (columns 8 n + 2 q, + 1): the four lanes of a row cover eight banks from
// 8 act on, so the four rows of a half-warp sit in distinct banks unless two actions differ by 4 (2-way); with a pitch of 128 every action would
// sit in the same banks (up to 4-way).
constexpr int kB2Bytes = 2 * 136 * kLine;                                  // one chunk of [H1 | 1], hi | lo
constexpr int kW3Pitch = kHidden + 8;
constexpr int kSA2 = 0, kSB2 = kSA2 + 2 * 128 * kLine, kSA3 = kSB2 + 2 * kB2Bytes, kSB3 = kSA3 + 2 * 128 * kLine, kSW1 = kSB3 + 2 * 8 * kLine;
constexpr int kSW3 = kSW1 + (kOffW2Hi - kOffW1Hi);                         // behind the W1 hi | lo panels of the forward image
constexpr int kSB1 = kSW3 + (kOutPad * kW3Pitch * 4 + 15) / 16 * 16, kSBar = kSB1 + kHidden * 4;
constexpr int kDwSmem = kSBar + 64 + 1024;
static_assert(kSB2 % 1024 == 0 && kB2Bytes % 1024 == 0 && kSA3 % 1024 == 0 && kSB3 % 1024 == 0 && kSW1 % 1024 == 0 && kSB1 % 16 == 0 &&
              kDwSmem <= 227 * 1024, "weight-gradient staging: 1024-byte aligned operands within the shared memory of one SM");

// gathered observation row of a virtual row (stored by the forward)
__device__ __forceinline__ const float* xg_row(const TcTrainParams& p, int net, int vr) {
  int agent, unit, off;
  decode_row(p.plan, net, vr, agent, unit, off);
  return p.xg + row_index(agent, unit, off, p.plan.units_per_agent, p.plan.unit_rows) * (size_t)p.x_pitch;
}

template <int K1>
__global__ void __launch_bounds__(kTcThreads, 1) tc_dw_kernel(TcTrainParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align_smem_1024(smem_raw);
  const float* w3f = reinterpret_cast<const float*>(smem + kSW3);
  const float* b1 = reinterpret_cast<const float*>(smem + kSB1);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kSBar);
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
  const uint32_t sb = smem_u32(smem);
  if (t == 0) {  // W1 hi | lo + b1 of the forward image: TMA bulk copies onto one mbarrier
    mbar_init(bar, 1); fence_mbar_init();
    const uint8_t* img = p.images + (size_t)net * kImageBytes;
    mbar_expect_tx(bar, (uint32_t)((kOffW2Hi - kOffW1Hi) + kHidden * 4));
    tma_image_range(sb + kSW1 - kOffW1Hi, img, kOffW1Hi, kOffW2Hi, bar);
    tma_bulk_g2s(sb + kSB1, img + kOffB1, kHidden * 4, bar);
  }
  const int A = p.lay.out, D = p.src.D;
  // constant lines of both B2 buffers: the ones line (hi 1, lo 0) of [H1 | 1] and the zero lines behind it; W3 copy
  for (int i = t; i < 2 * 8 * kChunk; i += kTcThreads) {
    const int b = i / (8 * kChunk), f = 128 + (i / kChunk) % 8, r = i % kChunk;
    stage_hl(smem + kSB2 + b * kB2Bytes, 136, f, r, f == 128 ? 1.f : 0.f);
  }
  {
    const float* w3src = reinterpret_cast<const float*>(p.images + (size_t)net * kImageBytes + kOffW3F);
    for (int i = t; i < kOutPad * kHidden; i += kTcThreads) reinterpret_cast<float*>(smem + kSW3)[(i / kHidden) * kW3Pitch + i % kHidden] = w3src[i];
  }
  __syncthreads();
  TSG(g_ts_dw, 1);
  float acc2[68], acc3[4];
#pragma unroll
  for (int i = 0; i < 68; ++i) acc2[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) acc3[i] = 0.f;
  float db3 = 0.f;   // warp a, lane 0: sum of dq[.][a]
  bool first = true;
  const int n_chunks = (row_end - row_begin + kChunk - 1) / kChunk;
  // this thread's H2 of chunk 0: element groups 4 (t / 64) + m of forward thread t % 64 of tile 0 (chunk c: + tile c / 2, + 64 (c % 2) threads)
  const float4* const h2s = p.h2s + h2_slab(p.plan, net, row_begin) * kH2TileF4 + 4 * (t >> 6) * 128 + (t & 63);
  const int cr = 16 * (warp & 1) + g;   // this thread's fragment rows of every chunk: cr and cr + 8
  int c = 0;
  do {   // n_chunks >= 1: with a zero-trip path (a for loop) ptxas serialises every wgmma of the kernel (C7515)
    TSG(g_ts_dw, 2 + c);   // chunk c: slots 2-29 (chunks past 27 land on 30 / 31, which the epilogue writes again)
    // ---- the chunk's rows' g and act (lane = row) and this thread's H2 fragment -> registers; their loads overlap the previous chunk's MMAs
    const int vr = row_begin + c * kChunk + lane;
    float gr = 0.f;
    int act = 0;
    if (vr < row_end) {
      int agent, unit, off;
      decode_row(p.plan, net, vr, agent, unit, off);
      const float* rp = p.rec + row_index(agent, unit, off, p.plan.units_per_agent, p.plan.unit_rows) * kRowRec;
      gr = rp[kRecG]; act = __float_as_int(rp[kRecAct]);
    }
    float4 h2q[4];
    {
      const float4* src = h2s + (size_t)(c >> 1) * kH2TileF4 + 64 * (c & 1);
#pragma unroll
      for (int m = 0; m < 4; ++m) h2q[m] = src[m * 128];
    }
    // ---- H1 of chunks c and c + 1 (even c): the 64 rows of warpgroup (c / 2) % 2 of tile c / 4, as the forward computed them
    const bool rebuild = (c & 1) == 0 && wg == ((c >> 1) & 1);
    const int r0 = row_begin + c * kChunk + 16 * wq + g, r1 = r0 + 8;
    float x[kMaxObsDim / 8][4], h1[64];
    if (rebuild) load_x_frag(r0 < row_end ? xg_row(p, net, r0) : nullptr, r1 < row_end ? xg_row(p, net, r1) : nullptr, D, tq, x);
    wg_wait<0>();
    fence_regs(acc2); fence_regs(acc3);
    // layer 1 behind the wait (its own wgmma.wait_group would wait for this warpgroup's chunk MMAs anyway); the x loads are already in flight
    if (rebuild) {
      if (first) { mbar_wait(bar, 0); first = false; }
      layer1_tile<K1>(h1, x, sb + kSW1, b1, tq);
    }
    __syncthreads();   // both warpgroups are done reading the previous chunk
#pragma unroll
    for (int k = 0; k < 2; ++k) {   // row cr + 8 k of the chunk: H2 (0 past the CTA's rows) and dH2 = g W3[act][j] relu'(H2)
      const int r = cr + 8 * k;
      const bool live = row_begin + c * kChunk + r < row_end;
      const float g_r = __shfl_sync(0xFFFFFFFFu, gr, r);
      const int act_r = __shfl_sync(0xFFFFFFFFu, act, r);
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const int j = 8 * (4 * (t >> 6) + m) + 2 * tq;
        const float2 w = *reinterpret_cast<const float2*>(w3f + act_r * kW3Pitch + j);
        const float h0 = live ? (k ? h2q[m].z : h2q[m].x) : 0.f, h1v = live ? (k ? h2q[m].w : h2q[m].y) : 0.f;
        stage_hl(smem + kSA2, 128, j, r, h0 > 0.f ? g_r * w.x : 0.f);
        stage_hl(smem + kSA2, 128, j + 1, r, h1v > 0.f ? g_r * w.y : 0.f);
        stage_hl(smem + kSA3, 128, j, r, h0);
        stage_hl(smem + kSA3, 128, j + 1, r, h1v);
      }
    }
    {
      const float dq = act == warp ? gr : 0.f;   // warp = output a
      stage_hl(smem + kSB3, 8, warp, lane, dq);
      float s = dq;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
      db3 += s;
    }
    if (rebuild) {   // this warp's rows are chunk c + (wq >> 1), rows 16 (wq & 1) + g and + 8 of it (0 past the CTA's rows)
      uint8_t* b2 = smem + kSB2 + (wq >> 1) * kB2Bytes;
      const int cr = 16 * (wq & 1) + g;
#pragma unroll
      for (int i = 0; i < 64; ++i) stage_hl(b2, 136, frag_col(i, tq), cr + ((i & 2) ? 8 : 0), (((i & 2) ? r1 : r0) < row_end) ? h1[i] : 0.f);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes, read by wgmma through the async proxy
    __syncthreads();
    wg_fence();
    const uint32_t m_off = (uint32_t)(wg * kWgRows * kLine), b2_off = (uint32_t)(kSB2 + (c & 1) * kB2Bytes);
#pragma unroll
    for (int term = 0; term < 3; ++term) {
      const uint32_t ah = term == 0 ? 1u : 0u, bh = term == 1 ? 1u : 0u;   // lo*hi, hi*lo, hi*hi
#pragma unroll
      for (int ks = 0; ks < kChunk / 8; ++ks) {
        const uint32_t ko = (uint32_t)(ks * 32);
        wgmma_ss_n136(acc2, sw128_desc(sb + kSA2 + ah * 128 * kLine + m_off + ko), sw128_desc(sb + b2_off + bh * 136 * kLine + ko), 1u);
        wgmma_ss_n8(acc3, sw128_desc(sb + kSA3 + ah * 128 * kLine + m_off + ko), sw128_desc(sb + kSB3 + bh * 8 * kLine + ko), 1u);
      }
    }
    wg_commit();
  } while (++c < n_chunks);
  wg_wait<0>();
  fence_regs(acc2); fence_regs(acc3);
  TSG(g_ts_dw, 30);
  // ---- accumulators -> this CTA's gradient sums ------------------------------------------------------------------------------------
  const NetLayout& L = p.lay;
#pragma unroll
  for (int i = 0; i < 64; i += 2) {   // columns n, n + 1 of W2 in one 8-byte store (L.w2 and n are even, the CTA pitch a multiple of 4 floats)
    const int m = wg * kWgRows + 16 * wq + g + ((i & 2) ? 8 : 0), n = frag_col(i, tq);
    *reinterpret_cast<float2*>(gs + L.w2 + m * kHidden + n) = make_float2(acc2[i], acc2[i + 1]);
  }
#pragma unroll
  for (int i = 64; i < 68; ++i) {
    const int m = wg * kWgRows + 16 * wq + g + ((i & 2) ? 8 : 0), n = frag_col(i, tq);
    if (n == kHidden) gs[L.b2 + m] = acc2[i];
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

int tc_train_init() {
  MARL_CUDA_TRY(cudaFuncSetAttribute(tc_dh1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDh1Smem));
  for (int D = 1; D <= kMaxObsDim; D += 8)
    if (int rc = with_k1(D, [](auto k1) {
          MARL_CUDA_TRY(cudaFuncSetAttribute(tc_dqn_fwd_kernel<decltype(k1)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFwdTrainSmem));
          MARL_CUDA_TRY(cudaFuncSetAttribute(tc_dw_kernel<decltype(k1)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, kDwSmem));
          return MARL_OK;
        }))
      return rc;
  return MARL_OK;
}

static TcTrainParams tc_params(const TrainParams& tp, const TcBuffers& buf) {
  TcTrainParams p; memset(&p, 0, sizeof(p));
  p.plan = tp.plan; p.src = tp.src; p.lay = tp.lay; p.images = buf.image; p.bwd_images = buf.bwd_image;
  p.h2s = reinterpret_cast<float4*>(buf.h2); p.rec = buf.rec; p.xg = buf.x; p.x_pitch = 8 * ((tp.src.D + 7) / 8);
  p.tq = tp.tq; p.td_ext = tp.td_ext; p.td_agent_stride = tp.td_agent_stride; p.gamma = tp.gamma; p.double_q = tp.double_q; p.huber = tp.huber;
  p.scratch = tp.scratch; p.scratch_pitch = tp.scratch_pitch; p.loss_part = tp.loss_part;
  return p;
}

// all three kernels walk the same episode-aligned row split, so the per-CTA partials line up with ReduceParams::cta_begin
int launch_tc_dqn_forward(const TrainParams& tp, const TcBuffers& buf, const uint8_t* tgt_images, float* tq_out, float* q_out, cudaStream_t st) {
  MARL_REQUIRE(tp.lay.in < kMaxObsDim, "tensor-core backward: observation width %d needs a spare column for the bias trick (max %d)", tp.lay.in, kMaxObsDim - 1);
  MARL_REQUIRE(tp.src.mode == 1, "tensor-core backward: rows must be gathered from the trajectory store (mode %d)", tp.src.mode);
  MARL_REQUIRE(tgt_images == nullptr || tq_out != nullptr, "tensor-core training forward: target images without an output buffer");
  {
    const RowPlan& pl = tp.plan;
    const size_t tiles = ((size_t)pl.slot_begin[pl.n_nets] * pl.units_per_agent * pl.unit_rows + kWgRows - 1) / kWgRows + pl.cta_begin[pl.n_nets];
    MARL_REQUIRE(tiles <= buf.h2_tiles, "tensor-core training forward: the H2 slabs need %zu tiles, %zu allocated", tiles, buf.h2_tiles);
  }
  TcTrainParams p = tc_params(tp, buf);
  p.tgt_images = tgt_images; p.tq_out = tq_out; p.q_out = q_out;
  return with_k1(tp.src.D, [&](auto k1) {
    MARL_CUDA_TRY(launch_pdl(tc_dqn_fwd_kernel<decltype(k1)::value>, dim3(tp.plan.cta_begin[tp.plan.n_nets]), dim3(kTcThreads), kFwdTrainSmem, st, p));
    return MARL_OK;
  });
}

int launch_tc_dqn_backward(const TrainParams& tp, const TcBuffers& buf, cudaStream_t st, cudaEvent_t after_dh1) {
  const TcTrainParams p = tc_params(tp, buf);
  const int grid = tp.plan.cta_begin[tp.plan.n_nets];
  MARL_CUDA_TRY(launch_pdl(tc_dh1_kernel, dim3(grid), dim3(kTcThreads), kDh1Smem, st, p));
  if (after_dh1) MARL_CUDA_TRY(cudaEventRecord(after_dh1, st));
  return with_k1(tp.src.D, [&](auto k1) {
    MARL_CUDA_TRY(launch_pdl(tc_dw_kernel<decltype(k1)::value>, dim3(grid), dim3(kTcThreads), kDwSmem, st, p));
    return MARL_OK;
  });
}

}  // namespace marl
