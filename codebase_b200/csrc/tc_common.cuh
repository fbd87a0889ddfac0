// tc_common.cuh -- Hopper (sm_90a) tensor-core primitives shared by the 3xTF32 kernels: warpgroup MMA (wgmma) wrappers, shared-memory
// matrix descriptors, mbarrier + TMA bulk copies, and the packed weight-image layout.
#pragma once
#include "learner.cuh"

namespace marl {

constexpr int kTcThreads = 256;                    // two warpgroups; warpgroup w owns rows [64 w, 64 w + 64) of every 128-row tile
constexpr int kWgRows = 64;                        // rows of one wgmma (M)
constexpr int kPanelBytes = kHidden * 128;         // 128 rows x 32 floats
// image layout (bytes): W1 hi | W1 lo | W2 hi (4 panels) | W2 lo | b1 | b2 | b3 | FP32 W3 [8][128]
constexpr int kOffW1Hi = 0, kOffW1Lo = kOffW1Hi + kPanelBytes, kOffW2Hi = kOffW1Lo + kPanelBytes, kOffW2Lo = kOffW2Hi + 4 * kPanelBytes;
constexpr int kOffB1 = kOffW2Lo + 4 * kPanelBytes, kOffB2 = kOffB1 + kHidden * 4, kOffB3 = kOffB2 + kHidden * 4;
constexpr int kOffW3F = kOffB3 + kOutPad * 4;      // plain FP32 copy of W3 [8][128]: the head runs on the CUDA cores
constexpr int kImageBytes = kOffW3F + kOutPad * kHidden * 4;
// backward image: W2^T as a K-major operand (rows = input features j1, K = output features j2), hi | lo
constexpr int kBwdImageBytes = 8 * kPanelBytes;
static_assert(kOffB1 % 16 == 0 && kOffW3F % 16 == 0 && kImageBytes % 16 == 0, "TMA bulk copies move multiples of 16 bytes");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// round to TF32 (10-bit mantissa), nearest with ties away from zero: what cvt.rna.tf32.f32 computes for finite inputs
__device__ __forceinline__ float tf32_rn(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }
// 3xTF32 operand split of values produced on the fly: hi = x with the 13 low mantissa bits cleared (exactly representable in TF32), lo = x - hi
// (exact in FP32, < 2^-10 |x|); the tensor core drops the low 13 bits of lo, i.e. at most 2^-20 |x| -- the order of the lo*lo term 3xTF32 omits.
__device__ __forceinline__ void tf32_split(float x, float& hi, float& lo) { hi = __uint_as_float(__float_as_uint(x) & 0xffffe000u); lo = x - hi; }
__device__ __forceinline__ void tf32_split_u(float x, uint32_t& hi, uint32_t& lo) { float h, l; tf32_split(x, h, l); hi = __float_as_uint(h); lo = __float_as_uint(l); }

// ---- weight image --------------------------------------------------------------------------------------------------
// The A operand of the forward and dH1 products comes from registers, in the wgmma accumulator layout of the previous layer: a thread holds
// features 2t and 2t + 1 of every group of 8 where the A fragment wants features t and t + 4.  The K order of every image is permuted to match:
// within each group of 8 features, the even ones first, then the odd ones.
__host__ __device__ __forceinline__ int kperm(int k) { return (k & ~7) | ((k & 1) << 2) | ((k & 7) >> 1); }
// element (row n, K position k) of a [rows][K] K-major SWIZZLE_128B operand -> byte offset inside its panel set (one panel per 32 K positions)
__device__ __forceinline__ int panel_offset(int n, int k, int panel_bytes) {
  const int p = k >> 5, c = (k >> 2) & 7, w = k & 3;
  return p * panel_bytes + n * 128 + ((c ^ (n & 7)) << 4) + (w << 2);
}
// One parameter (flat index j of a network, value x) -> its entries of the packed forward image `img` and, when present, of the
// backward image `bwd` (W2^T).  pack_weights_kernel writes whole images with it; adam_kernel keeps valid images current.
__device__ __forceinline__ void pack_param(const NetLayout& lay, int j, float x, uint8_t* img, uint8_t* bwd) {
  const float hi = tf32_rn(x), lo = tf32_rn(x - hi);
  if (j < lay.b1) {
    const int n = (j - lay.w1) / lay.in, k = (j - lay.w1) - n * lay.in, o = panel_offset(n, kperm(k), kPanelBytes);
    *reinterpret_cast<float*>(img + kOffW1Hi + o) = hi; *reinterpret_cast<float*>(img + kOffW1Lo + o) = lo;
  } else if (j < lay.w2) {
    reinterpret_cast<float*>(img + kOffB1)[j - lay.b1] = x;
  } else if (j < lay.b2) {
    const int n = (j - lay.w2) >> 7, k = (j - lay.w2) & 127, o = panel_offset(n, kperm(k), kPanelBytes);
    *reinterpret_cast<float*>(img + kOffW2Hi + o) = hi; *reinterpret_cast<float*>(img + kOffW2Lo + o) = lo;
    if (bwd != nullptr) {  // W2^T as a K-major operand: row = input feature, K = output feature
      const int ob = panel_offset(k, kperm(n), kPanelBytes);
      *reinterpret_cast<float*>(bwd + ob) = hi; *reinterpret_cast<float*>(bwd + 4 * kPanelBytes + ob) = lo;
    }
  } else if (j < lay.w3) {
    reinterpret_cast<float*>(img + kOffB2)[j - lay.b2] = x;
  } else if (j < lay.b3) {
    reinterpret_cast<float*>(img + kOffW3F)[j - lay.w3] = x;
  } else if (j < lay.P) {
    reinterpret_cast<float*>(img + kOffB3)[j - lay.b3] = x;
  }
}

// ---- optional phase timestamps (profiling builds: MARL_NVCC_DEFINES=-DMARL_TC_TIMESTAMPS) ------------------------------------------
// Thread 0 of every CTA stores %globaltimer (ns) and clock64() per probe slot into a per-kernel device buffer; tools/ts_timeline.py reads
// them back through marl_debug_timestamps (launch gaps, prologues, per-tile phases, tail skew).
#ifdef MARL_TC_TIMESTAMPS
constexpr int kTsgCtas = 160, kTsgSlots = 32;
#define TSG_DEFINE(name) static __device__ unsigned long long name[kTsgCtas][kTsgSlots][2];
#define TSG(name, slot) do { if (threadIdx.x == 0 && blockIdx.x < kTsgCtas && (slot) < kTsgSlots) { unsigned long long g_; \
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g_)); name[blockIdx.x][(slot)][0] = g_; name[blockIdx.x][(slot)][1] = (unsigned long long)clock64(); } } while (0)
#define TSG_GETTER(fn, name) int fn(unsigned long long* out) { return cudaMemcpyFromSymbol(out, name, sizeof(name)) == cudaSuccess ? 0 : -1; }
#else
#define TSG_DEFINE(name)
#define TSG(name, slot)
#define TSG_GETTER(fn, name) int fn(unsigned long long*) { return -1; }
#endif
int tsg_forward(unsigned long long* out); int tsg_fwd(unsigned long long* out); int tsg_dh1(unsigned long long* out); int tsg_dw(unsigned long long* out);
int tsg_adam(unsigned long long* out);

// dynamic shared memory rounded up to 1024 bytes (swizzle atoms), keeping the pointer in the shared address space so that the
// compiler emits LDS / STS rather than generic loads and stores
__device__ __forceinline__ uint8_t* align_smem_1024(uint8_t* raw) { return raw + ((1024u - ((uint32_t)__cvta_generic_to_shared(raw) & 1023u)) & 1023u); }

// ---- mbarrier + TMA bulk copy ----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// cp.async.bulk: one thread moves a contiguous, 16-byte aligned block global -> shared; completion is counted in bytes on an mbarrier
// (expect_tx by the issuing thread).  The packed weight images are byte-for-byte shared-memory images, so an image is a few instructions
// instead of a loop of per-thread copies, and the writes arrive through the async proxy, the one wgmma reads its operands through.
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// copy bytes [begin, end) of an image to the same offsets of its shared-memory copy, in pieces of at most 32 KB; the caller has armed `bar`
// with the total byte count of everything it sends to it (mbar_expect_tx, once)
__device__ __forceinline__ void tma_image_range(uint32_t smem_base, const uint8_t* src, int begin, int end, uint64_t* bar) {
  for (int o = begin; o < end; o += 32768) tma_bulk_g2s(smem_base + (uint32_t)o, src + o, (uint32_t)min(32768, end - o), bar);
}
// the forward image in the order the first tile needs it (one thread): bars[0] <- W1 + biases + FP32 W3, bars[1] <- W2
__device__ __forceinline__ void tma_forward_image(uint32_t smem_base, const uint8_t* src, uint64_t* bars) {
  mbar_expect_tx(bars + 0, (uint32_t)(kOffW2Hi + (kImageBytes - kOffB1)));
  tma_image_range(smem_base, src, kOffW1Hi, kOffW2Hi, bars + 0);
  tma_image_range(smem_base, src, kOffB1, kImageBytes, bars + 0);
  mbar_expect_tx(bars + 1, (uint32_t)(kOffB1 - kOffW2Hi));
  tma_image_range(smem_base, src, kOffW2Hi, kOffB1, bars + 1);
}

// ---- wgmma -----------------------------------------------------------------------------------------------------------
// K-major SWIZZLE_128B shared-memory matrix descriptor: start >> 4, LBO 16 B (unused by swizzled K-major operands), SBO 1024 B (one 8-row
// swizzle atom), layout type 1 (128-byte swizzle).  A k-step of 8 TF32 values inside an atom row is start + 32 bytes.
__device__ __forceinline__ uint64_t sw128_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// registers that an in-flight wgmma reads or writes: keep them where they are, and every use after this point, behind the wait that precedes it
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[N][4]) {
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) asm volatile("" : "+r"(r[i][j])::"memory");
}
// m64nNk8, D (F32) in registers; A from registers (RS, the tf32 fragment: rows lane/4 and +8 of the warp's 16, K t and t + 4) or from shared
// memory (SS); B from shared memory; both operands K-major.  scale_d == 0: D = A*B, else D += A*B.
__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss_n136(float (&d)[68], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %70, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n136k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67}, %68, %69, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss_n32(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ss_n8(float (&d)[4], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0, %1, %2, %3}, %4, %5, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

// 3xTF32 layer of a warpgroup, A in registers: D = A_lo*B_hi + A_hi*B_lo + A_hi*B_hi over `ksteps` (<= KSTEPS) steps of 8 K positions; B = hi / lo
// images of 32-position panels.  Waits for the MMAs before it returns.
template <int KSTEPS>
__device__ __forceinline__ void layer_rs(float (&d)[64], uint32_t (&ahi)[KSTEPS][4], uint32_t (&alo)[KSTEPS][4], uint32_t b_hi, uint32_t b_lo, int ksteps) {
  wg_fence();
#pragma unroll
  for (int term = 0; term < 3; ++term)
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks)
      if (ks < ksteps)
        wgmma_rs_n128(d, term == 0 ? alo[ks] : ahi[ks], sw128_desc((term == 1 ? b_lo : b_hi) + (uint32_t)((ks >> 2) * kPanelBytes + (ks & 3) * 32)),
                      (term | ks) ? 1u : 0u);
  wg_commit();
  wg_wait<0>();
  fence_regs(d); fence_regs(ahi); fence_regs(alo);
}

// ---- accumulator fragment of a warpgroup's 64 x 128 tile --------------------------------------------------------------
// Thread (warp w of the warpgroup, lane): rows 16 w + lane / 4 (element bit 1 clear) and + 8 (set); element i holds column 8 (i / 4) + 2 (lane % 4)
// + (i & 1).  Element pairs (4 ks, 4 ks + 2) / (4 ks + 1, 4 ks + 3) are exactly the A fragment of K step ks in the permuted K order (kperm).
__device__ __forceinline__ int frag_col(int i, int quad_lane) { return 8 * (i >> 2) + 2 * quad_lane + (i & 1); }
// values of a 64 x 128 fragment -> A operand registers (hi / lo) of the next product
__device__ __forceinline__ void frag_to_a(const float (&v)[64], uint32_t (&hi)[16][4], uint32_t (&lo)[16][4]) {
#pragma unroll
  for (int ks = 0; ks < 16; ++ks) {
    tf32_split_u(v[4 * ks + 0], hi[ks][0], lo[ks][0]); tf32_split_u(v[4 * ks + 2], hi[ks][1], lo[ks][1]);
    tf32_split_u(v[4 * ks + 1], hi[ks][2], lo[ks][2]); tf32_split_u(v[4 * ks + 3], hi[ks][3], lo[ks][3]);
  }
}
// head on the CUDA cores: q[row][a] = sum_j relu(D + b2)[row][j] W3[a][j] for the thread's two rows over its 32 columns, then over the four
// threads of the quad in a fixed order (xor 1, then xor 2); on return h holds relu(D + b2)
__device__ __forceinline__ void head_quad(float (&h)[64], const float* b2, const float* w3f, int out, int quad_lane, float (&q0)[kOutPad], float (&q1)[kOutPad]) {
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    const float2 bb = *reinterpret_cast<const float2*>(b2 + frag_col(i, quad_lane));
    h[i] = fmaxf(h[i] + bb.x, 0.f); h[i + 1] = fmaxf(h[i + 1] + bb.y, 0.f);
  }
#pragma unroll
  for (int a = 0; a < kOutPad; ++a) {
    float s0 = 0.f, s1 = 0.f;
    if (a < out) {
#pragma unroll
      for (int n = 0; n < 16; ++n) {
        const float2 w = *reinterpret_cast<const float2*>(w3f + a * kHidden + 8 * n + 2 * quad_lane);
        s0 = fmaf(h[4 * n + 1], w.y, fmaf(h[4 * n], w.x, s0));
        s1 = fmaf(h[4 * n + 3], w.y, fmaf(h[4 * n + 2], w.x, s1));
      }
      s0 += __shfl_xor_sync(0xFFFFFFFFu, s0, 1); s1 += __shfl_xor_sync(0xFFFFFFFFu, s1, 1);
      s0 += __shfl_xor_sync(0xFFFFFFFFu, s0, 2); s1 += __shfl_xor_sync(0xFFFFFFFFu, s1, 2);
    }
    q0[a] = s0; q1[a] = s1;
  }
}

// ---- the tensor-core training pass (tc_train.cu) ---------------------------------------------------------------------
// Row records [rows][kRowRec] floats: [0, 8) online outputs, [16, 20) / [20, 24) ReLU masks of H1 / H2 (training forward); [8] dLoss/dq[act],
// [9] act (int bits) (dH1 kernel).  Mask word q holds the columns of the fragment threads with lane % 4 == q: bit 2n + b = column 8n + 2q + b.
constexpr int kRowRec = 32;
constexpr int kRecG = 8, kRecAct = 9, kRecMask1 = 16, kRecMask2 = 20;
// a thread's ReLU mask words of its two fragment rows
__device__ __forceinline__ void frag_masks(const float (&h)[64], uint32_t& m0, uint32_t& m1) {
  m0 = 0; m1 = 0;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const uint32_t bit = (h[i] > 0.f ? 1u : 0u) << (((i >> 2) << 1) | (i & 1));
    if (i & 2) m1 |= bit; else m0 |= bit;
  }
}

struct TcTrainParams {
  RowPlan plan; RowSource src; NetLayout lay;
  const uint8_t* images;      // forward images [n_nets][kImageBytes]
  const uint8_t* bwd_images;  // backward images [n_nets][kBwdImageBytes]
  // H1, H2, dH1: feature-major [128][rows] (the weight-gradient kernel stages 32 consecutive rows of one feature per warp instruction)
  float* h1g; float* h2g; float* dh1g; size_t rows;
  float* rec;                 // [rows][kRowRec] row records
  float* xg;                  // [rows][kMaxObsDim] gathered observation rows: the weight-gradient kernel reads them without chasing the episode index again
  const float* tq; const float* td_ext; int td_agent_stride; float gamma; int double_q;
  float* scratch; int scratch_pitch; float* loss_part;
};

}  // namespace marl
