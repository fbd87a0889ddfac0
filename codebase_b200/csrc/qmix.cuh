// qmix.cuh -- the QMIX mixing network (marlbase/dqn/model.py:272-340) and its use in QMixNetwork._compute_loss (386-431).
//
//   Q_tot(q, s) = elu(q . |W1(s)| + b1(s)) . |w_final(s)| + V(s)      q: the agents' chosen (or target) Q-values, s: their observations concatenated
//   W1 = Linear(He -> N*E) o ReLU o Linear(S -> He), w_final likewise (-> E), b1 = Linear(S -> E), V = Linear(E -> 1) o ReLU o Linear(S -> E)
//
// The agents' networks stay on the tensor-core training pass: the mixer only replaces VDN's sum, i.e. it turns the agents' Q-values of every sampled
// (episode, step) into a TD error and hands dL/dq_a back through td_ext (per agent).  Work split:
//   qmix_pack_kernel   the online and the target mixer's weights, transposed per layer ([I][O]) -> two images (12 k floats each at N = 2, S = 30).
//   qmix_mix_kernel    a tile of 32 (episode b, step t) samples per CTA, lane = sample, the 8 warps share each layer's outputs; image and the tile's
//                      activations in shared memory (107 KB: two CTAs per SM).  Target: double-Q pick per agent at t + 1, target mixer on the state
//                      at t + 1.  Online: mixer on the state at t, delta = Q_tot - (r + gamma (1 - done) Q_tot_target), dL/dq_a -> td[a][b][t], and the
//                      back-propagated values at the OUTPUT of each of the mixer's seven linear layers next to those layers' inputs -> a per-sample
//                      record, stored field-major ([field][sample]: coalesced for this kernel's writes and the next kernel's reads).
//   qmix_wgrad2_kernel dW = sum over samples of (output gradient) x (input) for every layer's [O][I + 1 (bias)] matrix: one CTA per run of samples, the
//                      record read once, 4 x 8 register micro-tiles -> per-CTA partial sums (every parameter belongs to exactly one micro-tile).
//                      (qmix_wgrad_kernel: the first, tile-per-CTA form, kept behind MARL_QMIX_WGRAD_TILES=1 as a cross-check.)
//   qmix_reduce_kernel the chunks in fixed order -> gradient; the filled count next to it (Adam's 1 / filled.sum()).
// One-layer hypernetworks (hypernet_layers = 1): W1 = Linear(S -> N*E), w_final = Linear(S -> E), five linear layers (QmixLayout.hl, qmix_linears);
// W1 stays in global memory (read through L1 / L2), the rest of the image in shared memory.  standardise_returns splits qmix_mix_kernel into a
// target pass (returns) and an online pass around ret_ms_step (MODE 1 / 2); algorithm.td_lambda runs a target pass that writes the bootstrap values
// (MODE 3), the λ-return scan, then the online pass (MODE 2).
// The mixer's parameters take the shared Adam step WITHOUT gradient clipping: the reference clips self.critic.parameters() only (dqn/model.py:169-170).
#pragma once
#include "learner.cuh"
#include "dqn_heads.cuh"
#include "retms.cuh"

namespace marl {

constexpr int kQmixEmbedMax = 64, kQmixHypMax = 64, kQmixAgentsMax = 8, kQmixStateMax = 256, kQmixChunks = 32, kQmixMaxTiles = 512;

struct QmixLayout {   // offsets (floats) into the mixer's flat parameter vector (reference state_dict order) and into a sample's record
  int N, S, E, He, n, hl;   // hl: hypernetwork layers (1 or 2); He = 0 when hl == 1
  int w1a, b1a, w1b, b1b, wfa, bfa, wfb, bfb, wb, bb, wva, bva, wvb, bvb;
  int r_x, r_h1, r_h2, r_hv, r_dz1, r_draw1, r_dzf, r_drawf, r_dhb, r_dzv, r_dv, R;
  int res0;   // first parameter of the image that qmix_mix_kernel keeps in shared memory (hl == 1: W1 stays in global memory)
};

// hl == 2: hyper_w_1.{0,2}, hyper_w_final.{0,2}, hyper_b_1, V.{0,2}; record x | h1 | h2 | hv | dz1 | draw1 | dzf | drawf | dhb | dzv | dv.
// hl == 1: hyper_w_1 = Linear(S -> N*E) at w1b, hyper_w_final = Linear(S -> E) at wfb, then hyper_b_1, V.{0,2} (w1a / b1a / wfa / bfa and the
// record's h1, h2, dz1, dzf fields are unused, -1); record x | hv | draw1 | drawf | dhb | dzv | dv.
inline QmixLayout qmix_layout(int N, int S, int E, int He, int hl = 2) {
  QmixLayout L; L.N = N; L.S = S; L.E = E; L.He = hl == 2 ? He : 0; L.hl = hl;
  int o = 0;
  if (hl == 2) {
    L.w1a = o; o += He * S; L.b1a = o; o += He; L.w1b = o; o += N * E * He; L.b1b = o; o += N * E;
    L.wfa = o; o += He * S; L.bfa = o; o += He; L.wfb = o; o += E * He; L.bfb = o; o += E;
  } else {
    L.w1a = L.b1a = L.wfa = L.bfa = -1;
    L.w1b = o; o += N * E * S; L.b1b = o; o += N * E; L.wfb = o; o += E * S; L.bfb = o; o += E;
  }
  L.wb = o; o += E * S; L.bb = o; o += E; L.wva = o; o += E * S; L.bva = o; o += E; L.wvb = o; o += E; L.bvb = o; o += 1;
  L.n = o;
  L.res0 = hl == 2 ? 0 : N * E * S;
  int r = 0;
  if (hl == 2) {
    L.r_x = r; r += S; L.r_h1 = r; r += He; L.r_h2 = r; r += He; L.r_hv = r; r += E;
    L.r_dz1 = r; r += He; L.r_draw1 = r; r += N * E; L.r_dzf = r; r += He; L.r_drawf = r; r += E; L.r_dhb = r; r += E; L.r_dzv = r; r += E; L.r_dv = r; r += 1;
  } else {
    L.r_h1 = L.r_h2 = L.r_dz1 = L.r_dzf = -1;
    L.r_x = r; r += S; L.r_hv = r; r += E; L.r_draw1 = r; r += N * E; L.r_drawf = r; r += E; L.r_dhb = r; r += E; L.r_dzv = r; r += E; L.r_dv = r; r += 1;
  }
  L.R = r;
  return L;
}

// the mixer's linear layers (weight-gradient tables and the image pack): out / in width, record rows of the output gradient and of the input,
// weight and bias offsets.  Seven layers with two-layer hypernetworks, five with one.
struct QmixLin { int O, I, doff, ioff, woff, boff; };
__host__ __device__ inline int qmix_linears(const QmixLayout& L, QmixLin* out) {
  if (L.hl == 2) {
    out[0] = {L.He, L.S, L.r_dz1, L.r_x, L.w1a, L.b1a}; out[1] = {L.N * L.E, L.He, L.r_draw1, L.r_h1, L.w1b, L.b1b};
    out[2] = {L.He, L.S, L.r_dzf, L.r_x, L.wfa, L.bfa}; out[3] = {L.E, L.He, L.r_drawf, L.r_h2, L.wfb, L.bfb};
    out[4] = {L.E, L.S, L.r_dhb, L.r_x, L.wb, L.bb}; out[5] = {L.E, L.S, L.r_dzv, L.r_x, L.wva, L.bva}; out[6] = {1, L.E, L.r_dv, L.r_hv, L.wvb, L.bvb};
    return 7;
  }
  out[0] = {L.N * L.E, L.S, L.r_draw1, L.r_x, L.w1b, L.b1b}; out[1] = {L.E, L.S, L.r_drawf, L.r_x, L.wfb, L.bfb};
  out[2] = {L.E, L.S, L.r_dhb, L.r_x, L.wb, L.bb}; out[3] = {L.E, L.S, L.r_dzv, L.r_x, L.wva, L.bva}; out[4] = {1, L.E, L.r_dv, L.r_hv, L.wvb, L.bvb};
  return 5;
}

struct QmixTile { int o0, i0, O, I, doff, ioff, woff, boff; };   // a 32 x 32 tile of one linear layer's weight-gradient matrix ([O][I], bias = column I)

struct QmixParams {
  QmixLayout L;
  const float* q; const float* tq;   // [N][B][T+1][A] online / target Q-values of every gathered row
  TrajView traj; const int32_t* idx; int B, A, D; float gamma; int double_q;
  float huber;        // algorithm.huber_delta (> 0: the Huber TD loss of dqn_heads.cuh; <= 0: the squared error)
  const float* mix; const float* mix_tgt;
  float* rec;         // [R][B*T]
  float* td;          // [N][B][T] = dL/dq_a (un-normalised: x td_dloss(delta) filled)
  float* loss_part;   // [gridDim][4]
  // standardise_returns (two launches around ret_ms_step): the target pass writes ret[b][t], the online pass reads it back standardised
  const float* ret_ms; int n_stat;   // mean[n_stat] | var[n_stat], one column per batch entry (MODE 3: NULL without standardise_returns)
  float* ret;                        // [B][T]
  float* boot;                       // MODE 3 (algorithm.td_lambda): [B][T] the target mixer's Q_tot at t + 1
};

// ---- qmix_mix_kernel: 32 samples per CTA (lane = sample), 8 warps share each layer's outputs -----------------------------------------------------
// Shared memory: the mixer's image (weights TRANSPOSED, [I][O], so that a thread's four consecutive outputs are one 16-byte broadcast load and the
// transposed products of the backward read rows) + the tile's activations, field-major with a 33-float pitch (lane = sample: conflict-free).
constexpr int kQmTS = 32, kQmP = 33, kQmWarps = 8;

// image: same offsets as QmixLayout, every weight block transposed ([I][O]); built once per update by qmix_pack_kernel for the online and target mixer
__global__ void __launch_bounds__(256) qmix_pack_kernel(QmixLayout L, const float* __restrict__ mix, const float* __restrict__ mix_tgt, float* img, float* img_tgt) {
  const float* src = blockIdx.y ? mix_tgt : mix;
  float* dst = blockIdx.y ? img_tgt : img;
  QmixLin lin[7];
  const int nl = qmix_linears(L, lin);   // (in parameter order)
  for (int j = blockIdx.x * 256 + threadIdx.x; j < L.n; j += gridDim.x * 256) {
    int wo = lin[0].woff, O = lin[0].O, I = lin[0].I;   // the layer that holds j (constant indices: the table stays in registers)
#pragma unroll
    for (int k = 1; k < 7; ++k)
      if (k < nl && j >= lin[k].woff) { wo = lin[k].woff; O = lin[k].O; I = lin[k].I; }
    const int r = j - wo;
    if (r < O * I) { const int o = r / I, i = r - o * I; dst[wo + i * O + o] = src[j]; }
    else dst[j] = src[j];   // bias
  }
}

struct QmSmem { float *W, *X, *H1, *H2, *HV, *PRE, *RAWF, *RAW1, *QA, *RED, *RED2; };
__host__ __device__ inline int qm_act_rows(const QmixLayout& L) { return L.S + 2 * L.He + 3 * L.E + L.N * L.E + L.N + kQmWarps + L.N * kQmWarps; }
// the resident image (parameters res0 .. n) + the tile's activations (He = 0 with one-layer hypernetworks: no H1 / H2 rows)
__host__ __device__ inline size_t qm_smem_bytes(const QmixLayout& L) { return ((size_t)((L.n - L.res0 + 3) & ~3) + (size_t)qm_act_rows(L) * kQmP) * sizeof(float); }

// out[o][lane] = act(bias[o] + sum_i wT[i][o] in[i][lane]) for this warp's groups of 4 G consecutive outputs: one load of the input feeds 4 G FMAs,
// a weight load (16 bytes, the same address in every lane) four.  G = 2 whenever the layer is wide enough to keep all eight warps busy.
template <int G>
__device__ __forceinline__ void qm_layer_g(const float* __restrict__ wT, const float* __restrict__ bias, const float* in, float* out, int I, int O, bool relu, int warp, int lane) {
  for (int o0 = 4 * G * warp; o0 < O; o0 += 4 * G * kQmWarps) {
    float a[4 * G];
#pragma unroll
    for (int k = 0; k < 4 * G; ++k) a[k] = bias[o0 + k];
    const float* wp = wT + o0;
    const float* xp = in + lane;
#pragma unroll 4
    for (int i = 0; i < I; ++i, wp += O, xp += kQmP) {
      const float xv = *xp;
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float4 w = *reinterpret_cast<const float4*>(wp + 4 * g);
        a[4 * g] = fmaf(w.x, xv, a[4 * g]); a[4 * g + 1] = fmaf(w.y, xv, a[4 * g + 1]); a[4 * g + 2] = fmaf(w.z, xv, a[4 * g + 2]); a[4 * g + 3] = fmaf(w.w, xv, a[4 * g + 3]);
      }
    }
    float* op = out + o0 * kQmP + lane;
#pragma unroll
    for (int k = 0; k < 4 * G; ++k) op[k * kQmP] = relu ? fmaxf(a[k], 0.f) : a[k];
  }
}
__device__ __forceinline__ void qm_layer(const float* __restrict__ wT, const float* __restrict__ bias, const float* in, float* out, int I, int O, bool relu, int warp, int lane) {
  if ((O & 63) == 0) qm_layer_g<2>(wT, bias, in, out, I, O, relu, warp, lane);
  else qm_layer_g<1>(wT, bias, in, out, I, O, relu, warp, lane);
}
// rec[r_off + j][s] = (h[j][lane] > 0) sum_o d[o][lane] wT[j][o]: the gradient at a hypernetwork's hidden pre-activation (O a multiple of 4)
__device__ __forceinline__ void qm_layer_t(const float* __restrict__ wT, const float* d, const float* h, int I, int O, float* rec_col, int Sn, bool live, int warp, int lane) {
  for (int j0 = 4 * warp; j0 < I; j0 += 4 * kQmWarps) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    const float* w = wT + j0 * O;
#pragma unroll 2
    for (int o = 0; o < O; o += 4) {
      const float d0 = d[o * kQmP + lane], d1 = d[(o + 1) * kQmP + lane], d2 = d[(o + 2) * kQmP + lane], d3 = d[(o + 3) * kQmP + lane];
      const float4 u0 = *reinterpret_cast<const float4*>(w + o), u1 = *reinterpret_cast<const float4*>(w + O + o);
      const float4 u2 = *reinterpret_cast<const float4*>(w + 2 * O + o), u3 = *reinterpret_cast<const float4*>(w + 3 * O + o);
      a0 = fmaf(u0.x, d0, a0); a0 = fmaf(u0.y, d1, a0); a0 = fmaf(u0.z, d2, a0); a0 = fmaf(u0.w, d3, a0);
      a1 = fmaf(u1.x, d0, a1); a1 = fmaf(u1.y, d1, a1); a1 = fmaf(u1.z, d2, a1); a1 = fmaf(u1.w, d3, a1);
      a2 = fmaf(u2.x, d0, a2); a2 = fmaf(u2.y, d1, a2); a2 = fmaf(u2.z, d2, a2); a2 = fmaf(u2.w, d3, a2);
      a3 = fmaf(u3.x, d0, a3); a3 = fmaf(u3.y, d1, a3); a3 = fmaf(u3.z, d2, a3); a3 = fmaf(u3.w, d3, a3);
    }
    if (live) {
      rec_col[(size_t)j0 * Sn] = h[j0 * kQmP + lane] > 0.f ? a0 : 0.f; rec_col[(size_t)(j0 + 1) * Sn] = h[(j0 + 1) * kQmP + lane] > 0.f ? a1 : 0.f;
      rec_col[(size_t)(j0 + 2) * Sn] = h[(j0 + 2) * kQmP + lane] > 0.f ? a2 : 0.f; rec_col[(size_t)(j0 + 3) * Sn] = h[(j0 + 3) * kQmP + lane] > 0.f ? a3 : 0.f;
    }
  }
}

__device__ __forceinline__ float qmix_sgn(float x) { return (float)(x > 0.f) - (float)(x < 0.f); }   // torch.abs' gradient (0 at 0)

// Forward of the tile with the image in sm.W: the four state-fed layers, the hypernetworks' second layers, then Q_tot per sample.  On return
// PRE holds the ELU's argument and every thread of lane `lane` holds that sample's Q_tot.
__device__ __forceinline__ float qm_forward(const QmSmem& sm, const QmixLayout& L, int warp, int lane) {
  const float* W = sm.W;
  qm_layer(W + L.w1a, W + L.b1a, sm.X, sm.H1, L.S, L.He, true, warp, lane);
  qm_layer(W + L.wfa, W + L.bfa, sm.X, sm.H2, L.S, L.He, true, warp, lane);
  qm_layer(W + L.wva, W + L.bva, sm.X, sm.HV, L.S, L.E, true, warp, lane);
  qm_layer(W + L.wb, W + L.bb, sm.X, sm.PRE, L.S, L.E, false, warp, lane);
  __syncthreads();
  qm_layer(W + L.w1b, W + L.b1b, sm.H1, sm.RAW1, L.He, L.N * L.E, false, warp, lane);
  qm_layer(W + L.wfb, W + L.bfb, sm.H2, sm.RAWF, L.He, L.E, false, warp, lane);
  __syncthreads();
  float part = 0.f;
  for (int e = warp; e < L.E; e += kQmWarps) {
    float pe = sm.PRE[e * kQmP + lane];
    for (int a = 0; a < L.N; ++a) pe = fmaf(sm.QA[a * kQmP + lane], fabsf(sm.RAW1[(a * L.E + e) * kQmP + lane]), pe);
    sm.PRE[e * kQmP + lane] = pe;
    const float hid = pe > 0.f ? pe : expm1f(pe);
    part = fmaf(hid, fabsf(sm.RAWF[e * kQmP + lane]), part);
    part = fmaf(W[L.wvb + e], sm.HV[e * kQmP + lane], part);
  }
  sm.RED[warp * kQmP + lane] = part;
  __syncthreads();
  float y = W[L.bvb];
#pragma unroll
  for (int k = 0; k < kQmWarps; ++k) y += sm.RED[k * kQmP + lane];
  return y;
}

// One-layer hypernetworks: sm.W holds parameters res0 .. n (everything but W1's weights); W1 (transposed, [S][N*E]) is read from the global image
// w1g through L1 / L2 -- the same warp-uniform 16-byte loads as from shared memory.  The four layers all read the state only: one barrier.
__device__ __forceinline__ float qm_forward1(const QmSmem& sm, const QmixLayout& L, const float* __restrict__ w1g, int warp, int lane) {
  const float* W = sm.W;
  const int r0 = L.res0;
  qm_layer(W + (L.wva - r0), W + (L.bva - r0), sm.X, sm.HV, L.S, L.E, true, warp, lane);
  qm_layer(W + (L.wb - r0), W + (L.bb - r0), sm.X, sm.PRE, L.S, L.E, false, warp, lane);
  qm_layer(W + (L.wfb - r0), W + (L.bfb - r0), sm.X, sm.RAWF, L.S, L.E, false, warp, lane);
  qm_layer(w1g, W + (L.b1b - r0), sm.X, sm.RAW1, L.S, L.N * L.E, false, warp, lane);
  __syncthreads();
  float part = 0.f;
  for (int e = warp; e < L.E; e += kQmWarps) {
    float pe = sm.PRE[e * kQmP + lane];
    for (int a = 0; a < L.N; ++a) pe = fmaf(sm.QA[a * kQmP + lane], fabsf(sm.RAW1[(a * L.E + e) * kQmP + lane]), pe);
    sm.PRE[e * kQmP + lane] = pe;
    const float hid = pe > 0.f ? pe : expm1f(pe);
    part = fmaf(hid, fabsf(sm.RAWF[e * kQmP + lane]), part);
    part = fmaf(W[L.wvb - r0 + e], sm.HV[e * kQmP + lane], part);
  }
  sm.RED[warp * kQmP + lane] = part;
  __syncthreads();
  float y = W[L.bvb - r0];
#pragma unroll
  for (int k = 0; k < kQmWarps; ++k) y += sm.RED[k * kQmP + lane];
  return y;
}

// the tile's inputs: state = the agents' observations at step t + dt side by side; q_a = chosen Q (dt = 0) or the double-Q / max target pick (dt = 1).
// lane = sample (b, t, episode slot `ep` of this thread's sample); the rows are shared out over the warps
__device__ __forceinline__ void qm_load_inputs(const QmSmem& sm, const QmixParams& p, bool live, int b, int t, size_t ep, int dt, int warp, int lane) {
  const QmixLayout& L = p.L;
  const int T = p.traj.T;
  for (int a = 0; a < L.N; ++a) {
    const float* ob = p.traj.obs_row(ep, a, t + dt);
    for (int d = warp; d < p.D; d += kQmWarps) sm.X[(a * p.D + d) * kQmP + lane] = live ? ob[d] : 0.f;
  }
  for (int a = warp; a < L.N; a += kQmWarps) {
    float v = 0.f;
    if (live) {
      const size_t row = row_index(a, b, t + dt, p.B, T + 1);
      const float* q1 = p.q + row * p.A;
      if (dt == 0) v = q1[p.traj.act[p.traj.step_at(ep, a, t)]];
      else v = next_value(q1, p.tq + row * p.A, p.A, p.double_q);
    }
    sm.QA[a * kQmP + lane] = v;
  }
}

// HL: hypernetwork layers (the image's shared-memory part and the forward / backward follow the layout's table).  MODE 0: target and online pass
// in one launch.  standardise_returns needs the whole batch's returns before any TD error: MODE 1 runs the target pass only and writes
// ret[b][t] = r + gamma (Q_tot' sqrt(var[b]) + mean[b]) (1 - done) for every sample; ret_ms_step standardises them; MODE 2 runs the online
// pass against the standardised ret.  algorithm.td_lambda: MODE 3 runs the target pass only and writes boot[b][t] = Q_tot' (de-standardised as in
// MODE 1 when ret_ms is set); td_lambda_kernel (dqn.cu) turns it into the λ-returns in ret, and MODE 2 runs the online pass against them.
template <int HL, int MODE>
__global__ void __launch_bounds__(kQmWarps * 32, 2) qmix_mix_kernel(QmixParams p, const float* __restrict__ img, const float* __restrict__ img_tgt) {
  extern __shared__ __align__(16) float qsm[];
  const QmixLayout& L = p.L;
  QmSmem sm;
  sm.W = qsm;
  const int n_res = HL == 2 ? L.n : L.n - L.res0;   // image floats resident in shared memory
  float* o = qsm + ((n_res + 3) & ~3);
  sm.X = o; o += L.S * kQmP; sm.H1 = o; o += L.He * kQmP; sm.H2 = o; o += L.He * kQmP; sm.HV = o; o += L.E * kQmP; sm.PRE = o; o += L.E * kQmP;
  sm.RAWF = o; o += L.E * kQmP; sm.RAW1 = o; o += L.N * L.E * kQmP; sm.QA = o; o += L.N * kQmP; sm.RED = o; o += kQmWarps * kQmP; sm.RED2 = o;
  const int T = p.traj.T, Sn = p.B * T, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s0 = blockIdx.x * kQmTS, s = s0 + lane;
  const bool live = s < Sn;
  const int b = live ? s / T : 0, t = live ? s - b * T : 0;
  const size_t ep = (size_t)p.idx[b];
  const int n4 = (n_res + 3) >> 2, r4 = HL == 2 ? 0 : L.res0 >> 2;
  // ---- target: Q_tot' of the picks at t + 1 on the state at t + 1 ----
  float ytgt = 0.f;
  if constexpr (MODE != 2) {
    for (int i = threadIdx.x; i < n4; i += kQmWarps * 32) reinterpret_cast<float4*>(sm.W)[i] = reinterpret_cast<const float4*>(img_tgt)[r4 + i];
    qm_load_inputs(sm, p, live, b, t, ep, 1, warp, lane);
    __syncthreads();
    if constexpr (HL == 2) ytgt = qm_forward(sm, L, warp, lane);
    else ytgt = qm_forward1(sm, L, img_tgt + L.w1b, warp, lane);
    __syncthreads();
  }
  if constexpr (MODE == 1) {   // the target mixer's output de-standardised with the statistics so far (dqn/model.py:415-418), no FMA contraction
    if (live && warp == 0) {
      const float tq = unstandardise(ytgt, p.ret_ms[b], p.ret_ms[p.n_stat + b]);
      p.ret[s] = td_target_rn(p.traj.rew[p.traj.step_at(ep, 0, t)], p.gamma, tq, (float)p.traj.done[p.traj.done_at(ep, t + 1)]);
    }
  } else if constexpr (MODE == 3) {
    if (live && warp == 0) p.boot[s] = p.ret_ms ? unstandardise(ytgt, p.ret_ms[b], p.ret_ms[p.n_stat + b]) : ytgt;
  } else {
    // ---- online ----
    for (int i = threadIdx.x; i < n4; i += kQmWarps * 32) reinterpret_cast<float4*>(sm.W)[i] = reinterpret_cast<const float4*>(img)[r4 + i];
    qm_load_inputs(sm, p, live, b, t, ep, 0, warp, lane);
    __syncthreads();
    float y;
    if constexpr (HL == 2) y = qm_forward(sm, L, warp, lane);
    else y = qm_forward1(sm, L, img + L.w1b, warp, lane);
    const float filled = live ? (float)p.traj.filled[p.traj.filled_at(ep, t)] : 0.f;
    float ret;
    if constexpr (MODE == 2) ret = live ? p.ret[s] : 0.f;
    else ret = live ? td_target(p.traj.rew[p.traj.step_at(ep, 0, t)], p.gamma, ytgt, (float)p.traj.done[p.traj.done_at(ep, t + 1)]) : 0.f;
    const float delta = live ? y - ret : 0.f, dy = td_dloss(delta, p.huber) * filled;
    float* rc = p.rec + s;   // this sample's column of the field-major record
    if (live) {
      // the layers' inputs (x, h1, h2) -> record; rows are shared out over the warps
      for (int i = warp; i < L.S; i += kQmWarps) rc[(size_t)(L.r_x + i) * Sn] = sm.X[i * kQmP + lane];
      if constexpr (HL == 2)
        for (int j = warp; j < L.He; j += kQmWarps) { rc[(size_t)(L.r_h1 + j) * Sn] = sm.H1[j * kQmP + lane]; rc[(size_t)(L.r_h2 + j) * Sn] = sm.H2[j * kQmP + lane]; }
      if (warp == 0) rc[(size_t)L.r_dv * Sn] = dy;
    }
    const float* wvb = HL == 2 ? sm.W + L.wvb : sm.W + (L.wvb - L.res0);
    // per embedding unit: V's hidden layer, w_final, the ELU; PRE <- dL/d(ELU argument), RAWF <- dL/d(w_final before abs), RAW1 <- dL/d(W1 before abs)
    for (int e = warp; e < L.E; e += kQmWarps) {
      const float pe = sm.PRE[e * kQmP + lane], hid = pe > 0.f ? pe : expm1f(pe), rf = sm.RAWF[e * kQmP + lane], hv = sm.HV[e * kQmP + lane];
      const float dp = dy * fabsf(rf) * (pe > 0.f ? 1.f : hid + 1.f);
      const float drf = dy * hid * qmix_sgn(rf);
      if (live) {
        rc[(size_t)(L.r_hv + e) * Sn] = hv;
        rc[(size_t)(L.r_dzv + e) * Sn] = hv > 0.f ? dy * wvb[e] : 0.f;
        rc[(size_t)(L.r_drawf + e) * Sn] = drf;
        rc[(size_t)(L.r_dhb + e) * Sn] = dp;
      }
      if constexpr (HL == 2) sm.RAWF[e * kQmP + lane] = drf;
      sm.PRE[e * kQmP + lane] = dp;     // (this thread's own entries: the next loop reads them back without a barrier)
    }
    for (int a = 0; a < L.N; ++a) {
      const float qa = sm.QA[a * kQmP + lane];
      float dq = 0.f;
      for (int e = warp; e < L.E; e += kQmWarps) {
        const float dp = sm.PRE[e * kQmP + lane], r1 = sm.RAW1[(a * L.E + e) * kQmP + lane];
        dq = fmaf(dp, fabsf(r1), dq);
        const float d1 = dp * qa * qmix_sgn(r1);
        if constexpr (HL == 2) sm.RAW1[(a * L.E + e) * kQmP + lane] = d1;
        if (live) rc[(size_t)(L.r_draw1 + a * L.E + e) * Sn] = d1;
      }
      sm.RED2[(a * kQmWarps + warp) * kQmP + lane] = dq;
    }
    __syncthreads();
    for (int a = warp; a < L.N; a += kQmWarps) {   // dL/dq_a -> the agents' training pass
      float v = 0.f;
#pragma unroll
      for (int k = 0; k < kQmWarps; ++k) v += sm.RED2[(a * kQmWarps + k) * kQmP + lane];
      if (live) p.td[((size_t)a * p.B + b) * T + t] = v;
    }
    if constexpr (HL == 2) {   // the hypernetworks' hidden layers (one-layer hypernetworks stop at dRAW1 / dRAWF)
      qm_layer_t(sm.W + L.wfb, sm.RAWF, sm.H2, L.He, L.E, rc + (size_t)L.r_dzf * Sn, Sn, live, warp, lane);
      qm_layer_t(sm.W + L.w1b, sm.RAW1, sm.H1, L.He, L.N * L.E, rc + (size_t)L.r_dz1 * Sn, Sn, live, warp, lane);
    }
    // loss statistics of the tile (warp 0 holds every sample once)
    if (warp == 0) {
      float loss = td_loss(delta, p.huber) * filled, fill = filled;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) { loss += __shfl_xor_sync(0xFFFFFFFFu, loss, off); fill += __shfl_xor_sync(0xFFFFFFFFu, fill, off); }
      if (lane == 0) { p.loss_part[4 * blockIdx.x] = loss; p.loss_part[4 * blockIdx.x + 1] = fill; p.loss_part[4 * blockIdx.x + 2] = 0.f; p.loss_part[4 * blockIdx.x + 3] = 0.f; }
    }
  }
}

__global__ void __launch_bounds__(256) qmix_wgrad_kernel(const float* __restrict__ rec, int Sn, const QmixTile* __restrict__ tiles, int chunk_len, float* part, int n) {
  __shared__ float As[32][33], Bs[32][33];
  const QmixTile tl = tiles[blockIdx.x];
  const int chunk = blockIdx.y, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int s_begin = chunk * chunk_len, s_end = min(Sn, s_begin + chunk_len);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int s0 = s_begin; s0 < s_end; s0 += 32) {
    const int s = s0 + tx;
    const bool valid = s < s_end;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int o = tl.o0 + ty + 8 * k, i = tl.i0 + ty + 8 * k;
      As[tx][ty + 8 * k] = (valid && o < tl.O) ? rec[(size_t)(tl.doff + o) * Sn + s] : 0.f;
      Bs[tx][ty + 8 * k] = !valid ? 0.f : i < tl.I ? rec[(size_t)(tl.ioff + i) * Sn + s] : i == tl.I ? 1.f : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int ss = 0; ss < 32; ++ss) {
      const float bv = Bs[ss][tx];
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[k] = fmaf(As[ss][ty + 8 * k], bv, acc[k]);
    }
    __syncthreads();
  }
  float* dst = part + (size_t)chunk * n;
  const int i = tl.i0 + tx;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int o = tl.o0 + ty + 8 * k;
    if (o < tl.O) {
      if (i < tl.I) dst[tl.woff + o * tl.I + i] = acc[k];
      else if (i == tl.I) dst[tl.boff + o] = acc[k];
    }
  }
}

// ---- qmix_wgrad_kernel, second form: the record is read ONCE -----------------------------------------------------------------------------------
// A CTA owns a run of samples and every (o, i) of every layer: 32 samples of all R record fields at a time in shared memory ([field][33]), each thread
// accumulates two 4 (outputs) x 8 (inputs) micro-tiles in registers -- 12 shared loads per 32 FMAs, no re-reads of the record from L2 / DRAM (the
// tile form above reads every field once per tile that needs it: 137 MB instead of 55 MB, and is bound by its 5 shared loads per 4 FMAs).
// Column I of a layer is its bias: a constant-one field; out-of-range rows / columns read a constant-zero field (no branches in the inner loop).
struct QmixMicro { int d_row, n_o, x_row, i0, I, woff, boff, o0; };
constexpr int kQmMicroPerRound = 512;   // 2 per thread

inline int qmix_micro_tiles(const QmixLayout& L, QmixMicro* out, int cap) {
  QmixLin lays[7];
  const int nl = qmix_linears(L, lays);
  int n = 0;
  for (int k = 0; k < nl; ++k) {
    const QmixLin& l = lays[k];
    for (int o0 = 0; o0 < l.O; o0 += 4)
      for (int i0 = 0; i0 <= l.I; i0 += 8) {
        if (n == cap) return -1;
        out[n++] = QmixMicro{l.doff + o0, l.O - o0 < 4 ? l.O - o0 : 4, l.ioff + i0, i0, l.I, l.woff, l.boff, o0};
      }
  }
  return n;
}

__global__ void __launch_bounds__(256, 2) qmix_wgrad2_kernel(const float* __restrict__ rec, int Sn, int R, const QmixMicro* __restrict__ micro, int n_micro, int round, int per_cta,
                                                             float* part, int n) {
  extern __shared__ __align__(16) float fs[];   // [R + 2][33]: the record fields of 32 samples, then the zero and the one field
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, ZERO = R * kQmP, ONE = (R + 1) * kQmP;
  bool on[2]; int dr[2][4], xr[2][8];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int m = round * kQmMicroPerRound + q * 256 + (int)threadIdx.x;
    on[q] = m < n_micro;
    QmixMicro mt; mt.d_row = 0; mt.n_o = 0; mt.x_row = 0; mt.i0 = 0; mt.I = -1;
    if (on[q]) mt = micro[m];
#pragma unroll
    for (int k = 0; k < 4; ++k) dr[q][k] = k < mt.n_o ? (mt.d_row + k) * kQmP : ZERO;
#pragma unroll
    for (int k = 0; k < 8; ++k) { const int i = mt.i0 + k; xr[q][k] = i < mt.I ? (mt.x_row + k) * kQmP : i == mt.I ? ONE : ZERO; }
  }
  float acc[2][32];
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int k = 0; k < 32; ++k) acc[q][k] = 0.f;
  if (threadIdx.x < kQmP) { fs[ZERO + threadIdx.x] = 0.f; fs[ONE + threadIdx.x] = 1.f; }
  const int s_begin = blockIdx.x * per_cta, s_end = min(Sn, s_begin + per_cta);
  for (int s0 = s_begin; s0 < s_end; s0 += 32) {
    __syncthreads();
    const bool valid = s0 + lane < s_end;
    for (int f = warp; f < R; f += 8) fs[f * kQmP + lane] = valid ? rec[(size_t)f * Sn + s0 + lane] : 0.f;
    __syncthreads();
#pragma unroll 2
    for (int ss = 0; ss < 32; ++ss) {
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        float d[4], x[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) d[k] = fs[dr[q][k] + ss];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = fs[xr[q][k] + ss];
#pragma unroll
        for (int oo = 0; oo < 4; ++oo)
#pragma unroll
          for (int ii = 0; ii < 8; ++ii) acc[q][oo * 8 + ii] = fmaf(d[oo], x[ii], acc[q][oo * 8 + ii]);
      }
    }
  }
  float* dst = part + (size_t)blockIdx.x * n;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    if (!on[q]) continue;
    const QmixMicro mt = micro[round * kQmMicroPerRound + q * 256 + (int)threadIdx.x];
#pragma unroll
    for (int oo = 0; oo < 4; ++oo)
#pragma unroll
      for (int ii = 0; ii < 8; ++ii) {
        const int o = mt.o0 + oo, i = mt.i0 + ii;
        if (oo < mt.n_o) {
          if (i < mt.I) dst[mt.woff + o * mt.I + i] = acc[q][oo * 8 + ii];
          else if (i == mt.I) dst[mt.boff + o] = acc[q][oo * 8 + ii];
        }
      }
  }
}

// grad[0..n) = the chunks' partial sums in fixed order; grad[n..n+4) = (loss numerator, filled count, 0, 0) of this update
__global__ void __launch_bounds__(256) qmix_reduce_kernel(const float* __restrict__ part, int chunks, int n, float* grad, const float* __restrict__ loss_part, int n_loss_parts) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j < n) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;   // four independent chains (the loads of a chain are dependent on nothing but the index): fixed order
    int c = 0;
    for (; c + 3 < chunks; c += 4) {
      s0 += part[(size_t)c * n + j]; s1 += part[(size_t)(c + 1) * n + j]; s2 += part[(size_t)(c + 2) * n + j]; s3 += part[(size_t)(c + 3) * n + j];
    }
    for (; c < chunks; ++c) s0 += part[(size_t)c * n + j];
    grad[j] = (s0 + s1) + (s2 + s3);
  }
  if (blockIdx.x == 0 && threadIdx.x < 64) {
    const int which = threadIdx.x >> 5, l = threadIdx.x & 31;
    float x = 0.f;
    for (int c = l; c < n_loss_parts; c += 32) x += loss_part[4 * c + which];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, off);
    if (l == 0) { grad[n + which] = x; grad[n + 2 + which] = 0.f; }
  }
}

// tiles of the mixer's linear layers (host side)
inline int qmix_tiles(const QmixLayout& L, QmixTile* out) {
  QmixLin lays[7];
  const int nl = qmix_linears(L, lays);
  int n = 0;
  for (int k = 0; k < nl; ++k) {
    const QmixLin& l = lays[k];
    for (int o0 = 0; o0 < l.O; o0 += 32)
      for (int i0 = 0; i0 <= l.I; i0 += 32) {   // column I is the bias
        if (n == kQmixMaxTiles) return -1;
        out[n++] = QmixTile{o0, i0, l.O, l.I, l.doff, l.ioff, l.woff, l.boff};
      }
  }
  return n;
}

}  // namespace marl
