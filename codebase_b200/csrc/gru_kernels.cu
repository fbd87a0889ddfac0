// gru_kernels.cu -- sequence forward and BPTT backward of the recurrent agent networks (gru.cuh), FP32 FFMA.
//
// A CTA owns kGruSeqs = 16 sequences of one network for all of their steps; sequences are independent, so no grid-wide synchronisation
// is needed and each pass is one launch.  Thread j of each 128-thread half owns hidden unit j of 8 sequences: its three gate rows of
// W_ih / W_hh give r, z, n and h' of that unit without a cross-thread reduction.  The weights are read through L1 / L2 (W_ih + W_hh are
// 384 KB per network, more than shared memory holds); every weight a thread loads is used for 8 sequences.  A network of hidden width H < 128
// keeps the 128 threads per half: threads j >= H read a valid row (H - 1) and write zeros, weights are read with row stride H, and the weight
// gradients are written for units < H only, at their compact offsets (gru.cuh).
//
// The actor-critic learners add a loss-head kernel between the two: it reads the outputs the forward stored and hands the backward a dense dL/dout.
#include "gru.cuh"
#include "ac_heads.cuh"

namespace marl {

__device__ __forceinline__ float gru_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// sequence v of net -> (agent, unit)
__device__ __forceinline__ void gru_seq(const RowPlan& p, int net, int v, int& agent, int& unit) {
  const int slot = v / p.units_per_agent;
  agent = p.slot_agent[p.slot_begin[net] + slot];
  unit = v - slot * p.units_per_agent;
}

// KX: staged input columns per sequence (kMaxObsDim, or kMaxInDim for the wider inputs of the actor-critic learners)
template <int KX>
__global__ void __launch_bounds__(kGruThreads) gru_forward_kernel(GruFwdParams p) {
  __shared__ float xs[kGruSeqs][KX];
  __shared__ float x1[kGruSeqs][kHidden];
  __shared__ float hs[kGruSeqs][kHidden];
  const int net = blockIdx.y, j = threadIdx.x & (kHidden - 1), s0 = (threadIdx.x >> 7) * 8;
  const int nseq = (p.plan.slot_begin[net + 1] - p.plan.slot_begin[net]) * p.plan.units_per_agent;
  const int v0 = blockIdx.x * kGruSeqs;
  if (v0 >= nseq) return;   // uniform over the CTA
  const float* th = p.theta + (size_t)net * p.lay.P;
  const int D = p.lay.in, A = p.lay.out, steps = p.plan.unit_rows, B = p.plan.units_per_agent, H = p.lay.H;
  const bool live = j < H;               // unit j exists (else padding: it stays 0)
  const int jr = live ? j : H - 1;       // the weight row it reads
  for (int i = threadIdx.x; i < kGruSeqs * kHidden; i += kGruThreads) {
    const int s = i / kHidden, k = i - s * kHidden;
    float v = 0.f;
    if (p.h_in != nullptr && v0 + s < nseq && k < H) {
      int agent, unit; gru_seq(p.plan, net, v0 + s, agent, unit);
      v = p.h_in[((size_t)unit * p.src.N + agent) * H + k];
    }
    hs[s][k] = v;
  }
  const float* w1 = th + p.lay.w1 + jr * D;
  const float* wi = th + p.lay.wih + jr * H;
  const float* wh = th + p.lay.whh + jr * H;
  const float b1 = th[p.lay.b1 + jr];
  const float bir = th[p.lay.bih + jr], biz = th[p.lay.bih + H + jr], bin = th[p.lay.bih + 2 * H + jr];
  const float bhr = th[p.lay.bhh + jr], bhz = th[p.lay.bhh + H + jr], bhn = th[p.lay.bhh + 2 * H + jr];
  for (int t = 0; t < steps; ++t) {
    for (int i = threadIdx.x; i < kGruSeqs * KX; i += kGruThreads) {
      const int s = i / KX, k = i - s * KX;
      float v = 0.f;
      if (k < D && v0 + s < nseq) {
        int agent, unit; gru_seq(p.plan, net, v0 + s, agent, unit);
        v = src_row(p.src, agent, unit, t)[k];
      }
      xs[s][k] = v;
    }
    __syncthreads();
    {  // first_layer + ReLU
      float acc[8];
#pragma unroll
      for (int s = 0; s < 8; ++s) acc[s] = b1;
      for (int k = 0; k < D; ++k) {
        const float w = w1[k];
#pragma unroll
        for (int s = 0; s < 8; ++s) acc[s] = fmaf(w, xs[s0 + s][k], acc[s]);
      }
#pragma unroll
      for (int s = 0; s < 8; ++s) x1[s0 + s][j] = live ? fmaxf(acc[s], 0.f) : 0.f;
    }
    __syncthreads();
    float ar[8], az[8], ain[8], ahn[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) { ar[s] = 0.f; az[s] = 0.f; ain[s] = 0.f; ahn[s] = 0.f; }
#pragma unroll 2
    for (int k = 0; k < H; ++k) {
      const float wir = wi[k], wiz = wi[H * H + k], win = wi[2 * H * H + k];
      const float whr = wh[k], whz = wh[H * H + k], whn = wh[2 * H * H + k];
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        const float xv = x1[s0 + s][k], hv = hs[s0 + s][k];
        ar[s] = fmaf(whr, hv, fmaf(wir, xv, ar[s]));
        az[s] = fmaf(whz, hv, fmaf(wiz, xv, az[s]));
        ain[s] = fmaf(win, xv, ain[s]);
        ahn[s] = fmaf(whn, hv, ahn[s]);
      }
    }
    float hnew[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      float r = gru_sigmoid(ar[s] + bir + bhr), z = gru_sigmoid(az[s] + biz + bhz);
      float ghn = ahn[s] + bhn, n = tanhf(ain[s] + bin + r * ghn);
      hnew[s] = (1.f - z) * n + z * hs[s0 + s][j];
      if (!live) { r = 0.f; z = 0.f; ghn = 0.f; n = 0.f; hnew[s] = 0.f; }
      if (p.save != nullptr && v0 + s0 + s < nseq) {
        int agent, unit; gru_seq(p.plan, net, v0 + s0 + s, agent, unit);
        float* row = p.save + row_index(agent, unit, t, B, steps) * kGruSaveRow;
        row[j] = x1[s0 + s][j]; row[kHidden + j] = r; row[2 * kHidden + j] = z; row[3 * kHidden + j] = n; row[4 * kHidden + j] = ghn; row[5 * kHidden + j] = hnew[s];
      }
    }
    __syncthreads();   // every read of h is done
#pragma unroll
    for (int s = 0; s < 8; ++s) hs[s0 + s][j] = hnew[s];
    __syncthreads();
    if (threadIdx.x < kGruSeqs * kOutPad) {   // final_layer
      const int s = threadIdx.x / kOutPad, a = threadIdx.x - s * kOutPad;
      if (a < A && v0 + s < nseq) {
        const float* w3 = th + p.lay.w3 + a * H;
        float q = th[p.lay.b3 + a];
        for (int k = 0; k < H; ++k) q = fmaf(w3[k], hs[s][k], q);
        int agent, unit; gru_seq(p.plan, net, v0 + s, agent, unit);
        const size_t o = out_row(p.src, agent, unit, t, B, steps);
        p.q_out[o * A + a] = q;
      }
    }
  }
  if (p.h_out != nullptr) {
    for (int i = threadIdx.x; i < kGruSeqs * kHidden; i += kGruThreads) {
      const int s = i / kHidden, k = i - s * kHidden;
      if (v0 + s < nseq && k < H) {
        int agent, unit; gru_seq(p.plan, net, v0 + s, agent, unit);
        p.h_out[((size_t)unit * p.src.N + agent) * H + k] = hs[s][k];
      }
    }
  }
}

template <int KX>
struct GruBwdSmem {
  float dq[kGruSeqs][kOutPad];
  float x[kGruSeqs][KX];
  float x1[kGruSeqs][kHidden];        // first-layer output of step t
  float hp[kGruSeqs][kHidden];        // h_{t-1}
  float hc[kGruSeqs][kHidden];        // h_t
  float dx1[kGruSeqs][kHidden];
  float dgi[kGruSeqs][3 * kHidden];   // dL / d(W_ih x1 + b_ih), gate order r, z, n
  float dgh[kGruSeqs][3 * kHidden];   // dL / d(W_hh h + b_hh)
};

template <int KX>
__global__ void __launch_bounds__(kGruThreads) gru_backward_kernel(GruBwdParams p) {
  extern __shared__ float4 smem_raw[];
  GruBwdSmem<KX>& S = *reinterpret_cast<GruBwdSmem<KX>*>(smem_raw);
  const int j = threadIdx.x & (kHidden - 1), s0 = (threadIdx.x >> 7) * 8;
  int net, v_begin, v_end;
  cta_rows(p.plan, net, v_begin, v_end);   // unit_rows = 1: rows are sequences
  const float* th = p.theta + (size_t)net * p.lay.P;
  const int D = p.lay.in, A = p.lay.out, T = p.traj.T, B = p.B, H = p.lay.H;
  const bool live = j < H;               // unit j exists (else padding: every gradient through it is 0)
  const int jr = live ? j : H - 1;       // the weight column it reads
  float* out = p.scratch + (size_t)blockIdx.x * p.scratch_pitch;
  for (int e = threadIdx.x; e < p.lay.P; e += kGruThreads) out[e] = 0.f;
  __syncthreads();
  const float* w3 = th + p.lay.w3;
  const float* wi = th + p.lay.wih + jr;
  const float* wh = th + p.lay.whh + jr;
  for (int vt = v_begin; vt < v_end; vt += kGruSeqs) {
    float dhc[8];   // dL/dh_t carried from step t + 1
#pragma unroll
    for (int s = 0; s < 8; ++s) dhc[s] = 0.f;
    for (int t = T - 1; t >= 0; --t) {
      // (a) the step's saved state, observations and dL/dq
      for (int i = threadIdx.x; i < kGruSeqs * kHidden; i += kGruThreads) {
        const int s = i / kHidden, k = i - s * kHidden;
        float a = 0.f, b = 0.f, c = 0.f;
        if (vt + s < v_end) {
          int agent, unit; gru_seq(p.plan, net, vt + s, agent, unit);
          const float* row = p.save + row_index(agent, unit, t, B, T + 1) * kGruSaveRow;
          a = row[k]; b = row[5 * kHidden + k];
          if (t > 0) c = row[5 * kHidden + k - kGruSaveRow];
        }
        S.x1[s][k] = a; S.hc[s][k] = b; S.hp[s][k] = c;
      }
      for (int i = threadIdx.x; i < kGruSeqs * KX; i += kGruThreads) {
        const int s = i / KX, k = i - s * KX;
        float v = 0.f;
        if (k < D && vt + s < v_end) {
          int agent, unit; gru_seq(p.plan, net, vt + s, agent, unit);
          v = src_row(p.src, agent, unit, t)[k];
        }
        S.x[s][k] = v;
      }
      if (threadIdx.x < kGruSeqs * kOutPad) {
        const int s = threadIdx.x / kOutPad, a = threadIdx.x - s * kOutPad;
        float v = 0.f;
        if (a < A && vt + s < v_end) {
          int agent, unit; gru_seq(p.plan, net, vt + s, agent, unit);
          if (p.dout != nullptr) {
            v = p.dout[row_index(agent, unit, t, B, T + 1) * A + a];
          } else {
            if (p.traj.act[p.traj.step_at(p.idx[unit], agent, t)] == a) v = p.td[(size_t)agent * p.td_agent_stride + (size_t)unit * T + t];
          }
        }
        S.dq[s][a] = v;
      }
      __syncthreads();
      // (b) through final_layer and the gates of unit j
      float dhd[8];   // dL/dh_{t-1} through z * h_{t-1}
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        float r = 0.f, z = 0.f, n = 0.f, ghn = 0.f;
        if (vt + s0 + s < v_end) {
          int agent, unit; gru_seq(p.plan, net, vt + s0 + s, agent, unit);
          const float* row = p.save + row_index(agent, unit, t, B, T + 1) * kGruSaveRow;
          r = row[kHidden + j]; z = row[2 * kHidden + j]; n = row[3 * kHidden + j]; ghn = row[4 * kHidden + j];
        }
        float dh = dhc[s];
        for (int a = 0; a < A; ++a) dh = fmaf(w3[a * H + jr], S.dq[s0 + s][a], dh);
        if (!live) dh = 0.f;
        const float dn = dh * (1.f - z), dz = dh * (S.hp[s0 + s][j] - n);
        dhd[s] = dh * z;
        const float dnp = dn * (1.f - n * n), drp = dnp * ghn * r * (1.f - r), dzp = dz * z * (1.f - z);
        S.dgi[s0 + s][j] = drp; S.dgi[s0 + s][kHidden + j] = dzp; S.dgi[s0 + s][2 * kHidden + j] = dnp;
        S.dgh[s0 + s][j] = drp; S.dgh[s0 + s][kHidden + j] = dzp; S.dgh[s0 + s][2 * kHidden + j] = dnp * r;
      }
      __syncthreads();
      // (c) dL/dh_{t-1} = z dh + W_hh^T dgh,  dL/dx1 = W_ih^T dgi (masked by the ReLU)
      {
        float ah[8], ax[8];
#pragma unroll
        for (int s = 0; s < 8; ++s) { ah[s] = dhd[s]; ax[s] = 0.f; }
        for (int gate = 0; gate < 3; ++gate) {
          const float* uhp = wh + gate * H * H;
          const float* uip = wi + gate * H * H;
#pragma unroll 2
          for (int u = 0; u < H; ++u) {
            const float uh = uhp[u * H], ui = uip[u * H];
            const int g = gate * kHidden + u;
#pragma unroll
            for (int s = 0; s < 8; ++s) { ah[s] = fmaf(uh, S.dgh[s0 + s][g], ah[s]); ax[s] = fmaf(ui, S.dgi[s0 + s][g], ax[s]); }
          }
        }
#pragma unroll
        for (int s = 0; s < 8; ++s) { dhc[s] = live ? ah[s] : 0.f; S.dx1[s0 + s][j] = S.x1[s0 + s][j] > 0.f ? ax[s] : 0.f; }
      }
      __syncthreads();
      // (d) weight-gradient sums of this step over the tile's 16 sequences, added in fixed order
      for (int e = threadIdx.x; e < H * D; e += kGruThreads) {
        const int g = e / D, k = e - g * D;
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < kGruSeqs; ++s) acc = fmaf(S.dx1[s][g], S.x[s][k], acc);
        out[p.lay.w1 + e] += acc;
      }
      if (threadIdx.x < H) {
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < kGruSeqs; ++s) acc += S.dx1[s][threadIdx.x];
        out[p.lay.b1 + threadIdx.x] += acc;
      }
      // (padded index e: gate row g = gate * 128 + u, column k; stored at (gate * H + u) * H + k when u, k < H)
      for (int e = threadIdx.x; e < 3 * kHidden * kHidden; e += kGruThreads) {
        const int g = e >> 7, k = e & (kHidden - 1), u = g & (kHidden - 1);
        if (u >= H || k >= H) continue;
        float ai = 0.f, ah = 0.f;
#pragma unroll
        for (int s = 0; s < kGruSeqs; ++s) { ai = fmaf(S.dgi[s][g], S.x1[s][k], ai); ah = fmaf(S.dgh[s][g], S.hp[s][k], ah); }
        const int o = ((g >> 7) * H + u) * H + k;
        out[p.lay.wih + o] += ai;
        out[p.lay.whh + o] += ah;
      }
      for (int g = threadIdx.x; g < 3 * kHidden; g += kGruThreads) {
        const int u = g & (kHidden - 1);
        if (u >= H) continue;
        float ai = 0.f, ah = 0.f;
#pragma unroll
        for (int s = 0; s < kGruSeqs; ++s) { ai += S.dgi[s][g]; ah += S.dgh[s][g]; }
        out[p.lay.bih + (g >> 7) * H + u] += ai;
        out[p.lay.bhh + (g >> 7) * H + u] += ah;
      }
      for (int e = threadIdx.x; e < A * kHidden; e += kGruThreads) {
        const int a = e >> 7, k = e & (kHidden - 1);
        if (k >= H) continue;
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < kGruSeqs; ++s) acc = fmaf(S.dq[s][a], S.hc[s][k], acc);
        out[p.lay.w3 + a * H + k] += acc;
      }
      if (threadIdx.x < A) {
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < kGruSeqs; ++s) acc += S.dq[s][threadIdx.x];
        out[p.lay.b3 + threadIdx.x] += acc;
      }
      __syncthreads();
    }
  }
}

template <int HEAD>
__global__ void __launch_bounds__(kGruHeadThreads) gru_ac_head_kernel(GruHeadParams p) {
  __shared__ float red[4][kGruHeadThreads];
  const int T = p.traj.T, tid = threadIdx.x, i = blockIdx.x * kGruHeadThreads + tid;
  float st[4] = {0.f, 0.f, 0.f, 0.f};
  if (i < p.N * p.P * T) {
    RowCtx c;
    c.agent = i / (p.P * T);
    const int rem = i - c.agent * p.P * T;
    c.b = rem / T; c.tt = rem - c.b * T; c.T = T; c.A = p.A; c.B = p.P;
    const size_t ep = (size_t)p.idx[c.b];
    c.act = p.traj.act[p.traj.step_at(ep, c.agent, c.tt)];
    c.filled = (float)p.traj.filled[p.traj.filled_at(ep, c.tt)];
    c.rew = 0.f; c.done1 = 0.f;   // not read by the actor-critic heads
    const size_t row = row_index(c.agent, c.b, c.tt, p.P, T + 1);
    float dq[kOutPad];
#pragma unroll
    for (int o = 0; o < kOutPad; ++o) dq[o] = 0.f;
    if constexpr (HEAD == kHeadA2cCritic) head_a2c_critic(p.tp, c, p.q + row * p.A, dq, st);
    else head_a2c_actor(p.tp, c, p.q + row * p.A, dq, st);
#pragma unroll
    for (int o = 0; o < kOutPad; ++o)
      if (o < p.A) p.dq[row * p.A + o] = dq[o];
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) red[k][tid] = st[k];
  __syncthreads();
  for (int s = kGruHeadThreads / 2; s > 0; s >>= 1) {
    if (tid < s) {
#pragma unroll
      for (int k = 0; k < 4; ++k) red[k][tid] += red[k][tid + s];
    }
    __syncthreads();
  }
  if (tid < 4) p.loss_part[4 * blockIdx.x + tid] = red[tid][0];
}

int gru_kernels_init() {
  static bool done = false;
  if (!done) {
    MARL_CUDA_TRY(cudaFuncSetAttribute(gru_backward_kernel<kMaxObsDim>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GruBwdSmem<kMaxObsDim>)));
    MARL_CUDA_TRY(cudaFuncSetAttribute(gru_backward_kernel<kMaxInDim>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GruBwdSmem<kMaxInDim>)));
    done = true;
  }
  return MARL_OK;
}

int launch_gru_forward(const GruFwdParams& p, cudaStream_t st) {
  int most = 0;
  for (int k = 0; k < p.plan.n_nets; ++k) {
    const int n = (p.plan.slot_begin[k + 1] - p.plan.slot_begin[k]) * p.plan.units_per_agent;
    most = n > most ? n : most;
  }
  const dim3 grid((most + kGruSeqs - 1) / kGruSeqs, p.plan.n_nets);
  if (p.lay.in <= kMaxObsDim) gru_forward_kernel<kMaxObsDim><<<grid, kGruThreads, 0, st>>>(p);
  else gru_forward_kernel<kMaxInDim><<<grid, kGruThreads, 0, st>>>(p);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int launch_gru_backward(const GruBwdParams& p, cudaStream_t st) {
  const int grid = p.plan.cta_begin[p.plan.n_nets];
  if (p.lay.in <= kMaxObsDim) gru_backward_kernel<kMaxObsDim><<<grid, kGruThreads, sizeof(GruBwdSmem<kMaxObsDim>), st>>>(p);
  else gru_backward_kernel<kMaxInDim><<<grid, kGruThreads, sizeof(GruBwdSmem<kMaxInDim>), st>>>(p);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

int launch_gru_ac_head(const GruHeadParams& p, int head, cudaStream_t st) {
  const int blocks = gru_head_blocks(p.N, p.P, p.traj.T);
  if (head == kHeadA2cCritic) gru_ac_head_kernel<kHeadA2cCritic><<<blocks, kGruHeadThreads, 0, st>>>(p);
  else gru_ac_head_kernel<kHeadA2cActor><<<blocks, kGruHeadThreads, 0, st>>>(p);
  MARL_CUDA_TRY(cudaGetLastError());
  return MARL_OK;
}

}  // namespace marl
