// dqn_heads.cuh -- the TD rule of the DQN family (marlbase/dqn/model.py:138-163), shared by the fused FP32 training kernel (learner_kernels.cu),
// the tensor-core training pipeline (tc_train.cu), the column TD kernel (dqn.cu) and the QMIX mixer (qmix.cuh).
#pragma once
#include "common.cuh"

namespace marl {

// Bootstrap value of the next row (dqn/model.py:138-145): double_q: the target row tq at the first maximum of the online row qn; else max(tq).
__device__ __forceinline__ float next_value(const float* qn, const float* tq, int A, int double_q) {
  if (double_q) {
    int best = 0; float bv = qn[0];
    for (int o = 1; o < A; ++o) if (qn[o] > bv) { bv = qn[o]; best = o; }
    return tq[best];
  }
  float m = tq[0];
  for (int o = 1; o < A; ++o) m = fmaxf(m, tq[o]);
  return m;
}

// y = r + gamma next (1 - done[t + 1]) (dqn/model.py:152), free for the compiler to contract
__device__ __forceinline__ float td_target(float rew, float gamma, float next, float done1) { return rew + gamma * next * (1.f - done1); }

// The same target rounded step by step, no contraction: standardise_returns (dqn/model.py:147-152), whose returns feed the statistics
__device__ __forceinline__ float td_target_rn(float rew, float gamma, float next, float done1) {
  return __fadd_rn(rew, __fmul_rn(__fmul_rn(gamma, next), 1.f - done1));
}

// Loss of one TD error delta = Q - y and its derivative in Q.  huber <= 0: the reference's squared error (dqn/model.py:160-163), delta^2 and
// 2 delta.  huber > 0 (algorithm.huber_delta): torch.nn.functional.huber_loss with delta = huber, 0.5 delta^2 for |delta| < huber, else
// huber (|delta| - 0.5 huber), and clamp(delta, -huber, huber) -- half the squared error and half its gradient inside the band.
__device__ __forceinline__ float td_loss(float delta, float huber) {
  if (huber > 0.f) {
    const float ad = fabsf(delta);
    return ad < huber ? 0.5f * delta * delta : huber * (ad - 0.5f * huber);
  }
  return delta * delta;
}
__device__ __forceinline__ float td_dloss(float delta, float huber) { return huber > 0.f ? fminf(fmaxf(delta, -huber), huber) : 2.f * delta; }

// TD error of one row against its target y: returns dLoss/dQ[a] = td_dloss(delta) filled; s0 += td_loss(delta) filled, s1 += filled when the row
// counts the batch's filled steps (agent 0 / column 0) (dqn/model.py:160-163)
__device__ __forceinline__ float td_error(float q_act, float y, float filled, bool counts_filled, float& s0, float& s1, float huber) {
  const float delta = q_act - y;
  s0 += td_loss(delta, huber) * filled;
  if (counts_filled) s1 += filled;
  return td_dloss(delta, huber) * filled;
}

}  // namespace marl
