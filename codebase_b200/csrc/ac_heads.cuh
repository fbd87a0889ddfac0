// ac_heads.cuh -- loss heads of the actor-critic learners, shared by the fused MLP training kernel (learner_kernels.cu) and the head kernel of the
// recurrent parts (gru_kernels.cu).  One thread per (agent, env, step) row: `q` = the row's network outputs, results: dq[0..7] = dLoss/d(output)
// un-normalised, st[0..3] += loss statistics.
#pragma once
#include "learner.cuh"

namespace marl {

struct RowCtx { int agent, b, tt, T, A, B; int act; float rew, filled, done1; };

__device__ __forceinline__ void head_a2c_critic(const TrainParams& p, const RowCtx& c, const float* q, float (&dq)[kOutPad], float (&st)[4]) {
  const size_t i = ((size_t)c.agent * c.B + c.b) * c.T + c.tt;
  const float filled = c.filled;
  const float adv = p.returns[i] - q[0];                    // ac/model.py:214
  p.adv_out[i] = adv;
  st[3] += adv * adv * filled;                              // ac/model.py:221-222
  if (c.agent == 0) st[1] += filled;
  dq[0] = -2.f * adv * filled * p.value_coef;               // d(value_loss_coef * (R - V)^2)/dV
}

__device__ __forceinline__ void head_a2c_actor(const TrainParams& p, const RowCtx& c, const float* q, float (&dq)[kOutPad], float (&st)[4]) {
  const size_t i = ((size_t)c.agent * c.B + c.b) * c.T + c.tt;
  const int act = c.act;
  const float filled = c.filled;
  const float adv = p.adv[i];
  float m = q[0];
  for (int o = 1; o < c.A; ++o) m = fmaxf(m, q[o]);
  float s = 0.f;
  for (int o = 0; o < c.A; ++o) s += expf(q[o] - m);
  const float lse = m + logf(s);
  float ent = 0.f, pr[kOutPad], ls[kOutPad];
#pragma unroll
  for (int o = 0; o < kOutPad; ++o) {
    ls[o] = o < c.A ? q[o] - lse : 0.f;                     // Categorical(logits) normalisation (ac/model.py:142-144)
    pr[o] = o < c.A ? expf(ls[o]) : 0.f;
    ent -= pr[o] * ls[o];
  }
  float w = adv;   // dLoss/dlogp[act] = -w
  if (p.old_logp != nullptr) {
    // PPO clipped surrogate (ac/model.py:309-321).  torch.min sends the gradient to the smaller argument (half to each on a tie), clamp passes it
    // inside [1 - c, 1 + c]: d(-min(r adv, clamp(r) adv))/dlogp = -adv r k, k = 1 when the unclipped term is the minimum or r is inside the range.
    const float ratio = expf(ls[act] - p.old_logp[i]);
    const float lo = 1.f - p.ppo_clip, hi = 1.f + p.ppo_clip;
    const float surr1 = ratio * adv, surr2 = fminf(fmaxf(ratio, lo), hi) * adv;
    const float inrange = (ratio >= lo && ratio <= hi) ? 1.f : 0.f;
    const float k = surr1 < surr2 ? 1.f : (surr1 > surr2 ? inrange : 0.5f + 0.5f * inrange);
    st[0] += -fminf(surr1, surr2) * filled;
    w = adv * ratio * k;
  } else {
    st[0] += -ls[act] * adv * filled;                       // ac/model.py:216-219
  }
  st[2] += ent * filled;
#pragma unroll
  for (int o = 0; o < kOutPad; ++o)
    dq[o] = o < c.A ? filled * (w * (pr[o] - (o == act ? 1.f : 0.f)) + p.entropy_coef * pr[o] * (ls[o] + ent)) : 0.f;
}

}  // namespace marl
