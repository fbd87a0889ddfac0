// gru.cuh -- recurrent (GRU) agent networks of the DQN family (algorithm.model.use_rnn=True) and of the actor-critic learners
// (actor.use_rnn / critic.use_rnn): parameter layout, the sequence forward, the actor-critic loss head and the BPTT backward.  Replaces marlbase/utils/models.py:51-116 (RNNNetwork with layers = [H, H]:
// first_layer Linear(D, H) + ReLU, nn.GRU(H, H, num_layers=1), final_layer Linear(H, A)), 1 <= H <= 128.  The kernels keep 128 units per sequence;
// units >= H are padding that stays exactly 0 (zero input, r = z = 1/2, n = tanh(0) = 0, so h' = h / 2 = 0 from the zero state) and is never stored
// in the parameters or the gradients.
#pragma once
#include "learner.cuh"

namespace marl {

constexpr int kGruSeqs = 16;                 // sequences per CTA tile (two halves of 8, one per 128-thread half of the block)
constexpr int kGruThreads = 256;
constexpr int kGruSaveRow = 6 * kHidden;     // floats the online pass saves per row: x1 | r | z | n | W_hn h + b_hn | h' (128 each; units >= H hold 0)

// Flat parameters of one network in the reference's state_dict order; H = the hidden width.  weight_ih_l0 / weight_hh_l0 are [3H][H] with the
// gate blocks r, z, n at rows 0, H, 2H (torch's order).
struct GruLayout {
  int in, out, H;
  int w1, b1, wih, whh, bih, bhh, w3, b3, P;   // float offsets, P = total
  __host__ __device__ static GruLayout make(int in_, int out_, int hid = kHidden) {
    GruLayout l; l.in = in_; l.out = out_; l.H = hid;
    l.w1 = 0; l.b1 = l.w1 + hid * in_;
    l.wih = l.b1 + hid; l.whh = l.wih + 3 * hid * hid;
    l.bih = l.whh + 3 * hid * hid; l.bhh = l.bih + 3 * hid;
    l.w3 = l.bhh + 3 * hid; l.b3 = l.w3 + out_ * hid; l.P = l.b3 + out_;
    return l;
  }
};

// One launch runs every sequence of every network for all of its steps.  plan: slot lists of the networks, units_per_agent = B (training:
// one sequence per sampled episode and agent) or E (act step), unit_rows = steps per sequence (T + 1, or 1).  src: kRowsEpisode
// gathers through the replay indices, kRowsDense reads dense obs [E][N][D], the joint modes the rows of a centralised critic (learner.cuh).
struct GruFwdParams {
  RowPlan plan; RowSource src;
  const float* theta; GruLayout lay;
  const float* h_in;   // dense rows: [E][N][H] initial state (NULL: zeros); episode rows: always zeros (the reference's hiddens=None)
  float* h_out;        // dense rows: [E][N][H] final state (NULL: not written)
  float* q_out;        // dense rows: [E][N][A]; episode rows: [N][B][T+1][A]
  float* save;         // episode rows, online pass: [N][B][T+1][kGruSaveRow] for the backward (NULL: not saved)
};

// BPTT from dL/dq.  CTA c of net k (plan.cta_begin) owns a contiguous run of that net's sequences and writes the gradient sums of all eight
// tensors into scratch[c][0 .. P) in fixed order.
struct GruBwdParams {
  RowPlan plan; TrajView traj; const int32_t* idx; int B;
  const float* theta; GruLayout lay;
  const float* save;                    // the online pass's saved rows
  const float* td; int td_agent_stride; // DQN: 2 * delta * filled of the taken action at [agent * stride + b * T + t]
  const float* dout;                    // actor-critic: dense dL/dout [N][B][T+1][out] (rows t < T read); non-NULL replaces td
  RowSource src;                        // the rows the online pass read: kRowsEpisode (each agent's observations) or kRowsEpisodeJoint (centralised critic)
  float* scratch; int scratch_pitch;
};

// Loss head of a recurrent actor-critic part on the stored sequence outputs q [N][P][T+1][A]: one thread per (agent, env, t < T) runs
// head_a2c_critic or head_a2c_actor (ac_heads.cuh), writes dL/dq into dq (same layout) and block b's loss statistics into loss_part[b][0 .. 4)
// (fixed-order tree, no atomics).
constexpr int kGruHeadThreads = 256;
struct GruHeadParams {
  TrainParams tp;   // the head's fields: returns, adv_out, value_coef (critic); adv, entropy_coef, old_logp, ppo_clip (actor)
  TrajView traj; const int32_t* idx; int N, P, A;
  const float* q; float* dq;
  float* loss_part;
};
inline int gru_head_blocks(int N, int P, int T) { return (int)(((long long)N * P * T + kGruHeadThreads - 1) / kGruHeadThreads); }

int gru_kernels_init();
int launch_gru_forward(const GruFwdParams& p, cudaStream_t st);
int launch_gru_backward(const GruBwdParams& p, cudaStream_t st);
int launch_gru_ac_head(const GruHeadParams& p, int head, cudaStream_t st);

}  // namespace marl
