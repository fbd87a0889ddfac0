// traj.cuh -- device view of the trajectory store (marl_traj_view: the replay ring and the on-policy batch).  The env-step kernels write it,
// the learner kernels read it; both index it only through the functions below.  Episode-major, per ring slot ep < capacity:
//   obs float [cap][N][T+1][D]   act int32, rew float [cap][N][T]   done uint8 [cap][T+1]   filled uint8 [cap][T]
// (done[t]: observation t is terminal; filled[t]: step t was taken.)
#pragma once
#include "common.cuh"

namespace marl {

struct TrajView {
  float* obs; int32_t* act; float* rew; uint8_t* done; uint8_t* filled;   // all NULL: no store (an env step that records nothing)
  int capacity, N, T, D;
  // observation row of agent `agent` at step t <= T of slot ep
  __host__ __device__ __forceinline__ float* obs_row(size_t ep, int agent, int t) const { return obs + ((ep * N + agent) * (size_t)(T + 1) + t) * D; }
  // element (ep, agent, t < T) of act and rew
  __host__ __device__ __forceinline__ size_t step_at(size_t ep, int agent, int t) const { return (ep * N + agent) * T + t; }
  __host__ __device__ __forceinline__ size_t done_at(size_t ep, int t) const { return ep * (T + 1) + t; }
  __host__ __device__ __forceinline__ size_t filled_at(size_t ep, int t) const { return ep * T + t; }
};

inline TrajView traj_view(const marl_traj_view* t) {
  TrajView v = {};
  if (t) {
    v.obs = t->obs; v.act = t->act; v.rew = t->rew; v.done = t->done; v.filled = t->filled;
    v.capacity = t->capacity; v.N = t->n_agents; v.T = t->T; v.D = t->obs_dim;
  }
  return v;
}

}  // namespace marl
