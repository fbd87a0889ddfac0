/*
 * lbf_grid_oracle.c -- CPU restatement of Level-Based Foraging's grid observation (ForagingEnv._make_gym_obs with grid_observation=True,
 * DESIGN.md Appendix A), written from direct index arithmetic on the unpadded field.  TEST INFRASTRUCTURE ONLY: it checks the CUDA kernels
 * (lbf_step_kernel<true>, lbf_grid_obs_kernel) and is itself checked against tests/lbf_grid_ref.py, a literal transcription of upstream's
 * padded-array construction that shares no code with it.
 *
 * field: int8[rows*cols] food levels; players: int8[n_agents][4] = (row, col, level, 0); out: float[3][2*sight+1][2*sight+1] in C order.
 */
#include <stdint.h>

int lbf_grid_obs_dim(int sight) { return 3 * (2 * sight + 1) * (2 * sight + 1); }

void lbf_grid_obs_one(int rows, int cols, int n_agents, int sight, const int8_t* field, const int8_t* players, int agent, float* out) {
  const int W = 2 * sight + 1;
  const int top = players[4 * agent] - sight, left = players[4 * agent + 1] - sight;   /* field cell of window cell (0, 0) */
  for (int y = 0; y < W; ++y)
    for (int x = 0; x < W; ++x) {
      const int r = top + y, c = left + x;
      float level = 0.f, food = 0.f, access = 0.f;
      if (r >= 0 && r < rows && c >= 0 && c < cols) {
        int occupied = 0;
        for (int j = 0; j < n_agents; ++j)   /* a later player on the same cell overwrites an earlier one, as upstream's assignment loop does */
          if (players[4 * j] == r && players[4 * j + 1] == c) { level = (float)players[4 * j + 2]; occupied = 1; }
        food = (float)field[r * cols + c];
        access = (!occupied && field[r * cols + c] == 0) ? 1.f : 0.f;
      }
      out[0 * W * W + y * W + x] = level;
      out[1 * W * W + y * W + x] = food;
      out[2 * W * W + y * W + x] = access;
    }
}

/* E envs: field [E][rows*cols], players [E][N][4], out [E][N][D] */
void lbf_grid_obs_batch(int n_envs, int rows, int cols, int n_agents, int sight, const int8_t* field, const int8_t* players, float* out) {
  const int D = lbf_grid_obs_dim(sight);
  for (int e = 0; e < n_envs; ++e)
    for (int i = 0; i < n_agents; ++i)
      lbf_grid_obs_one(rows, cols, n_agents, sight, field + (long)e * rows * cols, players + (long)e * n_agents * 4, i,
                       out + ((long)e * n_agents + i) * D);
}
