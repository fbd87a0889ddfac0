/*
 * lbf_oracle.h -- CPU restatement of the Level-Based-Foraging transition + marlbase wrapper stack.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ may be imported, linked or executed by the product
 * path (codebase_b200/).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs use it, and only as the checker / CPU baseline.
 *
 * PARITY UNPINNED (env half): `ForagingEnv.step/reset` is NOT in the reference project -- it lives in the
 * third-party, un-vendored, unpinned pip package `lbforaging` (GitHub uoe-agents/lb-foraging, the
 * gymnasium-era 2.x/3.x line that registers the `-v3` ids; reference call sites
 * marlbase/utils/envs.py:27-37,90-92, consumer marlbase/dqn/train.py:203,217, marlbase/ac/train.py:30,79-81).
 * The reference holds no tests, fixtures or golden vectors for it, so this file restates the published
 * algorithm (SURVEY.md Appendix A) and IS the specification the CUDA kernel is compared against.
 * The wrapper half (TimeLimit / RecordEpisodeStatistics / CooperativeReward) follows
 * marlbase/utils/wrappers.py:13-45,106-108 and marlbase/utils/envs.py:93-109.
 */
#ifndef LBF_ORACLE_H
#define LBF_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Field-for-field the same meaning as marl_lbf_cfg in include/marl_b200.h, declared independently. */
typedef struct {
  int32_t rows, cols;          /* field_size */
  int32_t n_agents;            /* players */
  int32_t max_num_food;
  int32_t sight;               /* == rows for full observability, 2 for "-2s" ids */
  int32_t min_player_level, max_player_level;
  int32_t min_food_level;
  int32_t max_food_level;      /* <=0 : None -> sum of the (up to) 3 lowest player levels */
  int32_t max_episode_steps;   /* env-internal horizon (50 in the registered ids) */
  int32_t time_limit;          /* gymnasium TimeLimit wrapper (envs.py:95-96); 0 = absent */
  int32_t force_coop;
  int32_t normalize_reward;
  int32_t cooperative_reward;  /* CooperativeReward wrapper (wrappers.py:106-108, vdn.yaml:6-8) */
  double  penalty;
  int32_t observe_id;          /* ObserveID (wrappers.py:75-103) */
  int32_t standardise_rewards; /* StandardiseReward (wrappers.py:111-141), between RecordEpisodeStatistics and CooperativeReward (envs.py:97-109) */
  int32_t upstream_reset;      /* 1: stale previous-episode positions block cells during spawning; the two level-bound permutations consume draws */
} lbf_oracle_cfg;

/* Philox4x32-10 (Random123).  Pinned by the published known-answer vectors in tests/. */
void lbf_oracle_philox(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);

int  lbf_oracle_obs_dim(const lbf_oracle_cfg* c);

/* One env.  field: int8[rows*cols]; players: int8[n_agents][4] = (row, col, level, 0). */
void lbf_oracle_reset_one(const lbf_oracle_cfg* c, uint64_t seed, uint32_t env_gid, uint32_t episode_idx,
                          int8_t* field, int8_t* players, int32_t* food_spawned);
/* Raw env transition (no wrappers): rewards_raw are the python-float (f64) per-agent rewards. */
void lbf_oracle_step_one(const lbf_oracle_cfg* c, int8_t* field, int8_t* players, int32_t* step,
                         int32_t food_spawned, const int32_t* actions, double* rewards_raw,
                         int32_t* done, int32_t* truncated);
void lbf_oracle_obs_one(const lbf_oracle_cfg* c, const int8_t* field, const int8_t* players, int agent,
                        float* out);

/* Batched env + wrapper stack with exactly the semantics of marl_lbf_reset / marl_lbf_step. */
typedef struct {
  int8_t*   field;        /* [E][rows*cols] */
  int8_t*   players;      /* [E][N][4] */
  int32_t*  step;         /* [E] */
  int32_t*  food_spawned; /* [E] */
  float*    ep_return;    /* [E][N]  f32 accumulation (wrappers.py:33) */
  int32_t*  ep_len;       /* [E] */
  uint32_t* episode_idx;  /* [E] number of resets so far */
  uint8_t*  active;       /* [E] */
  float*    stdr;         /* [E][2N+1] StandardiseReward state: wmean[N] | t[N] | sumw (float32, like the wrapper's arrays); may be NULL without the flag */
  int32_t*  stdr_n;       /* [E] */
} lbf_oracle_state;

void lbf_oracle_reset(const lbf_oracle_cfg* c, int32_t n_envs, uint64_t seed, uint32_t env_gid0,
                      lbf_oracle_state* s, const uint8_t* reset_mask, float* obs_out);
void lbf_oracle_step(const lbf_oracle_cfg* c, int32_t n_envs, uint64_t seed, uint32_t env_gid0,
                     lbf_oracle_state* s, const int32_t* actions, float* obs_out, float* rew_out,
                     uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out,
                     int32_t autoreset);

#ifdef __cplusplus
}
#endif
#endif
