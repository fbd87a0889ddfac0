/*
 * marl_b200.h -- C ABI of libmarlb200.so, the H100 (sm_90a) native hot path behind marlbase's plugin surface.
 *
 * The reference (marl-book/codebase, `marlbase`) is 100 % Python and has NO FFI boundary of its own: its
 * plugin surface is Hydra `_target_` strings + Python duck typing (SURVEY.md §8b).  This header is therefore
 * the boundary a maintainer would bind (ctypes stub shown in INTEGRATION.md) to replace, one for one, the
 * Python call sites cited on each entry point below.  Citations are path:line in the reference project (marl-book/codebase).
 *
 * Conventions
 *   - every pointer argument documented "device" is a CUDA device pointer owned by the caller (a torch tensor);
 *     `stream` is a cudaStream_t passed as void*; calls enqueue work and return without synchronising;
 *   - return value 0 = ok, negative = MARL_E*; the message is in marl_last_error() (thread local);
 *   - handles are opaque, one host thread per GPU, not thread safe; no C++ / torch types cross the ABI;
 *   - there is NO CPU fallback: every entry point fails with MARL_ECUDA if no sm_90 (Hopper) device is present.
 */
#ifndef MARL_B200_H
#define MARL_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MARL_OK 0
#define MARL_EINVAL (-1)   /* bad argument / unsupported configuration */
#define MARL_ECUDA (-2)    /* CUDA runtime error (message has the cudaError string) */
#define MARL_ENOMEM (-3)

#define MARL_MAX_AGENTS 32
#define MARL_ABI_VERSION 1

int marl_version(void);
const char* marl_last_error(void);
/* Process-wide options: "tensor_core_forward" 1 (default) = forward-only passes on the tensor cores (wgmma) with the 3xTF32 split, 0 = FP32 FFMA;
 * "tensor_core_backward" 1 = the DQN-family training pass runs as the three-kernel wgmma pipeline (tc_train.cu), 0 = fused FP32 kernel. */
int marl_set_option(const char* name, int32_t value);
/* Profiling builds (-DMARL_TC_TIMESTAMPS): timeline probes of kernel `which` as uint64 [160 CTAs][32 slots][globaltimer ns, clock64] into HOST
 * memory; product builds return MARL_EINVAL. */
int marl_debug_timestamps(int32_t which, uint64_t* out);

/* ------------------------------------------------------------------------------------------------------
 * Level-Based Foraging, E environments per handle, one transition of all of them per launch.
 * Replaces `env.reset()` / `env.step(actions)` of the gym.make()'d third-party `lbforaging` ForagingEnv under
 * marlbase's wrapper stack:  marlbase/utils/envs.py:90-111 (single), :27-63 (AsyncVectorEnv), consumed at
 * marlbase/dqn/train.py:203,217 and marlbase/ac/train.py:30,79-81; wrappers marlbase/utils/wrappers.py:13-45
 * (RecordEpisodeStatistics), :106-108 (CooperativeReward); gymnasium TimeLimit at envs.py:95-96.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t rows, cols;          /* field_size */
  int32_t n_agents;            /* players (<= MARL_MAX_AGENTS) */
  int32_t max_num_food;
  int32_t sight;               /* == rows: full observability; 2 for the "-2s" ids */
  int32_t min_player_level, max_player_level;
  int32_t min_food_level;
  int32_t max_food_level;      /* <= 0: None -> sum of the (up to) 3 lowest player levels */
  int32_t max_episode_steps;   /* env-internal horizon (50 for the registered ids) */
  int32_t time_limit;          /* TimeLimit wrapper, env.time_limit in default.yaml:31; 0 = absent */
  int32_t force_coop;
  int32_t normalize_reward;
  int32_t cooperative_reward;  /* CooperativeReward wrapper (configs/algorithm/vdn.yaml:6-8) */
  double  penalty;
  int32_t observe_id;          /* ObserveID wrapper (marlbase/utils/wrappers.py:75-103, env.observe_id): one-hot agent id in front of every observation */
  int32_t standardise_rewards; /* StandardiseReward wrapper (wrappers.py:111-141, env.standardise_rewards): per-env running mean / variance, applied
                                  after RecordEpisodeStatistics (which keeps the raw rewards) and before CooperativeReward (envs.py:97-109) */
  int32_t upstream_reset;      /* 1: the two reset details of upstream lbforaging that the default leaves out -- (a) players that have not been re-placed
                                  yet still block their previous episode's cell (upstream never clears positions in reset()), (b) the two
                                  np_random.permutation() calls over the (identical) level bounds consume random draws (here: n - 1 Philox draws
                                  each, values unused).  0 (default): positions are cleared first and no draw is spent on the no-op permutations. */
  int32_t grid_observation;    /* 1: upstream's grid observation (the `Foraging-grid-*` ids, DESIGN.md Appendix A): layers agents | foods | access of the
                                  (2*sight+1)^2 window centred on the agent, field padded by `sight`, flattened in C order (FlattenObservation).
                                  1 <= sight <= 127; not with observe_id (ObserveID assumes a flattened observation space). */
} marl_lbf_cfg;

typedef struct marl_lbf marl_lbf;

/* Trajectory store: the device layout of BOTH the episode replay ring (marlbase/dqn/train.py:19-124,
 * capacity = buffer_size episodes) and the on-policy batch (marlbase/ac/train.py:36-52, capacity =
 * parallel_envs).  Episode-major so that one sampled episode of one agent is one contiguous run. */
typedef struct {
  float*   obs;     /* [capacity][N][T+1][obs_dim] */
  int32_t* act;     /* [capacity][N][T]            */
  float*   rew;     /* [capacity][N][T]            */
  uint8_t* done;    /* [capacity][T+1]             */
  uint8_t* filled;  /* [capacity][T]               */
  int32_t  capacity, n_agents, T, obs_dim;
} marl_traj_view;

int marl_lbf_create(const marl_lbf_cfg* cfg, int32_t n_envs, uint64_t seed, uint32_t env_gid0, int32_t device,
                    marl_lbf** out);
int marl_lbf_destroy(marl_lbf* env);
int marl_lbf_obs_dim(const marl_lbf_cfg* cfg);             /* 3*max_num_food + 3*n_agents (+ n_agents with observe_id); grid_observation: 3*(2*sight+1)^2 */
/* Overwrite the transition state (parity tests): host or device pointers are NOT mixed -- all device. */
int marl_lbf_set_state(marl_lbf* env, const int8_t* field /*[E][rows*cols] dense*/, const int8_t* players,
                       const int32_t* step, void* stream);

/* Copy the state out into caller-owned DEVICE buffers (any may be NULL): field dense int8[E][rows*cols],
 * players int8[E][N][4], step/food_spawned/ep_len int32[E], ep_return float[E][N], episode_idx uint32[E],
 * active uint8[E]. */
int marl_lbf_get_state(marl_lbf* env, int8_t* field, int8_t* players, int32_t* step, int32_t* food_spawned,
                       float* ep_return, int32_t* ep_len, uint32_t* episode_idx, uint8_t* active, void* stream);

/* env.reset(): reset_mask device uint8[E] or NULL (= all).  obs_out device float[E][N][obs_dim].
 * If `traj` is non-NULL also performs ReplayBuffer.init_episode (dqn/train.py:65-71): obs slot 0 of
 * ring slot (slot0 + e) % capacity. */
int marl_lbf_reset(marl_lbf* env, const uint8_t* reset_mask, float* obs_out, const marl_traj_view* traj,
                   int32_t slot0, void* stream);

/* env.step(actions): actions device int32[E][N].  Outputs (device): obs_out float[E][N][obs_dim] (the new
 * episode's first observation when autoreset fires, as gymnasium<1.0 vector envs do), rew_out float[E][N],
 * done_out/trunc_out uint8[E], final_ret_out float[E][N] + final_len_out int32[E] written only for envs whose
 * episode ended in this call (info["episode_returns"], info["episode_length"]). */
int marl_lbf_step(marl_lbf* env, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out,
                  uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out, int32_t autoreset,
                  void* stream);

/* Fused policy + transition + storage: one launch does, for every env,
 *   model.act      dqn/model.py:94-116 (policy=1: epsilon-greedy over `values`) or
 *                  ac/model.py:147-153 (policy=2: Categorical(logits=values).sample())
 *   env.step       (as marl_lbf_step)
 *   rb.add / batch_* writes   dqn/train.py:73-89, ac/train.py:90-99   (when traj != NULL)
 * values: device float[E][N][n_actions] produced by marl_mlp_forward on the current obs buffer.
 * actions_out (optional) receives the chosen actions. */
typedef struct {
  int32_t policy;                 /* 1 = eps-greedy on Q-values, 2 = categorical on logits */
  float   epsilon;
  int32_t n_actions;
  int32_t use_proper_termination; /* dqn/train.py:219-225 */
  int32_t autoreset;
  int32_t clear_stale;            /* 0 = reference behaviour (a reused ring slot keeps stale tail, SURVEY H6) */
  int32_t slot0;
} marl_rollout_args;

int marl_lbf_rollout_step(marl_lbf* env, const float* values, const marl_rollout_args* args,
                          const marl_traj_view* traj, float* obs_inout, float* rew_out, uint8_t* done_out,
                          uint8_t* trunc_out, float* final_ret_out, int32_t* final_len_out,
                          int32_t* actions_out, void* stream);

/* Frames of the current state (video recording; geometry and palette: DESIGN.md §4.8).  A frame is uint8 RGB [h][w][3] with
 * h = 1 + rows * 51 and w = 1 + cols * 51 (50-px cells, 1-px grid lines), as marl_lbf_frame_shape returns them.  marl_lbf_render writes the
 * frames of envs [env_first, env_first + n) to the DEVICE buffer frames uint8[n][h][w][3], in one launch; an empty range or one outside
 * [0, E) returns MARL_EINVAL. */
int marl_lbf_frame_shape(const marl_lbf_cfg* cfg, int32_t* h, int32_t* w);
int marl_lbf_render(marl_lbf* env, int32_t env_first, int32_t n, uint8_t* frames, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Multi-robot warehouse (RWARE), E environments per handle, one transition of all of them per launch.
 * Replaces `env.reset()` / `env.step(actions)` of the gym.make()'d third-party `rware` Warehouse (2.x, gymnasium; ids
 * `rware-{tiny,small,medium,large}-{N}ag[-easy|-hard]-v2`) under the same wrapper stack as marl_lbf_*.  Semantics: DESIGN.md Appendix B.
 * The entry points mirror the marl_lbf_* contracts; the trajectory view and the rollout arguments are the same structs.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t shelf_rows, shelf_columns;  /* grid = ((column_height + 1) * shelf_rows + 2) rows x (3 * shelf_columns + 1) columns */
  int32_t column_height;              /* 8 for the registered ids */
  int32_t n_agents;                   /* 1..31 */
  int32_t request_queue_size;         /* requested shelves at any time; 1 .. shelves - 1 */
  int32_t max_steps;                  /* env-internal horizon (terminates); 0 = none */
  int32_t max_inactivity_steps;       /* terminates after this many steps without a delivery; 0 = None */
  int32_t sensor_range;               /* 0..3; observation = 8 + 7 * (2r + 1)^2 floats */
  int32_t time_limit;                 /* TimeLimit wrapper (truncates); 0 = absent */
  int32_t cooperative_reward;         /* CooperativeReward wrapper */
  int32_t observe_id;                 /* ObserveID wrapper: one-hot agent id in front of every observation */
  int32_t standardise_rewards;        /* StandardiseReward wrapper, as marl_lbf_cfg.standardise_rewards */
} marl_rware_cfg;

typedef struct marl_rware marl_rware;

int marl_rware_create(const marl_rware_cfg* cfg, int32_t n_envs, uint64_t seed, uint32_t env_gid0, int32_t device, marl_rware** out);
int marl_rware_destroy(marl_rware* env);
int marl_rware_obs_dim(const marl_rware_cfg* cfg);   /* 8 + 7 * (2 * sensor_range + 1)^2 (+ n_agents with observe_id) */
/* Overwrite the transition state (device pointers): shelves uint8[E][rows*cols] (shelf id 1..255 at its current cell, 0 none; a carried shelf
 * sits at its carrier's cell), agents uint8[E][N][4] = (x, y, direction, carried shelf id or 0), requested uint32[E][8] (bit k: shelf k is
 * requested), step / inactive int32[E] (steps so far, steps since the last delivery).  Episode returns and lengths restart at 0. */
int marl_rware_set_state(marl_rware* env, const uint8_t* shelves, const uint8_t* agents, const uint32_t* requested, const int32_t* step,
                         const int32_t* inactive, void* stream);
/* Copy the state out into caller-owned DEVICE buffers (any may be NULL), in the layout of marl_rware_set_state plus ep_return float[E][N],
 * ep_len int32[E], episode_idx uint32[E], active uint8[E]. */
int marl_rware_get_state(marl_rware* env, uint8_t* shelves, uint8_t* agents, uint32_t* requested, int32_t* step, int32_t* inactive,
                         float* ep_return, int32_t* ep_len, uint32_t* episode_idx, uint8_t* active, void* stream);
/* as marl_lbf_reset */
int marl_rware_reset(marl_rware* env, const uint8_t* reset_mask, float* obs_out, const marl_traj_view* traj, int32_t slot0, void* stream);
/* as marl_lbf_step; actions outside 0..4 act as NOOP */
int marl_rware_step(marl_rware* env, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out, uint8_t* trunc_out,
                    float* final_ret_out, int32_t* final_len_out, int32_t autoreset, void* stream);
/* as marl_lbf_rollout_step with args->policy = 2 (categorical on logits); policy 1 (epsilon-greedy) returns MARL_EINVAL: no DQN-family
 * learner takes RWARE's observation width */
int marl_rware_rollout_step(marl_rware* env, const float* values, const marl_rollout_args* args, const marl_traj_view* traj,
                            float* obs_inout, float* rew_out, uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out,
                            int32_t* final_len_out, int32_t* actions_out, void* stream);
/* as marl_lbf_frame_shape / marl_lbf_render, with 30-px cells: h = 1 + rows * 31, w = 1 + cols * 31 */
int marl_rware_frame_shape(const marl_rware_cfg* cfg, int32_t* h, int32_t* w);
int marl_rware_render(marl_rware* env, int32_t env_first, int32_t n, uint8_t* frames, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Repeated matrix games (the `matrixgames` package: climbing, penalty-k), E environments per handle, one transition of all of them per launch.
 * Replaces `env.reset()` / `env.step(actions)` of the gym.make()'d `matrixgames` MatrixGame under the same wrapper stack as marl_lbf_*.
 * Semantics: DESIGN.md Appendix C.  Every player has the same action count A; the reward of a step is payoff[a_0, ..., a_{N-1}] for every
 * player.  The entry points mirror the marl_rware_* contracts; the trajectory view and the rollout arguments are the same structs.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t n_agents;                   /* players N = payoff.ndim, 1..32 */
  int32_t n_actions;                  /* actions A of every player, 1..8, with A^N <= 65536 */
  const double* payoff;               /* HOST pointer to the A^N payoffs in C order (entry sum_i a_i * A^(N-1-i)); create copies them */
  int32_t ep_length;                  /* terminates when the step count reaches it; >= 1 (25 for the registered ids) */
  int32_t last_action_state;          /* 1: observation = one-hot of every player's previous action (N * A), all zero after a reset;
                                         0 (`-nostate` ids): one constant feature, 0 */
  int32_t time_limit;                 /* TimeLimit wrapper (truncates); 0 = absent */
  int32_t cooperative_reward;         /* CooperativeReward wrapper */
  int32_t observe_id;                 /* ObserveID wrapper: one-hot agent id in front of every observation */
  int32_t standardise_rewards;        /* StandardiseReward wrapper, as marl_lbf_cfg.standardise_rewards */
} marl_matrix_cfg;

typedef struct marl_matrix marl_matrix;

int marl_matrix_create(const marl_matrix_cfg* cfg, int32_t n_envs, uint64_t seed, uint32_t env_gid0, int32_t device, marl_matrix** out);
int marl_matrix_destroy(marl_matrix* env);
int marl_matrix_obs_dim(const marl_matrix_cfg* cfg);   /* N * A with last_action_state, else 1 (+ n_agents with observe_id) */
/* Overwrite the transition state (device pointers): last_action int8[E][N] (each player's previous action, -1: none, as after a reset),
 * step int32[E] (steps so far).  Episode returns and lengths restart at 0. */
int marl_matrix_set_state(marl_matrix* env, const int8_t* last_action, const int32_t* step, void* stream);
/* Copy the state out into caller-owned DEVICE buffers (any may be NULL), in the layout of marl_matrix_set_state plus ep_return float[E][N],
 * ep_len int32[E], episode_idx uint32[E], active uint8[E]. */
int marl_matrix_get_state(marl_matrix* env, int8_t* last_action, int32_t* step, float* ep_return, int32_t* ep_len, uint32_t* episode_idx,
                          uint8_t* active, void* stream);
/* as marl_lbf_reset; a reset draws nothing */
int marl_matrix_reset(marl_matrix* env, const uint8_t* reset_mask, float* obs_out, const marl_traj_view* traj, int32_t slot0, void* stream);
/* as marl_lbf_step; an action outside 0..A-1 is played as action 0 */
int marl_matrix_step(marl_matrix* env, const int32_t* actions, float* obs_out, float* rew_out, uint8_t* done_out, uint8_t* trunc_out,
                     float* final_ret_out, int32_t* final_len_out, int32_t autoreset, void* stream);
/* as marl_lbf_rollout_step (policy 1 or 2); args->n_actions must equal A */
int marl_matrix_rollout_step(marl_matrix* env, const float* values, const marl_rollout_args* args, const marl_traj_view* traj,
                             float* obs_inout, float* rew_out, uint8_t* done_out, uint8_t* trunc_out, float* final_ret_out,
                             int32_t* final_len_out, int32_t* actions_out, void* stream);
/* as marl_lbf_frame_shape / marl_lbf_render: an N x A board of 40-px cells, h = 1 + N * 41, w = 1 + A * 41 */
int marl_matrix_frame_shape(const marl_matrix_cfg* cfg, int32_t* h, int32_t* w);
int marl_matrix_render(marl_matrix* env, int32_t env_first, int32_t n, uint8_t* frames, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Per-agent MLP sets and the DQN-family learner (IDQN, VDN).
 * Replaces marlbase/dqn/model.py QNetwork (14-196) / VDNetwork (199-269) and the network containers of
 * marlbase/utils/models.py:133-300.  Parameters are one flat float array [n_nets][P] in the reference's
 * state_dict order per network: network.0.weight [H][in], network.0.bias [H], network.2.weight [H][H],
 * network.2.bias [H], network.4.weight [out][H], network.4.bias [out]  (utils/models.py:35-44).
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t n_agents, n_nets;
  int32_t agent_net[MARL_MAX_AGENTS]; /* network of each agent: identity = independent (parameter_sharing False),
                                         all 0 = full sharing, else the seps indices (utils/models.py:189-196) */
  int32_t in_dim;                     /* flatdim(observation_space[i]) (or n_agents x it: centralised critic); 1..32 for marl_dqn_*,
                                         1..128 for marl_a2c_* (actor and critic) */
  int32_t hidden;                     /* layers = [hidden, hidden]: 1..128, default 128 (idqn.yaml:8-10).  Below 128 the parameters stay
                                         compact (H = hidden in the layouts above and below) and the FP32 kernels run, whatever the
                                         "tensor_core_*" options say */
  int32_t out_dim;                    /* n_actions (Q / logits) or 1 (state value) */
} marl_mlp_cfg;

typedef struct {
  float   lr;                             /* idqn.yaml:18 */
  float   gamma;                          /* idqn.yaml:19 */
  float   grad_clip;                      /* idqn.yaml:23, <= 0 disables clip_grad_norm_ */
  int32_t double_q;                       /* idqn.yaml:21 */
  float   target_update_interval_or_tau;  /* idqn.yaml:37: > 1 hard update every k updates, < 1 Polyak tau */
  float   beta1, beta2, eps;              /* torch.optim.Adam defaults 0.9, 0.999, 1e-8 (dqn/model.py:71) */
  int32_t mixer;                          /* 0 = independent learners (QNetwork), 1 = VDN sum (VDNetwork), 2 = QMIX (QMixNetwork) */
} marl_dqn_hp;

typedef struct marl_dqn marl_dqn;

/* The optimiser of a learner (algorithm.optimizer): the reference builds torch.optim.<name>(parameters, lr=cfg.lr) with torch's defaults for
 * everything else (marlbase/dqn/model.py:66-71,368-371, ac/model.py:103-109).  Each step runs per parameter on the gradient after
 * clip_grad_norm_ (g), with lr = hp.lr, as torch's single-tensor implementation does:
 *   MARL_OPT_ADAM     exp_avg (adam_m), exp_avg_sq (adam_v): Adam with bias correction; beta1, beta2, eps
 *   MARL_OPT_ADAMW    theta *= 1 - lr * weight_decay, then the Adam step
 *   MARL_OPT_RMSPROP  square_avg (adam_v): s = alpha * s + (1 - alpha) * g^2; theta -= lr * g / (sqrt(s) + eps)
 *   MARL_OPT_ADAGRAD  sum (adam_v): s += g^2; theta -= lr * g / (sqrt(s) + eps)   (lr_decay 0, initial accumulator 0)
 *   MARL_OPT_SGD      theta -= lr * g   (no state; momentum 0)
 * torch's defaults: Adam betas (0.9, 0.999), eps 1e-8; AdamW the same and weight_decay 0.01; RMSprop alpha 0.99, eps 1e-8; Adagrad eps 1e-10.
 * Fields an optimiser does not use are ignored. */
#define MARL_OPT_ADAM 0
#define MARL_OPT_ADAMW 1
#define MARL_OPT_RMSPROP 2
#define MARL_OPT_ADAGRAD 3
#define MARL_OPT_SGD 4
typedef struct {   /* the constants as torch holds them (Python floats); the step rounds them where torch does */
  int32_t kind;           /* MARL_OPT_* */
  double  beta1, beta2;   /* Adam, AdamW */
  double  alpha;          /* RMSprop */
  double  eps;            /* Adam, AdamW, RMSprop, Adagrad */
  double  weight_decay;   /* AdamW (decoupled) */
} marl_optimizer;

int marl_dqn_create(const marl_mlp_cfg* cfg, const marl_dqn_hp* hp, int32_t max_batch, int32_t max_T, int32_t device,
                    marl_dqn** out);
int marl_dqn_destroy(marl_dqn* q);
/* Device pointers to the flat parameter / optimiser state ([n_nets*P] floats each; grad has 4 extra floats:
 * loss numerator, filled count, 2 spare).  Initialise theta through these (orthogonal init is done by the caller). */
/* cfg.standardise_returns of the DQN family (marlbase/dqn/model.py:82-84,147-158; VDN 221-222,256-264; utils/standardise_stream.py): a
 * RunningMeanStd over the TD targets of every update -- target Q-values are de-standardised with the statistics so far, the statistics absorb the
 * batch's returns, the returns are standardised before the loss.  One column per agent; VDN and QMIX: one per batch entry (the reference's
 * reshape), so their updates must use batch == max_batch. */
int marl_dqn_standardise_returns(marl_dqn* q, int32_t enable);
int marl_dqn_ret_ms_ptrs(marl_dqn* q, float** ret_ms /* mean[n] | var[n] */, double** count, int32_t* n_stat);
/* device scratch of the last update's external TD head (parity tests), NULL where not allocated: bootstrap values v_{t+1} (td_lambda), TD targets
 * (standardised under standardise_returns), chosen Q-values, each [C][B][T] with C = n_agents (IDQN) or 1 (VDN, QMIX; QMIX leaves chosen
 * unwritten); and dLoss/dQ of the taken actions: IDQN, VDN [C][B][T], QMIX per agent [N][B][T] */
int marl_dqn_scratch_ptrs(marl_dqn* q, float** boot, float** ret, float** chosen, float** td);
/* algorithm.td_lambda of IDQN, VDN and QMIX (this project's option; the reference has only the one-step target): enable != 0 makes every later
 * update (marl_dqn_update, _update_grads, _update_n) use the TD(λ) target of `lambda` in [0, 1] over the sampled episode,
 *   G_t = r_t + γ (1 - d_{t+1}) ((1 - λ f_{t+1}) v_{t+1} + λ f_{t+1} G_{t+1}),  f_T = 0,
 * with v the learner's bootstrap value (double-Q or max, VDN: summed over agents, QMIX: the target mixer's Q_tot) -- λ = 0 is the one-step target.
 * Under standardise_returns the statistics absorb G.  enable == 0 restores the one-step target.  λ outside [0, 1] is refused. */
int marl_dqn_set_td_lambda(marl_dqn* q, int32_t enable, float lambda);
/* algorithm.huber_delta of IDQN, VDN and QMIX (this project's option; the reference has only the squared TD error): enable != 0 makes every later
 * update (marl_dqn_update, _update_grads, _update_n) use torch.nn.functional.huber_loss(Q, y, delta = `delta`) per TD error d = Q - y in place of
 * mse_loss: 0.5 d² for |d| < delta, else delta (|d| - 0.5 delta), gradient clamp(d, -delta, delta).  The logged loss is the Huber mean.  For a
 * large delta this is half the squared error and half its gradient.  enable == 0 restores the squared error.  A delta that is not a finite
 * number > 0 is refused. */
int marl_dqn_set_huber_delta(marl_dqn* q, int32_t enable, float delta);
/* QMixNetwork (marlbase/dqn/model.py:272-443, configs/algorithm/qmix.yaml): with hp.mixer == 2, call once after marl_dqn_create.  The mixing
 * network works on state = the agents' observations concatenated (state_dim = n_agents * in_dim); its parameters are one flat vector in the
 * reference's state_dict order (weight, bias each): hypernet_layers == 2: hyper_w_1.0, hyper_w_1.2, hyper_w_final.0, hyper_w_final.2, hyper_b_1,
 * V.0, V.2; hypernet_layers == 1: hyper_w_1, hyper_w_final, hyper_b_1, V.0, V.2 (hypernet_embed is then ignored).  Other values are refused.
 * marl_dqn_qmix_ptrs exposes parameters / target / Adam state / gradient (+ 4 statistics); initialise `mix` through it (nn.Linear defaults are the
 * caller's job), then marl_dqn_sync_target.  marl_dqn_update* then train agents and mixer with the one Adam step of the reference (the gradient
 * clip covers the agents' networks only, dqn/model.py:169-170); target updates (hard / Polyak) include the mixer (433-443). */
int marl_dqn_qmix_init(marl_dqn* q, int32_t embed_dim, int32_t hypernet_layers, int32_t hypernet_embed);
/* Host-only self-check of the two weight-gradient decompositions of the mixer (no device needed; tests/test_qmix.py): counts[0 .. n) and
 * counts[n .. 2n) = how many (micro-)tile entries write each of the n mixer parameters in the single-read form and in the tile form -- 1 everywhere.
 * counts == NULL just returns n. */
int marl_debug_qmix_coverage(int32_t n_agents, int32_t state_dim, int32_t embed_dim, int32_t hypernet_embed, int32_t* counts, int64_t cap,
                             int64_t* n_params);
/* The same self-check for either hypernetwork form (hypernet_layers 1 or 2; anything else is refused).  marl_debug_qmix_coverage is this with 2. */
int marl_debug_qmix_coverage_layers(int32_t n_agents, int32_t state_dim, int32_t embed_dim, int32_t hypernet_layers, int32_t hypernet_embed,
                                    int32_t* counts, int64_t cap, int64_t* n_params);
/* The tail every learner's update ends in (tests/test_optimizer_tail_gpu.py): the reduction of the per-CTA gradient partials, the clip, the optimiser
 * step and the target update, alone, through the launchers the learners use.
 * marl_debug_tail_shape: the fused tail's block shape for n parameters on `device` -- MARL_OK and pb (parameters per block), ns (CTA slices),
 * capacity (SMs x blocks per SM); MARL_EINVAL (capacity still written) when the learners would take the two-kernel tail. */
int marl_debug_tail_shape(int32_t n, int32_t opt_kind, int32_t device, int32_t* pb, int32_t* ns, int32_t* capacity);
typedef struct {
  int32_t n_nets, P, scratch_pitch, cta_begin[MARL_MAX_AGENTS + 1];   /* CTAs [cta_begin[k], cta_begin[k+1]) hold network k's partials */
  const float* scratch;   /* device [cta_begin[n_nets]][scratch_pitch] per-CTA partial gradient sums */
  const float* loss_part; /* device [n_loss_parts][4] per-CTA loss statistics */
  int32_t n_loss_parts, stats_accumulate;   /* stats_accumulate: add the statistics to grad[n .. n+4) instead of overwriting them */
  float* grad;            /* device [n_nets*P + 4], 16-byte aligned: the reduced gradient and the 4 statistics */
  float* sumsq;           /* device [ceil(n_nets*P / 64) + 1] per-block sums of squares */
  float *theta, *theta_tgt, *m, *v;   /* device [n_nets*P]; theta_tgt[0 .. tgt_n) mirrors theta[tgt_begin ..) */
  int32_t tgt_begin, tgt_n, target_mode; float tau;   /* target_mode 0 none, 1 hard copy, 2 Polyak with tau */
  float lr, grad_clip; int64_t step;   /* grad_clip <= 0: off; step = 1, 2, ... (bias corrections) */
  float* loss_out;        /* device [6] as marl_dqn_update's, or NULL */
} marl_debug_tail;
/* path 0: reduce_adam_kernel<0> with a fresh barrier counter (MARL_EINVAL without launching when no co-resident shape exists);
 *      1: grad_reduce_kernel + adam_kernel with the per-block sums of squares (the DQN family's fallback);
 *      2: the same without them (actor-critic learners, marl_dqn_update_apply, the QMIX mixer's step) */
int marl_debug_tail_run(const marl_debug_tail* t, const marl_optimizer* opt, int32_t path, int32_t device, void* stream);
int marl_dqn_qmix_ptrs(marl_dqn* q, float** mix, float** mix_tgt, float** adam_m, float** adam_v, float** grad, int64_t* n_params);
int marl_dqn_param_ptrs(marl_dqn* q, float** theta, float** theta_tgt, float** adam_m, float** adam_v, float** grad,
                        int64_t* n_params);
int marl_dqn_sync_target(marl_dqn* q, void* stream);        /* hard_update (dqn/model.py:195-196) */
/* MUST be called after writing through the pointers of marl_dqn_param_ptrs and before the next forward / update: cached derived
 * data (the packed tensor-core images of the online and target networks) is rebuilt on next use */
int marl_dqn_params_changed(marl_dqn* q);
/* model.act's network pass (dqn/model.py:96-99) for E envs at once: obs device float[E][N][in] -> q float[E][N][out] */
int marl_dqn_forward(marl_dqn* q, const float* obs, int32_t n_envs, int32_t use_target, float* q_out, void* stream);
/* np.random.randint(0, len(rb), batch) (dqn/train.py:95) from the Philox stream (seed, update_idx) */
int marl_replay_sample(uint64_t seed, uint64_t update_idx, int32_t batch, int32_t n_valid, int32_t* idx_out,
                       void* stream);
/* QNetwork.update (dqn/model.py:165-174) split at the point where data-parallel ranks exchange:
 *   _grads: rb.sample gather + _compute_loss + backward  -> un-normalised gradient sums in `grad`
 *   (caller may all-reduce grad[0 .. n_params+4) over ranks here)
 *   _apply: / filled.sum(), clip_grad_norm_, Adam.step, updates += 1, update_target; loss_out device float[6]
 *           = (loss, gradient norm before clipping, 0, 0, filled count, 0) or NULL */
int marl_dqn_update_grads(marl_dqn* q, const marl_traj_view* traj, const int32_t* episode_idx, int32_t batch,
                          void* stream);
int marl_dqn_update_apply(marl_dqn* q, float* loss_out, void* stream);
int marl_dqn_update(marl_dqn* q, const marl_traj_view* traj, const int32_t* episode_idx, int32_t batch,
                    float* loss_out, void* stream);
/* `rb.sample(); model.update()` (dqn/train.py:308-311) n_updates times without returning to Python */
int marl_dqn_update_n(marl_dqn* q, const marl_traj_view* traj, int32_t batch, int32_t n_valid, uint64_t seed,
                      uint64_t first_update_idx, int32_t n_updates, float* loss_out, void* stream);
int marl_dqn_counters(marl_dqn* q, int64_t* updates, int64_t* last_target_update);
/* Choose the optimiser (MLP and recurrent handles; QMIX: the mixer takes the same one, unclipped).  Without this call the handle runs Adam with
 * hp.beta1 / beta2 / eps.  Zeroes adam_m / adam_v (and the mixer's); refused (MARL_EINVAL) once the handle has taken an optimiser step. */
int marl_dqn_set_optimizer(marl_dqn* q, const marl_optimizer* opt);
/* Multi-GPU (one process per GPU on one NVLink node; replaces the torch.distributed all-reduce a data-parallel port of
 * dqn/train.py would add between loss.backward() and optimiser.step()): marl_dqn_peer_handle allocates this rank's exchange buffer
 * and writes its 64-byte CUDA IPC handle; the caller gathers all ranks' handles (rank-ordered, 64 bytes each) and passes them to
 * marl_dqn_peer_attach.  Afterwards marl_dqn_update / marl_dqn_update_n sum the gradients of all ranks over peer memory inside the
 * fused reduce + Adam kernel (identical parameters on every rank, no NCCL call); every rank must issue the same update calls.
 * MLP and recurrent handles whose parameters fit one wave of the fused tail (attach refuses the others); QMIX (call marl_dqn_qmix_init before
 * marl_dqn_peer_handle): the exchange slot is [agents' gradient sums | mixer's gradient sums | 4 statistics] and the mixer's step reads the all-rank sum. */
int marl_dqn_peer_handle(marl_dqn* q, void* handle_out64);
int marl_dqn_peer_attach(marl_dqn* q, int32_t rank, int32_t world, const void* handles);
/* *timed_out = 1 when an update's in-kernel exchange gave up waiting for a peer (bounded spin, ~10 s): results since are invalid.
 * The same flag is mirrored in loss_out[5] of every update.  Synchronises the device. */
int marl_dqn_peer_status(marl_dqn* q, int32_t* timed_out);
/* measurement hook (bench.py roofline leg): CUDA-event time of the training-kernel launches between enable=1 and enable=0 */
int marl_dqn_timing(marl_dqn* q, int32_t enable, float* total_ms, int32_t* count);
/* after marl_dqn_timing(q, 0, ..): the same window split over the three kernels of the tensor-core training pass, ms3[0..2] =
 * summed durations of (online forward + TD head, dH1 + dW1, the other weight gradients); *count = 0 if the window ran the fused FP32 kernel */
int marl_dqn_timing_kernels(marl_dqn* q, float* ms3, int32_t* count);
int marl_dqn_set_counters(marl_dqn* q, int64_t updates, int64_t last_target_update);

/* Recurrent agent networks (algorithm.model.use_rnn=True; marlbase/utils/models.py:51-130, RNNNetwork with layers = [H, H], H = cfg.hidden):
 * first_layer Linear(in, H) + ReLU, nn.GRU(H, H, num_layers=1) (gate order r, z, n), final_layer Linear(H, out), no activation
 * between the GRU and final_layer.  marl_dqn_create_rnn returns the same handle type; marl_dqn_param_ptrs then exposes [n_nets][P] floats,
 * per network in the reference's state_dict order: first_layer.weight [H][in], first_layer.bias [H], rnn.weight_ih_l0 [3H][H],
 * rnn.weight_hh_l0 [3H][H], rnn.bias_ih_l0 [3H], rnn.bias_hh_l0 [3H], final_layer.weight [out][H], final_layer.bias [out].
 * Training runs every sampled episode from a zero hidden state (dqn/model.py:127,133).  marl_dqn_update / _update_n / _update_grads +
 * _update_apply, standardise_returns, qmix_init, sync_target, the counters and marl_dqn_timing work unchanged (the timed window covers the
 * online sequence forward, the TD head and the backward; marl_dqn_timing_kernels reports count 0).  The "tensor_core_*" options do not apply
 * to recurrent handles (FP32 FFMA throughout); marl_dqn_forward refuses them; in_dim <= 32. */
int marl_dqn_create_rnn(const marl_mlp_cfg* cfg, const marl_dqn_hp* hp, int32_t max_batch, int32_t max_T, int32_t device,
                        marl_dqn** out);
/* One step of model.act's network pass (dqn/model.py:96-99) for E envs: obs device float[E][N][in], h_in / h_out device float[E][N][H]
 * (h_in == NULL: the zero state of init_hiddens; h_out == NULL: not written) -> q_out float[E][N][out].  h_in and h_out must not alias. */
int marl_dqn_forward_rnn(marl_dqn* q, const float* obs, int32_t n_envs, int32_t use_target, const float* h_in, float* h_out,
                         float* q_out, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Independent actor-critic learner (IA2C).  Replaces marlbase/ac/model.py A2CNetwork (22-246) with a
 * decentralised critic (ia2c.yaml:18), independent or shared per-agent networks.
 * theta = [actor nets | critic nets] flat, theta_tgt = target critic; per-net order as for marl_dqn.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
  float   lr;                             /* ia2c.yaml:29 */
  float   gamma;                          /* ia2c.yaml:34 */
  float   grad_clip;                      /* ia2c.yaml:31 (False -> 0) */
  int32_t n_steps;                        /* ia2c.yaml:33 */
  float   entropy_coef;                   /* ia2c.yaml:35 */
  float   value_loss_coef;                /* ia2c.yaml:36 */
  float   target_update_interval_or_tau;  /* ia2c.yaml:40; compared against the ENVIRONMENT step (ac/model.py:233-237) */
  float   beta1, beta2, eps;              /* Adam defaults */
} marl_a2c_hp;

typedef struct marl_a2c marl_a2c;

/* actor->in_dim and critic->in_dim: 1..128 (inputs wider than 32 always run the FP32 kernels, whatever "tensor_core_forward" says) */
int marl_a2c_create(const marl_mlp_cfg* actor, const marl_mlp_cfg* critic, const marl_a2c_hp* hp, int32_t max_envs,
                    int32_t max_T, int32_t device, marl_a2c** out);
int marl_a2c_destroy(marl_a2c* a);
int marl_a2c_param_ptrs(marl_a2c* a, float** theta, float** theta_tgt, float** adam_m, float** adam_v, float** grad,
                        int64_t* n_actor, int64_t* n_critic);
/* device scratch of the last update (parity tests): target values [N][P][T+1], n-step returns [N][P][T], advantages [N][P][T] */
int marl_a2c_scratch_ptrs(marl_a2c* a, float** target_values, float** returns, float** advantages);
int marl_a2c_sync_target(marl_a2c* a, void* stream);      /* soft_update(1.0) (ac/model.py:101,184-187) */
/* actor pass of A2CNetwork.act (ac/model.py:148-150): obs float[E][N][in] -> logits float[E][N][n_actions]; sampling
 * happens in marl_lbf_rollout_step(policy = 2) */
int marl_a2c_forward_actor(marl_a2c* a, const float* obs, int32_t n_envs, float* logits_out, void* stream);
int marl_a2c_forward_critic(marl_a2c* a, const float* obs, int32_t n_envs, int32_t use_target, float* values_out,
                            void* stream);
/* A2CNetwork.update (ac/model.py:189-246) on the on-policy batch held in a trajectory store of capacity >= n_envs
 * (slot e = env e), split where data-parallel ranks exchange grad[0 .. n_actor+n_critic+4):
 *   _grads: target-critic pass, n-step returns, critic + actor forward/loss/backward -> gradient sums + statistics
 *   _apply: / filled.sum(), optional clip, Adam over actor+critic, target sync when step % interval == 0;
 *           metrics_out device float[6] = (policy-gradient term, gradient norm, entropy, value_loss, filled count, 0) */
int marl_a2c_update_grads(marl_a2c* a, const marl_traj_view* batch, int32_t n_envs, void* stream);
int marl_a2c_update_apply(marl_a2c* a, int64_t step, float* metrics_out, void* stream);
int marl_a2c_update(marl_a2c* a, const marl_traj_view* batch, int32_t n_envs, int64_t step, float* metrics_out,
                    void* stream);
/* Choose the optimiser of actor and critic (one optimiser over both, as the reference's; MLP and recurrent handles).  Without this call the handle
 * runs Adam with hp.beta1 / beta2 / eps.  Zeroes adam_m / adam_v; refused (MARL_EINVAL) once the handle has taken an optimiser step. */
int marl_a2c_set_optimizer(marl_a2c* a, const marl_optimizer* opt);
/* cfg.standardise_returns of the actor-critic learners (marlbase/ac/model.py:112-114,195-204,272-281; utils/standardise_stream.py:6-43): a
 * RunningMeanStd(shape=(n_agents,)) over the n-step returns of every update -- the bootstrap values are de-standardised with the statistics so far,
 * the statistics absorb the batch's returns (all T x P of them, unmasked), the returns are standardised.  enable != 0 initialises them on first use. */
int marl_a2c_standardise_returns(marl_a2c* a, int32_t enable);
int marl_a2c_ret_ms_ptrs(marl_a2c* a, float** ret_ms /* mean[N] | var[N] */, double** count);
/* algorithm.gae_lambda (IA2C, IPPO, MAA2C, MAPPO): enable != 0 makes every later update (marl_a2c_update*, marl_ppo_update / _prepare) use the
 * λ-returns R_t = (1 - λ) Σ_{n>=1} λ^(n-1) G_t^(n) over the n-step returns G^(n) of compute_nstep_returns (the same masks, the same target-critic
 * values, de-standardised under standardise_returns) in place of the n_steps-step return; hp.n_steps is not read meanwhile.  λ = 0 is the one-step
 * return, λ = 1 the return to the end of the stored episode.  enable == 0 restores the n-step returns.  A λ outside [0, 1] is refused (MARL_EINVAL). */
int marl_a2c_set_gae_lambda(marl_a2c* a, int32_t enable, float lambda);
/* PPONetwork.update (marlbase/ac/model.py:265-352; configs/algorithm/ippo.yaml: num_epochs 4, ppo_clip 0.2, grad_clip 0.5) on an A2C handle:
 * n-step returns and the collecting policy's log-probabilities once, then num_epochs optimisation steps on the same batch with the clipped
 * surrogate; the target critic follows after the last epoch.  metrics_out: device float[6] as marl_a2c_update, averaged over the epochs. */
int marl_ppo_update(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, int64_t step, int32_t num_epochs, float ppo_clip,
                    float* metrics_out, void* stream);
/* marl_ppo_update split where data-parallel ranks exchange grad[0 .. n_actor+n_critic+4) once per epoch.  marl_ppo_update is exactly
 * marl_ppo_prepare followed by num_epochs x (marl_ppo_epoch_grads + marl_ppo_epoch_apply), so with nothing in between the results are the same bits.
 *   _prepare:     target-critic pass, n-step returns and the collecting policy's log-probabilities of the batch (kept until the next prepare;
 *                 the batch must not change before the last epoch)
 *   _epoch_grads: one epoch's critic + actor passes with the clipped surrogate -> gradient sums + statistics in grad
 *   _epoch_apply: / filled.sum(), optional clip, optimiser step (epoch = 0 .. num_epochs-1); the last epoch also updates the target critic for
 *                 `step` and writes the epochs' mean metrics to metrics_out (device float[6] as marl_ppo_update) */
int marl_ppo_prepare(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, void* stream);
int marl_ppo_epoch_grads(marl_a2c* h, float ppo_clip, void* stream);
int marl_ppo_epoch_apply(marl_a2c* h, int64_t step, int32_t epoch, int32_t num_epochs, float* metrics_out, void* stream);
/* Recurrent actor and / or critic (actor.use_rnn / critic.use_rnn; marlbase/utils/models.py:51-116 RNNNetwork with layers = [H, H], the
 * network and per-network parameter order of marl_dqn_create_rnn).  actor_rnn / critic_rnn != 0 make that part a GRU network; the other part stays
 * the MLP.  marl_a2c_param_ptrs then exposes [actor nets | critic nets], each part in its own layout.  Every update pass runs each env's episode
 * from the zero state (ac/model.py:189-246,265-352: hiddens=None): the target critic over all T+1 observations, the critic and the actor over the
 * first T.  marl_a2c_update, _update_grads + _update_apply, marl_ppo_update, standardise_returns, sync_target and scratch_ptrs work unchanged.
 * The "tensor_core_*" options do not apply to recurrent parts (FP32 FFMA); marl_a2c_forward_actor / _forward_critic refuse a recurrent part. */
int marl_a2c_create_rnn(const marl_mlp_cfg* actor, const marl_mlp_cfg* critic, const marl_a2c_hp* hp, int32_t actor_rnn, int32_t critic_rnn,
                        int32_t max_envs, int32_t max_T, int32_t device, marl_a2c** out);
/* One step of a recurrent part for E envs, carrying the hidden state (act, ac/model.py:147-153; get_value, 155-163).  which: 0 actor, 1 critic,
 * 2 target critic.  obs device float[E][N][in] (a centralised critic reads each env's N x in values), h_in / h_out device float[E][N][H]
 * (H: that part's hidden width)
 * (h_in == NULL: the zero state of init_*_hiddens; h_out == NULL: not written) -> out float[E][N][n_actions] (actor) or float[E][N][1].
 * h_in and h_out must not alias; a part that is not recurrent is refused. */
int marl_a2c_forward_rnn(marl_a2c* h, int32_t which, const float* obs, int32_t n_envs, const float* h_in, float* h_out, float* out,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MARL_B200_H */
