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
 * "tensor_core_backward" 1 = the DQN-family training pass runs as the three-kernel wgmma pipeline (tc_train.cu), 0 = fused FP32 kernel;
 * "split_exchange" (several ranks) 1 = gradient exchange split around the next update's target forward. */
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
} marl_lbf_cfg;

typedef struct marl_lbf marl_lbf;

/* Device-resident state, exposed for parity tests and checkpointing (all device pointers). */
typedef struct {
  int8_t*   field;        /* [E][field_pitch], row-major rows*cols cells then zero padding            */
  int8_t*   players;      /* [E][N][4] = (row, col, level, 0)                                        */
  int32_t*  step;         /* [E] current_step == TimeLimit's elapsed steps                           */
  int32_t*  food_spawned; /* [E] sum of food levels at reset (reward normaliser)                      */
  float*    ep_return;    /* [E][N] float32 running episode return (wrappers.py:33)                  */
  int32_t*  ep_len;       /* [E]                                                                     */
  uint32_t* episode_idx;  /* [E] resets performed so far                                             */
  uint8_t*  active;       /* [E] 0 after the episode ended when autoreset is off                     */
  int32_t   field_pitch;  /* bytes per env in `field` (rows*cols rounded up to 16)                    */
  int32_t   n_envs;
} marl_lbf_state;

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
int marl_lbf_obs_dim(const marl_lbf_cfg* cfg);             /* 3*max_num_food + 3*n_agents (+ n_agents with observe_id) */
int marl_lbf_state_ptrs(marl_lbf* env, marl_lbf_state* out);
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
  int32_t in_dim;                     /* flatdim(observation_space[i]) */
  int32_t hidden;                     /* layers = [hidden, hidden]; 128 (idqn.yaml:8-10) */
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

int marl_dqn_create(const marl_mlp_cfg* cfg, const marl_dqn_hp* hp, int32_t max_batch, int32_t max_T, int32_t device,
                    marl_dqn** out);
int marl_dqn_destroy(marl_dqn* q);
/* Device pointers to the flat parameter / optimiser state ([n_nets*P] floats each; grad has 4 extra floats:
 * loss numerator, filled count, 2 spare).  Initialise theta through these (orthogonal init is done by the caller). */
/* cfg.standardise_returns of the DQN family (marlbase/dqn/model.py:82-84,147-158; VDN 221-222,256-264; utils/standardise_stream.py): a
 * RunningMeanStd over the TD targets of every update -- target Q-values are de-standardised with the statistics so far, the statistics absorb the
 * batch's returns, the returns are standardised before the loss.  One column per agent; VDN: one per batch entry (the reference's reshape). */
int marl_dqn_standardise_returns(marl_dqn* q, int32_t enable);
int marl_dqn_ret_ms_ptrs(marl_dqn* q, float** ret_ms /* mean[n] | var[n] */, double** count, int32_t* n_stat);
/* QMixNetwork (marlbase/dqn/model.py:272-443, configs/algorithm/qmix.yaml): with hp.mixer == 2, call once after marl_dqn_create.  The mixing
 * network (hypernet_layers == 2) works on state = the agents' observations concatenated (state_dim = n_agents * in_dim); its parameters are one flat
 * vector in the reference's state_dict order: hyper_w_1.0, hyper_w_1.2, hyper_w_final.0, hyper_w_final.2, hyper_b_1, V.0, V.2 (weight, bias each).
 * marl_dqn_qmix_ptrs exposes parameters / target / Adam state / gradient (+ 4 statistics); initialise `mix` through it (nn.Linear defaults are the
 * caller's job), then marl_dqn_sync_target.  marl_dqn_update* then train agents and mixer with the one Adam step of the reference (the gradient
 * clip covers the agents' networks only, dqn/model.py:169-170); target updates (hard / Polyak) include the mixer (433-443). */
int marl_dqn_qmix_init(marl_dqn* q, int32_t embed_dim, int32_t hypernet_layers, int32_t hypernet_embed);
/* Host-only self-check of the two weight-gradient decompositions of the mixer (no device needed; tests/test_qmix.py): counts[0 .. n) and
 * counts[n .. 2n) = how many (micro-)tile entries write each of the n mixer parameters in the single-read form and in the tile form -- 1 everywhere.
 * counts == NULL just returns n. */
int marl_debug_qmix_coverage(int32_t n_agents, int32_t state_dim, int32_t embed_dim, int32_t hypernet_embed, int32_t* counts, int64_t cap,
                             int64_t* n_params);
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
/* Multi-GPU (one process per GPU on one NVLink node; replaces the torch.distributed all-reduce a data-parallel port of
 * dqn/train.py would add between loss.backward() and optimiser.step()): marl_dqn_peer_handle allocates this rank's exchange buffer
 * and writes its 64-byte CUDA IPC handle; the caller gathers all ranks' handles (rank-ordered, 64 bytes each) and passes them to
 * marl_dqn_peer_attach.  Afterwards marl_dqn_update / marl_dqn_update_n sum the gradients of all ranks over peer memory inside the
 * fused reduce + Adam kernel (identical parameters on every rank, no NCCL call); every rank must issue the same update calls. */
int marl_dqn_peer_handle(marl_dqn* q, void* handle_out64);
int marl_dqn_peer_attach(marl_dqn* q, int32_t rank, int32_t world, const void* handles);
/* *timed_out = 1 when an update's in-kernel exchange gave up waiting for a peer (bounded spin, ~10 s): results since are invalid.
 * The same flag is mirrored in loss_out[5] of every update.  Synchronises the device. */
int marl_dqn_peer_status(marl_dqn* q, int32_t* timed_out);
/* measurement hook (bench.py roofline leg): CUDA-event time of the training-kernel launches between enable=1 and enable=0 */
int marl_dqn_timing(marl_dqn* q, int32_t enable, float* total_ms, int32_t* count);
/* after marl_dqn_timing(q, 0, ..): the same window split over the three kernels of the tensor-core training pass, ms3[0..2] =
 * summed durations of (online forward + TD head, dH1, weight gradients); *count = 0 if the window ran the fused FP32 kernel */
int marl_dqn_timing_kernels(marl_dqn* q, float* ms3, int32_t* count);
int marl_dqn_set_counters(marl_dqn* q, int64_t updates, int64_t last_target_update);

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
/* cfg.standardise_returns of the actor-critic learners (marlbase/ac/model.py:112-114,195-204,272-281; utils/standardise_stream.py:6-43): a
 * RunningMeanStd(shape=(n_agents,)) over the n-step returns of every update -- the bootstrap values are de-standardised with the statistics so far,
 * the statistics absorb the batch's returns (all T x P of them, unmasked), the returns are standardised.  enable != 0 initialises them on first use. */
int marl_a2c_standardise_returns(marl_a2c* a, int32_t enable);
int marl_a2c_ret_ms_ptrs(marl_a2c* a, float** ret_ms /* mean[N] | var[N] */, double** count);
/* PPONetwork.update (marlbase/ac/model.py:265-352; configs/algorithm/ippo.yaml: num_epochs 4, ppo_clip 0.2, grad_clip 0.5) on an A2C handle:
 * n-step returns and the collecting policy's log-probabilities once, then num_epochs optimisation steps on the same batch with the clipped
 * surrogate; the target critic follows after the last epoch.  metrics_out: device float[6] as marl_a2c_update, averaged over the epochs. */
int marl_ppo_update(marl_a2c* h, const marl_traj_view* batch, int32_t n_envs, int64_t step, int32_t num_epochs, float ppo_clip,
                    float* metrics_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MARL_B200_H */
