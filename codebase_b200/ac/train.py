"""IA2C training driver on the GPU path -- drop-in for marlbase/ac/train.py `main(envs, eval_env, logger, time_limit,
**cfg)` (`algorithm._target_: ac.train.main`, configs/algorithm/ia2c.yaml:6).

Loop structure of the reference (ac/train.py:170-204) with every stage on the device:

    reference                                                   here
    ------------------------------------------------------      --------------------------------------------------------------
    _collect_trajectories: AsyncVectorEnv (10 processes),        env.reset(batch); T x [marl_a2c_forward_actor + marl_lbf_rollout_step
      model.act -> envs.step -> masked writes with `running`       (policy 2, frozen after each env's first episode end == `running`)]
    model.update(batch, step)                                    marl_a2c_update (target critic, n-step returns, critic + actor passes, Adam)
    if step - last_eval >= eval_interval: log TRAINING infos     same (AC never runs eval_env, ac/train.py:184-186)
    updates += 1; step += t * parallel_envs                      same, t = longest episode of the batch
"""
from __future__ import annotations

import time
from pathlib import Path

import torch

from .. import distributed
from ..config import Config, instantiate
from ..native_env import TrajStore
from ..utils import video
from ..utils.envs import episode_info


class Collector:
    """_collect_trajectories (ac/train.py:24-119) for all envs at once; the on-policy Batch lives in a TrajStore of capacity P."""

    def __init__(self, envs, model, time_limit, use_proper_termination=False):
        self.env, self.model, self.T, self.proper = envs.native, model, int(time_limit), bool(use_proper_termination)
        self.batch = TrajStore(self.env.E, self.env.N, self.T, self.env.D, self.env.device)
        self.logits = torch.empty(self.env.E, self.env.N, model.n_actions, dtype=torch.float32, device=self.env.device)
        # recurrent actor: two [E][N][H] hidden-state buffers used in turn (step input, step output)
        self.rnn = bool(getattr(model, "actor_rnn", False))
        if self.rnn:
            self.h = [torch.zeros(self.env.E, self.env.N, model.actor_hidden, dtype=torch.float32, device=self.env.device) for _ in range(2)]

    def collect(self):
        env, b = self.env, self.batch
        # fresh, all-zero batch_* tensors on every call (ac/train.py:36-52): compute_nstep_returns never looks at `filled`, so rows after an
        # early episode end must read as reward 0 / zero observation, not as the previous batch's longer episode in the same slot
        b.obs.zero_(); b.act.zero_(); b.rew.zero_(); b.filled.zero_(); b.done.zero_()
        env.reset(traj=b, slot0=0)
        if self.rnn:   # every env starts its episode here: init_actor_hiddens at the start of each collection (ac/train.py:69-77)
            self.h[0].zero_()
        for t in range(self.T):
            if self.rnn:
                self.model.logits(env.obs, out=self.logits, h=self.h[t & 1], h_out=self.h[(t + 1) & 1])
            else:
                self.model.logits(env.obs, out=self.logits)
            env.rollout_step(self.logits, policy=2, traj=b, slot0=0, use_proper_termination=self.proper)
        return env.final_len, env.final_ret


def iteration_env_steps(t, P, dp) -> int:
    """Env steps of one iteration on all ranks, as the reference counts them (ac/train.py:201): longest episode t of each rank's batch x P."""
    return dp.sum_int(int(t) * int(P))


def record_episodes(env, model, n_timesteps, path):
    """marlbase/ac/train.py:122-150 on a one-env B200VecEnv: `n_timesteps` frames of episodes sampled from the policy to the mp4 file `path`
    (utils.video.record_policy); an episode ends on done or truncated."""
    return video.record_policy(env, n_timesteps, path, model.logits, 2, 0.0, model.actor_hidden if model.actor_rnn else 0)


def main(envs, eval_env, logger, time_limit, **cfg):
    cfg = Config(cfg)
    P = envs.num_envs
    dp = distributed.current()
    video_env = None
    if cfg.video_interval and eval_env is not None:   # rank 0 records
        video.require_encoder()
        video_env = video.recording_env(eval_env)
    from ..dqn.train import check_iteration_budget

    check_iteration_budget(P * dp.world, time_limit, cfg.total_steps, cfg.eval_interval)
    model = instantiate(cfg.model, envs.single_observation_space, envs.single_action_space, cfg, max_envs=P, max_episode_length=time_limit)
    dp.sync_learner(model)
    logger.watch(model)
    collector = Collector(envs, model, time_limit, cfg.use_proper_termination)
    step = updates = last_eval = last_save = last_video = 0
    while step < cfg.total_steps + 1:
        t0 = time.perf_counter()
        final_len, final_ret = collector.collect()
        if dp.active:   # `step` is global: the target critic's `step % interval == 0` sync fires on every rank at once
            metrics = model.update_allreduce(collector.batch, P, step, dp.all_reduce_)
        else:
            metrics = model.update_from_store(collector.batch, P, step)
        t = int(final_len.max().item())
        if (step - last_eval) >= cfg.eval_interval:
            ln, ret = final_len.cpu().numpy(), final_ret.cpu().numpy()
            per_episode = (time.perf_counter() - t0) / P
            infos = []
            for ln_r, ret_r, per_r in dp.gather_objects((ln, ret, per_episode)):   # the training episodes of every rank
                infos += [episode_info(ret_r[i], ln_r[i], per_r) for i in range(len(ln_r))]
            infos.append(model.metrics_dict(metrics))
            infos.append({"updates": updates, "environment_steps": step})
            logger.log_metrics(infos)
            last_eval = step
        if cfg.save_interval and (step - last_save) >= cfg.save_interval and dp.is_main:
            Path("checkpoints").mkdir(exist_ok=True)
            torch.save(model.state_dict(), f"checkpoints/model_s{step}.pt")
            last_save = step
        if video_env is not None and (step - last_video) >= cfg.video_interval:
            record_episodes(video_env, model, cfg.video_frames, f"./videos/step-{step}.mp4")
            last_video = step
        updates += 1
        step += iteration_env_steps(t, P, dp)
    envs.close()
    if video_env is not None:
        video_env.close()
    return dict(environment_steps=step, updates=updates)
