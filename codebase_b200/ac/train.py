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

from ..config import Config, instantiate
from ..lbf import TrajStore
from ..utils.envs import episode_info


class Collector:
    """_collect_trajectories (ac/train.py:24-119) for all envs at once; the on-policy Batch lives in a TrajStore of capacity P."""

    def __init__(self, envs, model, time_limit, use_proper_termination=False):
        self.env, self.model, self.T, self.proper = envs.native, model, int(time_limit), bool(use_proper_termination)
        self.batch = TrajStore(self.env.E, self.env.N, self.T, self.env.D, self.env.device)
        self.logits = torch.empty(self.env.E, self.env.N, model.n_actions, dtype=torch.float32, device=self.env.device)

    def collect(self):
        env, b = self.env, self.batch
        # fresh, all-zero batch_* tensors on every call (ac/train.py:36-52): compute_nstep_returns never looks at `filled`, so rows after an
        # early episode end must read as reward 0 / zero observation, not as the previous batch's longer episode in the same slot
        b.obs.zero_(); b.act.zero_(); b.rew.zero_(); b.filled.zero_(); b.done.zero_()
        env.reset(traj=b, slot0=0)
        for _ in range(self.T):
            self.model.logits(env.obs, out=self.logits)
            env.rollout_step(self.logits, policy=2, traj=b, slot0=0, use_proper_termination=self.proper)
        return env.final_len, env.final_ret


def main(envs, eval_env, logger, time_limit, **cfg):
    cfg = Config(cfg)
    P = envs.num_envs
    from ..dqn.train import check_iteration_budget

    check_iteration_budget(P, time_limit, cfg.total_steps, cfg.eval_interval)
    model = instantiate(cfg.model, envs.single_observation_space, envs.single_action_space, cfg, max_envs=P, max_episode_length=time_limit)
    logger.watch(model)
    collector = Collector(envs, model, time_limit, cfg.use_proper_termination)
    step = updates = last_eval = last_save = 0
    while step < cfg.total_steps + 1:
        t0 = time.perf_counter()
        final_len, final_ret = collector.collect()
        metrics = model.update_from_store(collector.batch, P, step)
        t = int(final_len.max().item())
        if (step - last_eval) >= cfg.eval_interval:
            ln, ret = final_len.cpu().numpy(), final_ret.cpu().numpy()
            per_episode = (time.perf_counter() - t0) / P
            infos = [episode_info(ret[i], ln[i], per_episode) for i in range(P)]
            infos.append(model.metrics_dict(metrics))
            infos.append({"updates": updates, "environment_steps": step})
            logger.log_metrics(infos)
            last_eval = step
        if cfg.save_interval and (step - last_save) >= cfg.save_interval:
            Path("checkpoints").mkdir(exist_ok=True)
            torch.save(model.state_dict(), f"checkpoints/model_s{step}.pt")
            last_save = step
        if cfg.video_interval:
            raise NotImplementedError("algorithm.video_interval: video recording is out of scope of the GPU hot path")
        updates += 1
        step += t * P
    envs.close()
    return dict(environment_steps=step, updates=updates)
