"""IDQN / VDN training driver on the GPU path -- drop-in for marlbase/dqn/train.py `main(env, eval_env, logger,
time_limit, **cfg)` (`algorithm._target_: dqn.train.main`, configs/algorithm/idqn.yaml:4).

Same loop structure as the reference (dqn/train.py:298-343), vectorised over E = env.parallel_envs instances:

    reference (1 env)                                   here (E envs, all on device)
    -----------------------------------------------     ---------------------------------------------------------------
    _collect_trajectory: reset; act/step/rb.add  x<=T   env.reset(ring); T x [marl_dqn_forward + marl_lbf_rollout_step]
    step += t                                           step += sum of the E episode lengths
    if step > training_start and rb.can_sample(B):      same condition
        rb.sample(B); model.update(batch)                   marl_dqn_update_n: `updates_per_iteration` x (sample + update);
                                                            default E, i.e. the reference's one update per collected episode
    every eval_interval: 100 eval episodes (eps 0.05)   one batch of `eval_episodes` envs through the same fused kernels
    logger.log_metrics(infos)                           identical list-of-dicts -> identical results.csv columns

Exploration / replay sampling draw from Philox streams keyed by `seed` (the reference's Python `random` stream is not
seeded by run.py and cannot be reproduced -- SURVEY F6).
"""
from __future__ import annotations

import logging
import time
from pathlib import Path

import torch

from .. import _native as nat
from .. import distributed
from ..config import Config, instantiate
from ..native_env import TrajStore
from ..utils import video
from ..utils.envs import episode_info


def epsilon_schedule(decay_style, decay_over, eps_start, eps_end, exp_decay_rate, total_steps):
    """marlbase/dqn/train.py:127-174 (same validation, same arithmetic in Python floats)."""
    import math

    assert decay_style in ["linear", "lin", "exponential", "exp"], "decay_style must be one of 'linear' or 'exponential'"
    assert 0 <= eps_start <= 1 and 0 <= eps_end <= 1, "eps must be in [0, 1]"
    assert eps_start >= eps_end, "eps_start must be >= eps_end"
    assert 0 < decay_over <= 1, "decay_over must be in (0, 1]"
    assert total_steps > 0, "total_steps must be > 0"
    assert exp_decay_rate > 0, "eps_decay must be > 0"
    if decay_style in ["linear", "lin"]:
        return lambda steps_done: max(eps_end + (eps_start - eps_end) * (1 - steps_done / (total_steps * decay_over)), eps_end)
    eps_decay = (eps_start - eps_end) / (total_steps * decay_over) * exp_decay_rate
    return lambda steps_done: max(eps_end + (eps_start - eps_end) * math.exp(-eps_decay * steps_done), eps_end)


def check_iteration_budget(parallel_envs, time_limit, total_steps, eval_interval, eps_decay_over=1.0):
    """The reference's schedules are written for ONE env (a 25-step episode per iteration).  One vectorised iteration here is up to
    parallel_envs * time_limit env steps, and epsilon / evaluation / the loop condition are only looked at between iterations: warn when a
    configuration makes them degenerate (e.g. parallel_envs=4096 with the reference's total_steps=100_000 would be ONE iteration at eps=1)."""
    import warnings

    per_iter = int(parallel_envs) * int(time_limit)
    need = 20 * per_iter
    problems = []
    if total_steps * eps_decay_over < need:
        problems.append(f"fewer than 20 iterations inside the epsilon decay (total_steps * eps_decay_over = {int(total_steps * eps_decay_over)})")
    if eval_interval and eval_interval < per_iter:
        problems.append(f"eval_interval={eval_interval} is shorter than one iteration")
    if problems:
        warnings.warn(f"env.parallel_envs={parallel_envs} x time_limit={time_limit} = {per_iter} env steps per iteration: " + "; ".join(problems) +
                      f" -- raise algorithm.total_steps to >= {int(need / max(eps_decay_over, 1e-9))} (and the intervals with it) or lower env.parallel_envs", UserWarning, stacklevel=2)


class Collector:
    """_collect_trajectory (dqn/train.py:202-237) for every env of a B200VecEnv at once, episode-synchronous: all envs reset,
    step until each one's episode ended (at most `time_limit` steps, finished envs freeze), trajectories land in the ring."""

    def __init__(self, env, model, time_limit, use_proper_termination=False, clear_stale=False):
        self.env, self.model, self.T = env.native, model, int(time_limit)
        self.proper, self.clear_stale = bool(use_proper_termination), bool(clear_stale)
        self.q = torch.empty(self.env.E, self.env.N, model.n_actions, dtype=torch.float32, device=self.env.device)
        # recurrent networks: two [E][N][H] hidden-state buffers used in turn (step input, step output)
        self.rnn = bool(getattr(model, "use_rnn", False))
        if self.rnn:
            self.h = [torch.zeros(self.env.E, self.env.N, model.hidden, dtype=torch.float32, device=self.env.device) for _ in range(2)]

    def collect(self, rb: TrajStore | None, slot0: int, epsilon: float):
        env = self.env
        env.reset(traj=rb, slot0=slot0)
        if self.rnn:   # every env starts a new episode here: the reference's init_hiddens at each episode start (dqn/train.py:210)
            self.h[0].zero_()
        for t in range(self.T):
            if self.rnn:
                self.model.q_values(env.obs, out=self.q, h=self.h[t & 1], h_out=self.h[(t + 1) & 1])
            else:
                self.model.q_values(env.obs, out=self.q)
            env.rollout_step(self.q, policy=1, epsilon=epsilon, traj=rb, slot0=slot0, use_proper_termination=self.proper, clear_stale=self.clear_stale)
        return env.final_len, env.final_ret  # device tensors: every env finished exactly one episode


def _episode_infos(final_len, final_ret, seconds):
    ln, ret = final_len.cpu().numpy(), final_ret.cpu().numpy()
    per_episode = seconds / max(len(ln), 1)
    return [episode_info(ret[i], ln[i], per_episode) for i in range(len(ln))]


def iteration_env_steps(final_len, dp) -> int:
    """Env steps of one iteration on all ranks: the sum of every collected episode's length.  Then step, epsilon, training_start, the intervals
    and the loop condition agree on every rank; this host collective also keeps a rank out of an in-kernel exchange while rank 0 evaluates or saves."""
    return dp.sum_int(final_len.sum().item())


def attach_peer_exchange(model, dp) -> bool:
    """Several ranks, each on its own device: sum the gradients inside the fused reduce + Adam kernel over peer memory (IDQN / VDN / QMIX, MLP or
    recurrent, whose parameters fit one wave of the fused tail).  All ranks or none: attach_peers agrees on the outcome on every rank, and a
    refusal anywhere makes every rank use the all-reduce between the two calls.  Never with ranks that share a device: the exchange's bounded
    spin assumes co-resident peers."""
    if not (dp.active and dp.own_device):
        return False
    try:
        model.attach_peers()
    except nat.NativeError as e:  # e.g. no peer access between the devices, or too many parameters for one wave of the fused tail
        logging.warning("%s: one all-reduce per update", e)
        return False
    return True


def record_episodes(env, model, n_timesteps, path, epsilon):
    """marlbase/dqn/train.py:239-261 on a one-env B200VecEnv: `n_timesteps` frames of epsilon-greedy episodes to the mp4 file `path`
    (utils.video.record_policy).  An episode ends on done or truncated; the reference ignores truncation here and would step past its TimeLimit,
    while the step kernel freezes a finished env."""
    return video.record_policy(env, n_timesteps, path, model.q_values, 1, epsilon, model.hidden if model.use_rnn else 0)


def main(env, eval_env, logger, time_limit, **cfg):
    cfg = Config(cfg)
    E = env.num_envs
    dp = distributed.current()
    video_env = None
    if cfg.video_interval and eval_env is not None:   # rank 0 records
        video.require_encoder()
        video_env = video.recording_env(eval_env)
    check_iteration_budget(E * dp.world, time_limit, cfg.total_steps, cfg.eval_interval, cfg.eps_decay_over)
    model = instantiate(cfg.model, env.single_observation_space, env.single_action_space, cfg, max_batch=cfg.batch_size, max_episode_length=time_limit)
    dp.sync_learner(model)
    peer = attach_peer_exchange(model, dp)
    logger.watch(model)
    capacity = int(cfg.buffer_size)
    if capacity < E:
        raise ValueError(f"algorithm.buffer_size ({capacity} episodes) must hold at least one episode per env (env.parallel_envs={E})")
    rb = TrajStore(capacity, env.n_agents, time_limit, env.cfg.obs_dim, env.native.device)
    eps_sched = epsilon_schedule(cfg.eps_decay_style, cfg.eps_decay_over, cfg.eps_start, cfg.eps_end, cfg.eps_exp_decay_rate, cfg.total_steps)
    collector = Collector(env, model, time_limit, cfg.use_proper_termination, cfg.get("replay_clear_stale", False))
    evaluator = Collector(eval_env, model, time_limit) if eval_env is not None else None
    updates_per_iteration = int(cfg.get("updates_per_iteration") or E)
    # replay sampling stream: one per rank
    seed = int(cfg.get("seed_for_sampling", 0) or env.native.seed) + 7919 * dp.rank

    updates = step = pos = 0
    last_eval = last_save = last_video = 0
    metrics_dev = None
    while step < cfg.total_steps + 1:
        final_len, _ = collector.collect(rb, pos % capacity, eps_sched(step))
        step += iteration_env_steps(final_len, dp)
        pos += E
        if step > cfg.training_start and pos >= cfg.batch_size:
            if dp.active and not peer:
                metrics_dev = model.update_n_allreduce(rb, int(cfg.batch_size), min(pos, capacity), seed, updates, updates_per_iteration, dp.all_reduce_)
            else:
                metrics_dev = model.update_n(rb, int(cfg.batch_size), min(pos, capacity), seed, updates, updates_per_iteration)
            updates += updates_per_iteration
        else:
            metrics_dev = None

        if cfg.eval_interval and (step - last_eval) >= cfg.eval_interval and evaluator is not None:
            t0 = time.perf_counter()
            ln, ret = evaluator.collect(None, 0, cfg.eps_evaluation)
            torch.cuda.synchronize()
            infos = _episode_infos(ln, ret, time.perf_counter() - t0)
            if metrics_dev is not None:
                infos.append({"loss": float(metrics_dev[0].item())})
            infos.append({"updates": updates, "environment_steps": step, "epsilon": eps_sched(step)})
            logger.log_metrics(infos)
            last_eval = step

        # here, like evaluation: the other ranks wait in the next iteration's host collective, not in the in-kernel peer exchange
        if video_env is not None and (step - last_video) >= cfg.video_interval:
            record_episodes(video_env, model, cfg.video_frames, f"./videos/step-{step}.mp4", cfg.eps_evaluation)
            last_video = step

        if cfg.save_interval and (step - last_save) >= cfg.save_interval and dp.is_main:
            Path("checkpoints").mkdir(exist_ok=True)
            torch.save(model.state_dict(), f"checkpoints/model_s{step}.pt")
            last_save = step

    env.close()
    if video_env is not None:
        video_env.close()
    return dict(environment_steps=step, updates=updates)
