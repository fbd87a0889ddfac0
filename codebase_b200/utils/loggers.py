"""results.csv logging with the reference's schema -- restates marlbase/utils/loggers.py (squash_info 14-36, Logger 39-109,
FileSystemLogger 140-169) on plain dict configs (omegaconf is not a dependency here)."""
from __future__ import annotations

import json
import logging
import math
import time
from datetime import timedelta
from hashlib import sha256

import numpy as np
import pandas as pd
import yaml


def squash_info(info):
    """loggers.py:14-36: a key seen once is copied; otherwise mean_/std_ of np.array(v).sum() per entry."""
    new_info = {}
    keys = set(k for i in info for k in i.keys())
    keys.discard("TimeLimit.truncated")
    keys.discard("terminal_observation")
    for key in keys:
        values = [d[key] for d in info if key in d]
        if len(values) == 1:
            new_info[key] = values[0]
            continue
        sums = [np.array(v).sum() for v in values]
        head, _, tail = key.rpartition("/")
        pre = head + "/" if head else ""
        new_info[f"{pre}mean_{tail}"] = np.mean(sums)
        new_info[f"{pre}std_{tail}"] = np.std(sums)
    return new_info


class Logger:
    def __init__(self, project_name, cfg):
        plain = cfg.to_dict() if hasattr(cfg, "to_dict") else dict(cfg)
        self.config_hash = sha256(json.dumps({k: v for k, v in plain.items() if k != "seed"}, sort_keys=True, default=str).encode("utf8")).hexdigest()[-10:]
        self._total_steps = plain["algorithm"]["total_steps"]
        self._start_time = time.time()
        self._prev_time = None
        self._prev_steps = (0, 0)
        self.last_fps = None

    def log_metrics(self, metrics):
        raise NotImplementedError

    def print_progress(self, updates, steps, mean_returns, episodes):
        self.info(f"Updates {updates}, Environment timesteps {steps}")
        now = time.time()
        elapsed = now - self._prev_time if self._prev_time else None
        from_start = timedelta(seconds=math.ceil(now - self._start_time))
        completed = steps / self._total_steps
        if elapsed:
            ups = (updates - self._prev_steps[0]) / elapsed
            fps = (steps - self._prev_steps[1]) / elapsed
            self.last_fps = fps
            self.info(f"UPS: {ups:.2f}, FPS: {fps:.2f} (wall time)")
            eta = from_start * (1 - completed) / completed if completed > 0 else timedelta(0)
            self.info(f"Elapsed Time: {from_start}")
            self.info(f"Estim. Time Left: {timedelta(seconds=math.ceil(eta.total_seconds()))}")
        self.info(f"Completed: {100 * completed:.2f}%")
        self._prev_steps = (updates, steps)
        self._prev_time = time.time()
        self.info(f"Last {episodes} episodes with mean returns: {mean_returns:.3f}")
        self.info("-------------------------------------------")

    def watch(self, model):
        logging.debug(model)

    def info(self, *a, **k):
        return logging.info(*a, **k)

    def warning(self, *a, **k):
        return logging.warning(*a, **k)

    def get_state(self):
        return None


class NullLogger(Logger):
    """The logger of data-parallel ranks other than 0: writes nothing (rank 0 logs the metrics of every rank)."""

    def log_metrics(self, metrics):
        pass


class FileSystemLogger(Logger):
    def __init__(self, project_name, cfg):
        super().__init__(project_name, cfg)
        self.results_path, self.config_path = "results.csv", "config.yaml"
        with open(self.config_path, "w") as f:
            yaml.safe_dump(cfg.to_dict() if hasattr(cfg, "to_dict") else dict(cfg), f)

    def log_metrics(self, metrics):
        d = squash_info(metrics)
        df = pd.DataFrame.from_dict([d])[["environment_steps"] + sorted(k for k in d if k != "environment_steps")]
        with open(self.results_path, "a") as f:
            df.to_csv(f, header=f.tell() == 0, index=False)
        self.print_progress(d["updates"], d["environment_steps"], d["mean_episode_returns"], len(metrics) - 1)

    def get_state(self):
        return pd.read_csv(self.results_path, index_col=0)
