"""Timings of video recording (DESIGN.md §4.8):

    python tools/video_time.py [--out DIR]

prints the GPU's name and power limit, then
  * the render kernel per frame, CUDA events over many launches after a warm-up, at 1 and 4 096 envs per launch on Foraging 8x8 and 15x15
    and on rware tiny and large (random boards), with the frame bytes written per second;
  * the wall time of one 500-frame recording (IDQN on Foraging-8x8-2p-3f-v3, time limit 25), split into rollout plus render, device-to-host
    copies and encoding.
Writes the same numbers as JSON to DIR/video_time.json when --out is given.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # pragma: no cover
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def make_env(kind: str, E: int):
    from codebase_b200.lbf import LbfConfig, NativeLbf
    from codebase_b200.rware import NativeRware, parse_rware_id

    if kind.startswith("lbf"):
        side = int(kind[3:])
        env = NativeLbf(LbfConfig(rows=side, cols=side, n_agents=4, max_num_food=5, sight=2), E, seed=1)
    else:
        env = NativeRware(parse_rware_id(f"rware-{kind[6:]}-4ag-v2"), E, seed=1)
    env.reset()
    if kind.startswith("lbf"):   # a few steps so boards differ
        for _ in range(5):
            env.step(torch.randint(0, 6, (E, env.N), dtype=torch.int32, device="cuda"), autoreset=True)
    return env


def time_render(kind: str, E: int) -> dict:
    env = make_env(kind, E)
    out = torch.empty(E, *env.frame_shape, dtype=torch.uint8, device="cuda")
    launches = 200 if E == 1 else 10
    for _ in range(3):
        env.render(0, E, out=out)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        env.render(0, E, out=out)
    b.record()
    torch.cuda.synchronize()
    launch_us = a.elapsed_time(b) * 1e3 / launches
    frame_bytes = int(np.prod(env.frame_shape))
    res = dict(env=kind, envs=E, frame=list(env.frame_shape), launch_us=round(launch_us, 2), us_per_frame=round(launch_us / E, 3),
               write_GBps=round(E * frame_bytes / (launch_us * 1e-6) / 1e9, 1))
    env.close()
    del out
    torch.cuda.empty_cache()
    return res


def time_recording(frames: int = 500) -> dict:
    from codebase_b200.config import compose, instantiate, call
    from codebase_b200.dqn.train import record_episodes
    from codebase_b200.utils import video

    cfg = compose(["+algorithm=idqn", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "seed=0", "env.parallel_envs=8"])
    eval_env = call(cfg.env, seed=0, env_gid0=1 << 30)
    model = instantiate(cfg.algorithm.model, eval_env.single_observation_space, eval_env.single_action_space, cfg.algorithm, max_batch=32,
                        max_episode_length=25)
    venv = video.recording_env(eval_env)
    import tempfile

    with tempfile.TemporaryDirectory() as d:
        record_episodes(venv, model, 50, os.path.join(d, "warm.mp4"), 0.05)   # warm-up: module loads, encoder start
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rec = record_episodes(venv, model, frames, os.path.join(d, "v.mp4"), 0.05)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        size = os.path.getsize(os.path.join(d, "v.mp4"))
    d2h, enc = rec.seconds["d2h"], rec.seconds["encode"]
    return dict(frames=frames, frame=list(venv.native.frame_shape), wall_s=round(wall, 4), rollout_render_s=round(wall - d2h - enc, 4),
                d2h_s=round(d2h, 4), encode_s=round(enc, 4), mp4_bytes=size)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    info = gpu_info()
    print("GPU:", info)
    res = dict(gpu=info, render=[], recording=None)
    for kind in ("lbf8", "lbf15", "rware-tiny", "rware-large"):
        for E in (1, 4096):
            r = time_render(kind, E)
            res["render"].append(r)
            print(json.dumps(r))
    res["recording"] = time_recording()
    print(json.dumps(res["recording"]))
    print("GPU (again):", gpu_info())
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "video_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
