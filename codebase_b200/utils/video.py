"""Episode videos -- drop-in for marlbase/utils/video.py (`VideoRecorder(fps=30)`: reset / record_frame / save) and the recording loop of the
reference's `record_episodes` (marlbase/dqn/train.py:239-261, marlbase/ac/train.py:122-150).

Frames are drawn on the device by the env's render kernel (DESIGN.md §4.8) into a device ring of at most RING_FRAMES frames (and RING_BYTES);
a full ring is copied to the host and encoded, so host memory holds one ring however long the recording.  The encoder is OpenCV's `mp4v`
VideoWriter (the reference's imageio is not a dependency here); it writes to a temporary file that `save` moves into place.  The video's frame
size is the frame's rounded up to even (a black row or column pads an odd side), as MPEG-4 Part 2 requires.
"""
from __future__ import annotations

import os
import shutil
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

RING_FRAMES = 256
RING_BYTES = 256 << 20
# env_gid0 of the one-env recording copy of the evaluation env: its own Philox streams, apart from training (ranks from 0), evaluation (1 << 30)
# and codebase_b200.eval (1 << 29)
VIDEO_GID0 = 3 << 29


def require_encoder():
    """Import OpenCV, or fail with the reason: called before training starts when videos are requested, not at the first recording."""
    try:
        import cv2
    except ImportError as e:
        raise ImportError("video recording (algorithm.video_interval, eval video_frames=) encodes mp4 files with OpenCV: "
                          f"`import cv2` failed ({e}); install opencv-python or leave videos off") from e
    return cv2


class VideoRecorder:
    def __init__(self, fps=30):
        self.fps = fps
        self._cv2 = require_encoder()
        self._ring = None
        self._writer = self._tmp = None
        self.reset()

    def reset(self):
        if self._writer is not None:
            self._writer.release()
        if self._tmp is not None and os.path.exists(self._tmp):
            os.remove(self._tmp)
        self._writer = self._tmp = None
        self._n = self.frames = 0
        self.seconds = {"d2h": 0.0, "encode": 0.0}   # device-to-host copies and encoding so far

    def record_frame(self, env):
        """Appends env 0's frame of `env` (a B200VecEnv, or its native handle)."""
        native = getattr(env, "native", env)
        shape = native.frame_shape
        if self._ring is None or tuple(self._ring.shape[1:]) != shape or self._ring.device != native.device:
            if self._n:
                raise ValueError(f"frame shape {shape} differs from the recording's {tuple(self._ring.shape[1:])}")
            size = max(1, min(RING_FRAMES, RING_BYTES // (shape[0] * shape[1] * shape[2])))
            self._ring = torch.empty(size, *shape, dtype=torch.uint8, device=native.device)
        native.render(0, 1, out=self._ring[self._n:self._n + 1])
        self._n += 1
        self.frames += 1
        if self._n == self._ring.shape[0]:
            self._flush()

    def _flush(self):
        if not self._n:
            return
        t0 = time.perf_counter()
        host = self._ring[:self._n].cpu().numpy()
        t1 = time.perf_counter()
        h, w = host.shape[1:3]
        if self._writer is None:
            fd, self._tmp = tempfile.mkstemp(suffix=".mp4")
            os.close(fd)
            self._writer = self._cv2.VideoWriter(self._tmp, self._cv2.VideoWriter_fourcc(*"mp4v"), float(self.fps), (w + (w & 1), h + (h & 1)))
            if not self._writer.isOpened():
                raise RuntimeError(f"OpenCV cannot open an mp4v VideoWriter for {w}x{h} frames")
        # MPEG-4 Part 2 codes even sizes only (an odd frame would lose its last row or column): a black row / column pads an odd side
        img = np.zeros((h + (h & 1), w + (w & 1), 3), np.uint8)
        for f in host:
            img[:h, :w] = f[..., ::-1]   # the frames are RGB, OpenCV writes BGR
            self._writer.write(img)
        self.seconds["d2h"] += t1 - t0
        self.seconds["encode"] += time.perf_counter() - t1
        self._n = 0

    def save(self, filename):
        if not self.frames:
            raise ValueError("VideoRecorder.save: no frames recorded")
        self._flush()
        self._writer.release()
        self._writer = None
        shutil.move(self._tmp, str(filename))
        self._tmp = None


def recording_env(eval_env):
    """The env videos are recorded on: a one-env copy of the evaluation env's config and seed with its own env_gid0, so the training env, the
    evaluation env and every Philox stream of training are untouched."""
    from .envs import B200VecEnv

    native = eval_env.native
    return B200VecEnv(eval_env.cfg, 1, native.seed, VIDEO_GID0, native.device_index)


def record_policy(env, n_timesteps, path, forward, policy, epsilon=0.0, hidden=0):
    """The reference's record_episodes loop on a one-env B200VecEnv: exactly `n_timesteps` frames; when the episode is over, reset and record
    the reset frame, otherwise take one step and record the new frame.  An episode is over on `done or truncated` (the step kernel freezes a
    finished env; the DQN reference ignores truncation here and would step past its TimeLimit).

    forward(obs, out=..., h=..., h_out=...): the network pass (QNetwork.q_values, A2CNetwork.logits); policy 1 acts epsilon-greedily on its
    output, 2 samples the categorical, both inside the env's rollout step.  hidden > 0: a recurrent network of that width, whose state is zeroed
    at every reset."""
    native = env.native
    if native.E != 1:
        raise ValueError(f"record_policy records a one-env B200VecEnv (got {native.E} envs); see recording_env")
    recorder = VideoRecorder()
    out = torch.empty(1, native.N, native.A, dtype=torch.float32, device=native.device)
    h = [torch.zeros(1, native.N, hidden, dtype=torch.float32, device=native.device) for _ in range(2)] if hidden else None
    done, cur = True, 0
    for _ in range(int(n_timesteps)):
        if done:
            native.reset()
            if h:
                h[0].zero_()
                cur = 0
            done = False
        else:
            if h:
                forward(native.obs, out=out, h=h[cur], h_out=h[cur ^ 1])
                cur ^= 1
            else:
                forward(native.obs, out=out)
            native.rollout_step(out, policy=policy, epsilon=epsilon)
            done = bool((native.done[0] | native.trunc[0]).item())
        recorder.record_frame(native)
    Path(path).parent.mkdir(parents=True, exist_ok=True)
    recorder.save(path)
    return recorder
