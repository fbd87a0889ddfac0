"""GPU: the render kernels against the numpy oracle (tests/render_ref.py, DESIGN.md §4.8), bit for bit; the recorder loop of both learner
families; `algorithm.video_interval` in all seven drivers (recording leaves training untouched); `eval video_frames=`."""
import os

import numpy as np
import pandas as pd
import pytest
import torch

from tests import render_ref as rr

pytestmark = pytest.mark.gpu


def random_lbf(env, rng, max_level=99):
    E, (R, C), N = env.E, (env.cfg.rows, env.cfg.cols), env.N
    field = np.where(rng.random((E, R * C)) < 0.15, rng.integers(1, max_level + 1, (E, R * C)), 0).astype(np.int8)
    players = np.zeros((E, N, 4), np.int8)
    players[..., 0] = rng.integers(0, R, (E, N))
    players[..., 1] = rng.integers(0, C, (E, N))
    players[..., 2] = rng.integers(1, max_level + 1, (E, N))
    if N > 1:   # some shared cells
        players[::3, 1, :2] = players[::3, 0, :2]
    env.set_state(torch.from_numpy(field), torch.from_numpy(players), torch.zeros(E, dtype=torch.int32))
    return [rr.lbf_frame(field[e].reshape(R, C), players[e, :, :3].astype(np.int64)) for e in range(E)]


def random_rware(env, rng):
    E, R, C, N = env.E, env.cfg.rows, env.cfg.cols, env.N
    shelves = np.where(rng.random((E, R * C)) < 0.4, rng.integers(1, 256, (E, R * C)), 0).astype(np.uint8)
    agents = np.zeros((E, N, 4), np.uint8)
    for e in range(E):
        cells = rng.choice(R * C, N, replace=False)
        agents[e, :, 0], agents[e, :, 1] = cells % C, cells // C
        agents[e, :, 2] = rng.integers(0, 4, N)
        loaded = rng.random(N) < 0.5
        ids = rng.integers(1, 256, N)
        agents[e, :, 3] = np.where(loaded, ids, 0)
        shelves[e, cells[loaded]] = ids[loaded]   # a carried shelf sits at its carrier's cell
    req = rng.integers(0, 2**32, (E, 8), dtype=np.uint64).astype(np.uint32)
    env.set_state(torch.from_numpy(shelves), torch.from_numpy(agents), torch.from_numpy(req.view(np.int32)), torch.zeros(E, dtype=torch.int32),
                  torch.zeros(E, dtype=torch.int32))
    return [rr.rware_frame(shelves[e].reshape(R, C), agents[e].astype(np.int64), req[e]) for e in range(E)]


def lbf_env(rows, n_agents, E, grid=False):
    from codebase_b200.lbf import LbfConfig, NativeLbf

    cfg = LbfConfig(rows=rows, cols=rows, n_agents=n_agents, max_num_food=3, sight=2 if grid else rows, grid_observation=int(grid))
    return NativeLbf(cfg, E, seed=0)


def rware_env(size, n_agents, E):
    from codebase_b200.rware import NativeRware, parse_rware_id

    return NativeRware(parse_rware_id(f"rware-{size}-{n_agents}ag-v2"), E, seed=0)


@pytest.mark.parametrize("rows, n_agents, grid", [(5, 1, False), (6, 2, False), (8, 3, True), (10, 4, False), (12, 5, True), (15, 7, False),
                                                  (17, 6, True), (20, 9, False)])
def test_lbf_frames_match_the_oracle(rows, n_agents, grid):
    env = lbf_env(rows, n_agents, 12, grid)
    want = random_lbf(env, np.random.default_rng(rows * 10 + n_agents))
    got = env.render(0, env.E).cpu().numpy()
    assert env.frame_shape == want[0].shape == (1 + 51 * rows, 1 + 51 * rows, 3)
    for e in range(env.E):
        assert np.array_equal(got[e], want[e]), (e, np.argwhere((got[e] != want[e]).any(-1))[:5])


@pytest.mark.parametrize("size, n_agents", [("tiny", 1), ("tiny", 4), ("small", 8), ("medium", 13), ("large", 19)])
def test_rware_frames_match_the_oracle(size, n_agents):
    env = rware_env(size, n_agents, 10)
    want = random_rware(env, np.random.default_rng(n_agents))
    got = env.render(0, env.E).cpu().numpy()
    assert env.frame_shape == want[0].shape == (1 + 31 * env.cfg.rows, 1 + 31 * env.cfg.cols, 3)
    for e in range(env.E):
        assert np.array_equal(got[e], want[e]), (e, np.argwhere((got[e] != want[e]).any(-1))[:5])


@pytest.mark.parametrize("kind", ["lbf", "rware"])
def test_one_launch_equals_single_launches_and_touches_only_its_frames(kind):
    env = lbf_env(7, 3, 9) if kind == "lbf" else rware_env("tiny", 4, 9)
    (random_lbf if kind == "lbf" else random_rware)(env, np.random.default_rng(5))
    all_frames = env.render(0, env.E)
    for e in range(env.E):
        assert torch.equal(env.render(e, 1)[0], all_frames[e])
    fb = int(np.prod(env.frame_shape))
    for off in (0, 5, 16 + 3):   # the frames' start at every phase of a 16-byte store
        buf = torch.full((off + 4 * fb + 64,), 0xAB, dtype=torch.uint8, device="cuda")
        env.render(3, 4, out=buf[off:off + 4 * fb].view(4, *env.frame_shape))
        assert (buf[:off] == 0xAB).all() and (buf[off + 4 * fb:] == 0xAB).all()
        assert torch.equal(buf[off:off + 4 * fb].view(4, *env.frame_shape), all_frames[3:7])


@pytest.mark.parametrize("kind", ["lbf", "rware"])
def test_bad_ranges_are_refused(kind):
    import ctypes as C

    from codebase_b200 import _native as nat

    env = lbf_env(5, 2, 4) if kind == "lbf" else rware_env("tiny", 2, 4)
    buf = torch.empty(8, device="cuda", dtype=torch.uint8)
    for first, n in ((-1, 1), (4, 1), (3, 2), (0, 5), (0, 0), (2, -1), (2**31 - 1, 2)):
        with pytest.raises(nat.NativeError, match="range"):
            nat.check(env._c_render(env._h, C.c_int32(first), C.c_int32(n), nat.ptr(buf), nat.stream_ptr()), "render")
    with pytest.raises(nat.NativeError, match="range"):
        env.render(3, 2)
    with pytest.raises(nat.NativeError, match="NULL"):
        nat.check(env._c_render(env._h, C.c_int32(0), C.c_int32(1), C.c_void_p(None), nat.stream_ptr()), "render")
    with pytest.raises(nat.NativeError, match="NULL"):
        nat.check(env._c_render(C.c_void_p(None), C.c_int32(0), C.c_int32(1), C.c_void_p(None), nat.stream_ptr()), "render")


# ---- the recorder loop ------------------------------------------------------------------------------------------------------------------
def build(alg, env_name, extra, time_limit=10):
    from codebase_b200.config import Config, call, compose, instantiate

    cfg = compose([f"+algorithm={alg}", f"env.name={env_name}", f"env.time_limit={time_limit}", "seed=0", "env.parallel_envs=8"] + extra)
    eval_cfg = Config(cfg.env.to_dict())
    eval_env = call(eval_cfg, seed=0, env_gid0=1 << 30)
    a = cfg.algorithm
    kw = dict(max_batch=a.get("batch_size", 128)) if alg in ("idqn", "vdn", "qmix") else dict(max_envs=8)
    model = instantiate(a.model, eval_env.single_observation_space, eval_env.single_action_space, a, max_episode_length=time_limit, **kw)
    return cfg, eval_env, model


@pytest.mark.parametrize("alg, env_name, extra", [
    ("idqn", "lbforaging:Foraging-8x8-2p-3f-v3", []),
    ("idqn", "lbforaging:Foraging-8x8-2p-3f-v3", ["algorithm.model.use_rnn=True"]),
    ("ippo", "lbforaging:Foraging-8x8-2p-3f-v3", ["algorithm.model.actor.use_rnn=True"]),
    ("mappo", "lbforaging:Foraging-8x8-2p-3f-v3", ["algorithm.model.actor.use_rnn=True"]),
    ("ippo", "rware:rware-tiny-4ag-v2", ["algorithm.model.actor.use_rnn=True"]),
    ("mappo", "rware:rware-tiny-1ag-v2", ["algorithm.model.actor.use_rnn=True"]),   # 4 agents: a 284-wide joint observation, over the critic's 128
])
def test_record_episodes(tmp_path, monkeypatch, alg, env_name, extra):
    """Exactly video_frames frames; frame 0 is what render() shows after reset; a new episode (reset frame) starts exactly after a frame whose
    step ended with done | trunc; the mp4 decodes to the frame count and the frame size rounded up to even."""
    import cv2

    from codebase_b200.ac import train as ac_train
    from codebase_b200.dqn import train as dqn_train
    from codebase_b200.utils import video

    cfg, eval_env, model = build(alg, env_name, extra)
    venv = video.recording_env(eval_env)
    seen = []
    orig = video.VideoRecorder.record_frame

    def spy(self, env):
        st = env.get_state()
        seen.append((env.render(0, 1)[0].cpu().numpy(), int(st["episode_idx"][0]), int(st["step"][0]), bool(env.done[0] | env.trunc[0])))
        return orig(self, env)

    monkeypatch.setattr(video.VideoRecorder, "record_frame", spy)
    n = 57
    path = tmp_path / "v" / "rec.mp4"
    if alg == "idqn":
        dqn_train.record_episodes(venv, model, n, str(path), 0.05)
    else:
        ac_train.record_episodes(venv, model, n, str(path))
    assert len(seen) == n
    fresh = video.recording_env(eval_env)
    fresh.native.reset()
    assert np.array_equal(seen[0][0], fresh.render())
    assert seen[0][2] == 0
    # frame k is a reset frame when the episode index moved; one follows exactly a stepped frame whose step ended with done | trunc (a reset
    # frame's flags are the previous episode's)
    reset = [True] + [seen[k][1] != seen[k - 1][1] for k in range(1, n)]
    for k in range(1, n):
        assert reset[k] == (not reset[k - 1] and seen[k - 1][3]), k
        assert seen[k][2] == (0 if reset[k] else seen[k - 1][2] + 1), k
    starts = sum(reset)
    assert starts >= 3   # time_limit 10: the boundaries were exercised
    cap = cv2.VideoCapture(str(path))
    count = 0
    while cap.read()[0]:
        count += 1
    H, W, _ = venv.native.frame_shape
    assert count == n and int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)) == W + W % 2 and int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)) == H + H % 2


# ---- drivers ---------------------------------------------------------------------------------------------------------------------------------
WALL_TIME_COLUMNS = {"mean_episode_time", "std_episode_time"}


@pytest.mark.parametrize("alg", ["idqn", "vdn", "qmix", "ia2c", "ippo", "maa2c", "mappo"])
def test_video_interval_leaves_training_untouched(tmp_path, monkeypatch, alg):
    from codebase_b200 import run

    dqn = alg in ("idqn", "vdn", "qmix")
    args = [f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=64", "seed=0",
            "algorithm.total_steps=12000", "algorithm.eval_interval=2000", "algorithm.eval_episodes=32"]
    if dqn:
        args += ["algorithm.batch_size=64", "algorithm.buffer_size=1024", "algorithm.updates_per_iteration=8", "algorithm.training_start=1000"]
    frames = {}
    for video_on in (False, True):
        out = tmp_path / ("on" if video_on else "off")
        monkeypatch.chdir(tmp_path)
        run.main(args + [f"run_dir={out}"] + (["algorithm.video_interval=4000", "algorithm.video_frames=30"] if video_on else []))
        frames[video_on] = pd.read_csv(out / "results.csv")
        vids = sorted(os.listdir(out / "videos")) if (out / "videos").exists() else []
        assert bool(vids) == video_on and all(v.startswith("step-") and v.endswith(".mp4") for v in vids)
    off, on = frames[False], frames[True]
    cols = [c for c in off.columns if c not in WALL_TIME_COLUMNS]
    assert list(off.columns) == list(on.columns) and len(off) >= 3
    pd.testing.assert_frame_equal(off[cols], on[cols], check_exact=True)


@pytest.mark.parametrize("alg", ["idqn", "ippo"])
def test_eval_video_frames(tmp_path, monkeypatch, alg):
    import cv2

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    extra = ["algorithm.batch_size=64", "algorithm.buffer_size=1024", "algorithm.updates_per_iteration=8"] if alg == "idqn" else []
    run.main([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=64", "seed=0",
              "algorithm.total_steps=6000", "algorithm.eval_interval=3000", "algorithm.save_interval=3000", f"run_dir={out}"] + extra)
    monkeypatch.chdir(tmp_path)
    plain = ev.main([f"path={out}", "episodes=16", "seed=3"])
    assert "video" not in plain and not os.path.exists(f"{out}/eval.mp4")
    with_video = ev.main([f"path={out}", "episodes=16", "seed=3", "video_frames=40"])
    assert with_video.pop("video") == os.path.abspath(f"{out}/eval.mp4")
    assert with_video == plain
    cap = cv2.VideoCapture(f"{out}/eval.mp4")
    count = 0
    while cap.read()[0]:
        count += 1
    assert count == 40
