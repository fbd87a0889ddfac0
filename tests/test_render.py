"""CPU: known-answer boards for the frame oracle (tests/render_ref.py, DESIGN.md §4.8), the host side of `eval video_frames=` and the encoder."""
import numpy as np
import pytest

from tests import render_ref as rr

FOOD, AGENT = rr.LBF["food"], rr.LBF["agent"]


def lbf_px(frame, r, c, lx, ly):
    return tuple(int(v) for v in frame[1 + 51 * r + ly, 1 + 51 * c + lx])


def rw_px(frame, x, y, lx, ly):
    return tuple(int(v) for v in frame[1 + 31 * y + ly, 1 + 31 * x + lx])


def test_frame_size_grid_lines_and_palette_at_cell_centres():
    field = np.zeros((8, 8), np.int8)
    field[2, 3] = 2
    players = np.array([[5, 6, 1], [0, 0, 2]])
    f = rr.lbf_frame(field, players)
    assert f.shape == (409, 409, 3) == rr.frame_shape(8, 8, 50) and f.dtype == np.uint8
    assert rr.frame_shape(20, 20, 50)[:2] == (1021, 1021) and rr.frame_shape(11, 10, 30)[:2] == (342, 311)
    for k in range(9):
        assert (f[51 * k] == 0).all() and (f[:, 51 * k] == 0).all()
    assert lbf_px(f, 2, 3, 25, 25) == FOOD and lbf_px(f, 5, 6, 25, 25) == AGENT and lbf_px(f, 0, 0, 25, 25) == AGENT
    assert lbf_px(f, 4, 4, 25, 25) == rr.WHITE and (f[1:51, 1:51][:, :, 0] != 0).any()
    # disc edges: radius 16 (food) / 20 (agent) around the corner (25, 25), measured from pixel centres
    assert lbf_px(f, 2, 3, 25, 9) == FOOD and lbf_px(f, 2, 3, 25, 8) == rr.WHITE      # dy = 2*(9-25)+1 = -31: 961 <= 1024; -33: 1089
    assert lbf_px(f, 5, 6, 25, 5) == AGENT and lbf_px(f, 5, 6, 25, 4) == rr.WHITE     # -39: 1521 <= 1600; -41: 1681
    # badge ring: black between radii 9 and 11 around (37, 37), white inside
    assert lbf_px(f, 2, 3, 37, 47) == rr.BLACK and lbf_px(f, 2, 3, 37, 45) == rr.WHITE and lbf_px(f, 2, 3, 37, 48) == rr.WHITE


@pytest.mark.parametrize("level, ink, blank", [
    (1, [(36, 32), (34, 34), (34, 40), (38, 41)], [(34, 32), (38, 32), (38, 36)]),        # ".#." / "##." / ... / "###", box x 34..39, y 32..41
    (9, [(34, 32), (38, 38), (34, 36)], [(36, 34), (34, 38), (36, 38)]),                  # "#.#" row 1, "..#" row 3
    (10, [(30, 34), (32, 32), (38, 32), (42, 36)], [(36, 32), (37, 40), (40, 36), (30, 32)]),   # "1" at x 30..35, gap 36..37, "0" at 38..43
    (23, [(30, 32), (34, 34), (30, 38), (42, 38), (38, 36)], [(30, 34), (32, 34), (38, 34), (38, 38)]),
])
def test_badge_digits(level, ink, blank):
    field = np.zeros((5, 5), np.int8)
    field[2, 2] = level
    f = rr.lbf_frame(field, np.array([[0, 4, 1]]))
    for lx, ly in ink:
        assert lbf_px(f, 2, 2, lx, ly) == rr.BLACK, (level, lx, ly)
    for lx, ly in blank:
        assert lbf_px(f, 2, 2, lx, ly) == rr.WHITE, (level, lx, ly)
    # the agent's badge shows its own level
    g = rr.lbf_frame(np.zeros((5, 5), np.int8), np.array([[2, 2, level]]))
    tile = lambda fr: fr[1 + 102:1 + 102 + 50, 1 + 102:1 + 102 + 50]   # noqa: E731
    badge = rr.disc(50, 37, 37, 11)
    assert (tile(f)[badge] == tile(g)[badge]).all() and lbf_px(g, 2, 2, 25, 25) == AGENT


def test_shared_cell_draws_the_higher_index_last():
    field = np.zeros((6, 6), np.int8)
    both = rr.lbf_frame(field, np.array([[3, 3, 2], [3, 3, 17]]))
    second = rr.lbf_frame(field, np.array([[0, 0, 2], [3, 3, 17]]))
    assert (both[1 + 153:1 + 203, 1 + 153:1 + 203] == second[1 + 153:1 + 203, 1 + 153:1 + 203]).all()
    swapped = rr.lbf_frame(field, np.array([[3, 3, 17], [3, 3, 2]]))
    assert not (swapped == both).all()


def rware_board():
    rows, cols = 11, 10   # tiny
    shelves = np.zeros((rows, cols), np.uint8)
    shelves[1, 1], shelves[1, 2], shelves[5, 4] = 1, 2, 3
    req = np.zeros(8, np.uint32)
    req[0] = 1 << 2
    return shelves, req


@pytest.mark.parametrize("d, line, off", [
    (rr.UP, [(14, 5), (15, 14)], [(14, 15), (16, 10)]), (rr.DOWN, [(14, 15), (15, 24)], [(14, 14), (16, 20)]),
    (rr.LEFT, [(5, 14), (14, 15)], [(15, 14), (10, 16)]), (rr.RIGHT, [(15, 14), (24, 15)], [(14, 14), (20, 16)]),
])
def test_rware_directions(d, line, off):
    shelves, req = rware_board()
    f = rr.rware_frame(shelves, np.array([[7, 3, d, 0]]), req)
    assert f.shape == (342, 311, 3)
    for lx, ly in line:
        assert rw_px(f, 7, 3, lx, ly) == rr.BLACK
    for lx, ly in off:
        assert rw_px(f, 7, 3, lx, ly) == rr.RWARE["agent"]
    assert rw_px(f, 7, 3, 15, 4) == rr.WHITE and rw_px(f, 7, 3, 2, 2) == rr.WHITE   # outside the disc (radius 10), no shelf


def test_rware_shelves_loads_and_goals():
    shelves, req = rware_board()
    f = rr.rware_frame(shelves, np.array([[4, 5, rr.UP, 3], [2, 1, rr.LEFT, 0]]), req)
    assert rw_px(f, 1, 1, 2, 2) == rr.RWARE["shelf"] and rw_px(f, 1, 1, 27, 27) == rr.RWARE["shelf"]
    assert rw_px(f, 1, 1, 1, 1) == rr.WHITE and rw_px(f, 1, 1, 28, 28) == rr.WHITE        # 2-px inset
    assert rw_px(f, 2, 1, 2, 2) == rr.RWARE["shelf_requested"]                             # shelf 2 is requested
    assert rw_px(f, 2, 1, 15, 20) == rr.RWARE["agent"]                                     # unloaded agent over a shelf
    assert rw_px(f, 4, 5, 15, 20) == rr.RWARE["agent_loaded"] and rw_px(f, 4, 5, 2, 2) == rr.RWARE["shelf"]   # carried shelf under its carrier
    for x in (4, 5):   # goals (cols/2 - 1, rows - 1), (cols/2, rows - 1)
        assert rw_px(f, x, 10, 0, 0) == rr.RWARE["goal"] and rw_px(f, x, 10, 29, 29) == rr.RWARE["goal"]
    assert rw_px(f, 3, 10, 15, 15) == rr.WHITE
    g = rr.rware_frame(shelves, np.array([[4, 10, rr.DOWN, 0]]), req)
    assert rw_px(g, 4, 10, 15, 20) == rr.BLACK and rw_px(g, 4, 10, 20, 15) == rr.RWARE["agent"] and rw_px(g, 4, 10, 1, 1) == rr.RWARE["goal"]


def test_eval_video_frames_argument():
    from codebase_b200 import eval as ev

    assert ev.parse_args(["path=x"]) == dict(path="x", load_step=None, seed=None, episodes=None)
    assert ev.parse_args(["path=x", "video_frames=40"]) == dict(path="x", load_step=None, seed=None, episodes=None, video_frames=40)
    with pytest.raises(ValueError):
        ev.parse_args(["path=x", "frames=40"])


class _FrameSource:
    """Stands in for a native env handle: `render` fills the recorder's ring slot with an oracle frame of the next board."""

    def __init__(self, frames):
        import torch

        self.frames, self.k, self.device = frames, 0, torch.device("cpu")
        self.frame_shape = frames[0].shape

    def render(self, env_first, n, out):
        import torch

        out.copy_(torch.from_numpy(self.frames[self.k])[None])
        self.k += 1
        return out


def test_video_recorder_ring_flushes_and_mp4_decodes(tmp_path, monkeypatch):
    """VideoRecorder: frames pass through a ring of RING_FRAMES (5 here: 12 frames are two full flushes and a partial one), are written BGR
    through OpenCV's mp4v VideoWriter, and decode to the same count, size and colours."""
    cv2 = pytest.importorskip("cv2")
    from codebase_b200.utils import video

    assert video.require_encoder() is cv2
    monkeypatch.setattr(video, "RING_FRAMES", 5)
    field = np.zeros((4, 4), np.int8)
    field[1, 1] = 3
    frames = [rr.lbf_frame(field, np.array([[k % 4, 3, 1]])) for k in range(12)]
    src = _FrameSource(frames)
    rec = video.VideoRecorder(fps=30)
    for _ in frames:
        rec.record_frame(src)
    assert rec.frames == 12 and rec._ring.shape[0] == 5 and rec._n == 2
    path = tmp_path / "sub" / "v.mp4"
    path.parent.mkdir()
    rec.save(path)
    cap = cv2.VideoCapture(str(path))
    got = []
    while True:
        ok, img = cap.read()
        if not ok:
            break
        got.append(img[..., ::-1])
    # MPEG-4 Part 2 codes even sizes: the odd 205 x 205 frames gain a black row and column
    assert len(got) == 12 and got[0].shape == (206, 206, 3) and (got[0][205] < 40).all() and (got[0][:, 205] < 40).all()
    # a lossy codec: colours compared loosely, but red and blue must not be swapped
    food = got[0][1 + 51 + 25, 1 + 51 + 25].astype(int)
    assert np.abs(food - np.array(FOOD)).max() < 40 and food[0] > food[2]
    with pytest.raises(ValueError):
        video.VideoRecorder().save(tmp_path / "empty.mp4")
