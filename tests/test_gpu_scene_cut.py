"""F15 on the GPU: rb_scene_cut_scores against the numpy oracle of tests/test_scene_cut.py bit for bit (sizes, frame
counts, uniform, identical and disjoint frames, a dirty histogram buffer, graph replay), and scene_cut end to end on a
clip of two shots -- shifted crops of tests/data/frame_0016.png and of its negative -- through
video_interpolate(fps=...), video_interpolate(ts=...), video(warm_start=True) and infer_raft.py --scene-cut."""
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from test_gpu_video import _files
from test_gpu_video_interp import _model, _weights
from test_scene_cut import oracle, oracle_cuts

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "data", "frame_0016.png")


def _scores(frames):
    from networks.utils import scene_cut_scores
    s, h = scene_cut_scores(torch.from_numpy(np.ascontiguousarray(frames)).cuda(), return_hist=True)
    return s.cpu().numpy(), h.cpu().numpy()


def _check(frames):
    s, h = _scores(frames)
    ws, wh = oracle(frames)
    assert h.dtype == np.int32 and np.array_equal(h, wh)
    assert s.dtype == np.float32 and np.array_equal(s.view(np.uint32), ws.view(np.uint32)), (s, ws)
    return s


def _natural(n, H, W, seed):
    """n frames of a slow pan over frame_0016.png at H x W, with a little noise."""
    import cv2
    rng = np.random.default_rng(seed)
    src = cv2.imread(SRC)
    out = []
    for k in range(n):
        img = cv2.resize(np.roll(src, 5 * k, axis=1), (W, H), interpolation=cv2.INTER_AREA).astype(np.int16)
        out.append(np.clip(img + rng.integers(-6, 7, img.shape), 0, 255).astype(np.uint8))
    return np.stack(out)


# ---- rb_scene_cut_scores -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(1, 1), (1, 611), (587, 1), (37, 53), (127, 4099), (436, 1024), (1080, 1920)])
def test_scores_equal_oracle(cuda, H, W):
    s = _check(_natural(3, H, W, seed=H * 7 + W))
    if H * W > 1000:
        assert (s > 0).all() and (s < 0.5).all()  # a pan: close histograms, not equal ones


def test_frame_counts(cuda):
    rng = np.random.default_rng(7)
    for n in range(2, 34):
        f = rng.integers(0, 256, (n, 19, 23, 3), dtype=np.uint8)
        f[: n // 2] >>= 2  # darker frames: scores away from 0 and 1
        _check(f)


def test_uniform_identical_disjoint(cuda):
    H, W = 1080, 1920
    colours = [(0, 0, 0), (0, 0, 0), (31, 31, 31), (32, 31, 31), (255, 255, 255), (128, 64, 200), (128, 64, 200)]
    uni = np.stack([np.broadcast_to(np.array(c, np.uint8), (H, W, 3)) for c in colours])
    s, h = _scores(uni)
    assert s.tolist() == [0.0, 0.0, 1.0, 1.0, 1.0, 0.0]  # one pixel bin each: equal or disjoint
    assert (h.max(axis=1) == H * W).all() and (h.sum(axis=1) == H * W).all()
    _check(uni[:, :436, :1024])
    same = np.repeat(_natural(1, 436, 1024, seed=1), 4, axis=0)
    assert _check(same).tolist() == [0.0, 0.0, 0.0]
    rng = np.random.default_rng(8)
    low = rng.integers(0, 128, (436, 1024, 3), dtype=np.uint8)   # levels 0..3 in every channel
    high = rng.integers(128, 256, (436, 1024, 3), dtype=np.uint8)  # levels 4..7
    assert _check(np.stack([low, high, low, high.copy()])).tolist() == [1.0, 1.0, 1.0]


def test_dirty_histogram_and_graph_replay(cuda):
    """The call zeroes hist itself, and a captured CUDA graph replays it to the same bits."""
    from raft_b200 import capi
    frames = torch.from_numpy(_natural(5, 64, 96, seed=9)).cuda()
    want_s, want_h = oracle(frames.cpu().numpy())
    hist = torch.full((5, 512), 12345, dtype=torch.int32, device="cuda")
    scores = torch.full((4,), -1.0, device="cuda")

    def call():
        capi.check(capi.lib.rb_scene_cut_scores(capi.ptr(frames), 5, 64, 96, capi.ptr(hist), capi.ptr(scores),
                                                capi.stream()))

    call()
    assert np.array_equal(hist.cpu().numpy(), want_h) and np.array_equal(scores.cpu().numpy(), want_s)
    stream = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        call()
    hist.fill_(-7)
    scores.fill_(2.0)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(hist.cpu().numpy(), want_h) and np.array_equal(scores.cpu().numpy(), want_s)


def test_wrapper_refusals(cuda):
    from networks.utils import scene_cut_scores
    f = torch.zeros(3, 8, 8, 3, dtype=torch.uint8, device="cuda")
    for bad in (f.cpu(), f.float(), f[:1], f[..., :2], f[0]):
        with pytest.raises(ValueError, match="scene_cut_scores"):
            scene_cut_scores(bad)


# ---- the clip: two shots ---------------------------------------------------------------------------------------------
SHOTS = "ABBBBAAAABAAB"  # frame k's shot; 12 pairs, cuts at 0, 4 (mid-pass at batch 3), 8 (last pair of a pass at batch
CUTS = [0, 4, 8, 9, 11]  # 3), 8 and 9 (frame 9 is a one-frame shot) and 11 (the last pair)
N_FRAMES = len(SHOTS)


@pytest.fixture(scope="module")
def cut_dir(tmp_path_factory):
    import cv2
    src = cv2.imread(SRC)
    d = tmp_path_factory.mktemp("cutframes")
    for k, shot in enumerate(SHOTS):
        crop = src[100 + k:100 + k + 124, 200 + 3 * k:200 + 3 * k + 150]
        cv2.imwrite(str(d / f"frame_{k:04d}.png"), crop if shot == "A" else 255 - crop)
    return str(d)


def _decoded(d):
    import cv2
    from raft_b200.video import list_frames
    return np.stack([cv2.imread(p) for p in list_frames(d)])


def _threshold(d):
    """Midway between the largest within-shot score and the smallest cut score, both from the oracle."""
    s = oracle(_decoded(d))[0]
    within, at = [float(s[k]) for k in range(N_FRAMES - 1) if k not in CUTS], [float(s[k]) for k in CUTS]
    assert max(within) < min(at), (within, at)
    thr = (max(within) + min(at)) / 2
    assert max(within) < thr < min(at) and oracle_cuts(s, thr) == CUTS
    return thr


class _Spy:
    """The model's engine, recording the items of every interpolate_sequence_at call and counting the
    interpolate_sequence calls."""

    def __init__(self, engine):
        self._engine, self.at, self.seq = engine, [], 0

    def __getattr__(self, name):
        return getattr(self._engine, name)

    def interpolate_sequence_at(self, frames, items, **kw):
        self.at.append(list(items))
        return self._engine.interpolate_sequence_at(frames, items, **kw)

    def interpolate_sequence(self, frames, ts, **kw):
        self.seq += 1
        return self._engine.interpolate_sequence(frames, ts, **kw)


def _spied():
    m = _model()
    spy = _Spy(m.engine())
    m.engine = lambda: spy
    return m, spy


def test_clip_scores(cuda, cut_dir):
    _check(_decoded(cut_dir))
    _threshold(cut_dir)


def test_fps_scene_cut(cuda, cut_dir, tmp_path):
    import cv2
    from raft_b200.video import cut_copy, fps_schedule, video_interpolate
    thr, frames = _threshold(cut_dir), _decoded(cut_dir)
    video_interpolate(_model(), cut_dir, str(tmp_path / "plain"), batch=3, fps=(24, 60))
    plain = _files(str(tmp_path / "plain"))
    runs = []
    for batch, workers in ((1, 0), (3, 4), (8, 4), (8, 0)):
        m, spy = _spied()
        out = str(tmp_path / f"b{batch}w{workers}")
        paths, cuts = video_interpolate(m, cut_dir, out, batch=batch, workers=workers, fps=(24, 60), scene_cut=thr)
        assert cuts == CUTS and [os.path.basename(p) for p in paths] == sorted(plain)
        want = [[(k - p.frames[0], t) for _, k, t in p.items if k not in CUTS]
                for p in fps_schedule(N_FRAMES, 24, 60, batch)]
        assert spy.at == [w for w in want if w], batch  # no cut item reached the engine; all-cut passes made no call
        if batch == 1:
            assert len(spy.at) < len(want)
        runs.append(_files(out))
    assert all(r == runs[0] for r in runs)
    n_cut = 0
    for n, name in enumerate(sorted(plain)):
        s = Fraction(n * 24, 60)
        k = s.numerator // s.denominator
        if s.denominator != 1 and k in CUTS:
            got = cv2.imread(os.path.join(str(tmp_path / "b3w4"), name))
            assert np.array_equal(got, frames[cut_copy(k, float(s - k))]), n
            assert runs[0][name] != plain[name], n  # the blend of two shots is gone
            n_cut += 1
        else:
            assert runs[0][name] == plain[name], n
    assert n_cut == 2 * len(CUTS)  # 24 -> 60 puts two frames strictly inside every pair


def test_ts_scene_cut(cuda, cut_dir, tmp_path):
    import cv2
    from raft_b200.video import cut_copy, frame_number, interp_schedule, video_interpolate
    thr, frames = _threshold(cut_dir), _decoded(cut_dir)
    ts = [0.25, 0.5, 0.75]
    video_interpolate(_model(), cut_dir, str(tmp_path / "plain"), ts=ts, batch=3)
    plain = _files(str(tmp_path / "plain"))
    runs = []
    for batch, workers in ((1, 4), (3, 0), (8, 4)):
        m, spy = _spied()
        out = str(tmp_path / f"b{batch}w{workers}")
        paths, cuts = video_interpolate(m, cut_dir, out, ts=ts, batch=batch, workers=workers, scene_cut=thr)
        assert cuts == CUTS and len(paths) == len(plain)
        live = [p for p in interp_schedule(N_FRAMES, batch) if any(k is not None and k not in CUTS for k in p.pairs)]
        assert spy.seq == len(live) and not spy.at, batch
        runs.append(_files(out))
    assert all(r == runs[0] for r in runs)
    for k in range(N_FRAMES - 1):
        for j, t in enumerate(ts):
            name = f"frame_{frame_number(k, 3, j):06d}.png"
            if k in CUTS:
                got = cv2.imread(os.path.join(str(tmp_path / "b3w0"), name))
                assert np.array_equal(got, frames[cut_copy(k, t)]), (k, t)
            else:
                assert runs[0][name] == plain[name], (k, t)
        assert runs[0][f"frame_{frame_number(k, 3):06d}.png"] == plain[f"frame_{frame_number(k, 3):06d}.png"]


def test_threshold_one_changes_nothing(cuda, cut_dir, tmp_path):
    from raft_b200.video import video_interpolate
    m = _model()
    for kw in ({"fps": (24, 60)}, {"ts": [0.5]}):
        a, b = str(tmp_path / "a"), str(tmp_path / "b")
        plain = video_interpolate(m, cut_dir, a, batch=3, **kw)
        paths, cuts = video_interpolate(m, cut_dir, b, batch=3, scene_cut=1.0, **kw)
        assert cuts == [] and [os.path.basename(p) for p in paths] == [os.path.basename(p) for p in plain]
        assert _files(a) == _files(b), kw


def test_warm_video_scene_cut(cuda, cut_dir, tmp_path):
    from raft_b200.video import list_frames, video
    thr, frames = _threshold(cut_dir), _decoded(cut_dir)
    m = _model()
    npy = tmp_path / "npy"
    paths, cuts = video(m, cut_dir, str(tmp_path / "png"), batch=1, warm_start=True, scene_cut=thr, npy=str(npy))
    assert cuts == CUTS and len(paths) == 2 * (N_FRAMES - 1)
    files = list_frames(cut_dir)
    shots, start = [], 0
    for k in CUTS + [N_FRAMES - 1]:
        shots.append(list(range(start, k + 1)))
        start = k + 1
    shots = [s for s in shots if len(s) > 1]
    assert shots == [[1, 2, 3, 4], [5, 6, 7, 8], [10, 11]]
    for i, shot in enumerate(shots):  # each shot's chain is the chain of video(warm_start=True) on the shot alone
        d = tmp_path / f"shot{i}"
        video(m, [files[f] for f in shot], str(d / "png"), batch=1, warm_start=True, npy=str(d / "npy"))
        for j in range(len(shot) - 1):
            got = np.load(str(npy / f"flow_{shot[j]:06d}.npy"))
            want = np.load(str(d / "npy" / f"flow_{j:06d}.npy"))
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (shot, j)
    for k in CUTS:  # a pair across a cut runs cold
        want = m.forward(frames[k:k + 1], frames[k + 1:k + 2]).cpu().numpy()[0]
        assert np.array_equal(np.load(str(npy / f"flow_{k:06d}.npy")).view(np.uint32), want.view(np.uint32)), k
    # warm-started without cuts, pair 1 (after the cut at 0) differs from its cold flow: the restart is visible
    video(m, cut_dir, str(tmp_path / "warm"), batch=1, warm_start=True, npy=str(tmp_path / "warm_npy"))
    assert not np.array_equal(np.load(str(tmp_path / "warm_npy" / "flow_000001.npy")),
                              np.load(str(npy / "flow_000001.npy")))
    with pytest.raises(ValueError, match="warm_start"):
        video(m, cut_dir, str(tmp_path / "x"), batch=3, scene_cut=thr)
    with pytest.raises(ValueError, match="scene_cut"):
        video(m, cut_dir, str(tmp_path / "x"), batch=1, warm_start=True, scene_cut=1.5)


def test_cli_scene_cut(cuda, cut_dir, tmp_path):
    from raft_b200.video import video_interpolate
    thr = _threshold(cut_dir)
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    out = tmp_path / "cli"
    argv = [sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", cut_dir, "--out", str(out),
            "--load", npz, "--iters", "4", "--input-fps", "24", "--fps", "60", "--keep-size", "--batch", "3",
            "--scene-cut", repr(thr)]
    r = subprocess.run(argv, cwd=tmp_path, env=dict(os.environ, PYTHONNOUSERSITE="1"), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "scene cuts: 5 at pairs 0 4 8 9 11" in r.stdout.splitlines(), r.stdout
    video_interpolate(_model(), cut_dir, str(tmp_path / "api"), batch=8, fps=(24, 60), scene_cut=thr)
    assert _files(str(out)) == _files(str(tmp_path / "api"))
