"""F13 on the GPU: RaftEngine.forward_sequence_bidirectional against per-pair forward / forward_bidirectional calls bit for
bit, rb_flow_reverse_multi against per-step rb_flow_reverse and tests/interp_oracle.py, rb_frame_synthesize_pairs against
rb_frame_synthesize and the uint8 restatement (tests/test_video_interp.py), interpolate_sequence against per-pair
interpolate, mode alternation, and video_interpolate / infer_raft.py --path --interpolate end to end on shifted crops of
tests/data/frame_0016.png."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import interp_oracle as O
from test_gpu_video import _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)
from test_video_interp import quantise, synthesize_u8

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_WEIGHTS = {}


def _weights(small):
    from raft_b200 import synth
    if small not in _WEIGHTS:
        _WEIGHTS[small] = synth.make_weights(small)
    return _WEIGHTS[small]


def _model(small=False, iters=4, **kw):
    from networks.RAFT import RAFT
    return RAFT(None, SimpleNamespace(small=small), iters=iters, device="cuda:0", **kw).load(_weights(small))


def _same(a, b):
    a, b = (x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x) for x in (a, b))
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b)


def _check_bidirectional(m, frames):
    fw, bw, ofw, obw = m.forward_sequence_bidirectional(frames)
    T = len(frames) - 1
    assert fw.shape[0] == bw.shape[0] == ofw.shape[0] == obw.shape[0] == T
    for k in range(T):
        a, b = frames[k:k + 1], frames[k + 1:k + 2]
        assert _same(fw[k], m.forward(a, b)[0]), k
        assert _same(bw[k], m.forward(b, a)[0]), k
        want = m.forward_bidirectional(a, b)
        assert _same(ofw[k], want[2][0]) and _same(obw[k], want[3][0]), k
    none = m.forward_sequence_bidirectional(frames, check=False)
    assert none[2] is None and none[3] is None and _same(none[0], fw) and _same(none[1], bw)


# ---- forward_sequence_bidirectional ------------------------------------------------------------------------------
VARIANTS = {"default": {}, "upstream": {"upstream": True}, "mixed": {"mixed_precision": True},
            "volume_free": {"volume_free": True}}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("small", [False, True])
def test_bidirectional_sequence_equals_pairs(cuda, small, variant):
    _check_bidirectional(_model(small, **VARIANTS[variant]), _frames(3, 125, 150, seed=4000))  # odd size, T = 2


@pytest.mark.parametrize("T", [1, 2, 5])
def test_bidirectional_sequence_lengths(cuda, T):
    _check_bidirectional(_model(), _frames(T + 1, 64, 96, seed=4100 + T))


@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("input_size", [None, (128, 160)])
def test_bidirectional_sequence_frame_inputs(cuda, u8, input_size):
    _check_bidirectional(_model(input_size=input_size), _frames(4, 100, 140, seed=4200, u8=u8))


# ---- rb_flow_reverse_multi ---------------------------------------------------------------------------------------
def _reverse_multi(flow, steps):
    from raft_b200 import capi
    from raft_b200.engine import _floats
    lib, P = capi.lib, capi.ptr
    B, H, W = flow.shape[:3]
    n = len(steps)
    nbytes = capi.size_query(lib.rb_flow_reverse_multi_workspace_bytes, n, B, H, W)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=flow.device)
    ft = torch.empty(n, B, H, W, 2, device=flow.device)
    em = torch.empty(2, n, B, H, W, dtype=torch.uint8, device=flow.device)
    capi.check(lib.rb_flow_reverse_multi(P(flow), _floats(steps), n, P(ft), P(em[0]), P(em[1]), B, H, W, P(ws), nbytes,
                                         capi.stream()))
    return ft.cpu().numpy(), em[0].cpu().numpy(), em[1].cpu().numpy()


@pytest.mark.parametrize("B,H,W", [(3, 37, 53), (2, 1, 29), (1, 23, 1), (2, 64, 96)])
def test_reverse_multi_equals_single_steps(cuda, B, H, W):
    from networks.utils import reverse_flow
    rng = np.random.default_rng(B * 100 + H + W)
    f = (rng.normal(0, 3, (B, H, W, 2)) * rng.uniform(0.2, 2, (B, 1, 1, 2))).astype(np.float32)
    if H * W > 1:
        for v in (np.nan, np.inf, -np.inf):
            f.reshape(-1)[rng.choice(f.size, 3, replace=False)] = v
    # 0, ordinary steps, negative, raft-small's x8 and 1e6 (every source leaves the frame and clamps to the border)
    steps = [0.0, 0.25, 0.5, 1.0 / 3.0, -0.75, 8 * 0.625, 1e6]
    flow = torch.from_numpy(f).cuda()
    ft, em, mu = _reverse_multi(flow, steps)
    for i, s in enumerate(steps):
        one = [x.cpu().numpy() for x in reverse_flow(flow, s)]
        assert _same(ft[i], one[0]) and _same(em[i], one[1]) and _same(mu[i], one[2]), s
        ref = O.reverse_flow(f, time_step=s)
        assert _same(ft[i], ref[0]) and _same(em[i], ref[1]) and _same(mu[i], ref[2]), s


# ---- rb_frame_synthesize_pairs -----------------------------------------------------------------------------------
def _synth_pairs(i0, i1, f0, f1, e0, e1, ts, u8, bgr, pad=(0, 0)):
    from raft_b200 import capi
    from raft_b200.engine import _floats
    lib, P = capi.lib, capi.ptr
    B, Hp, Wp = i0.shape[:3]
    H, W = f0.shape[2:4]
    out = torch.empty(len(ts), B, H, W, 3, dtype=torch.uint8 if u8 else torch.float32, device="cuda")
    capi.check(lib.rb_frame_synthesize_pairs(P(i0), P(i1), Hp, Wp, pad[0], pad[1], P(f0), P(f1), P(e0), P(e1),
                                             _floats(ts), len(ts), P(out), int(u8), int(bgr), B, H, W, capi.stream()))
    return out.cpu().numpy()


def test_synthesize_pairs(cuda):
    from networks.utils import synthesize
    rng = np.random.default_rng(9)
    ts = [0.0, 0.25, 1.0 / 3.0, 0.5, 1.0]
    n, B, H, W = len(ts), 3, 31, 47
    i0, i1 = (rng.uniform(-0.1, 1.1, (B, H, W, 3)).astype(np.float32) for _ in range(2))  # clamps at both ends
    i0[0, 3, 4] = np.nan  # NaN through the blend -> 0
    i1[1, 5, 6] = np.inf
    f0, f1 = (rng.normal(0, 4, (n, B, H, W, 2)).astype(np.float32) for _ in range(2))
    e0, e1 = ((rng.random((n, B, H, W)) < 0.3).astype(np.uint8) for _ in range(2))
    g = [torch.from_numpy(a).cuda() for a in (i0, i1, f0, f1, e0, e1)]
    fp = _synth_pairs(*g, ts, False, False)
    for i, t in enumerate(ts):
        one = synthesize(g[0], g[1], g[2][i], g[3][i], g[4][i], g[5][i], t).cpu().numpy()
        assert _same(fp[i], one), t
        for bgr in (False, True):
            want = synthesize_u8(i0, i1, f0[i], f1[i], e0[i], e1[i], t, bgr)
            assert _same(_synth_pairs(*g, ts, True, bgr)[i], want), (t, bgr)
    u8 = _synth_pairs(*g, ts, True, False)
    assert _same(u8, quantise(fp)) and (u8 == 0).any() and (u8 == 255).any()
    assert _same(_synth_pairs(*g, ts, True, True), u8[..., ::-1])


# ---- interpolate_sequence ----------------------------------------------------------------------------------------
def _check_interp_sequence(m, frames, ts):
    got = m.interpolate_sequence(frames, ts)
    got_u8 = m.interpolate_sequence(frames, ts, uint8=True)
    assert got.shape == (len(ts), len(frames) - 1) + frames.shape[1:3] + (3,)
    for k in range(len(frames) - 1):
        want = m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], ts)[:, 0]
        assert _same(got[:, k], want), k
        assert _same(got_u8[:, k], quantise(want.cpu().numpy())), k
    assert _same(m.interpolate_sequence(frames, ts, uint8=True, bgr=True), got_u8.flip(-1))
    return got


@pytest.mark.parametrize("small", [False, True])
def test_interpolate_sequence_equals_pairs(cuda, small):
    _check_interp_sequence(_model(small), _frames(4, 60, 100, seed=4300), [0.25, 0.5, 0.8])
    _check_interp_sequence(_model(small, upstream=True), _frames(3, 125, 150, seed=4310), [0.5])


def test_interpolate_chunk_bound_changes_no_bit(cuda, monkeypatch):
    from raft_b200 import engine
    frames = _frames(4, 64, 96, seed=4400)
    ts = [i / 8 for i in range(1, 8)]
    m = _model()
    whole = m.interpolate_sequence(frames, ts)
    pair = m.interpolate(frames[:2], frames[1:3], ts)
    monkeypatch.setattr(engine, "REVERSE_WS_BOUND", 1)  # one time per chunk
    assert _same(m.interpolate_sequence(frames, ts), whole)
    assert _same(m.interpolate(frames[:2], frames[1:3], ts), pair)
    monkeypatch.setattr(engine, "REVERSE_WS_BOUND",
                        engine.capi.size_query(engine.capi.lib.rb_flow_reverse_multi_workspace_bytes, 3, 3, 64, 96))
    assert _same(m.interpolate_sequence(frames, ts), whole)  # chunks of 3, 3, 1


def test_full_size(cuda):
    frames = _frames(3, 436, 1024, seed=4500)
    m = _model()
    _check_bidirectional(m, frames)
    _check_interp_sequence(m, frames, [0.5])


# ---- mode alternation --------------------------------------------------------------------------------------------
def test_alternating_modes(cuda):
    frames = _frames(5, 72, 104, seed=4600)
    other = _frames(2, 72, 104, seed=4700)
    l, r = other[:1], other[1:]
    ts = [0.3, 0.6]
    ref = _model()
    want_seq = ref.interpolate_sequence(frames, ts)
    want_bi = ref.forward_sequence_bidirectional(frames)
    whole = ref.forward_sequence(frames)
    m = _model()
    got = [m.forward_sequence(frames[:3])]  # T = 2, then a carry across the new mode
    assert _same(m.interpolate_sequence(frames, ts), want_seq)
    assert _same(m.forward(l, r), _model().forward(l, r))
    assert _same(m.interpolate(l, r, ts), _model().interpolate(l, r, ts))
    got.append(m.forward_sequence(frames[3:5], carry=True))
    assert _same(torch.cat(got), whole)
    for a, b in zip(m.forward_sequence_bidirectional(frames), want_bi):
        assert _same(a, b)
    assert _same(m.forward_sequence(frames[:3]), whole[:2])
    assert _same(m.interpolate_sequence(frames, ts), want_seq)
    assert _same(m.forward_sequence_bidirectional(frames[:3])[0], whole[:2])  # another T
    assert _same(m.interpolate_sequence(frames, ts), want_seq)


# ---- video_interpolate and the CLI -------------------------------------------------------------------------------
def _decoded(d):
    import cv2
    from raft_b200.video import list_frames
    return np.stack([cv2.imread(p) for p in list_frames(d)])


def test_video_interpolate_end_to_end(cuda, frame_dir, tmp_path):
    from raft_b200.video import frame_number, video_interpolate
    m = _model()
    frames = _decoded(frame_dir)
    ts = [0.25, 0.5, 0.75]
    runs = {}
    for batch, workers in ((1, 0), (3, 4), (8, 4), (8, 0)):
        out = tmp_path / f"b{batch}w{workers}"
        written = video_interpolate(m, frame_dir, str(out), ts, batch=batch, workers=workers)
        assert len(written) == (len(frames) - 1) * (len(ts) + 1) + 1
        assert sorted(os.listdir(out)) == [os.path.basename(p) for p in written]
        runs[(batch, workers)] = _files(str(out))
    first = next(iter(runs.values()))
    assert all(r == first for r in runs.values())
    import cv2
    out = tmp_path / "b8w4"
    for k in range(len(frames)):
        assert np.array_equal(cv2.imread(str(out / f"frame_{frame_number(k, 3):06d}.png")), frames[k]), k
    for k in range(len(frames) - 1):
        want = quantise(m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], ts).cpu().numpy()[:, 0])
        for j in range(len(ts)):
            assert np.array_equal(cv2.imread(str(out / f"frame_{frame_number(k, 3, j):06d}.png")), want[j]), (k, j)
    with pytest.raises(ValueError, match="strictly increasing"):
        video_interpolate(m, frame_dir, str(tmp_path / "x"), [0.5, 0.5])


def test_cli_path_interpolate(cuda, frame_dir, tmp_path):
    import cv2
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    frames = _decoded(frame_dir)
    paths = sorted(os.listdir(frame_dir))
    for keep in (True, False):
        out = tmp_path / f"out{int(keep)}"
        argv = [sys.executable, cli, "--path", frame_dir, "--out", str(out), "--load", npz, "--iters", "4",
                "--interpolate", "0.5", "--batch", "4"] + (["--keep-size"] if keep else [])
        r = subprocess.run(argv, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        assert sorted(os.listdir(out)) == [f"frame_{n:06d}.png" for n in range(2 * len(frames) - 1)]
        for k in (0, 4, len(frames) - 1):
            want = frames[k] if keep else cv2.resize(frames[k], dsize=(1024, 432))
            assert np.array_equal(cv2.imread(str(out / f"frame_{2 * k:06d}.png")), want), (keep, k)
        for k in (0, 5):  # the single-pair CLI's PNG of the same pair
            one = tmp_path / f"one{int(keep)}_{k}"
            one.mkdir()
            argv = [sys.executable, cli, "--im1", os.path.join(frame_dir, paths[k]), "--im2",
                    os.path.join(frame_dir, paths[k + 1]), "--load", npz, "--iters", "4", "--interpolate", "0.5"]
            r = subprocess.run(argv + (["--keep-size"] if keep else []), cwd=one, env=env, capture_output=True, text=True,
                               timeout=600)
            assert r.returncode == 0, r.stderr[-3000:]
            assert (out / f"frame_{2 * k + 1:06d}.png").read_bytes() == (one / "raft_interp_0.png").read_bytes(), (keep, k)
