"""F14 on the GPU: rb_flow_reverse_items against per-item rb_flow_reverse_multi and tests/interp_oracle.py,
rb_frame_synthesize_items against per-item rb_frame_synthesize_pairs, RaftEngine.interpolate_sequence_at against
per-pair interpolate bit for bit, chunk-bound invariance, mode alternation, and video_interpolate(fps=...) /
infer_raft.py --path --input-fps --fps end to end on shifted crops of tests/data/frame_0016.png."""
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

import interp_oracle as O
from test_gpu_video import _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)
from test_gpu_video_interp import _decoded, _model, _reverse_multi, _same, _synth_pairs, _weights
from test_video_interp import quantise

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- rb_flow_reverse_items ---------------------------------------------------------------------------------------
def _reverse_items(flow, samples, steps):
    from raft_b200 import capi
    from raft_b200.engine import _floats, _ints
    lib, P = capi.lib, capi.ptr
    B, H, W = flow.shape[:3]
    n = len(steps)
    nbytes = capi.size_query(lib.rb_flow_reverse_multi_workspace_bytes, n, 1, H, W)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=flow.device)
    ft = torch.empty(n, H, W, 2, device=flow.device)
    em = torch.empty(2, n, H, W, dtype=torch.uint8, device=flow.device)
    capi.check(lib.rb_flow_reverse_items(P(flow), B, _ints(samples), _floats(steps), n, P(ft), P(em[0]), P(em[1]), H, W,
                                         P(ws), nbytes, capi.stream()))
    return ft.cpu().numpy(), em[0].cpu().numpy(), em[1].cpu().numpy()


@pytest.mark.parametrize("B,H,W,n", [(3, 37, 53, 64), (2, 1, 29, 9), (1, 23, 1, 5), (4, 64, 96, 1), (3, 31, 45, 13)])
def test_reverse_items_equals_multi(cuda, B, H, W, n):
    rng = np.random.default_rng(B * 1000 + H * 10 + W + n)
    f = (rng.normal(0, 3, (B, H, W, 2)) * rng.uniform(0.2, 2, (B, 1, 1, 2))).astype(np.float32)
    if H * W > 1:
        for v in (np.nan, np.inf, -np.inf):
            f.reshape(-1)[rng.choice(f.size, 3, replace=False)] = v
    if B > 1:  # one sample whose every source lands on the same border pixels: collisions there, holes elsewhere
        f[-1] = np.float32(1e4)
    samples = [int(s) for s in rng.integers(0, B, n)]  # repeated and unsorted
    if n > 2:
        samples[:3] = [B - 1, 0, B - 1]
    # 0, ordinary steps, negative, raft-small's x8 and 1e6 (every source leaves the frame and clamps to the border)
    steps = [float(np.float32(s)) for s in rng.choice([0.0, 0.25, 0.5, 1.0 / 3.0, -0.75, 8 * 0.6, 1e6], n)]
    flow = torch.from_numpy(f).cuda()
    ft, em, mu = _reverse_items(flow, samples, steps)
    for i, (b, s) in enumerate(zip(samples, steps)):
        one = _reverse_multi(flow[b:b + 1], [s])
        assert _same(ft[i], one[0][0, 0]) and _same(em[i], one[1][0, 0]) and _same(mu[i], one[2][0, 0]), (i, b, s)
        ref = O.reverse_flow(f[b:b + 1], time_step=s)
        assert _same(ft[i], ref[0][0]) and _same(em[i], ref[1][0]) and _same(mu[i], ref[2][0]), (i, b, s)
    if B > 1 and H * W > 1:
        assert any(e.any() for e in em) and any(m.any() for m in mu)  # holes and collisions were exercised


# ---- rb_frame_synthesize_items -----------------------------------------------------------------------------------
def _synth_items(i0, i1, f0, f1, e0, e1, samples, ts, u8, bgr, pad=(0, 0)):
    from raft_b200 import capi
    from raft_b200.engine import _floats, _ints
    lib, P = capi.lib, capi.ptr
    B, Hp, Wp = i0.shape[:3]
    H, W = f0.shape[1:3]
    out = torch.empty(len(ts), H, W, 3, dtype=torch.uint8 if u8 else torch.float32, device="cuda")
    capi.check(lib.rb_frame_synthesize_items(P(i0), P(i1), Hp, Wp, pad[0], pad[1], P(f0), P(f1), P(e0), P(e1),
                                             _ints(samples), _floats(ts), len(ts), P(out), int(u8), int(bgr), B, H, W,
                                             capi.stream()))
    return out.cpu().numpy()


def test_synthesize_items_equals_pairs(cuda):
    rng = np.random.default_rng(19)
    B, H, W, top, left = 3, 31, 47, 2, 3
    samples = [2, 0, 0, 1, 2, 1, 0, 2, 2]
    ts = [0.0, 0.25, 1.0 / 3.0, 0.5, 1.0, 0.7, 0.1, 0.9, 0.5]
    n = len(ts)
    i0, i1 = (rng.uniform(-0.1, 1.1, (B, H + 5, W + 4, 3)).astype(np.float32) for _ in range(2))  # clamps at both ends
    i0[0, 5, 6] = np.nan  # NaN through the blend -> 0
    i1[2, 7, 8] = np.inf
    f0, f1 = (rng.normal(0, 4, (n, H, W, 2)).astype(np.float32) for _ in range(2))
    e0, e1 = ((rng.random((n, H, W)) < 0.3).astype(np.uint8) for _ in range(2))
    g = [torch.from_numpy(a).cuda() for a in (i0, i1, f0, f1, e0, e1)]
    for u8, bgr in ((False, False), (True, False), (True, True)):
        got = _synth_items(*g, samples, ts, u8, bgr, (top, left))
        for i, (b, t) in enumerate(zip(samples, ts)):
            want = _synth_pairs(g[0][b:b + 1], g[1][b:b + 1], *(x[i:i + 1, None] for x in g[2:]), [t], u8, bgr,
                                (top, left))
            assert _same(got[i], want[0, 0]), (u8, bgr, i)
        if u8:
            assert (got == 0).any() and (got == 255).any()


# ---- interpolate_sequence_at -------------------------------------------------------------------------------------
ITEMS = [(2, 0.4), (0, 0.8), (1, 0.2), (0, 0.4), (2, 1.0), (1, 0.0), (0, 0.4), (1, 0.6)]


def _check_at(m, frames, items):
    got = m.interpolate_sequence_at(frames, items)
    got_u8 = m.interpolate_sequence_at(frames, items, uint8=True)
    assert got.shape[0] == len(items) and got.dtype == torch.float32 and got_u8.dtype == torch.uint8
    for i, (k, t) in enumerate(items):
        want = m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], t)[0]
        assert _same(got[i], want), (k, t)
        assert _same(got_u8[i], quantise(want.cpu().numpy())), (k, t)
    assert _same(m.interpolate_sequence_at(frames, items, uint8=True, bgr=True), got_u8.flip(-1))
    return got


@pytest.mark.parametrize("upstream", [False, True])
@pytest.mark.parametrize("small", [False, True])
def test_interpolate_sequence_at_equals_pairs(cuda, small, upstream):
    if upstream:
        _check_at(_model(small, upstream=True), _frames(4, 125, 150, seed=5000), ITEMS)
    else:
        _check_at(_model(small), _frames(4, 60, 100, seed=5010), ITEMS)  # odd: replicate padding on both axes


@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("input_size", [None, (128, 160)])
def test_interpolate_sequence_at_frame_inputs(cuda, u8, input_size):
    _check_at(_model(input_size=input_size), _frames(4, 100, 140, seed=5100, u8=u8), ITEMS[:5])


def test_interpolate_sequence_at_refusals(cuda):
    m = _model()
    frames = _frames(3, 64, 96, seed=5200)
    for bad in ([], [(2, 0.5)], [(-1, 0.5)], [(0, 1.5)], [(0, float("nan"))]):
        with pytest.raises(ValueError):
            m.interpolate_sequence_at(frames, bad)
    with pytest.raises(ValueError, match="uint8"):
        m.interpolate_sequence_at(frames, [(0, 0.5)], bgr=True)


def test_interpolate_sequence_at_chunk_bound_changes_no_bit(cuda, monkeypatch):
    from raft_b200 import engine
    frames = _frames(4, 64, 96, seed=5300)
    rng = np.random.default_rng(5300)
    items = [(int(k), float(t)) for k, t in zip(rng.integers(0, 3, 70), rng.random(70))]  # 70 > RB_INTERP_MAX_STEPS
    m = _model()
    whole = m.interpolate_sequence_at(frames, items)
    seq = m.interpolate_sequence(frames, [0.25, 0.5])
    monkeypatch.setattr(engine, "REVERSE_WS_BOUND", 1)  # one item per chunk
    assert _same(m.interpolate_sequence_at(frames, items), whole)
    monkeypatch.setattr(engine, "REVERSE_WS_BOUND",
                        engine.capi.size_query(engine.capi.lib.rb_flow_reverse_multi_workspace_bytes, 3, 1, 64, 96))
    assert _same(m.interpolate_sequence_at(frames, items), whole)  # chunks of 3
    assert _same(m.interpolate_sequence(frames, [0.25, 0.5]), seq)  # one time (3 pairs) per chunk
    for i in (0, 33, 69):
        k, t = items[i]
        assert _same(whole[i], m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], t)[0]), i


def test_alternating_modes(cuda):
    frames = _frames(5, 72, 104, seed=5400)
    other = _frames(2, 72, 104, seed=5500)
    l, r = other[:1], other[1:]
    ts = [0.3, 0.6]
    items = [(3, 0.5), (0, 0.25), (3, 0.75)]
    ref = _model()
    want_at = ref.interpolate_sequence_at(frames, items)
    want_seq = ref.interpolate_sequence(frames, ts)
    want_bi = ref.forward_sequence_bidirectional(frames)
    want_fw, want_i = ref.forward(l, r), ref.interpolate(l, r, ts)
    whole = ref.forward_sequence(frames)
    m = _model()
    got = [m.forward_sequence(frames[:3])]  # T = 2, then a carry across the other modes
    assert _same(m.interpolate_sequence_at(frames, items), want_at)
    assert _same(m.interpolate_sequence(frames, ts), want_seq)
    assert _same(m.interpolate_sequence_at(frames, items), want_at)
    assert _same(m.forward(l, r), want_fw)
    assert _same(m.interpolate(l, r, ts), want_i)
    got.append(m.forward_sequence(frames[3:5], carry=True))
    assert _same(torch.cat(got), whole)
    for a, b in zip(m.forward_sequence_bidirectional(frames), want_bi):
        assert _same(a, b)
    assert _same(m.interpolate_sequence_at(frames, items[:1]), want_at[:1])  # another item count
    assert _same(m.interpolate_sequence_at(frames[2:5], [(1, 0.5)])[0], ref.interpolate(frames[3:4], frames[4:5], 0.5)[0])
    assert _same(m.interpolate_sequence_at(frames, items), want_at)


# ---- video_interpolate(fps=...) and the CLI ----------------------------------------------------------------------
def _check_fps_files(out, frames, m, fin, fout):
    """Every file of a conversion: input frame s at an integer s, else the quantised interpolate of its pair."""
    import cv2
    ratio = Fraction(fin) / Fraction(fout)
    n_out = (len(frames) - 1) * Fraction(fout) / Fraction(fin)
    n_out = n_out.numerator // n_out.denominator + 1
    assert sorted(os.listdir(out)) == [f"frame_{n:06d}.png" for n in range(n_out)]
    for n in range(n_out):
        s = n * ratio
        k = s.numerator // s.denominator
        got = cv2.imread(os.path.join(out, f"frame_{n:06d}.png"))
        if s.denominator == 1:
            assert np.array_equal(got, frames[k]), n
        else:
            want = quantise(m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], float(s - k)).cpu().numpy()[0])
            assert np.array_equal(got, want), n


def test_video_interpolate_fps(cuda, frame_dir, tmp_path):
    from raft_b200.video import video_interpolate
    m = _model()
    frames = _decoded(frame_dir)
    runs = {}
    for batch, workers in ((1, 0), (3, 4), (8, 4)):
        out = tmp_path / f"b{batch}w{workers}"
        written = video_interpolate(m, frame_dir, str(out), batch=batch, workers=workers, fps=(24, 60))
        assert sorted(os.listdir(out)) == [os.path.basename(p) for p in written]
        runs[(batch, workers)] = _files(str(out))
    first = next(iter(runs.values()))
    assert all(r == first for r in runs.values())
    _check_fps_files(str(tmp_path / "b3w4"), frames, m, 24, 60)
    for kw in ({}, {"ts": [0.5], "fps": (24, 60)}, {"fps": (60, 24)}, {"fps": (24, 24)}):
        with pytest.raises(ValueError):
            video_interpolate(m, frame_dir, str(tmp_path / "x"), **kw)


def test_cli_path_fps(cuda, frame_dir, tmp_path):
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    runs = []
    for batch in (1, 8):
        out = tmp_path / f"out{batch}"
        argv = [sys.executable, cli, "--path", frame_dir, "--out", str(out), "--load", npz, "--iters", "4",
                "--input-fps", "24", "--fps", "60", "--keep-size", "--batch", str(batch)]
        r = subprocess.run(argv, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        runs.append(_files(str(out)))
    assert runs[0] == runs[1]
    _check_fps_files(str(tmp_path / "out8"), _decoded(frame_dir), _model(), 24, 60)
