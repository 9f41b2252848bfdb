"""F16 on the GPU: rb_frame_synthesize_pairs_resized / _items_resized against the composition of the existing entries
(rb_frames_prepare, rb_flow_resize, a gather of the masks, rb_frame_synthesize_pairs / _items) and tests/native_oracle.py
bit for bit; RaftEngine's native=True against native=False at equal sizes and against the composition from
forward_bidirectional flows at other sizes; video_interpolate(native=True) and infer_raft.py --native-frames /
--flow-size end to end on shifted crops of tests/data/frame_0016.png."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import native_oracle as N
from test_gpu_video import _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)
from test_gpu_video_interp import _decoded, _model, _same, _weights
from test_video_interp import quantise

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")


# ---- the entries -------------------------------------------------------------------------------------------------
def _resized(i0, i1, f0, f1, e0, e1, ts, u8, bgr, samples=None):
    """One call of the new entries: pairs ([n,B,H,W,...] flows) or items (samples, [n,H,W,...] flows)."""
    from raft_b200 import capi
    from raft_b200.engine import _floats, _ints
    lib, P = capi.lib, capi.ptr
    B, Hs, Ws = i0.shape[:3]
    H, W = f0.shape[-3:-1]
    n = len(ts)
    shape = (n, B, Hs, Ws, 3) if samples is None else (n, Hs, Ws, 3)
    out = torch.empty(shape, dtype=torch.uint8 if u8 else torch.float32, device="cuda")
    args = (P(i0), P(i1), int(i0.dtype == torch.uint8), Hs, Ws, P(f0), P(f1), P(e0), P(e1), H, W)
    if samples is None:
        capi.check(lib.rb_frame_synthesize_pairs_resized(*args, _floats(ts), n, P(out), int(u8), int(bgr), B,
                                                         capi.stream()))
    else:
        capi.check(lib.rb_frame_synthesize_items_resized(*args, _ints(samples), _floats(ts), n, P(out), int(u8),
                                                         int(bgr), B, capi.stream()))
    return out


def _composition(i0, i1, f0, f1, e0, e1, ts, u8, bgr, samples=None):
    """The spec through the existing entries: prepare, rb_flow_resize, a gather of the masks, then the plain blend."""
    from raft_b200 import capi
    from raft_b200.engine import _floats, _ints
    from networks.utils import resize_flow
    lib, P = capi.lib, capi.ptr
    B, Hs, Ws = i0.shape[:3]
    H, W = f0.shape[-3:-1]
    n = len(ts)
    frames = []
    for x in (i0, i1):
        if x.dtype == torch.uint8:
            y = torch.empty(x.shape, dtype=torch.float32, device="cuda")
            capi.check(lib.rb_frames_prepare(P(x), 1, P(y), B, Hs, Ws, 0, 0, 0, 0, capi.stream()))
            x = y
        frames.append(x)
    ys = torch.from_numpy(N.nearest_index(H, Hs)).cuda()
    xs = torch.from_numpy(N.nearest_index(W, Ws)).cuda()
    flows = [resize_flow(f.reshape(-1, H, W, 2), (Hs, Ws)).contiguous() for f in (f0, f1)]
    masks = [e.reshape(-1, H, W)[:, ys][:, :, xs].contiguous() for e in (e0, e1)]
    shape = (n, B, Hs, Ws, 3) if samples is None else (n, Hs, Ws, 3)
    out = torch.empty(shape, dtype=torch.uint8 if u8 else torch.float32, device="cuda")
    args = (P(frames[0]), P(frames[1]), Hs, Ws, 0, 0, P(flows[0]), P(flows[1]), P(masks[0]), P(masks[1]))
    if samples is None:
        capi.check(lib.rb_frame_synthesize_pairs(*args, _floats(ts), n, P(out), int(u8), int(bgr), B, Hs, Ws,
                                                 capi.stream()))
    else:
        capi.check(lib.rb_frame_synthesize_items(*args, _ints(samples), _floats(ts), n, P(out), int(u8), int(bgr), B,
                                                 Hs, Ws, capi.stream()))
    return out


def _inputs(rng, B, H, W, Hs, Ws, n, frames_u8):
    if frames_u8:
        i0, i1 = (rng.integers(0, 256, (B, Hs, Ws, 3)).astype(np.uint8) for _ in range(2))
    else:
        i0, i1 = (rng.uniform(-0.1, 1.1, (B, Hs, Ws, 3)).astype(np.float32) for _ in range(2))  # clamps at both ends
    f0, f1 = (rng.normal(0, 3, (n, H, W, 2)).astype(np.float32) for _ in range(2))
    if H * W > 2:
        f0.reshape(-1)[rng.choice(f0.size, 3, replace=False)] = [np.nan, 1e6, -1e7]  # NaN and far out of the frame
        f1.reshape(-1)[rng.choice(f1.size, 2, replace=False)] = [np.nan, -np.inf]
    e0, e1 = ((rng.random((n, H, W)) < 0.3).astype(np.uint8) for _ in range(2))
    return i0, i1, f0, f1, e0, e1


SIZES = [((432, 1024), (1080, 1920)), ((37, 53), (100, 141)), ((100, 141), (37, 53)), ((40, 60), (40, 60)),
         ((1, 29), (7, 40)), ((23, 1), (30, 5)), ((16, 24), (16, 57))]


@pytest.mark.parametrize("frames_u8", [True, False])
@pytest.mark.parametrize("net,size", SIZES)
def test_resized_equals_composition(cuda, net, size, frames_u8):
    (H, W), (Hs, Ws) = net, size
    big = Hs * Ws > 1e6
    rng = np.random.default_rng(H * 7 + Ws + frames_u8)
    B = 2 if big else 3
    samples = [2, 0, 0, 1, 2, 1, 0, 2, 2] if not big else [1, 0, 1]
    ts = [0.0, 0.25, 1.0 / 3.0, 0.5, 1.0, 0.7, 0.1, 0.9, 0.5][:len(samples)]
    n = len(samples)
    arrays = _inputs(rng, B, H, W, Hs, Ws, n, frames_u8)
    g = [torch.from_numpy(a).cuda() for a in arrays]
    for u8, bgr in ((False, False), (True, True)):
        got = _resized(*g, ts, u8, bgr, samples)
        assert got.shape == (n, Hs, Ws, 3)
        assert _same(got, _composition(*g, ts, u8, bgr, samples)), (u8, bgr)
        # pairs: the first B * len(pt) flows as [len(pt), B, ...]
        pt = ts[:n // B]
        pg = g[:2] + [x[:len(pt) * B].reshape((len(pt), B) + x.shape[1:]) for x in g[2:]]
        assert _same(_resized(*pg, pt, u8, bgr), _composition(*pg, pt, u8, bgr)), (u8, bgr)


def test_resized_items_up_to_max_steps(cuda):
    rng = np.random.default_rng(64)
    B, H, W, Hs, Ws, n = 3, 20, 30, 45, 70, 64
    g = [torch.from_numpy(a).cuda() for a in _inputs(rng, B, H, W, Hs, Ws, n, True)]
    samples = [(7 * i) % 3 for i in range(n)]  # repeated and unsorted
    ts = [float(np.float32(t)) for t in rng.random(n)]
    ts[:2] = [0.0, 1.0]
    for u8, bgr in ((False, False), (True, False), (True, True)):
        assert _same(_resized(*g, ts, u8, bgr, samples), _composition(*g, ts, u8, bgr, samples)), (u8, bgr)


@pytest.mark.parametrize("frames_u8", [True, False])
@pytest.mark.parametrize("net,size", [((13, 17), (29, 41)), ((29, 41), (13, 17)), ((1, 9), (5, 14)), ((11, 1), (4, 6)),
                                      ((12, 16), (12, 16))])
def test_resized_equals_oracle(cuda, net, size, frames_u8):
    (H, W), (Hs, Ws) = net, size
    rng = np.random.default_rng(H * 13 + Ws)
    B, ts = 2, [0.0, 0.3, 0.5, 1.0]
    n = len(ts) * B
    arrays = _inputs(rng, B, H, W, Hs, Ws, n, frames_u8)
    i0, i1, f0, f1, e0, e1 = arrays
    g = [torch.from_numpy(a).cuda() for a in arrays]
    pg = g[:2] + [x.reshape((len(ts), B) + x.shape[1:]) for x in g[2:]]
    pairs = _resized(*pg, ts, False, False).cpu().numpy()
    pairs_u8 = _resized(*pg, ts, True, True).cpu().numpy()
    for j, t in enumerate(ts):
        rows = slice(j * B, (j + 1) * B)
        want = N.synthesize_resized(i0, i1, f0[rows], f1[rows], e0[rows], e1[rows], t)
        assert _same(pairs[j], want), t
        assert _same(pairs_u8[j], quantise(want, bgr=True)), t
        for b in range(B):  # items: every (sample, t) of the pairs call
            one = _resized(*g[:2], *(x[j * B + b:j * B + b + 1] for x in g[2:]), [t], False, False, [b])
            assert _same(one[0], pairs[j, b]), (t, b)


# ---- the engine --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("variant", ["things", "small", "upstream"])
def test_native_at_equal_size_equals_default(cuda, variant, u8):
    small = variant == "small"
    upstream = variant == "upstream"
    H, W = (125, 150) if upstream else (60, 100)
    m = _model(small, upstream=upstream, input_size=(H, W))
    frames = _frames(4, H, W, seed=6000, u8=u8)
    l, r = frames[:2], frames[1:3]
    ts, items = [0.0, 0.3, 1.0], [(2, 0.4), (0, 0.8), (1, 0.0), (2, 1.0)]
    assert _same(m.interpolate(l, r, ts, native=True), m.interpolate(l, r, ts))
    for u in (False, True):
        assert _same(m.interpolate_sequence(frames, ts, uint8=u, native=True), m.interpolate_sequence(frames, ts, uint8=u))
        assert _same(m.interpolate_sequence_at(frames, items, uint8=u, native=True),
                     m.interpolate_sequence_at(frames, items, uint8=u))


@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("u8", [True, False])
def test_native_equals_spec_from_bidirectional_flows(cuda, small, u8):
    from networks.utils import reverse_flow, synthesize_resized
    m = _model(small, input_size=(64, 96))
    frames = _frames(2, 100, 140, seed=6100, u8=u8)
    l, r = frames[:1], frames[1:]
    ts = [0.3, 0.5]
    got = m.interpolate(l, r, ts, native=True)
    assert got.shape == (2, 1, 100, 140, 3)
    fw, bw = (f.clone() for f in m.forward_bidirectional(l, r, check=False)[:2])
    s = 8.0 if small else 1.0
    raw = [torch.from_numpy(x).cuda() for x in (l, r)]
    for i, t in enumerate(ts):
        ft0, e0 = reverse_flow(fw, s * t)[:2]
        ft1, e1 = reverse_flow(bw, s * (1.0 - t))[:2]
        want = synthesize_resized(*raw, ft0, ft1, e0, e1, t)
        assert _same(got[i], want), t
        assert _same(synthesize_resized(*raw, ft0, ft1, e0, e1, t, uint8=True), quantise(want.cpu().numpy())), t


@pytest.mark.parametrize("u8", [True, False])
def test_native_sequence_equals_pairs(cuda, u8):
    m = _model(input_size=(64, 96))
    frames = _frames(4, 90, 130, seed=6200, u8=u8)
    ts = [0.0, 0.25, 0.5, 1.0]
    items = [(2, 0.4), (0, 0.0), (1, 1.0), (0, 0.4), (2, 0.9)]
    seq = m.interpolate_sequence(frames, ts, native=True)
    seq_u8 = m.interpolate_sequence(frames, ts, uint8=True, native=True)
    at = m.interpolate_sequence_at(frames, items, native=True)
    at_u8 = m.interpolate_sequence_at(frames, items, uint8=True, native=True)
    assert seq.shape == (4, 3, 90, 130, 3) and at.shape == (5, 90, 130, 3)
    for k in range(3):
        want = m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], ts, native=True)[:, 0]
        assert _same(seq[:, k], want), k
        assert _same(seq_u8[:, k], quantise(want.cpu().numpy())), k
    for i, (k, t) in enumerate(items):
        want = m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], t, native=True)[0]
        assert _same(at[i], want), (k, t)
        assert _same(at_u8[i], quantise(want.cpu().numpy())), (k, t)
    if u8:  # t = 0 and t = 1 give the frames themselves, byte for byte
        for k in range(3):
            assert _same(seq_u8[0, k], frames[k]) and _same(seq_u8[3, k], frames[k + 1]), k
        assert _same(at_u8[1], frames[0]) and _same(at_u8[2], frames[2])


def test_native_without_input_size_changes_nothing(cuda):
    m = _model()
    frames = _frames(3, 60, 100, seed=6300)
    assert _same(m.interpolate(frames[:1], frames[1:2], [0.5], native=True), m.interpolate(frames[:1], frames[1:2], [0.5]))
    assert _same(m.interpolate_sequence(frames, [0.5], uint8=True, native=True),
                 m.interpolate_sequence(frames, [0.5], uint8=True))
    assert _same(m.interpolate_sequence_at(frames, [(1, 0.3)], native=True), m.interpolate_sequence_at(frames, [(1, 0.3)]))


# ---- video_interpolate and the CLI -------------------------------------------------------------------------------
SIZE = (72, 96)  # the frame_dir frames are 124x150


def _run_cli(argv, cwd):
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, CLI] + argv, cwd=cwd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]


def test_video_interpolate_native(cuda, frame_dir, tmp_path):
    import cv2
    from raft_b200.video import frame_number, list_frames, video_interpolate
    m = _model(input_size=SIZE)
    frames = _decoded(frame_dir)
    ts = [0.25, 0.5]
    runs = {}
    for batch, workers in ((1, 0), (3, 4), (8, 4)):
        out = tmp_path / f"ts_b{batch}w{workers}"
        video_interpolate(m, frame_dir, str(out), ts, batch=batch, workers=workers, native=True)
        runs[(batch, workers)] = _files(str(out))
    first = next(iter(runs.values()))
    assert all(r == first for r in runs.values())
    out = str(tmp_path / "ts_b3w4")
    for k in range(len(frames) - 1):
        assert np.array_equal(cv2.imread(os.path.join(out, f"frame_{frame_number(k, 2):06d}.png")), frames[k]), k
        want = quantise(m.interpolate(frames[k:k + 1], frames[k + 1:k + 2], ts, native=True).cpu().numpy()[:, 0])
        for j in range(2):
            got = cv2.imread(os.path.join(out, f"frame_{frame_number(k, 2, j):06d}.png"))
            assert got.shape == frames[k].shape and np.array_equal(got, want[j]), (k, j)
    assert np.array_equal(cv2.imread(os.path.join(out, f"frame_{frame_number(len(frames) - 1, 2):06d}.png")), frames[-1])

    # the single-pair CLI's --native-frames PNGs of pair 3 are the same bytes
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    paths = list_frames(frame_dir)
    cwd = tmp_path / "pair"
    cwd.mkdir()
    _run_cli(["--im1", paths[3], "--im2", paths[4], "--load", npz, "--iters", "4", "--interpolate", "0.25", "0.5",
              "--native-frames", "--flow-size", str(SIZE[0]), str(SIZE[1])], str(cwd))
    for j in range(2):
        assert (cwd / f"raft_interp_{j}.png").read_bytes() == first[f"frame_{frame_number(3, 2, j):06d}.png"], j

    # frame-rate conversion, and scene-cut copies at the decoded size
    fps_runs = {}
    for batch, workers in ((1, 0), (8, 4)):
        out = tmp_path / f"fps_b{batch}w{workers}"
        video_interpolate(m, frame_dir, str(out), batch=batch, workers=workers, fps=(24, 60), native=True)
        fps_runs[(batch, workers)] = _files(str(out))
    fps_first = next(iter(fps_runs.values()))
    assert all(r == fps_first for r in fps_runs.values())
    got = cv2.imread(str(tmp_path / "fps_b1w0" / "frame_000001.png"))  # s = 0.4 between frames 0 and 1
    want = quantise(m.interpolate(frames[:1], frames[1:2], 0.4, native=True).cpu().numpy()[0])
    assert np.array_equal(got, want)
    assert np.array_equal(cv2.imread(str(tmp_path / "fps_b1w0" / "frame_000005.png")), frames[2])
    cut_out = tmp_path / "cuts"
    _, cuts = video_interpolate(m, frame_dir, str(cut_out), [0.25, 0.75], batch=3, native=True, scene_cut=0.0)
    assert cuts
    k = cuts[0]
    for j, src in ((0, k), (1, k + 1)):
        assert np.array_equal(cv2.imread(str(cut_out / f"frame_{frame_number(k, 2, j):06d}.png")), frames[src]), j

    # the CLI over the directory writes the same files
    cli_out = tmp_path / "cli"
    _run_cli(["--path", frame_dir, "--out", str(cli_out), "--load", npz, "--iters", "4", "--input-fps", "24", "--fps",
              "60", "--native-frames", "--flow-size", str(SIZE[0]), str(SIZE[1]), "--batch", "3"], str(tmp_path))
    cli_files = _files(str(cli_out))
    assert cli_files == fps_first
    assert all(cv2.imread(str(cli_out / n)).shape == frames[0].shape for n in cli_files)
