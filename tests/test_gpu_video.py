"""F11 on the GPU: rb_flow_to_color against the oracle (tests/flowviz_oracle.py: bit for bit on every non-ambiguous pixel,
within 1 LSB on the ambiguous ones), its batch invariance and argument errors; RaftEngine.forward_sequence against
per-pair forward calls bit for bit (fresh, carry, interleaved with the pair modes, warm-started), its carry errors; and
raft_b200.video / infer_raft.py --path end to end on shifted crops of tests/data/frame_0016.png."""
import ctypes
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import flowviz_oracle
from test_video import _golden_cases, raft_like

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


def _color(flows, clip=None, bgr=False):
    from networks.utils import flow_to_color
    return flow_to_color(torch.from_numpy(np.ascontiguousarray(flows)).cuda(), clip, bgr).cpu().numpy()


# ---- rb_flow_to_color ---------------------------------------------------------------------------------------------
def test_golden_cases(cuda):
    n = 0
    for name, flow, clip, _ in _golden_cases():
        if flow.dtype != np.float32:
            continue
        for bgr in (False, True):
            flowviz_oracle.assert_matches(_color(flow[None], clip, bgr), flow[None], clip, bgr)
            n += 1
    assert n >= 10


def test_clip_on_raft_like_flows(cuda):
    rng = np.random.default_rng(5)
    f = np.stack([raft_like(rng, 64, 80) for _ in range(2)])
    for clip in (0.0, 3.0, 25.0):
        flowviz_oracle.assert_matches(_color(f, clip, True), f, clip, True)


def test_zero_flow_and_single_pixel(cuda):
    z = np.zeros((1, 7, 9, 2), np.float32)
    got = _color(z)
    flowviz_oracle.assert_matches(got, z)
    assert (got == 255).all()
    one = np.zeros((1, 31, 17, 2), np.float32)
    one[0, 12, 5] = (-3.25, 1.5)
    for bgr in (False, True):
        flowviz_oracle.assert_matches(_color(one, None, bgr), one, None, bgr)


def test_raft_flow_full_size(cuda):
    from raft_b200 import synth
    m = _model()
    l, r = synth.make_batch(1, 436, 1024)
    flow = m.forward(l, r)
    host = flow.cpu().numpy()
    from networks.utils import flow_to_color
    amb = flowviz_oracle.assert_matches(flow_to_color(flow, convert_to_bgr=True).cpu().numpy(), host, None, True)
    assert amb < host.size // 200


def test_batch_equals_per_sample(cuda):
    rng = np.random.default_rng(11)
    f = np.stack([raft_like(rng, 45, 300) * s for s in (1.0, 0.01, 40.0, 3.0)])
    f[2, 7, 9] = 500.0  # one sample with an outlier that sets its own maximum
    whole = _color(f, None, True)
    for b in range(len(f)):
        assert np.array_equal(whole[b], _color(f[b:b + 1], None, True)[0]), b
    flowviz_oracle.assert_matches(whole, f, None, True)


def test_argument_errors(cuda):
    from networks.utils import flow_to_color
    from raft_b200 import capi
    lib = capi.lib
    f = torch.zeros(2, 8, 8, 2, device="cuda")
    out = torch.empty(2, 8, 8, 3, dtype=torch.uint8, device="cuda")
    nbytes = capi.size_query(lib.rb_flow_to_color_workspace_bytes, 2, 8, 8)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    st = capi.stream()
    P = capi.ptr
    assert lib.rb_flow_to_color(None, 2, 8, 8, 0, 0.0, 0, P(out), P(ws), nbytes, st) == -2
    assert lib.rb_flow_to_color(P(f), 2, 8, 8, 0, 0.0, 0, None, P(ws), nbytes, st) == -2
    assert lib.rb_flow_to_color(P(f), 0, 8, 8, 0, 0.0, 0, P(out), P(ws), nbytes, st) == -1
    assert lib.rb_flow_to_color(P(f), 2, 8, -1, 0, 0.0, 0, P(out), P(ws), nbytes, st) == -1
    assert lib.rb_flow_to_color(P(f), 2, 8, 8, 1, float("nan"), 0, P(out), P(ws), nbytes, st) == -2
    assert lib.rb_flow_to_color(P(f), 2, 8, 8, 0, 0.0, 0, P(out), P(ws), nbytes - 1, st) == -5
    assert lib.rb_flow_to_color_workspace_bytes(2, 8, 8, None) == -2
    assert lib.rb_flow_to_color_workspace_bytes(2, 0, 8, ctypes.byref(ctypes.c_size_t())) == -1
    for bad in (f.cpu(), f[..., :1], f.double(), f[0]):
        with pytest.raises(ValueError):
            flow_to_color(bad)


# ---- forward_sequence --------------------------------------------------------------------------------------------
def _frames(n, H, W, seed=3000, u8=True):
    rng = np.random.default_rng(seed)
    from raft_b200 import synth
    base, _ = synth.make_batch(1, H + 4 * n, W + 4 * n, seed0=seed)
    out = []
    for k in range(n):  # a camera pan with a little noise
        y, x = 2 * k + int(rng.integers(0, 2)), 3 * k
        out.append(base[0, y:y + H, x:x + W])
    f = np.stack(out).astype(np.float32)
    return (np.clip(np.rint(f * 255), 0, 255).astype(np.uint8) if u8 else f)


def _per_pair(m, frames, **kw):
    return [m.forward(frames[k:k + 1], frames[k + 1:k + 2], **kw) for k in range(len(frames) - 1)]


def _assert_pairs(got, frames, m):
    want = _per_pair(m, frames)
    assert got.shape[0] == len(want)
    for k, w in enumerate(want):
        assert torch.equal(got[k], w[0]), k


VARIANTS = {"default": {}, "upstream": {"upstream": True}, "mixed": {"mixed_precision": True}}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("small", [False, True])
def test_sequence_equals_pairs(cuda, small, variant):
    m = _model(small, **VARIANTS[variant])
    frames = _frames(4, 125, 150)  # not a multiple of 8; >= 121 for the upstream lookup
    _assert_pairs(m.forward_sequence(frames), frames, m)


@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("input_size", [None, (128, 160)])
def test_sequence_frame_inputs(cuda, u8, input_size):
    m = _model(input_size=input_size)
    frames = _frames(4, 100, 140, seed=3100, u8=u8)
    _assert_pairs(m.forward_sequence(frames), frames, m)
    t = torch.from_numpy(frames).cuda()  # CUDA frames
    _assert_pairs(m.forward_sequence(t), frames, m)


@pytest.mark.parametrize("T", [1, 8])
def test_sequence_lengths(cuda, T):
    m = _model()
    frames = _frames(T + 1, 64, 96, seed=3200 + T)
    _assert_pairs(m.forward_sequence(frames), frames, m)


def test_carry_equals_one_fresh_call(cuda):
    frames = _frames(10, 72, 104, seed=3300)
    whole = _model().forward_sequence(frames)  # T = 9
    m = _model()
    parts = [m.forward_sequence(frames[:4])] + [m.forward_sequence(frames[i:i + 3], carry=True) for i in (4, 7)]
    assert torch.equal(torch.cat(parts), whole)
    one = _model()  # T = 1 carries
    parts = [one.forward_sequence(frames[:2])] + [one.forward_sequence(frames[i:i + 1], carry=True) for i in range(2, 10)]
    assert torch.equal(torch.cat(parts), whole)


def test_carry_across_pair_modes(cuda):
    """forward, forward_bidirectional and interpolate at the same frame size between carry calls break nothing, and their
    results equal those of fresh models."""
    frames = _frames(10, 72, 104, seed=3400)
    other = _frames(2, 72, 104, seed=3500)
    l, r = other[:1], other[1:]
    whole = _model().forward_sequence(frames)
    m = _model()
    got = [m.forward_sequence(frames[:4])]
    assert torch.equal(m.forward(l, r), _model().forward(l, r))
    got.append(m.forward_sequence(frames[4:7], carry=True))
    for a, b in zip(m.forward_bidirectional(l, r), _model().forward_bidirectional(l, r)):
        assert torch.equal(a, b)
    assert torch.equal(m.forward(l.astype(np.float32) / 255, r.astype(np.float32) / 255),
                       _model().forward(l.astype(np.float32) / 255, r.astype(np.float32) / 255))
    assert torch.equal(m.interpolate(l, r, 0.5), _model().interpolate(l, r, 0.5))
    got.append(m.forward_sequence(frames[7:10], carry=True))
    assert torch.equal(torch.cat(got), whole)
    assert torch.equal(m.forward(l, r), _model().forward(l, r))


def test_carry_errors(cuda):
    frames = _frames(5, 64, 96, seed=3600)
    m = _model()
    with pytest.raises(ValueError, match="none before"):
        m.forward_sequence(frames[:3], carry=True)
    m.forward_sequence(frames[:4])  # T = 3
    with pytest.raises(ValueError, match="another T"):
        m.forward_sequence(frames[:2], carry=True)
    with pytest.raises(ValueError, match="frame size"):
        m.forward_sequence(_frames(3, 64, 104), carry=True)
    with pytest.raises(ValueError, match="dtype"):
        m.forward_sequence(frames[:3].astype(np.float32) / 255, carry=True)
    m.forward_sequence(frames[2:5], carry=True)  # still continues
    big = _frames(2, 80, 96)
    m.forward(big[:1], big[1:])  # another frame size releases the sequence buffers
    with pytest.raises(ValueError, match="released"):
        m.forward_sequence(frames[:3], carry=True)
    m.forward_sequence(frames[:4])
    m.mixed_precision = True
    with pytest.raises(ValueError, match="mixed_precision"):
        m.forward_sequence(frames[:3], carry=True)
    m.mixed_precision = False
    m.upstream = True
    with pytest.raises(ValueError, match="upstream"):
        m.forward_sequence(frames[:3], carry=True)


def test_warm_stream_equals_forward_chain(cuda):
    from networks.utils import forward_interpolate
    frames = _frames(6, 72, 104, seed=3700)
    m, ref = _model(), _model()
    init, rinit = None, None
    for k in range(5):
        if k == 0:
            low, flow = m.forward_sequence(frames[:2], return_low=True)
        else:
            low, flow = m.forward_sequence(frames[k + 1:k + 2], carry=True, flow_init=init, return_low=True)
        rlow, rflow = ref.forward(frames[k:k + 1], frames[k + 1:k + 2], flow_init=rinit, return_low=True)
        assert torch.equal(flow, rflow) and torch.equal(low, rlow), k
        init, rinit = forward_interpolate(low), forward_interpolate(rlow)
    # a zero flow_init is the cold start
    z = torch.zeros(3, 9, 13, 2)
    assert torch.equal(m.forward_sequence(frames[:4], flow_init=z), torch.cat(_per_pair(ref, frames[:4])))


# ---- video() and the CLI -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def frame_dir(tmp_path_factory):
    import cv2
    src = cv2.imread(os.path.join(ROOT, "tests", "data", "frame_0016.png"))
    d = tmp_path_factory.mktemp("frames")
    for k in range(10):
        cv2.imwrite(str(d / f"frame_{k:04d}.png"), src[100 + k:100 + k + 124, 200 + 3 * k:200 + 3 * k + 150])
    return str(d)


def _decoded(d):
    import cv2
    from raft_b200.video import list_frames
    return np.stack([cv2.imread(p) for p in list_frames(d)])


def _files(d):
    return {n: open(os.path.join(d, n), "rb").read() for n in sorted(os.listdir(d))}


def _check_outputs(out, flo, frames, m, **kw):
    import cv2
    from flow_utils import read_flo
    want = [f.cpu().numpy()[0] for f in _per_pair(m, frames, **kw)] if not kw else None
    for k in range(len(frames) - 1):
        png = cv2.imread(os.path.join(out, f"flow_{k:06d}.png"))
        flow = read_flo(os.path.join(flo, f"flow_{k:06d}.flo"))
        if want is not None:
            assert np.array_equal(flow, want[k]), k
        flowviz_oracle.assert_matches(png[None], flow[None], None, True)


@pytest.mark.parametrize("batch", [1, 3, 8])
def test_video_end_to_end(cuda, frame_dir, tmp_path, batch):
    from raft_b200.video import video
    m = _model()
    frames = _decoded(frame_dir)
    a, b = tmp_path / "a", tmp_path / "b"
    wa = video(m, frame_dir, str(a / "png"), batch=batch, workers=4, flo=str(a / "flo"), npy=str(a / "npy"))
    assert len(wa) == 3 * 9
    _check_outputs(str(a / "png"), str(a / "flo"), frames, m)
    for k in range(9):
        assert np.array_equal(np.load(str(a / "npy" / f"flow_{k:06d}.npy")),
                              m.forward(frames[k:k + 1], frames[k + 1:k + 2]).cpu().numpy()[0])
    video(m, frame_dir, str(b / "png"), batch=batch, workers=0, flo=str(b / "flo"), npy=str(b / "npy"))
    for sub in ("png", "flo", "npy"):
        assert _files(str(a / sub)) == _files(str(b / sub)), sub


def test_video_warm_and_native_flow(cuda, frame_dir, tmp_path):
    import cv2
    from flow_utils import read_flo
    from networks.utils import forward_interpolate, resize_flow
    from raft_b200.video import video
    frames = _decoded(frame_dir)
    m = _model(input_size=(128, 160))
    video(m, frame_dir, str(tmp_path / "png"), batch=1, warm_start=True, flo=str(tmp_path / "flo"), native_flow=True)
    ref, init = _model(input_size=(128, 160)), None
    for k in range(9):
        low, flow = ref.forward(frames[k:k + 1], frames[k + 1:k + 2], flow_init=init, return_low=True)
        init = forward_interpolate(low)
        want = resize_flow(flow, frames.shape[1:3]).cpu().numpy()[0]
        got = read_flo(str(tmp_path / "flo" / f"flow_{k:06d}.flo"))
        assert np.array_equal(got, want), k
        png = cv2.imread(str(tmp_path / "png" / f"flow_{k:06d}.png"))
        flowviz_oracle.assert_matches(png[None], want[None], None, True)
    with pytest.raises(ValueError):
        video(m, frame_dir, str(tmp_path / "x"), batch=8, warm_start=True)


def _mixed_sizes(frame_dir, tmp_path):
    """A copy of frame_dir whose frame_0006.png is 8 rows short."""
    import cv2
    import shutil
    d = tmp_path / "mixed"
    shutil.copytree(frame_dir, d)
    bad = d / "frame_0006.png"
    cv2.imwrite(str(bad), cv2.imread(str(bad))[:-8])
    return str(d)


def test_video_size_mismatch_names_file(cuda, frame_dir, tmp_path):
    from raft_b200.video import video
    with pytest.raises(ValueError, match="frame_0006.png"):
        video(_model(), _mixed_sizes(frame_dir, tmp_path), str(tmp_path / "out"), batch=3, workers=2)


@pytest.mark.parametrize("entry,kw", [("video_interpolate", {"ts": [0.5]}), ("video_track", {"grid": 16})],
                         ids=["video_interpolate", "video_track"])
def test_interpolate_and_track_size_mismatch_names_file(cuda, frame_dir, tmp_path, entry, kw):
    import raft_b200.video as rv
    with pytest.raises(ValueError, match="frame_0006.png"):
        getattr(rv, entry)(_model(), _mixed_sizes(frame_dir, tmp_path), str(tmp_path / "out"), batch=3, workers=2, **kw)


@pytest.mark.parametrize("workers", [0, 4])
def test_video_write_error_reaches_caller(cuda, frame_dir, tmp_path, workers):
    from raft_b200.video import video
    out = tmp_path / "out"
    (out / "flow_000004.png").mkdir(parents=True)  # cv2.imwrite cannot write over a directory
    with pytest.raises(OSError, match="flow_000004.png"):
        video(_model(), frame_dir, str(out), batch=3, workers=workers)


def test_cli_path(cuda, frame_dir, tmp_path):
    import cv2
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    base = [sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", frame_dir, "--load", npz,
            "--iters", "4"]
    cli = base + ["--out", str(tmp_path / "out"), "--flo", str(tmp_path / "flo"), "--keep-size", "--batch", "4"]
    r = subprocess.run(cli, cwd=tmp_path, env=dict(os.environ, PYTHONNOUSERSITE="1"), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert sorted(os.listdir(tmp_path / "out")) == [f"flow_{k:06d}.png" for k in range(9)]
    _check_outputs(str(tmp_path / "out"), str(tmp_path / "flo"), _decoded(frame_dir), _model())
    # the default: frames resized to 432x1024 on the GPU
    r = subprocess.run(base + ["--out", str(tmp_path / "full")], cwd=tmp_path,
                       env=dict(os.environ, PYTHONNOUSERSITE="1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert cv2.imread(str(tmp_path / "full" / "flow_000000.png")).shape == (432, 1024, 3)
    assert len(os.listdir(tmp_path / "full")) == 9
