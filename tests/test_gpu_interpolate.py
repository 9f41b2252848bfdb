"""F6: frame interpolation on the GPU.

rb_flow_reverse must equal the reference's flow reversal (tests/golden/reverse_flow.npz) and the numpy restatement
(tests/interp_oracle.py) bit for bit, be batch-invariant, deterministic and graph-capturable; rb_frame_synthesize must
equal its restatement bit for bit; RAFT.interpolate must equal the restatements applied to forward_bidirectional's flows,
return the frames themselves at t = 0 and 1, and give fresh results when it alternates with the other modes."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import interp_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reverse_flow.npz")
NAMES = sorted({k.split("/")[0] for k in np.load(GOLDEN).files})


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b)


def _np(ts):
    return [t.cpu().numpy() for t in ts]


@pytest.mark.parametrize("name", NAMES)
def test_mirror_equals_reference(cuda, name):
    import flow_utils
    g = np.load(GOLDEN)
    res = flow_utils.reverse_flow_avg_skip_static(g[f"{name}/flow"], g[f"{name}/bg"], g[f"{name}/im0"],
                                                  float(g[f"{name}/time_step"]))
    for k, r in enumerate(res):
        assert _same(r, g[f"{name}/out{k}"]), (name, k)


def _gpu(flow, ts, bg=None, im0=None):
    from networks.utils import reverse_flow
    dev = torch.device("cuda:0")
    t = [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (flow, bg, im0)]
    return _np(reverse_flow(t[0], ts, t[1], t[2]))


def _check_restatement(flow, ts, bg=None, im0=None):
    got = _gpu(flow, ts, bg, im0)
    ref = O.reverse_flow(flow, bg, im0, ts)
    ref = ref[:3] + (ref[3].astype(np.uint8), ref[4])
    for k, (g, r) in enumerate(zip(got, ref)):
        assert _same(g, r), (k, int((g != r).sum()))
    return got


def _flows(rng, B, H, W, special=True):
    f = (rng.normal(0, 3, (B, H, W, 2)) * rng.uniform(0.2, 2, (B, 1, 1, 2))).astype(np.float32)  # differs per sample
    if special:
        for v in (np.nan, np.inf, -np.inf):
            f.reshape(-1)[rng.choice(f.size, 7, replace=False)] = v
    return f


@pytest.mark.parametrize("ts", [1.0, 0.5, 1.0 / 3.0, -0.5, 8 * 0.25])
@pytest.mark.parametrize("B,H,W", [(3, 37, 53), (3, 1, 29), (2, 23, 1), (1, 1, 1)])
def test_reverse_equals_restatement(cuda, B, H, W, ts):
    rng = np.random.default_rng(B * 7 + H * 3 + W)
    _check_restatement(_flows(rng, B, H, W, special=H * W > 1), ts)


@pytest.mark.parametrize("u8", [True, False])
def test_reverse_static_images(cuda, u8):
    rng = np.random.default_rng(11)
    B, H, W = 3, 29, 41
    flow = _flows(rng, B, H, W)
    if u8:
        im0 = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
        bg = ((im0.astype(np.int64) + rng.integers(-12, 13, (B, H, W, 1))) % 256).astype(np.uint8)
    else:
        im0 = rng.uniform(0, 255, (B, H, W, 3)).astype(np.float32)
        bg = (im0 + rng.normal(0, 6, (B, H, W, 1))).astype(np.float32)
    got = _check_restatement(flow, 0.5, bg, im0)
    assert 0 < got[3].sum() < got[3].size


@pytest.mark.parametrize("H,W", [(64, 96), (436, 1024)])
def test_reverse_all_sources_on_one_pixel(cuda, H, W):
    """Every source lands on (0, 0) with magnitudes 1e-3 .. 1e3: one thread sums H*W values in raster order."""
    rng = np.random.default_rng(H)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    mag = (10.0 ** rng.uniform(-3, 3, (H, W, 2))).astype(np.float32)
    flow = np.stack([-(xx + mag[..., 0]), -(yy + mag[..., 1])], -1)[None].astype(np.float32)
    got = _check_restatement(flow, 1.0)
    assert got[1].sum() == H * W - 1 and got[2][0, 0, 0] == 1


def test_reverse_raft_flow_full_size(cuda):
    from networks.RAFT import RAFT
    from raft_b200 import synth
    H, W = 436, 1024
    l, r = synth.make_batch(1, H, W)
    m = RAFT((H, W, 3), SimpleNamespace(small=False), iters=4, device=cuda).load(synth.make_weights(False))
    flow = m.forward(l, r).cpu().numpy()
    for ts in (0.5, 1.0):
        _check_restatement(flow, ts)


def test_batched_deterministic_and_graph_captured(cuda):
    from networks.utils import reverse_flow
    rng = np.random.default_rng(3)
    B, H, W = 3, 45, 67
    flow = torch.from_numpy(_flows(rng, B, H, W)).to(cuda)
    a = _np(reverse_flow(flow, 0.75))
    b = _np(reverse_flow(flow, 0.75))
    assert all(_same(x, y) for x, y in zip(a, b))
    for i in range(B):
        one = _np(reverse_flow(flow[i:i + 1], 0.75))
        assert all(_same(x, y[i:i + 1]) for x, y in zip(one, a))
    reverse_flow(flow, 0.75)  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = reverse_flow(flow, 0.75)
    g.replay()
    torch.cuda.synchronize()
    assert all(_same(x, y) for x, y in zip(_np(outs), a))


def test_synthesize_equals_restatement(cuda):
    from networks.utils import synthesize
    rng = np.random.default_rng(4)
    B, H, W = 3, 31, 47
    i0, i1 = (rng.uniform(0, 1, (B, H, W, 3)).astype(np.float32) for _ in range(2))
    f0, f1 = (_flows(rng, B, H, W) * np.float32(3) for _ in range(2))  # many leave the frame; NaN and +-inf
    e0, e1 = ((rng.random((B, H, W)) < 0.3).astype(np.uint8) for _ in range(2))
    assert ((e0 == 1) & (e1 == 1)).any() and ((e0 == 1) & (e1 == 0)).any() and ((e0 == 0) & (e1 == 1)).any()
    dev = cuda
    for t in (0.0, 0.25, 1.0 / 3.0, 0.5, 1.0):
        got = synthesize(*(torch.from_numpy(a).to(dev) for a in (i0, i1, f0, f1, e0, e1)), t).cpu().numpy()
        assert _same(got, O.synthesize(i0, i1, f0, f1, e0, e1, t)), t
    with pytest.raises(ValueError):
        synthesize(*(torch.from_numpy(a).to(dev) for a in (i0, i1, f0, f1, e0, e1)), 1.5)


def _model(p, small, H, W, B, cuda):
    from networks.RAFT import RAFT
    return RAFT((H, W, 3), SimpleNamespace(small=small), iters=4, batch=B, device=cuda).load(p)


def _frames(B, H, W, u8, seed0=None):
    from raft_b200 import synth
    l, r = synth.make_batch(B, H, W) if seed0 is None else synth.make_batch(B, H, W, seed0=seed0)
    if u8:
        l, r = (np.round(l * 255).astype(np.uint8), np.round(r * 255).astype(np.uint8))
    return l, r


def _as_f32(x):
    return x.astype(np.float32) / np.float32(255) if x.dtype == np.uint8 else x


def _expected(fw, bw, l, r, t, small):
    s = 8.0 if small else 1.0
    f0, e0 = O.reverse_flow(fw, time_step=s * t)[:2]
    f1, e1 = O.reverse_flow(bw, time_step=s * (1.0 - t))[:2]
    return O.synthesize(_as_f32(l), _as_f32(r), f0, f1, e0, e1, t)


@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("H,W", [(64, 96), (60, 100)])
def test_interpolate(cuda, small, H, W):
    from raft_b200 import synth
    p = synth.make_weights(small)
    B = 2
    for u8 in (False, True):
        l, r = _frames(B, H, W, u8)
        m = _model(p, small, H, W, B, cuda)
        fw, bw, _, _ = (None if x is None else x.cpu().numpy() for x in
                        _model(p, small, H, W, B, cuda).forward_bidirectional(l, r, check=False))
        ends = m.interpolate(l, r, [0.0, 1.0]).cpu().numpy()
        assert ends.shape == (2, B, H, W, 3) and ends.dtype == np.float32
        assert _same(ends[0], _as_f32(l)) and _same(ends[1], _as_f32(r)), u8
        ts = [0.25, 0.5, 0.75]
        many = m.interpolate(l, r, ts).cpu().numpy()
        for k, t in enumerate(ts):
            one = m.interpolate(l, r, t).cpu().numpy()
            assert one.shape == (B, H, W, 3) and _same(one, many[k]), t
            assert _same(many[k], _expected(fw, bw, l, r, t, small)), (u8, t)
    with pytest.raises(ValueError):
        m.interpolate(l, r, 1.25)
    with pytest.raises(ValueError):
        m.interpolate(l, r, [0.5, -0.1])


def test_alternating_modes_give_fresh_results(cuda):
    """forward, forward_bidirectional and interpolate each keep their buffers and graph on one engine: an alternating
    sequence (different frames on every call) equals fresh models."""
    from raft_b200 import synth
    small, B, H, W = False, 1, 60, 100
    p = synth.make_weights(small)
    frames = [_frames(B, H, W, False, seed0=s) for s in (3000, 3100, 3200, 3300, 3400)]
    calls = [("i", frames[0]), ("f", frames[1]), ("b", frames[2]), ("i", frames[3]), ("f", frames[4]), ("i", frames[1])]

    def call(m, kind, lr):
        if kind == "f":
            return (m.forward(*lr),)
        if kind == "b":
            return m.forward_bidirectional(*lr)
        return (m.interpolate(*lr, [0.3, 0.6]),)

    one = _model(p, small, H, W, B, cuda)
    for kind, lr in calls:
        got = call(one, kind, lr)
        want = call(_model(p, small, H, W, B, cuda), kind, lr)
        for g, w in zip(got, want):
            assert torch.equal(g, w), kind
    # a new frame size drops the parked buffers and still gives fresh results
    l, r = _frames(B, 64, 96, False)
    assert torch.equal(one.interpolate(l, r, 0.5), _model(p, small, 64, 96, B, cuda).interpolate(l, r, 0.5))


def test_cli_interpolate(cuda, tmp_path, monkeypatch):
    import cv2
    import infer_raft
    from raft_b200 import synth
    l, r = synth.make_batch(1, 60, 100)
    for name, img in (("a.png", l[0]), ("b.png", r[0])):
        cv2.imwrite(str(tmp_path / name), (img * 255).astype(np.uint8))
    p = synth.make_weights(False)
    np.savez(tmp_path / "w.npz", **p)
    monkeypatch.chdir(tmp_path)
    base = ["--im1", "a.png", "--im2", "b.png", "--load", "w.npz", "--iters", "3", "--keep-size"]
    assert infer_raft.main(base + ["--npy", "plain.npy"]) == 0
    assert not os.path.exists("raft_interp_0.png")
    assert infer_raft.main(base + ["--npy", "f.npy", "--interpolate", "0", "0.5", "1"]) == 0
    assert np.array_equal(np.load("f.npy"), np.load("plain.npy"))
    a, b = cv2.imread("a.png"), cv2.imread("b.png")
    frames = [cv2.imread(f"raft_interp_{k}.png") for k in range(3)]
    assert all(f is not None and f.shape == (60, 100, 3) for f in frames)
    # frames are decoded to [0,1] fp32 and written as rint(255 x): the end points round-trip exactly
    assert np.array_equal(frames[0], a) and np.array_equal(frames[2], b)
    m = _model(p, False, 60, 100, 1, cuda)
    m.iters = 3
    want = m.interpolate(np.float32(a)[None] / 255.0, np.float32(b)[None] / 255.0, 0.5).cpu().numpy()[0]
    assert np.array_equal(frames[1], np.clip(np.rint(255.0 * want), 0, 255).astype(np.uint8))
    with pytest.raises(SystemExit):
        infer_raft.main(base + ["--interpolate", "1.5"])
