"""F6 on the CPU: the numpy restatements of the frame-interpolation kernels (tests/interp_oracle.py) against the
reference's flow reversal (tests/golden/reverse_flow.npz, written by oracle/make_reverseflow_golden.py from the
unmodified reference function), against analytic cases, and the argument checks of the C calls."""
import ctypes
import os

import numpy as np
import pytest

import interp_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reverse_flow.npz")


def _golden_cases():
    g = np.load(GOLDEN)
    return g, sorted({k.split("/")[0] for k in g.files})


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


@pytest.mark.parametrize("name", _golden_cases()[1])
def test_restatement_equals_reference_bit_for_bit(name):
    g = np.load(GOLDEN)
    flow, bg, im0, ts = g[f"{name}/flow"], g[f"{name}/bg"], g[f"{name}/im0"], float(g[f"{name}/time_step"])
    ft, empty, multi, static, eroded = O.reverse_one(flow, bg, im0, ts)
    ref = [g[f"{name}/out{k}"] for k in range(5)]
    assert ref[0].dtype == np.float32 and np.array_equal(_bits(ft), _bits(ref[0])), name
    assert np.array_equal(empty, ref[1]) and np.array_equal(multi, ref[2]) and np.array_equal(eroded, ref[4])
    assert ref[3].dtype == np.int64 and np.array_equal(static.astype(np.int64)[..., None], ref[3])


def test_golden_covers_the_cases():
    g, names = _golden_cases()
    steps = {float(g[f"{n}/time_step"]) for n in names}
    assert {1.0, 0.5, 1.0 / 3.0, 0.0, -0.5} <= steps
    assert g["all_static/out1"].all() and not g["all_static/out0"].any()   # everything empty, filled with +0
    assert g["one_source/out1"].sum() == g["one_source/out1"].size - 1
    assert g["converge/out1"].sum() == g["converge/out1"].size - 1          # every source on one pixel
    s = g["u8_static/out3"]
    assert 0 < s.sum() < s.size and g["f32_images/out3"].any()
    assert g["row/flow"].shape[0] == 1 and g["column/flow"].shape[1] == 1
    # the converge case: the sum depends on the order (a sorted-order sum gives other bits)
    flow = g["converge/flow"].reshape(-1, 2)
    fwd = np.float32(0)
    for v in -flow[:, 0]:
        fwd = np.float32(fwd + v)
    srt = np.float32(0)
    for v in np.sort(-flow[:, 0]):
        srt = np.float32(srt + v)
    assert fwd != srt


def test_nan_sources_are_skipped():
    """The one divergence from the reference (which raises in int(np.round(nan))): a NaN source is skipped, exactly as
    the reference skips an infinite one."""
    rng = np.random.default_rng(5)
    flow = rng.normal(0, 2, (13, 17, 2)).astype(np.float32)
    nan, inf = flow.copy(), flow.copy()
    idx = rng.choice(flow.size, 30, replace=False)
    nan.reshape(-1)[idx] = np.nan
    inf.reshape(-1)[idx] = np.inf
    a, b = O.reverse_one(nan, time_step=0.5), O.reverse_one(inf, time_step=0.5)
    for x, y in zip(a, b):
        assert np.array_equal(_bits(x), _bits(y))
    assert np.isfinite(a[0]).all()


def _random_frames(rng, B, H, W):
    return rng.uniform(0, 1, (B, H, W, 3)).astype(np.float32), rng.uniform(0, 1, (B, H, W, 3)).astype(np.float32)


def test_synthesis_endpoints_are_the_frames():
    rng = np.random.default_rng(6)
    B, H, W = 2, 19, 23
    i0, i1 = _random_frames(rng, B, H, W)
    fw = rng.normal(0, 3, (B, H, W, 2)).astype(np.float32)
    bw = rng.normal(0, 3, (B, H, W, 2)).astype(np.float32)
    for t, want in ((0.0, i0), (1.0, i1)):
        f0, e0 = O.reverse_flow(fw, time_step=t)[:2]
        f1, e1 = O.reverse_flow(bw, time_step=1.0 - t)[:2]
        got = O.synthesize(i0, i1, f0, f1, e0, e1, t)
        assert np.array_equal(_bits(got), _bits(want)), t


@pytest.mark.parametrize("d", [2, 4, 6])
def test_translation_midpoint_is_half_shift(d):
    """I1 is I0 moved right by d pixels, the flows are exactly +-d: the middle frame is I0 moved by d/2, bit for bit,
    wherever both reversed flows have sources (columns d/2 .. W-1-d/2)."""
    rng = np.random.default_rng(d)
    B, H, W = 1, 11, 29
    i0 = rng.uniform(0, 1, (B, H, W, 3)).astype(np.float32)
    i1 = rng.uniform(0, 1, (B, H, W, 3)).astype(np.float32)
    i1[:, :, d:] = i0[:, :, :-d]
    fw = np.zeros((B, H, W, 2), np.float32)
    fw[..., 0] = d
    bw = -fw
    f0, e0 = O.reverse_flow(fw, time_step=0.5)[:2]
    f1, e1 = O.reverse_flow(bw, time_step=0.5)[:2]
    assert (f0[..., 0] == -d / 2).all() and (f1[..., 0] == d / 2).all()  # holes filled from their neighbours
    mid = O.synthesize(i0, i1, f0, f1, e0, e1, 0.5)
    h = d // 2
    assert np.array_equal(_bits(mid[:, :, h:W - h]), _bits(i0[:, :, 0:W - 2 * h]))


def test_synthesis_weights_of_empty_pixels():
    rng = np.random.default_rng(8)
    B, H, W = 1, 6, 7
    i0, i1 = _random_frames(rng, B, H, W)
    z = np.zeros((B, H, W, 2), np.float32)
    e0 = np.zeros((B, H, W), np.uint8)
    e1 = np.zeros((B, H, W), np.uint8)
    e0[0, 1], e1[0, 2], e0[0, 3], e1[0, 3] = 1, 1, 1, 1
    out = O.synthesize(i0, i1, z, z, e0, e1, 0.25)
    w0, w1 = np.float32(0.75), np.float32(0.25)
    assert np.array_equal(out[0, 1], (w1 * i1[0, 1]) / w1)  # frame 0 empty: frame 1 only
    assert np.array_equal(out[0, 2], (w0 * i0[0, 2]) / w0)  # frame 1 empty: frame 0 only
    assert np.array_equal(out[0, 0], (w0 * i0[0, 0] + w1 * i1[0, 0]) / np.float32(1))
    both = (np.float32(0.75) * i0[0, 3] + np.float32(0.25) * i1[0, 3]) / np.float32(1)
    assert np.array_equal(out[0, 3], both)


def test_mirror_refuses_other_dtypes():
    import flow_utils
    assert "torch" not in vars(flow_utils)  # flow_to_color stays pure numpy
    flow = np.zeros((4, 5, 2), np.float32)
    im = np.zeros((4, 5, 3), np.uint8)
    with pytest.raises(TypeError):
        flow_utils.reverse_flow_avg_skip_static(flow.astype(np.float64), im, im)
    with pytest.raises(TypeError):
        flow_utils.reverse_flow_avg_skip_static(flow, im.astype(np.int32), im.astype(np.int32))


def test_argument_checks():
    """Bad arguments return RB_ERR_* with a message before any CUDA call (the pointers are host addresses)."""
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG, WORKSPACE = -1, -2, -5
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = ctypes.c_float

    def refused(rc, code, *words):
        assert rc == code, (rc, code)
        msg = lib.rb_last_error()
        assert all(w in msg for w in words), msg

    def rev(flow=p, bg=None, im0=None, u8=0, C=0, ts=1.0, ft=p, empty=p, multi=p, B=1, H=4, W=4, ws=p, nbytes=1 << 20):
        return lib.rb_flow_reverse(flow, bg, im0, u8, C, f(ts), ft, empty, multi, None, None, B, H, W, ws, nbytes, None)

    for kw in ({"flow": None}, {"ft": None}, {"empty": None}, {"multi": None}, {"ws": None}):
        refused(rev(**kw), BAD_ARG, b"rb_flow_reverse", b"null")
    refused(rev(bg=p), BAD_ARG, b"both")
    refused(rev(im0=p), BAD_ARG, b"both")
    refused(rev(bg=p, im0=p, C=0), BAD_SHAPE, b"img_channels")
    for ts in (float("nan"), float("inf"), -float("inf"), 1e300):
        refused(rev(ts=ts), BAD_ARG, b"time_step")
    for B, H, W in ((0, 4, 4), (1, 0, 4), (1, 4, -1)):
        refused(rev(B=B, H=H, W=W), BAD_SHAPE, b"bad shape")
    refused(rev(B=1, H=65535, W=65537), BAD_SHAPE, b"2^32")  # B*H*W + 1 == 2^32
    refused(rev(B=2, H=32768, W=65536), BAD_SHAPE, b"2^32")
    refused(rev(nbytes=64), WORKSPACE, b"too small")
    out = ctypes.c_size_t()
    refused(lib.rb_flow_reverse_workspace_bytes(1, 4, 4, None), BAD_ARG, b"null")
    refused(lib.rb_flow_reverse_workspace_bytes(1, 0, 4, ctypes.byref(out)), BAD_SHAPE, b"bad shape")
    refused(lib.rb_flow_reverse_workspace_bytes(1, 65535, 65537, ctypes.byref(out)), BAD_SHAPE, b"2^32")

    def syn(frames=p, Hp=8, Wp=8, top=0, left=0, f0=p, f1=p, e0=p, e1=p, t=0.5, out=p, B=1, H=8, W=8):
        return lib.rb_frame_synthesize(frames, Hp, Wp, top, left, f0, f1, e0, e1, f(t), out, B, H, W, None)

    for kw in ({"frames": None}, {"f0": None}, {"f1": None}, {"e0": None}, {"e1": None}, {"out": None}):
        refused(syn(**kw), BAD_ARG, b"rb_frame_synthesize", b"null")
    for t in (-0.01, 1.01, float("nan"), float("inf")):
        refused(syn(t=t), BAD_ARG, b"[0, 1]")
    for B, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, -2)):
        refused(syn(B=B, H=H, W=W), BAD_SHAPE, b"bad shape")
    for Hp, Wp, top, left in ((7, 8, 0, 0), (8, 7, 0, 0), (9, 8, 2, 0), (8, 9, 0, 2), (8, 8, -1, 0), (8, 8, 0, -1)):
        refused(syn(Hp=Hp, Wp=Wp, top=top, left=left), BAD_SHAPE, b"outside")
