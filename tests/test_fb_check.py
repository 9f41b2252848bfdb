"""Forward-backward consistency check (F5): analytic cases on the fp32 numpy restatement (tests/fb_oracle.py), its
agreement with the fp64 form, and the argument checks of rb_flow_fb_check, which come before any CUDA call."""
import ctypes

import numpy as np
import pytest

from fb_oracle import fb_check, fb_check_f64


def _const(B, H, W, fx, fy):
    f = np.empty((B, H, W, 2), np.float32)
    f[..., 0], f[..., 1] = fx, fy
    return f


def test_zero_flows_are_consistent():
    z = np.zeros((2, 5, 7, 2), np.float32)
    a, b = fb_check(z, z)
    assert a.dtype == np.uint8 and a.shape == (2, 5, 7) and not a.any() and not b.any()


@pytest.mark.parametrize("t", [1, 3, 6])
def test_integer_translation_leaves_exactly_t_columns(t):
    B, H, W = 2, 6, 9
    a, b = fb_check(_const(B, H, W, t, 0), _const(B, H, W, -t, 0))
    assert (a[..., :W - t] == 0).all() and (a[..., W - t:] == 2).all()  # x + t > W-1 on the last t columns
    assert (b[..., t:] == 0).all() and (b[..., :t] == 2).all()  # x - t < 0 on the first t columns
    # the same vertically
    a, b = fb_check(_const(B, H, W, 0, 2), _const(B, H, W, 0, -2))
    assert (a[:, :H - 2] == 0).all() and (a[:, H - 2:] == 2).all()
    assert (b[:, 2:] == 0).all() and (b[:, :2] == 2).all()


def test_perturbation_far_beyond_alpha2_is_occluded():
    B, H, W = 1, 6, 9
    fw, bw = _const(B, H, W, 2, 0), _const(B, H, W, -2, 0)
    bw[0, 3, 4] = (3.0, 0.0)  # fw(3,2) lands on (3,4): |f + b| = 5, m = 0.01 (4 + 9) + 0.5
    a, b = fb_check(fw, bw)
    assert a[0, 3, 2] == 1
    assert ((a == 1).sum(), (a[..., :W - 2] == 0).sum()) == (1, H * (W - 2) - 1)
    # and backwards: bw(3,4) = +3 lands on (3,7) where fw = +2, |3 + 2|^2 = 25 > 0.01 (9 + 4) + 0.5
    assert b[0, 3, 4] == 1 and (b == 1).sum() == 1


def test_threshold_sides():
    """fw = 0 samples bw at the pixel itself: d = v^2, m = 0.01 v^2 + 0.5, so the mask flips at v = sqrt(0.5 / 0.99)."""
    vt = np.sqrt(0.5 / 0.99)
    for v, want in ((vt - 1e-4, 0), (vt + 1e-4, 1), (-(vt - 1e-4), 0), (-(vt + 1e-4), 1)):
        a, _ = fb_check(_const(1, 3, 3, 0, 0), _const(1, 3, 3, v, 0))
        assert (a == want).all(), (v, want)
        a, _ = fb_check(_const(1, 3, 3, 0, 0), _const(1, 3, 3, 0, v))
        assert (a == want).all(), (v, want)
    # in fp32: the last value on the consistent side and the next float up straddle the real threshold within rounding
    vs = np.float32(vt) + np.arange(-64, 65, dtype=np.float32) * np.spacing(np.float32(vt))
    bw = np.zeros((1, 1, vs.size, 2), np.float32)
    bw[0, 0, :, 0] = vs
    (a, d, m), _ = fb_check(np.zeros_like(bw), bw, return_terms=True)
    flip = np.flatnonzero(a[0, 0] == 1)
    assert flip.size and (a[0, 0, :flip[0]] == 0).all() and (a[0, 0, flip[0]:] == 1).all()
    lo, hi = float(vs[flip[0] - 1]), float(vs[flip[0]])
    assert d[0, 0, flip[0] - 1] <= m[0, 0, flip[0] - 1] and d[0, 0, flip[0]] > m[0, 0, flip[0]]
    assert abs(lo - vt) < 1e-6 and abs(hi - vt) < 1e-6


def test_flow_scale_equals_prescaled_flow():
    rng = np.random.default_rng(0)
    fw = rng.uniform(-6, 6, (2, 9, 13, 2)).astype(np.float32)
    bw = (-fw + rng.normal(0, 0.5, fw.shape)).astype(np.float32)
    ref = fb_check(fw, bw)
    got = fb_check(fw / np.float32(8), bw / np.float32(8), flow_scale=8.0)  # /8 and x8 are exact in binary
    assert all(np.array_equal(r, g) for r, g in zip(ref, got))
    assert {0, 1, 2} <= set(np.unique(ref[0]))


@pytest.mark.parametrize("shape", [(2, 1, 7), (2, 5, 1), (1, 1, 1)])
def test_degenerate_frames_stay_in_range(shape):
    B, H, W = shape
    rng = np.random.default_rng(1)
    fw = rng.uniform(-2, 2, shape + (2,)).astype(np.float32)
    bw = rng.uniform(-2, 2, shape + (2,)).astype(np.float32)
    for f, b in ((fw, bw), (np.zeros_like(fw), np.zeros_like(bw))):
        a, c = fb_check(f, b)
        assert a.shape == c.shape == shape
    a, c = fb_check(np.zeros_like(fw), np.zeros_like(bw))
    assert not a.any() and not c.any()
    # on a single row (column) any vertical (horizontal) motion leaves the frame
    a, _ = fb_check(_const(B, H, W, 0.0, 0.25 if H == 1 else 0.0) + _const(B, H, W, 0.25 if W == 1 else 0.0, 0.0),
                    np.zeros_like(fw))
    assert (a == 2).all()


def test_nan_flow_leaves_the_frame_and_nan_samples_are_consistent():
    fw = np.zeros((1, 4, 4, 2), np.float32)
    bw = np.zeros_like(fw)
    fw[0, 1, 1, 0] = np.nan
    bw[0, 2, 2, 1] = np.nan
    a, b = fb_check(fw, bw)
    assert a[0, 1, 1] == 2 and b[0, 2, 2] == 2
    assert a[0, 2, 2] == 0 and b[0, 1, 1] == 0  # d = NaN: "d > m" is false


def test_fp32_agrees_with_fp64_away_from_rounding():
    rng = np.random.default_rng(2)
    B, H, W = 3, 31, 47
    fw = rng.uniform(-8, 8, (B, H, W, 2)).astype(np.float32)
    bw = (-fw + rng.normal(0, 0.8, fw.shape)).astype(np.float32)
    (a32, d32, m32), (b32, e32, n32) = fb_check(fw, bw, return_terms=True)
    (a64, d64, m64), (b64, e64, n64) = fb_check_f64(fw, bw, return_terms=True)
    # the 2-class: the fp32 target x + f differs from the fp64 one only near the frame's edges
    xs = np.arange(W)[None, None, :] + fw[..., 0].astype(np.float64)
    ys = np.arange(H)[None, :, None] + fw[..., 1].astype(np.float64)
    near_edge = np.minimum.reduce([np.abs(xs), np.abs(xs - (W - 1)), np.abs(ys), np.abs(ys - (H - 1))]) < 1e-5
    assert np.array_equal((a32 == 2)[~near_edge], (a64 == 2)[~near_edge])
    both_in = (a32 != 2) & (a64 != 2)
    clear = both_in & (np.abs(d64 - m64) > 1e-4 * (1 + m64))
    assert clear.sum() > 0.9 * both_in.sum() and (a32 == 1)[clear].any() and (a32 == 0)[clear].any()
    assert np.array_equal(a32[clear], a64[clear])
    assert np.abs(d32 - d64)[both_in].max() < 1e-4 * (1 + np.abs(d64[both_in]).max())
    clear_b = (b32 != 2) & (b64 != 2) & (np.abs(e64 - n64) > 1e-4 * (1 + n64))
    assert np.array_equal(b32[clear_b], b64[clear_b])


def test_argument_checks_before_any_cuda_call():
    from raft_b200 import capi
    lib = capi.lib
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ok = dict(ff=p, fb=p, of=p, ob=p, B=1, H=4, W=4, s=1.0, a1=0.01, a2=0.5)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.rb_flow_fb_check(a["ff"], a["fb"], a["of"], a["ob"], a["B"], a["H"], a["W"], a["s"], a["a1"], a["a2"],
                                    None)

    cases = [(dict(ff=None), -2), (dict(fb=None), -2), (dict(of=None), -2), (dict(ob=None), -2),
             (dict(B=0), -1), (dict(H=0), -1), (dict(W=-3), -1),
             (dict(s=0.0), -2), (dict(s=-8.0), -2), (dict(s=float("nan")), -2), (dict(s=float("inf")), -2),
             (dict(a1=-0.01), -2), (dict(a1=float("nan")), -2), (dict(a1=float("inf")), -2),
             (dict(a2=-0.5), -2), (dict(a2=float("nan")), -2), (dict(a2=float("inf")), -2)]
    for kw, code in cases:
        assert call(**kw) == code, kw
        assert b"rb_flow_fb_check" in lib.rb_last_error(), kw
