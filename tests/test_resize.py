"""F3 resize on the CPU: the numpy restatements of rb_frames_resize / rb_flow_resize (tests/resize_oracle.py) against the
reference's cv2.resize and resize_flow (tests/golden/resize.npz, written by oracle/make_resize_golden.py), against live
cv2.resize over a seeded sweep of shapes, and the argument checks of the C calls."""
import ctypes

import numpy as np
import pytest

import resize_oracle as O

CASES = O.golden_cases()


def _golden_input(mk, kind, case, H, W):
    if kind == "flow":
        return mk.flow_f32(H, W, bool(case))
    return (mk.frames_u8 if kind == "u8" else mk.frames_f32)(1, H, W)[0]


@pytest.mark.parametrize("kind,case,H,W,Ho,Wo", CASES, ids=lambda v: str(v))
def test_restatement_equals_reference_bit_for_bit(kind, case, H, W, Ho, Wo):
    g, mk = np.load(O.GOLDEN), O.golden_maker()
    x = _golden_input(mk, kind, case, H, W)
    if kind == "flow":
        out = O.resize_flow(x, Ho, Wo)
    else:
        out = O.resize_u8(x, Ho, Wo) if kind == "u8" else O.resize_f32(x, Ho, Wo)
    assert O.equals_golden(g, O.golden_key(kind, case, H, W, Ho, Wo), out)


def test_golden_covers_the_cases():
    shapes = {(H, W, Ho, Wo) for kind, _, H, W, Ho, Wo in CASES if kind == "u8"}
    assert {(436, 1024, 432, 1024), (1080, 1920, 432, 1024), (375, 1242, 432, 1024), (64, 96, 432, 1024)} <= shapes
    for axis in (0, 1):  # down, up and identity on each axis, with the other axis unchanged
        same = [s for s in shapes if s[1 - axis] == s[3 - axis]]
        assert any(s[axis] > s[2 + axis] for s in same) and any(s[axis] < s[2 + axis] for s in same)
        assert any(s[axis] == s[2 + axis] for s in same)
    assert any(H == 1 for H, _, _, _ in shapes) and any(W == 1 for _, W, _, _ in shapes)
    assert any(Ho % 8 and Wo % 8 for _, _, Ho, Wo in shapes) and any(H % 2 and W % 2 for H, W, _, _ in shapes)
    flows = {(case, H, W, Ho, Wo) for kind, case, H, W, Ho, Wo in CASES if kind == "flow"}
    assert (1, 432, 1024, 436, 1024) in flows and (1, 1, 12, 7, 5) in flows and (1, 12, 1, 5, 7) in flows
    g = np.load(O.GOLDEN)
    nan_case = g[O.golden_key("flow", 1, 43, 61, 80, 33)]
    assert np.isnan(nan_case).any() and np.isinf(nan_case).any()


def _sweep_shapes(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        H, W = int(rng.integers(1, 70)), int(rng.integers(1, 70))
        Ho, Wo = int(rng.integers(1, 100)), int(rng.integers(1, 100))
        if i % 7 == 0:
            Ho = H
        if i % 7 == 1:
            Wo = W
        out.append((H, W, Ho, Wo))
    return out


def test_restatements_equal_live_cv2_sweep():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(20261015)
    for H, W, Ho, Wo in _sweep_shapes(150, 1):
        u = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(cv2.resize(u, (Wo, Ho)), O.resize_u8(u, Ho, Wo)), (H, W, Ho, Wo)
        f = rng.random((H, W, 3), dtype=np.float32)
        assert np.array_equal(cv2.resize(f, (Wo, Ho)), O.resize_f32(f, Ho, Wo)), (H, W, Ho, Wo)
        fl = rng.normal(0, 20, (H, W)).astype(np.float32)
        k = max(1, fl.size // 16)
        for val in (np.nan, np.inf, -np.inf):
            fl.flat[rng.integers(0, fl.size, k)] = val
        with np.errstate(invalid="ignore"):
            assert np.array_equal(cv2.resize(fl, (Wo, Ho)), O.resize_f32(fl, Ho, Wo), equal_nan=True), (H, W, Ho, Wo)


def test_float_restatement_equals_cv2_at_cli_sizes():
    """IPP's float64 coordinates matter at large indices: OpenCV's own fp32-coordinate code differs there."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for H, W in ((436, 1024), (1080, 1920), (375, 1242), (64, 96)):
        f = rng.random((H, W, 3), dtype=np.float32)
        ref = cv2.resize(f, (1024, 432))
        assert np.array_equal(ref, O.resize_f32(f, 432, 1024)), (H, W)
        if H != 64:
            assert not np.array_equal(ref, O.resize_f32_opencv(f, 432, 1024)), (H, W)


def test_opencv_float_path_equals_cv2_without_ipp():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    was = cv2.useOptimized()
    try:
        cv2.setUseOptimized(False)
        for H, W, Ho, Wo in _sweep_shapes(40, 2) + [(436, 1024, 432, 1024), (375, 1242, 432, 1024)]:
            f = rng.random((H, W, 3), dtype=np.float32)
            assert np.array_equal(cv2.resize(f, (Wo, Ho)), O.resize_f32_opencv(f, Ho, Wo)), (H, W, Ho, Wo)
    finally:
        cv2.setUseOptimized(was)


def test_vertical_rounding_is_the_simd_form():
    """The scalar rounding (b0 S0 + b1 S1 + 2^21) >> 22 disagrees with cv2 on many values; the SIMD form does not."""
    cv2 = pytest.importorskip("cv2")
    u = np.random.default_rng(5).integers(0, 256, (436, 1024, 3), dtype=np.uint8)
    ref = cv2.resize(u, (1024, 432))
    x0, x1, a0, a1 = O._axis_u8(1024, 1024, True)
    y0, y1, b0, b1 = O._axis_u8(436, 432, False)
    S = u.astype(np.int64)[:, x0] * a0[None, :, None] + u.astype(np.int64)[:, x1] * a1[None, :, None]
    scalar = (b0[:, None, None] * S[y0] + b1[:, None, None] * S[y1] + (1 << 21)) >> 22
    assert np.count_nonzero(scalar != ref) > 1000
    assert np.array_equal(O.resize_u8(u, 432, 1024), ref)


def test_upscale_border_rows_keep_their_fraction():
    """Upscaling: rows -1 and H are clamped but their coefficients kept (OpenCV's vertical rule); dropping the fraction
    like the horizontal rule changes the first and last rows."""
    cv2 = pytest.importorskip("cv2")
    u = np.random.default_rng(6).integers(0, 256, (375, 1242, 3), dtype=np.uint8)
    ref = cv2.resize(u, (1024, 432))
    assert np.array_equal(O.resize_u8(u, 432, 1024), ref)
    x0, x1, a0, a1 = O._axis_u8(1242, 1024, True)
    y0, y1, b0, b1 = O._axis_u8(375, 432, True)  # the horizontal rule on rows
    S = u.astype(np.int64)[:, x0] * a0[None, :, None] + u.astype(np.int64)[:, x1] * a1[None, :, None]
    r = (((b0[:, None, None] * (S[y0] >> 4)) >> 16) + ((b1[:, None, None] * (S[y1] >> 4)) >> 16) + 2) >> 2
    bad = np.argwhere(r != ref)
    assert len(bad) and set(np.unique(bad[:, 0])) <= {0, 1, 430, 431}


def test_fmaf_is_exactly_rounded():
    rng = np.random.default_rng(8)
    a, b = rng.random(100000, dtype=np.float32), rng.normal(0, 1, 100000).astype(np.float32)
    c = rng.normal(0, 1e-3, 100000).astype(np.float32)
    r = O.fmaf(a, b, c)
    from fractions import Fraction
    for i in range(0, 100000, 997):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo, hi = np.nextafter(r[i], np.float32(-np.inf)), np.nextafter(r[i], np.float32(np.inf))
        err = abs(Fraction(float(r[i])) - exact)
        assert err <= abs(Fraction(float(lo)) - exact) and err <= abs(Fraction(float(hi)) - exact)
    # a tie that float64 double rounding gets wrong: (1 + u)(1 - u + u^2) = 1 + u^3 with u = 2^-12, so the exact sum is
    # 1 + 2^-24 + 2^-60, just above the midpoint of 1 and 1 + 2^-23; float64 rounds it onto the midpoint (then to even)
    a, b = np.float32(1 + 2 ** -12), np.float32((1 - 2 ** -12 + 2 ** -24) * 2 ** -24)
    assert np.float32(a.astype(np.float64) * b + 1.0) == np.float32(1)
    assert O.fmaf(a, b, np.float32(1)) == np.float32(1 + 2 ** -23)


def test_frames_resize_pads_after_resizing():
    u = O.golden_maker().frames_u8(2, 37, 53)
    out = O.frames_resize(u, 45, 61, pad=(1, 2, 3, 0))
    core = (O.resize_u8(u, 45, 61).astype(np.float32) / np.float32(255)).astype(np.float32)
    assert out.shape == (2, 48, 64, 3) and out.dtype == np.float32
    assert np.array_equal(out[:, 1:46, 3:], core)
    assert np.array_equal(out[:, 0], out[:, 1]) and np.array_equal(out[:, 47], out[:, 45])
    assert np.array_equal(out[:, :, 0], out[:, :, 3])


def test_resize_flow_scales_u_by_width_and_v_by_height():
    flow = np.zeros((20, 30, 2), np.float32)
    flow[..., 0], flow[..., 1] = 1.0, 1.0
    out = O.resize_flow(flow, 60, 45)  # twice the height, 1.5 times the width
    assert np.all(out[..., 0] == np.float32(1.5)) and np.all(out[..., 1] == np.float32(3.0))


def test_argument_checks():
    """Bad arguments return RB_ERR_* with a message before any CUDA call (host pointers: a launch would fail instead)."""
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG = -1, -2
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def refused(rc, code, *words):
        assert rc == code, (rc, code)
        msg = lib.rb_last_error()
        assert all(w in msg for w in words), msg

    refused(lib.rb_frames_resize(None, 1, p, 2, 37, 53, 40, 40, 0, 0, 0, 0, None), BAD_ARG, b"rb_frames_resize", b"null")
    refused(lib.rb_frames_resize(p, 0, None, 2, 37, 53, 40, 40, 0, 0, 0, 0, None), BAD_ARG, b"rb_frames_resize", b"null")
    for B, H, W, Ho, Wo in ((0, 37, 53, 40, 40), (1, 0, 53, 40, 40), (1, 37, -1, 40, 40), (1, 37, 53, 0, 40),
                            (1, 37, 53, 40, -5)):
        refused(lib.rb_frames_resize(p, 1, p, B, H, W, Ho, Wo, 0, 0, 0, 0, None), BAD_SHAPE, b"rb_frames_resize", b"shape")
        refused(lib.rb_flow_resize(p, p, B, H, W, Ho, Wo, None), BAD_SHAPE, b"rb_flow_resize", b"shape")
    for pads in ((-1, 0, 0, 0), (0, -1, 0, 0), (0, 0, -1, 0), (0, 0, 0, -3)):
        refused(lib.rb_frames_resize(p, 1, p, 2, 37, 53, 40, 40, *pads, None), BAD_SHAPE, b"rb_frames_resize", b"pad")
    refused(lib.rb_frames_resize(p, 1, p, 1, 1 << 16, 1 << 15, 40, 40, 0, 0, 0, 0, None), BAD_SHAPE, b"too large")
    refused(lib.rb_flow_resize(None, p, 1, 4, 4, 4, 4, None), BAD_ARG, b"rb_flow_resize", b"null")
    refused(lib.rb_flow_resize(p, None, 1, 4, 4, 4, 4, None), BAD_ARG, b"rb_flow_resize", b"null")
    refused(lib.rb_flow_resize(p, p, 1, 4, 4, 1 << 16, 1 << 15, None), BAD_SHAPE, b"too large")
