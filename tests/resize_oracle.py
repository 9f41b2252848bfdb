"""numpy restatements of the bilinear resize the reference calls (cv2.resize, default INTER_LINEAR, OpenCV 4.13 with
its bundled Intel IPP), which csrc/resize.cu reproduces bit for bit.  cv2 runs two different algorithms:

uint8 (OpenCV's own fixed-point code; IPP is not used for 8-bit bilinear):
  - per axis f = fl32((d + 0.5) * scale - 0.5) with scale = 1 / (dst / src) in float64, s = floor(f), f -= s;
  - horizontally a source index below 0 or at or above W - 1 is clamped and its fraction set to 0; vertically only
    the row index is clamped (rows -1 and H become 0 and H - 1) and the fraction is KEPT -- the upscaling border rule;
  - coefficients rint((1 - f) * 2048), rint(f * 2048); horizontal int32 sum S;
  - vertical rounding of the SIMD path: ((b0 * (S0 >> 4)) >> 16 + (b1 * (S1 >> 4)) >> 16 + 2) >> 2.

float32 (IPP's linear resize):
  - per axis c = (d + 0.5) * (src / dst) - 0.5 in float64, s = floor(c), w = fl32(c - s) (the fraction of the float64
    coordinate, so it keeps the precision OpenCV's fl32 coordinate loses at large indices);
  - indices clamped to the frame (replicate border), w kept;
  - horizontal pass, then vertical, each fmaf(w, p1 - p0, p0) with p1 - p0 rounded to fp32, except that a column
    whose two taps clamping made the same pixel copies it (an inf there stays inf; the same case in the vertical pass
    does compute inf - inf = NaN).
  cv2 does not use IPP when the source is a single row or column, nor with cv2.setUseOptimized(False): then OpenCV's
  own float code runs (resize_f32_opencv): the uint8 path's coordinates and clamping, p0 * (1 - f) + p1 * f
  horizontally with the columns whose right tap is clamped copied from one tap, S0 * (1 - f) + S1 * f vertically.
  A same-size resize is a copy."""
import hashlib
import importlib.util
import os

import numpy as np

F32 = np.float32


def _coords_f32(src, dst):
    """OpenCV's coordinate: float32 f, integer s, fraction f - s (resize.cpp, resizeGeneric)."""
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * (1.0 / (dst / src)) - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    return s, (f - s.astype(F32)).astype(F32)


def _axis_u8(src, dst, clamp_fraction):
    s, f = _coords_f32(src, dst)
    if clamp_fraction:
        out = (s < 0) | (s >= src - 1)
        f = np.where(out, F32(0), f)
        s = np.clip(s, 0, src - 1)
    w0 = np.rint((F32(1) - f) * F32(2048)).astype(np.int64)
    w1 = np.rint(f * F32(2048)).astype(np.int64)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), w0, w1


def _batched(img):
    img = np.asarray(img)
    if img.ndim == 2:
        return img[None, :, :, None], lambda r: r[0, :, :, 0]
    if img.ndim == 3:
        return img[None], lambda r: r[0]
    return img, lambda r: r


def resize_u8(img, Ho, Wo):
    """cv2.resize(img, (Wo, Ho)) for uint8 [H,W], [H,W,C] or a batch [B,H,W,C]."""
    x, unbatch = _batched(img)
    assert x.dtype == np.uint8
    H, W = x.shape[1:3]
    x0, x1, a0, a1 = _axis_u8(W, Wo, True)
    y0, y1, b0, b1 = _axis_u8(H, Ho, False)
    I = x.astype(np.int64)
    S = I[:, :, x0] * a0[None, None, :, None] + I[:, :, x1] * a1[None, None, :, None]  # [B,H,Wo,C] int32 range
    S0, S1 = S[:, y0] >> 4, S[:, y1] >> 4
    bb0, bb1 = b0[None, :, None, None], b1[None, :, None, None]
    r = (((bb0 * S0) >> 16) + ((bb1 * S1) >> 16) + 2) >> 2
    return unbatch(np.clip(r, 0, 255).astype(np.uint8))


def fmaf(a, b, c):
    """fp32 fused multiply-add, exactly rounded: a * b is exact in float64 (two 24-bit significands), the float64 sum
    is exact up to one rounding whose error TwoSum recovers, and that error only matters when the float64 sum lands
    exactly on a float32 tie."""
    a, b, c = (np.asarray(v, dtype=np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bp = s - c
        e = (p - bp) + (c - (s - bp))  # TwoSum: s + e == p + c exactly (finite operands)
        r = s.astype(F32)
        rd = r.astype(np.float64)
        other = np.where(s > rd, np.nextafter(r, F32(np.inf)), np.nextafter(r, F32(-np.inf))).astype(np.float64)
        tie = np.isfinite(s) & (s != rd) & (2 * s == rd + other)
        # on a tie, round towards the exact value: away from r if the exact sum lies beyond s, as seen from r
        beyond = np.where(s > rd, e > 0, e < 0)
        return np.where(tie & (e != 0), np.where(beyond, other, rd), r.astype(np.float64)).astype(F32)


def _axis_f32(src, dst):
    c = (np.arange(dst, dtype=np.float64) + 0.5) * (src / dst) - 0.5
    s = np.floor(c)
    w = (c - s).astype(F32)
    s = s.astype(np.int64)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), w


def _lerp(p0, p1, w, same):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(same, p0, fmaf(w, (p1 - p0).astype(F32), p0))


def resize_f32(img, Ho, Wo):
    """cv2.resize(img, (Wo, Ho)) for float32 [H,W], [H,W,C] or a batch [B,H,W,C] (IPP's linear resize)."""
    x, unbatch = _batched(img)
    assert x.dtype == np.float32
    H, W = x.shape[1:3]
    if (H, W) == (Ho, Wo):
        return unbatch(x.copy())
    if H == 1 or W == 1:
        return resize_f32_opencv(img, Ho, Wo)
    x0, x1, wx = _axis_f32(W, Wo)
    y0, y1, wy = _axis_f32(H, Ho)
    cx, cy = (x0 == x1)[None, None, :, None], (y0 == y1)[None, :, None, None]
    S = _lerp(x[:, :, x0], x[:, :, x1], wx[None, None, :, None], False)  # [B,H,Wo,C]
    Sc = np.broadcast_to(x[:, :, x0], S.shape)  # border columns: the pixel itself
    T0 = np.where(cx & ~cy, Sc[:, y0], S[:, y0])
    T1 = np.where(cx & ~cy, Sc[:, y1], S[:, y1])
    return unbatch(np.where(cy & ~cx, T0, _lerp(T0, T1, wy[None, :, None, None], False)))


def resize_f32_opencv(img, Ho, Wo):
    """cv2.resize for float32 with IPP off (cv2.setUseOptimized(False)): OpenCV's own float code."""
    x, unbatch = _batched(img)
    H, W = x.shape[1:3]
    if (H, W) == (Ho, Wo):
        return unbatch(x.copy())
    sx, fx = _coords_f32(W, Wo)
    out = (sx < 0) | (sx >= W - 1)
    fx = np.where(out, F32(0), fx)
    sx = np.clip(sx, 0, W - 1)
    sy, fy = _coords_f32(H, Ho)
    x0, x1 = sx, np.clip(sx + 1, 0, W - 1)
    y0, y1 = np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1)
    ax, ay = fx[None, None, :, None], fy[None, :, None, None]
    with np.errstate(invalid="ignore", over="ignore"):
        one_tap = (sx >= W - 1)[None, None, :, None]  # OpenCV's xmax: from there on one tap, S[sx] * 1
        S = np.where(one_tap, x[:, :, x0], (x[:, :, x0] * (F32(1) - ax) + x[:, :, x1] * ax).astype(F32))
        return unbatch((S[:, y0] * (F32(1) - ay) + S[:, y1] * ay).astype(F32))


def frames_resize(frames, Ho, Wo, pad=(0, 0, 0, 0)):
    """rb_frames_resize: [B,H,W,3] uint8 or fp32 frames -> cv2 resize to Ho x Wo, /255 for uint8 (correctly rounded
    fp32 division), then replicate pad (top, bottom, left, right) -> [B,Ho+pt+pb,Wo+pl+pr,3] fp32."""
    frames = np.asarray(frames)
    if frames.dtype == np.uint8:
        r = (resize_u8(frames, Ho, Wo).astype(F32) / F32(255)).astype(F32)
    else:
        r = resize_f32(frames, Ho, Wo)
    t, b, l, rr = pad
    return np.pad(r, ((0, 0), (t, b), (l, rr), (0, 0)), mode="edge")


def resize_flow(flow, Ho, Wo):
    """rb_flow_resize / the reference's flow_utils.resize_flow for [B,H,W,2] or [H,W,2] float32 flows: each channel
    resized like cv2, then u *= Wo / W and v *= Ho / H as float32 multiplies (numpy >= 2: a python float is weak)."""
    x, unbatch = _batched(flow)
    H, W = x.shape[1:3]
    r = resize_f32(x.astype(F32), Ho, Wo)
    with np.errstate(invalid="ignore", over="ignore"):
        r[..., 0] = r[..., 0] * F32(Wo / float(W))
        r[..., 1] = r[..., 1] * F32(Ho / float(H))
    return unbatch(r)


# ---- the goldens of oracle/make_resize_golden.py (tests/golden/resize.npz) ----------------------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize.npz")


def golden_maker():
    """oracle/make_resize_golden.py as a module: its input formulas (frames_u8, frames_f32, flow_f32)."""
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "make_resize_golden.py")
    spec = importlib.util.spec_from_file_location("make_resize_golden", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def golden_cases():
    """[(kind, case, H, W, Ho, Wo)]: kind 'u8' / 'f32' (frames) or 'flow'; case the NaN/inf flag of flows."""
    out = set()
    for k in np.load(GOLDEN).files:
        parts = k.split("/")
        (H, W), (Ho, Wo) = (tuple(int(v) for v in s.split("x")) for s in parts[2].split("->"))
        kind, case = (parts[1], None) if parts[0] == "frames" else ("flow", int(parts[1]))
        out.add((kind, case, H, W, Ho, Wo))
    return sorted(out, key=str)


def golden_key(kind, case, H, W, Ho, Wo):
    return (f"flow/{case}" if kind == "flow" else f"frames/{kind}") + f"/{H}x{W}->{Ho}x{Wo}"


def canonical_nan(arr):
    """NaN payloads differ between x86 (inf - inf is the negative default NaN) and the GPU: compare every NaN as one."""
    arr = np.array(arr)
    if arr.dtype == np.float32:
        arr[np.isnan(arr)] = np.float32(np.nan)
    return arr


def equals_golden(g, key, arr):
    """Bit for bit (every NaN as one NaN): the stored array, or the SHA-256 of the bytes of large outputs."""
    arr = np.ascontiguousarray(canonical_nan(arr))
    if key + "/sha256" in g.files:
        return tuple(g[key + "/shape"]) == arr.shape and \
            hashlib.sha256(arr.tobytes()).digest() == g[key + "/sha256"].tobytes()
    ref = canonical_nan(g[key])
    return ref.dtype == arr.dtype and ref.shape == arr.shape and ref.tobytes() == arr.tobytes()
