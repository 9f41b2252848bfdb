"""numpy restatements of the frame-interpolation kernels (csrc/interp.cu), for the tests.

reverse_flow is rb_flow_reverse: the reference's flow_utils.py:166 reverse_flow_avg_skip_static under numpy >= 2, with
the raster-order splat written as np.add.at (unbuffered, applied in index order) and the hole fill vectorised through
the nearest non-empty index per row and column.  synthesize is rb_frame_synthesize in the kernel's operation order.
Both are fp32 where the kernels are, so the kernels must reproduce them bit for bit.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def static_mask(bg, im0):
    """[..., C] images -> [...] bool: every channel differs by < 10 (uint8 images: the wrapped difference)."""
    bg, im0 = np.asarray(bg), np.asarray(im0)
    if bg.dtype == np.uint8 and im0.dtype == np.uint8:
        d = bg - im0  # wraps, and np.abs of a uint8 is the identity
    else:
        d = np.abs(bg.astype(f32) - im0.astype(f32))
    return np.all(d < 10, axis=-1)


def _nearest(nonempty, axis, reverse):
    """Index along `axis` of the nearest non-empty pixel at or before (reverse: at or after) each pixel; -1 if none."""
    n = nonempty.shape[axis]
    idx = np.arange(n).reshape([-1 if a == axis else 1 for a in range(nonempty.ndim)])
    if not reverse:
        return np.maximum.accumulate(np.where(nonempty, idx, -1), axis=axis)
    r = np.flip(np.minimum.accumulate(np.flip(np.where(nonempty, idx, n), axis), axis=axis), axis)
    return np.where(r == n, -1, r)


def erode5(mask):
    """5x5 minimum over the window clipped to the image."""
    H, W = mask.shape
    p = np.pad(mask, 2, constant_values=1)
    out = np.ones_like(mask)
    for dy in range(5):
        for dx in range(5):
            out = np.minimum(out, p[dy:dy + H, dx:dx + W])
    return out


def reverse_one(flow01, bg=None, im0=None, time_step=1.0):
    """One [H,W,2] flow -> (flow_t f32 [H,W,2], empty u8, multi u8, static bool [H,W], eroded empty u8)."""
    flow01 = np.asarray(flow01, dtype=f32)
    H, W = flow01.shape[:2]
    st = np.zeros((H, W), bool) if bg is None else static_mask(bg, im0)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.where(st[..., None], f32(np.inf), flow01) * f32(time_step)
        px = f[..., 0].astype(np.float64) + np.arange(W)
        py = f[..., 1].astype(np.float64) + np.arange(H)[:, None]
    ok = np.isfinite(px) & np.isfinite(py)
    rx = np.clip(np.rint(np.where(ok, px, 0)), 0, W - 1).astype(np.int64)
    ry = np.clip(np.rint(np.where(ok, py, 0)), 0, H - 1).astype(np.int64)
    tgt = (ry * W + rx)[ok]  # boolean indexing keeps raster order
    acc = np.zeros((H * W, 2), f32)
    np.add.at(acc, tgt, -f[ok])
    count = np.bincount(tgt, minlength=H * W)
    with np.errstate(invalid="ignore", divide="ignore"):
        ft = np.where(count[:, None] > 0, (acc.astype(np.float64) / count[:, None]).astype(f32), acc).reshape(H, W, 2)
    empty = (count == 0).reshape(H, W)
    nonempty = ~empty
    s = np.zeros((H, W, 2), f32)
    n = np.zeros((H, W), np.int64)
    yy, xx = np.mgrid[0:H, 0:W]
    up = _nearest(nonempty, 0, False)
    down = _nearest(nonempty, 0, True)
    left = _nearest(nonempty, 1, False)
    right = _nearest(nonempty, 1, True)
    for idx, col in ((up, True), (down, True), (left, False), (right, False)):
        found = idx >= 0
        src = ft[np.where(found, idx, 0), xx] if col else ft[yy, np.where(found, idx, 0)]
        s = np.where(found[..., None], s + src, s)
        n += found
    with np.errstate(invalid="ignore", divide="ignore"):
        fill = np.where(n[..., None] > 0, s / n[..., None].astype(f32), f32(0))
    ft = np.where(empty[..., None], fill, ft).astype(f32)
    empty_u8 = empty.astype(np.uint8)
    return ft, empty_u8, (count > 1).reshape(H, W).astype(np.uint8), st, erode5(empty_u8)


def reverse_flow(flow01, bg=None, im0=None, time_step=1.0):
    """Batched [B,H,W,2] form: five [B,...] arrays (see reverse_one)."""
    outs = [reverse_one(flow01[b], None if bg is None else bg[b], None if im0 is None else im0[b], time_step)
            for b in range(len(flow01))]
    return tuple(np.stack(o) for o in zip(*outs))


def _sample(img, F):
    """Bilinear sample of img [B,H,W,3] at p + F (clamped, NaN -> 0), the arithmetic of rb_flow_fb_check."""
    B, H, W, _ = img.shape
    qx = np.fmin(np.fmax(np.arange(W, dtype=f32)[None, None, :] + F[..., 0], f32(0)), f32(W - 1))
    qy = np.fmin(np.fmax(np.arange(H, dtype=f32)[None, :, None] + F[..., 1], f32(0)), f32(H - 1))
    fx0, fy0 = np.floor(qx), np.floor(qy)
    x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = qx - fx0, qy - fy0
    cx, cy = f32(1) - ax, f32(1) - ay
    bi = np.arange(B)[:, None, None]
    out = np.empty(img.shape, f32)
    for c in range(3):
        v = img[..., c]
        t0 = cx * v[bi, y0, x0] + ax * v[bi, y0, x1]
        t1 = cx * v[bi, y1, x0] + ax * v[bi, y1, x1]
        out[..., c] = t0 * cy + t1 * ay
    return out


def synthesize(frame0, frame1, flow_t0, flow_t1, empty0, empty1, t):
    """[B,H,W,3] frames, [B,H,W,2] flows from time t, [B,H,W] empty masks -> [B,H,W,3] fp32."""
    frame0, frame1 = np.asarray(frame0, f32), np.asarray(frame1, f32)
    flow_t0, flow_t1 = np.asarray(flow_t0, f32), np.asarray(flow_t1, f32)
    t = f32(t)
    s = f32(1) - t
    w0 = np.where(np.asarray(empty0) != 0, f32(0), s)
    w1 = np.where(np.asarray(empty1) != 0, f32(0), t)
    both = (w0 == 0) & (w1 == 0)
    w0, w1 = np.where(both, s, w0)[..., None], np.where(both, t, w1)[..., None]
    with np.errstate(invalid="ignore", over="ignore"):
        return ((w0 * _sample(frame0, flow_t0) + w1 * _sample(frame1, flow_t1)) / (w0 + w1)).astype(f32)
