"""numpy restatement of the forward-backward consistency check rb_flow_fb_check (csrc/consistency.cu), for the tests.

fb_check is fp32 in the kernel's operation order -- every operation rounded on its own, left to right, no FMA -- so the
kernel must reproduce it bit for bit.  fb_check_f64 is the same formula in fp64, the reference for the fp32 rounding.
Masks: 0 = consistent, 1 = inconsistent (occluded), 2 = the flow leaves the frame.
"""
from __future__ import annotations

import numpy as np


def _direction(f, b, s, a1, a2, dt):
    """One direction for [B,H,W,2] flows f (checked) and b (sampled) -> (mask, d, m); d = m = NaN where mask == 2."""
    f, b = np.asarray(f, dtype=dt), np.asarray(b, dtype=dt)
    s, a1, a2, one = dt(s), dt(a1), dt(a2), dt(1)
    B, H, W, _ = f.shape
    fx, fy = s * f[..., 0], s * f[..., 1]
    qx = np.arange(W, dtype=dt)[None, None, :] + fx
    qy = np.arange(H, dtype=dt)[None, :, None] + fy
    with np.errstate(invalid="ignore"):
        inside = (qx >= 0) & (qx <= dt(W - 1)) & (qy >= 0) & (qy <= dt(H - 1))  # NaN -> outside
    qx, qy = np.where(inside, qx, dt(0)), np.where(inside, qy, dt(0))
    fx0, fy0 = np.floor(qx), np.floor(qy)
    x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = qx - fx0, qy - fy0
    cx, cy = one - ax, one - ay
    bi = np.arange(B)[:, None, None]

    def bilerp(c):
        v = b[..., c]
        t0 = cx * v[bi, y0, x0] + ax * v[bi, y0, x1]
        t1 = cx * v[bi, y1, x0] + ax * v[bi, y1, x1]
        return t0 * cy + t1 * ay

    with np.errstate(invalid="ignore", over="ignore"):
        bx, by = s * bilerp(0), s * bilerp(1)
        ex, ey = fx + bx, fy + by
        d = ex * ex + ey * ey
        m = a1 * (((fx * fx + fy * fy) + bx * bx) + by * by) + a2
        mask = np.where(inside, (d > m).astype(np.uint8), np.uint8(2)).astype(np.uint8)
    nan = dt(np.nan)
    return mask, np.where(inside, d, nan), np.where(inside, m, nan)


def fb_check(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5, flow_scale=1.0, return_terms=False):
    """fp32, bit-exact with the kernel.  -> (occ_fw, occ_bw) [B,H,W] uint8; return_terms: ((occ, d, m) fw, (occ, d, m) bw)."""
    fw = _direction(flow_fw, flow_bw, flow_scale, alpha1, alpha2, np.float32)
    bw = _direction(flow_bw, flow_fw, flow_scale, alpha1, alpha2, np.float32)
    return (fw, bw) if return_terms else (fw[0], bw[0])


def fb_check_f64(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5, flow_scale=1.0, return_terms=False):
    """The same formula evaluated in fp64 (inputs widened exactly)."""
    fw = _direction(flow_fw, flow_bw, flow_scale, alpha1, alpha2, np.float64)
    bw = _direction(flow_bw, flow_fw, flow_scale, alpha1, alpha2, np.float64)
    return (fw, bw) if return_terms else (fw[0], bw[0])
