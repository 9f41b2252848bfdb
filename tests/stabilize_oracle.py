"""numpy restatements of F22 (rb_global_motion: the same 8 sums, weights and rounds in fp64) and F23
(rb_frames_warp_affine, bit for bit), and analytic flows of known similarities for the recovery tests."""
import numpy as np

from raft_b200.stabilize import MOTION_CAUCHY, MOTION_MIN_WEIGHT, MOTION_ROUNDS

F32 = np.float32


def points(Hn, Wn, Hs, Ws):
    """The centred frame-pixel positions (px, py) [Hn,Wn] of the network pixels and the axis scales (sx, sy)."""
    sx, sy = Ws / Wn, Hs / Hn
    j, i = np.meshgrid(np.arange(Wn, dtype=np.float64), np.arange(Hn, dtype=np.float64))
    return (j + 0.5) * sx - 0.5 - 0.5 * (Ws - 1), (i + 0.5) * sy - 0.5 - 0.5 * (Hs - 1), sx, sy


def sums(px, py, qx, qy, w):
    """The 8 weighted sums of the normal equations, in rb_global_motion's order."""
    return np.array([w.sum(), (w * px).sum(), (w * py).sum(), (w * (px * px + py * py)).sum(),
                     (w * (px * qx + py * qy)).sum(), (w * (px * qy - py * qx)).sum(), (w * qx).sum(),
                     (w * qy).sum()])


def abs_sums(px, py, qx, qy, w):
    """The sums of the terms' magnitudes: the scale a reordered sum's rounding error is relative to."""
    a = np.abs
    return np.array([a(w).sum(), a(w * px).sum(), a(w * py).sum(), a(w * (px * px + py * py)).sum(),
                     (a(w * px * qx) + a(w * py * qy)).sum(), (a(w * px * qy) + a(w * py * qx)).sum(), a(w * qx).sum(),
                     a(w * qy).sum()])


def solve(s):
    """(a, b, tx, ty, singular) of the 8 sums, closed form."""
    S, X, Y, P, U, V, Qx, Qy = s
    den = P * S - X * X - Y * Y
    if not (S > 0) or not (den > 1e-9 * P * S):
        return 1.0, 0.0, 0.0, 0.0, True
    a = (U * S - X * Qx - Y * Qy) / den
    b = (V * S - X * Qy + Y * Qx) / den
    return a, b, (Qx - a * X + b * Y) / S, (Qy - b * X - a * Y) / S, False


def round_sums(flow, occ, hw, flow_scale=1.0, m=None, c=MOTION_CAUCHY):
    """The 8 sums (and their magnitude sums) of one pair's round: flow [Hn,Wn,2] fp32, occ [Hn,Wn] uint8; m = the previous
    round's (a, b, tx, ty), None for round 0."""
    Hn, Wn, _ = flow.shape
    Hs, Ws = hw
    px, py, sx, sy = points(Hn, Wn, Hs, Ws)
    u, v = flow[..., 0].astype(np.float64), flow[..., 1].astype(np.float64)
    ok = (occ == 0) & np.isfinite(u) & np.isfinite(v)
    u, v = np.where(ok, u, 0.0), np.where(ok, v, 0.0)
    qx, qy = px + flow_scale * (u * sx), py + flow_scale * (v * sy)
    w = ok.astype(np.float64)
    if m is not None:
        ex = (m[0] * px - m[1] * py + m[2] - qx) * (Wn / Ws)
        ey = (m[1] * px + m[0] * py + m[3] - qy) * (Hn / Hs)
        w = w / (1.0 + (ex * ex + ey * ey) / (c * c))
    return sums(px, py, qx, qy, w), abs_sums(px, py, qx, qy, w)


def global_motion(flow, occ, hw, flow_scale=1.0, rounds=MOTION_ROUNDS, c=MOTION_CAUCHY, min_weight=MOTION_MIN_WEIGHT):
    """rb_global_motion in fp64 numpy: flow [B,Hn,Wn,2] fp32, occ [B,Hn,Wn] uint8, hw = (Hs, Ws).  Returns (params [B,4],
    weight [B], flags [B] uint8, sums [B,8] of the last round, abs_sums [B,8] of the last round)."""
    B, Hn, Wn, _ = flow.shape
    out = np.zeros((B, 4)), np.zeros(B), np.zeros(B, np.uint8), np.zeros((B, 8)), np.zeros((B, 8))
    for b in range(B):
        m, flag = (1.0, 0.0, 0.0, 0.0), False
        for r in range(rounds + 1):
            s, a = round_sums(flow[b], occ[b], hw, flow_scale, m if r > 0 else None, c)
            if r == 0:
                out[1][b] = s[0] / (Hn * Wn)
                flag = not out[1][b] >= min_weight
            if not flag:
                *mm, flag = solve(s)
            m = tuple(mm) if not flag else (1.0, 0.0, 0.0, 0.0)
        out[0][b], out[2][b], out[3][b], out[4][b] = m, flag, s, a
    return out


def similarity_flow(M, Hn, Wn, Hs, Ws, flow_scale=1.0):
    """The network-grid flow [Hn,Wn,2] fp32 of the similarity M = (a, b, tx, ty) in centred frame pixels: each point p
    moves to M p, expressed in network pixels and divided by flow_scale."""
    px, py, sx, sy = points(Hn, Wn, Hs, Ws)
    a, b, tx, ty = M
    u = (a * px - b * py + tx - px) / sx / flow_scale
    v = (b * px + a * py + ty - py) / sy / flow_scale
    return np.stack([u, v], -1).astype(F32)


def corner_error(M, N, hw):
    """The largest distance between where two similarities (a, b, tx, ty) take the frame's four corners."""
    H, W = hw
    hx, hy = 0.5 * (W - 1), 0.5 * (H - 1)
    c = np.array([[-hx, -hy], [hx, -hy], [-hx, hy], [hx, hy]])

    def apply(m):
        a, b, tx, ty = m
        return np.stack([a * c[:, 0] - b * c[:, 1] + tx, b * c[:, 0] + a * c[:, 1] + ty], -1)
    return float(np.hypot(*(apply(M) - apply(N)).T).max())


def warp(frames, A):
    """rb_frames_warp_affine bit for bit: frames [F,H,W,C] uint8, A [F,2,3] fp64 -> [F,H,W,C] uint8."""
    F, H, W, C = frames.shape
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    out = np.empty_like(frames)
    for f in range(F):
        m = A[f]
        sx = (m[0, 0] * x + m[0, 1] * y) + m[0, 2]
        sy = (m[1, 0] * x + m[1, 1] * y) + m[1, 2]
        with np.errstate(invalid="ignore"):
            fx = np.minimum(np.maximum(np.nan_to_num(sx.astype(F32), nan=0.0), F32(0)), F32(W - 1))
            fy = np.minimum(np.maximum(np.nan_to_num(sy.astype(F32), nan=0.0), F32(0)), F32(H - 1))
        x0, y0 = np.floor(fx).astype(np.int64), np.floor(fy).astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
        ax, ay = (fx - x0.astype(F32)).astype(F32), (fy - y0.astype(F32)).astype(F32)
        cx, cy = F32(1) - ax, F32(1) - ay
        img = frames[f].astype(F32)
        v00, v01, v10, v11 = img[y0, x0], img[y0, x1], img[y1, x0], img[y1, x1]
        t0 = cx[..., None] * v00 + ax[..., None] * v01
        t1 = cx[..., None] * v10 + ax[..., None] * v11
        v = t0 * cy[..., None] + t1 * ay[..., None]
        out[f] = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    return out
