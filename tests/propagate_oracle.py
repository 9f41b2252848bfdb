"""numpy restatement of keyframe label propagation (csrc/propagate.cu: rb_flow_accumulate / _backward and
rb_labels_propagate), for the tests.

Everything is fp32 in the kernels' operation order -- every operation rounded on its own, left to right, no FMA -- so the
kernels must reproduce it bit for bit.  The per-pixel resize of the displacement is tests/resize_oracle.py's resize_flow.
Status: 0 consistent at every step back to the keyframe, 1 occluded at some step, 2 entered through the frame edge at
some step (the larger value wins).
"""
from __future__ import annotations

import numpy as np

from resize_oracle import resize_flow

F32 = np.float32
CONSISTENT, OCCLUDED, EDGE = 0, 1, 2


def _taps(qx, qy, H, W):
    """bilerp_at: the taps and weights of points inside [0, W-1] x [0, H-1]."""
    fx0, fy0 = np.floor(qx), np.floor(qy)
    x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = (qx - fx0).astype(F32), (qy - fy0).astype(F32)
    return x0, x1, y0, y1, ax, ay, (F32(1) - ax).astype(F32), (F32(1) - ay).astype(F32)


def _bilerp(v, t):
    """bilerp1 of the [H,W] channel v at the taps t."""
    x0, x1, y0, y1, ax, ay, cx, cy = t
    t0 = cx * v[y0, x0] + ax * v[y0, x1]
    t1 = cx * v[y1, x0] + ax * v[y1, x1]
    return t0 * cy + t1 * ay


def step(pull, test, prev_acc, prev_st, s=1.0, a1=0.01, a2=0.5):
    """One accumulation step: pull / test [H,W,2] (the flow from this frame to the chain's previous one, and the opposite
    flow of that pair), the previous row (prev_acc [H,W,2], prev_st [H,W]) -> (acc [H,W,2] fp32, status [H,W] uint8)."""
    H, W = pull.shape[:2]
    s, a1, a2 = F32(s), F32(a1), F32(a2)
    pull, test, prev_acc = (np.asarray(a, dtype=F32) for a in (pull, test, prev_acc))
    with np.errstate(invalid="ignore", over="ignore"):
        fx, fy = s * pull[..., 0], s * pull[..., 1]
        px = np.broadcast_to(np.arange(W, dtype=F32)[None, :], (H, W))
        py = np.broadcast_to(np.arange(H, dtype=F32)[:, None], (H, W))
        qx, qy = px + fx, py + fy
        inside = (qx >= 0) & (qx <= F32(W - 1)) & (qy >= 0) & (qy <= F32(H - 1))  # NaN -> outside
        cx = np.where(inside, qx, np.fmin(np.fmax(qx, F32(0)), F32(W - 1))).astype(F32)  # fmaxf(NaN, 0) = 0
        cy = np.where(inside, qy, np.fmin(np.fmax(qy, F32(0)), F32(H - 1))).astype(F32)
        dx = np.where(inside, fx, cx - px).astype(F32)
        dy = np.where(inside, fy, cy - py).astype(F32)
        t = _taps(cx, cy, H, W)
        bx, by = s * _bilerp(test[..., 0], t), s * _bilerp(test[..., 1], t)
        ex, ey = fx + bx, fy + by
        d = ex * ex + ey * ey
        m = a1 * (((fx * fx + fy * fy) + bx * bx) + by * by) + a2
        st = np.where(inside, (d > m).astype(np.uint8), np.uint8(EDGE))
        acc = np.stack([dx + _bilerp(prev_acc[..., 0], t), dy + _bilerp(prev_acc[..., 1], t)], -1).astype(F32)
    x0, x1, y0, y1, ax, ay = t[:6]
    nx, ny = np.where(ax > F32(0.5), x1, x0), np.where(ay > F32(0.5), y1, y0)
    return acc, np.maximum(st, np.asarray(prev_st, dtype=np.uint8)[ny, nx]).astype(np.uint8)


def accumulate(flow_fw, flow_bw, acc, status, start=0, n_steps=None, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """rb_flow_accumulate: flows [T,H,W,2]; acc [n_steps+1,H,W,2] and status [n_steps+1,H,W] with row `start` the input
    -> copies with rows start+1 .. n_steps written."""
    T = np.shape(flow_fw)[0]
    n_steps = T if n_steps is None else int(n_steps)
    acc, status = np.array(acc, dtype=F32), np.array(status, dtype=np.uint8)
    for r in range(start + 1, n_steps + 1):
        acc[r], status[r] = step(flow_bw[r - 1], flow_fw[r - 1], acc[r - 1], status[r - 1], flow_scale, alpha1, alpha2)
    return acc, status


def accumulate_backward(flow_fw, flow_bw, acc, status, start=0, n_steps=None, flow_scale=1.0, alpha1=0.01,
                        alpha2=0.5):
    """rb_flow_accumulate_backward: as accumulate, rows start-1 .. 0 written (step r+1 -> r pulls with flow_fw[r])."""
    acc, status = np.array(acc, dtype=F32), np.array(status, dtype=np.uint8)
    for r in range(start - 1, -1, -1):
        acc[r], status[r] = step(flow_fw[r], flow_bw[r], acc[r + 1], status[r + 1], flow_scale, alpha1, alpha2)
    return acc, status


def keyframe_rows(n_rows, H, W, key_row):
    """acc / status of n_rows rows with zeros (and status 0) at key_row and garbage elsewhere, as the kernels get them."""
    acc = np.full((n_rows, H, W, 2), np.nan, F32)
    status = np.full((n_rows, H, W), 77, np.uint8)
    acc[key_row], status[key_row] = 0, 0
    return acc, status


def vote(key, ox, oy):
    """The label vote at origins (ox, oy) inside the [Hs,Ws] key: each distinct label of the four taps scores the sum of
    its weights in tap order 00, 01, 10, 11; the largest wins, a tie goes to the smaller label."""
    Hs, Ws = key.shape
    x0, x1, y0, y1, ax, ay, cx, cy = _taps(ox, oy, Hs, Ws)
    lab = [key[y0, x0], key[y0, x1], key[y1, x0], key[y1, x1]]
    w = [cx * cy, ax * cy, cx * ay, ax * ay]
    best = lab[0].copy()
    top = np.full(ox.shape, -1, F32)
    for i in range(4):
        score = np.zeros(ox.shape, F32)
        for j in range(4):
            score = np.where(lab[j] == lab[i], score + w[j], score).astype(F32)
        better = (score > top) | ((score == top) & (lab[i] < best))
        top, best = np.where(better, score, top), np.where(better, lab[i], best)
    return best.astype(np.uint8)


def propagate(acc, status, key):
    """rb_labels_propagate: acc [n,H,W,2], status [n,H,W] at the network size, key [Hs,Ws] uint8 -> (labels [n,Hs,Ws],
    status [n,Hs,Ws]) uint8."""
    acc, status, key = np.asarray(acc, dtype=F32), np.asarray(status, dtype=np.uint8), np.asarray(key, dtype=np.uint8)
    n, H, W = acc.shape[:3]
    Hs, Ws = key.shape
    A = resize_flow(acc, Hs, Ws)
    px = np.arange(Ws, dtype=F32)[None, :]
    py = np.arange(Hs, dtype=F32)[:, None]
    ny = (((2 * np.arange(Hs, dtype=np.int64) + 1) * H) // (2 * Hs))[:, None]
    nx = (((2 * np.arange(Ws, dtype=np.int64) + 1) * W) // (2 * Ws))[None, :]
    labels = np.empty((n, Hs, Ws), np.uint8)
    st = np.empty((n, Hs, Ws), np.uint8)
    for i in range(n):
        with np.errstate(invalid="ignore", over="ignore"):
            ox, oy = (px + A[i, ..., 0]).astype(F32), (py + A[i, ..., 1]).astype(F32)
            cx = np.fmin(np.fmax(ox, F32(0)), F32(Ws - 1)).astype(F32)
            cy = np.fmin(np.fmax(oy, F32(0)), F32(Hs - 1)).astype(F32)
            moved = ~((cx == ox) & (cy == oy))
        st[i] = np.where(moved, np.uint8(EDGE), status[i][ny, nx])
        labels[i] = vote(key, cx, cy)
    return labels, st


def reversed_clip(flow_fw, flow_bw):
    """The clip played backward: fw'[k] = flow_bw[T-1-k], bw'[k] = flow_fw[T-1-k]."""
    return np.ascontiguousarray(flow_bw[::-1]), np.ascontiguousarray(flow_fw[::-1])
