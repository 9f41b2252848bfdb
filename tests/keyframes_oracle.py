"""numpy restatement of several-keyframe label propagation (csrc/propagate.cu: rb_labels_propagate_keys, and
raft_b200.video.keyframe_rows), for the tests.

Per side the work is propagate_oracle.propagate's (resize_flow of the row, origin, clamp, status at the nearest network
pixel, the four taps of the key); the vote over the eight weighted candidates is fp32, every operation rounded on its
own, left to right, so the kernel must reproduce it bit for bit.
"""
from __future__ import annotations

import numpy as np

from propagate_oracle import EDGE, _taps
from resize_oracle import resize_flow

F32 = np.float32
NONE = 3  # no keyframe reaches the pixel


def side(acc, status, key):
    """One side of one row: acc [H,W,2], status [H,W] at the network size, key [Hs,Ws] -> (labels [4,Hs,Ws], weights
    [4,Hs,Ws] fp32, S [Hs,Ws] uint8) in tap order 00, 01, 10, 11."""
    H, W = acc.shape[:2]
    Hs, Ws = key.shape
    A = resize_flow(np.asarray(acc, dtype=F32)[None], Hs, Ws)[0]
    px = np.arange(Ws, dtype=F32)[None, :]
    py = np.arange(Hs, dtype=F32)[:, None]
    ny = (((2 * np.arange(Hs, dtype=np.int64) + 1) * H) // (2 * Hs))[:, None]
    nx = (((2 * np.arange(Ws, dtype=np.int64) + 1) * W) // (2 * Ws))[None, :]
    with np.errstate(invalid="ignore", over="ignore"):
        ox, oy = (px + A[..., 0]).astype(F32), (py + A[..., 1]).astype(F32)
        cx = np.fmin(np.fmax(ox, F32(0)), F32(Ws - 1)).astype(F32)
        cy = np.fmin(np.fmax(oy, F32(0)), F32(Hs - 1)).astype(F32)
        moved = ~((cx == ox) & (cy == oy))
    S = np.where(moved, np.uint8(EDGE), np.asarray(status, dtype=np.uint8)[ny, nx]).astype(np.uint8)
    x0, x1, y0, y1, ax, ay, bx, by = _taps(cx, cy, Hs, Ws)
    lab = np.stack([key[y0, x0], key[y0, x1], key[y1, x0], key[y1, x1]])
    w = np.stack([bx * by, ax * by, bx * ay, ax * ay]).astype(F32)
    return lab, w, S


def vote(lab, w):
    """The vote of N candidates (lab [N,...], w [N,...] fp32): each scores the sum, left to right, of the weights of the
    candidates carrying its label; the largest wins, a tie goes to the smaller label."""
    best = lab[0].copy()
    top = np.full(lab.shape[1:], -1, F32)
    for i in range(len(lab)):
        score = np.zeros(lab.shape[1:], F32)
        for j in range(len(lab)):
            score = np.where(lab[j] == lab[i], score + w[j], score).astype(F32)
        better = (score > top) | ((score == top) & (lab[i] < best))
        top, best = np.where(better, score, top), np.where(better, lab[i], best)
    return best.astype(np.uint8)


def propagate_keys(acc_a, status_a, acc_b, status_b, keys, rows):
    """rb_labels_propagate_keys: acc_* [n,H,W,2], status_* [n,H,W], keys [m,Hs,Ws], rows [n,4] (slot_a, slot_b, w_a,
    w_b) -> (labels [n,Hs,Ws], status [n,Hs,Ws]) uint8."""
    keys = np.asarray(keys, dtype=np.uint8)
    m, Hs, Ws = keys.shape
    n = len(rows)
    labels = np.zeros((n, Hs, Ws), np.uint8)
    st = np.full((n, Hs, Ws), NONE, np.uint8)
    for r in range(n):
        sa, sb, wa, wb = (int(v) for v in rows[r])
        a = side(acc_a[r], status_a[r], keys[sa]) if 0 <= sa < m else None
        b = side(acc_b[r], status_b[r], keys[sb]) if 0 <= sb < m else None
        if a is None and b is None:
            continue
        if a is None or b is None:
            lab, w, S = a if b is None else b
            labels[r], st[r] = vote(lab, w), S
            continue
        (la, wa_, Sa), (lb, wb_, Sb) = a, b
        both = vote(np.concatenate([la, lb]), np.concatenate([wa_ * F32(wa), wb_ * F32(wb)]).astype(F32))
        labels[r] = np.where(Sa == Sb, both, np.where(Sa < Sb, vote(la, wa_), vote(lb, wb_)))
        st[r] = np.minimum(Sa, Sb)
    return labels, st


def keyframe_rows(F, keys, cuts=()):
    """The rules of raft_b200.video.keyframe_rows read literally, frame by frame: [F,4] int32."""
    keys, cuts = list(keys), set(cuts)
    rows = np.zeros((F, 4), np.int32)
    for t in range(F):
        before = [i for i, k in enumerate(keys) if k <= t]
        after = [j for j, k in enumerate(keys) if k > t]
        a = before[-1] if before and not any(c in cuts for c in range(keys[before[-1]], t)) else -1
        b = after[0] if after and not any(c in cuts for c in range(t, keys[after[0]])) else -1
        if t in keys:
            b = -1
        wa = keys[b] - t if a >= 0 and b >= 0 else 0
        wb = t - keys[a] if a >= 0 and b >= 0 else 0
        rows[t] = (a, b, wa, wb)
    return rows
