"""numpy restatement of the video-denoising kernels rb_denoise_merge and rb_noise_sums (csrc/denoise.cu), bit for bit:
every fp32 operation rounded on its own in the kernel's order (numpy float32 arithmetic does not contract), the chain
step tests/track_oracle.py's, the pixel-centre maps tests/inpaint_oracle.py's."""
from __future__ import annotations

import numpy as np

from inpaint_oracle import _remap
from raft_b200.denoise import H, MAX_WINDOW, PATCH, SEARCH

F32 = np.float32
R = SEARCH + PATCH  # samples at integer offsets -R .. R around a match


def samples(img, ox, oy):
    """The replicate-padded frame img [Hs,Ws,3] uint8 sampled at (ox, oy) + delta for the (2R+1)^2 integer offsets delta,
    with (ox, oy)'s bilinear weights: [N,2R+1,2R+1,3] fp32."""
    Hs, Ws = img.shape[:2]
    x0, y0 = np.floor(ox).astype(np.int64), np.floor(oy).astype(np.int64)
    ax, ay = (ox - x0.astype(F32)).astype(F32), (oy - y0.astype(F32)).astype(F32)
    cx, cy = (F32(1) - ax).astype(F32), (F32(1) - ay).astype(F32)
    taps = np.arange(-R, R + 2)
    cols = np.clip(x0[:, None] + taps, 0, Ws - 1)
    rows = np.clip(y0[:, None] + taps, 0, Hs - 1)
    v = img[rows[:, :, None], cols[:, None, :]].astype(F32)  # [N,6,6,3]
    h = (cx[:, None, None, None] * v[:, :, :-1]) + (ax[:, None, None, None] * v[:, :, 1:])  # [N,6,5,3]
    return (h[:, :-1] * cy[:, None, None, None]) + (h[:, 1:] * ay[:, None, None, None])


def _merge(S, ref, two_var, den, acc, wsum):
    """The (2 SEARCH + 1)^2 candidates of one frame's samples S added to (acc [N,3], wsum [N]) in raster order."""
    P = 2 * PATCH + 1
    for sy in range(2 * SEARCH + 1):
        for sx in range(2 * SEARCH + 1):
            d = np.zeros(len(S), F32)
            for uy in range(P):
                for ux in range(P):
                    for c in range(3):
                        e = S[:, sy + uy, sx + ux, c] - ref[:, uy, ux, c]
                        d = d + e * e
            d = d / F32(P * P * 3)
            num = np.maximum(d - two_var, F32(0))
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                x = np.where(num > 0, num / den, F32(0)).astype(F32)
            om = F32(1) - x
            w = np.where(x < 1, om * om, F32(0)).astype(F32)
            acc += w[:, None] * S[:, sy + PATCH, sx + PATCH]
            wsum += w


def denoise_merge(frames, fw, bw, rows, sigma, s=1.0, a1=0.01, a2=0.5):
    """rb_denoise_merge: frames [F,Hs,Ws,3] uint8, fw / bw [F-1,Hn,Wn,2] fp32, rows [n,3], sigma > 0 ->
    (out [n,Hs,Ws,3] uint8, support [n,Hs,Ws] uint8)."""
    from track_oracle import step
    frames = np.asarray(frames)
    F, Hs, Ws, _ = frames.shape
    Hn, Wn = (fw.shape[1:3] if fw is not None and len(fw) else (Hs, Ws))
    sg = F32(sigma)
    two_var = F32(2) * (sg * sg)
    hs = F32(H) * sg
    den = hs * hs
    n = len(rows)
    out = np.zeros((n, Hs, Ws, 3), np.uint8)
    support = np.zeros((n, Hs, Ws), np.uint8)
    ys, xs = (a.reshape(-1) for a in np.mgrid[0:Hs, 0:Ws])
    N = len(xs)
    pu = np.arange(-PATCH, PATCH + 1)
    for r, (t, nf, nb) in enumerate(np.asarray(rows).tolist()):
        if not 0 <= t < F:
            continue
        img = frames[t]
        ry = np.clip(ys[:, None] + pu, 0, Hs - 1)
        rx = np.clip(xs[:, None] + pu, 0, Ws - 1)
        ref = img[ry[:, :, None], rx[:, None, :]].astype(F32)  # [N,3,3,3]
        acc, wsum = np.zeros((N, 3), F32), np.zeros(N, F32)
        _merge(samples(img, xs.astype(F32), ys.astype(F32)), ref, two_var, den, acc, wsum)
        sup = np.zeros(N, np.int64)
        px, py = _remap(xs, Wn / Ws, Wn), _remap(ys, Hn / Hs, Hn)
        for direction, m in ((1, min(max(nf, 0), MAX_WINDOW, F - 1 - t)), (-1, min(max(nb, 0), MAX_WINDOW, t))):
            live, qx, qy = np.arange(N), px.copy(), py.copy()
            for k in range(1, m + 1):
                pair = t + k - 1 if direction > 0 else t - k
                pull, test = (fw[pair], bw[pair]) if direction > 0 else (bw[pair], fw[pair])
                nx, ny, st = step(pull, test, qx[live], qy[live], s, a1, a2)
                keep = st == 0
                live = live[keep]
                if not len(live):
                    break
                qx[live], qy[live] = nx[keep], ny[keep]
                ox, oy = _remap(qx[live], Ws / Wn, Ws), _remap(qy[live], Hs / Hn, Hs)
                a, w = acc[live], wsum[live]
                _merge(samples(frames[t + direction * k], ox, oy), ref[live], two_var, den, a, w)
                acc[live], wsum[live] = a, w
                sup[live] += 1
        out[r] = np.clip(np.rint(acc / wsum[:, None]), 0, 255).astype(np.uint8).reshape(Hs, Ws, 3)
        support[r] = sup.reshape(Hs, Ws)
    return out, support


def noise_sums(frames):
    """rb_noise_sums: frames [N,H,W,3] uint8 -> [N,3] int64 sums of |I * M| over the interior pixels."""
    f = np.asarray(frames).astype(np.int64)
    M = np.array([[1, -2, 1], [-2, 4, -2], [1, -2, 1]], np.int64)
    H, W = f.shape[1:3]
    conv = np.zeros((f.shape[0], H - 2, W - 2, 3), np.int64)
    for i in range(3):
        for j in range(3):
            conv += M[i, j] * f[:, i:i + H - 2, j:j + W - 2]
    return np.abs(conv).sum(axis=(1, 2))
