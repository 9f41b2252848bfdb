"""numpy restatement of the motion-segmentation kernels (csrc/motionseg.cu): rb_homography_motion's per-round sums and
Cholesky solve in fp64 (to rounding: the kernel's fixed reduction order is not restated), and rb_motion_evidence /
rb_motion_segment bit for bit -- every fp64 and fp32 operation rounded on its own in the kernel's order, the chain step
tests/track_oracle.py's, the pixel-centre map tests/inpaint_oracle.py's."""
from __future__ import annotations

import numpy as np

import stabilize_oracle as SO
from inpaint_oracle import _remap
from raft_b200.motionseg import CAUCHY, MAX_WINDOW, ROUNDS, TAU

F32, F64 = np.float32, np.float64
TRI = [(r, c) for r in range(8) for c in range(r, 8)]  # the upper triangle's order in the sums, after S


def geometry(Hn, Wn, Hs, Ws, fs):
    """The kernels' per-field constants: (sx, sy, cx, cy, isx, isy, fs, L, invL)."""
    L = 0.5 * max(Ws, Hs)
    return Ws / Wn, Hs / Hn, 0.5 * (Ws - 1), 0.5 * (Hs - 1), Wn / Ws, Hn / Hs, float(F32(fs)), L, 1.0 / L


def points(flow, hw, fs):
    """Normalised points (x, y) and targets (qx, qy) [Hn,Wn] fp64 of one field, and its geometry, each operation rounded
    in rb_motion_evidence's order."""
    Hn, Wn = flow.shape[:2]
    sx, sy, cx, cy, isx, isy, fs, L, invL = g = geometry(Hn, Wn, hw[0], hw[1], fs)
    i, j = (a.astype(F64) for a in np.mgrid[0:Hn, 0:Wn])
    px, py = ((j + 0.5) * sx - 0.5) - cx, ((i + 0.5) * sy - 0.5) - cy
    qx = (px + fs * (flow[..., 0].astype(F64) * sx)) * invL
    qy = (py + fs * (flow[..., 1].astype(F64) * sy)) * invL
    return px * invL, py * invL, qx, qy, g


def project(h, x, y):
    """(X, Y, z) of H (x, y, 1), each sum left to right."""
    h = np.asarray(h, F64).reshape(9)
    return (h[0] * x + h[1] * y) + h[2], (h[3] * x + h[4] * y) + h[5], (h[6] * x + h[7] * y) + 1.0


def usable(flow, occ):
    return (occ == 0) & np.isfinite(flow[..., 0]) & np.isfinite(flow[..., 1])


def round_sums(flow, occ, hw, fs, h, c=CAUCHY):
    """One round's 45 sums of one field under the previous estimate h, and the sums of their terms' magnitudes."""
    x, y, qx, qy, g = points(flow, hw, fs)
    L, isx, isy = g[7], g[4], g[5]
    X, Y, z = project(h, x, y)
    with np.errstate(all="ignore"):
        ex, ey = (X / z - qx) * (L * isx), (Y / z - qy) * (L * isy)
        r2 = ex * ex + ey * ey
        w = 1.0 / (1.0 + r2 / (c * c)) / (z * z)
    ok = usable(flow, occ) & (z > 0) & np.isfinite(r2)
    w, x, y, qx, qy = w[ok], x[ok], y[ok], qx[ok], qy[ok]
    zero, one = np.zeros_like(x), np.ones_like(x)
    ax = [x, y, one, zero, zero, zero, -x * qx, -y * qx]
    ay = [zero, zero, zero, x, y, one, -x * qy, -y * qy]
    terms = [w] + [w * (ax[r] * ax[c] + ay[r] * ay[c]) for r, c in TRI] + [w * (ax[r] * qx + ay[r] * qy) for r in range(8)]
    return np.array([t.sum() for t in terms]), np.array([np.abs(t).sum() for t in terms])


def solve(s):
    """The 8 x 8 system of the sums by Cholesky in fp64 (the kernel's pivot rule), or None when singular."""
    if not s[0] > 0:
        return None
    A = np.zeros((8, 8))
    for k, (r, c) in enumerate(TRI):
        A[r, c] = A[c, r] = s[1 + k]
    Lm = np.zeros((8, 8))
    for j in range(8):
        d = A[j, j] - np.dot(Lm[j, :j], Lm[j, :j])
        if not d > 1e-12 * A[j, j]:
            return None
        Lm[j, j] = np.sqrt(d)
        for i in range(j + 1, 8):
            Lm[i, j] = (A[i, j] - np.dot(Lm[i, :j], Lm[j, :j])) / Lm[j, j]
    yv = np.zeros(8)
    for i in range(8):
        yv[i] = (s[37 + i] - np.dot(Lm[i, :i], yv[:i])) / Lm[i, i]
    h = np.zeros(8)
    for i in range(7, -1, -1):
        h[i] = (yv[i] - np.dot(Lm[i + 1:, i], h[i + 1:])) / Lm[i, i]
    return h if np.isfinite(h).all() else None


def similarity_h(m, L):
    a, b, tx, ty = m
    return np.array([[a, -b, tx / L], [b, a, ty / L], [0, 0, 1]], F64)


def homography(flow, occ, hw, fs, sim, sim_flags, rounds=ROUNDS, c=CAUCHY):
    """rb_homography_motion of B fields -> (H [B,3,3], flags [B] uint8, sums [B,45] and abs_sums [B,45] of the last
    round, prev [B,3,3]: the estimate the last round started from)."""
    B = len(flow)
    L = 0.5 * max(hw)
    H, flags = np.zeros((B, 3, 3)), np.zeros(B, np.uint8)
    S, A, P = np.zeros((B, 45)), np.zeros((B, 45)), np.zeros((B, 3, 3))
    for b in range(B):
        h0 = np.eye(3) if sim_flags[b] else similarity_h(sim[b], L)
        h, flag = h0, 2 if sim_flags[b] else 0
        for _ in range(rounds):
            P[b] = h
            S[b], A[b] = round_sums(flow[b], occ[b], hw, fs, h, c)
            if flag:
                continue
            sol = solve(S[b])
            if sol is None:
                h, flag = h0, 1
            else:
                h = np.append(sol, 1.0).reshape(3, 3)
        H[b], flags[b] = h, flag
    return H, flags, S, A, P


def fit(flow, occ, hw, fs, rounds=ROUNDS):
    """F22 then F34 on a batch of fields, as raft_b200.motionseg.fit_fields: (H, flags)."""
    sim, _, sflags, _, _ = SO.global_motion(flow, occ, hw, fs)
    return homography(flow, occ, hw, fs, sim, sflags, rounds)[:2]


def field_e(flow, occ, h, hw, fs, tau):
    """e [Hn,Wn] fp32 of one field and where it counts (before the flag and cut rules), bit for bit."""
    x, y, qx, qy, g = points(flow, hw, fs)
    isx, isy, L = g[4], g[5], g[7]
    X, Y, z = project(h, x, y)
    with np.errstate(all="ignore"):
        dx = ((X / z - qx) * L) * isx
        dy = ((Y / z - qy) * L) * isy
        r2 = (dx * dx + dy * dy).astype(F32)
        t2 = F32(tau) * F32(tau)
        e = (r2 / (r2 + t2)).astype(F32)
    e = np.where((z > 0) & np.isfinite(r2), e, F32(1)).astype(F32)
    return e, usable(flow, occ)


def evidence(fw, bw, ofw, obw, H, flags, hw, fs=1.0, cuts=None, tau=TAU):
    """rb_motion_evidence: [T+1,Hn,Wn,2] fp32 (N, C), bit for bit."""
    T, Hn, Wn = fw.shape[:3]
    cut = np.zeros(T, bool) if cuts is None else np.asarray(cuts).astype(bool)
    ev = np.zeros((T + 1, Hn, Wn, 2), F32)
    for t in range(T + 1):
        N, C = np.zeros((Hn, Wn), F32), np.zeros((Hn, Wn), F32)
        for k, field, flow, occ in ((t, t, fw, ofw), (t - 1, T + t - 1, bw, obw)):
            if not 0 <= k < T or flags[field] > 1 or cut[k]:
                continue
            e, ok = field_e(flow[k], occ[k], H[field], hw, fs, tau)
            N = np.where(ok, N + e, N).astype(F32)
            C = np.where(ok, C + F32(1), C).astype(F32)
        ev[t, ..., 0], ev[t, ..., 1] = N, C
    return ev


def _sample_ev(ev, qx, qy):
    """The bilinear sample of (N, C) [Hn,Wn,2] at points inside the grid, fb_sample.cuh's bilerp1 order."""
    Hn, Wn = ev.shape[:2]
    x0, y0 = np.floor(qx).astype(np.int64), np.floor(qy).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, Wn - 1), np.minimum(y0 + 1, Hn - 1)
    ax, ay = (qx - x0.astype(F32)).astype(F32), (qy - y0.astype(F32)).astype(F32)
    cx, cy = F32(1) - ax, F32(1) - ay
    out = []
    for c in range(2):
        v = ev[..., c]
        t0 = cx * v[y0, x0] + ax * v[y0, x1]
        t1 = cx * v[y1, x0] + ax * v[y1, x1]
        out.append((t0 * cy + t1 * ay).astype(F32))
    return out


def segment(ev, fw, bw, hw, rows, s=1.0, a1=0.01, a2=0.5):
    """rb_motion_segment: (mask [n,Hs,Ws] uint8, status [n,Hs,Ws] uint8), bit for bit."""
    from track_oracle import step
    F, Hn, Wn = ev.shape[:3]
    Hs, Ws = hw
    ys, xs = (a.reshape(-1) for a in np.mgrid[0:Hs, 0:Ws])
    px, py = _remap(xs, Wn / Ws, Wn), _remap(ys, Hn / Hs, Hn)
    n = len(rows)
    mask, status = np.zeros((n, Hs, Ws), np.uint8), np.ones((n, Hs, Ws), np.uint8)
    for r, (t, nf, nb) in enumerate(np.asarray(rows).tolist()):
        if not 0 <= t < F:
            mask[r] = 0
            continue
        num, den = _sample_ev(ev[t], px, py)
        for direction, m in ((1, min(max(nf, 0), MAX_WINDOW, F - 1 - t)), (-1, min(max(nb, 0), MAX_WINDOW, t))):
            live, qx, qy = np.arange(len(xs)), px.copy(), py.copy()
            for k in range(1, m + 1):
                pair = t + k - 1 if direction > 0 else t - k
                pull, test = (fw[pair], bw[pair]) if direction > 0 else (bw[pair], fw[pair])
                nx, ny, st = step(pull, test, qx[live], qy[live], s, a1, a2)
                keep = st == 0
                live = live[keep]
                if not len(live):
                    break
                qx[live], qy[live] = nx[keep], ny[keep]
                en, ec = _sample_ev(ev[t + direction * k], qx[live], qy[live])
                num[live] = (num[live] + en).astype(F32)
                den[live] = (den[live] + ec).astype(F32)
        mask[r] = ((den > 0) & (F32(2) * num >= den)).reshape(Hs, Ws)
        status[r] = (den <= 0).reshape(Hs, Ws)
    return mask, status


def segment_clip(fw, bw, ofw, obw, hw, rows, fs=1.0, cuts=(), tau=TAU, a1=0.01, a2=0.5):
    """The whole of RaftEngine.segment_motion after the flow pass: (mask, status, H [2T,3,3], flags [2T], ev)."""
    T = len(fw)
    H, flags = fit(np.concatenate([fw, bw]), np.concatenate([ofw, obw]), hw, fs)
    cut = np.zeros(T, np.uint8)
    cut[list(cuts)] = 1
    ev = evidence(fw, bw, ofw, obw, H, flags, hw, fs, cut, tau)
    mask, status = segment(ev, fw, bw, hw, rows, fs, a1, a2)
    return mask, status, H, flags, ev
