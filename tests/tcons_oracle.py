"""numpy restatement of the temporal-consistency kernels rb_tcons_terms, rb_screened_poisson and rb_warp_error
(csrc/temporal.cu), bit for bit: every fp32 operation is a numpy float32 operation rounded on its own in the kernel's
order, every fp64 dot product follows the kernel's fixed reduction tree.  The step is tests/track_oracle.py's, the
pixel-centre maps tests/inpaint_oracle.py's, the bilinear sample tests/stabfill_oracle.py's.  Also the fp64 sparse
solve the solver is held to."""
import numpy as np

from inpaint_oracle import _children, _colours, _nbrs, _prolong, _remap
from raft_b200.inpaint import fill_levels
from raft_b200.temporal import EPS, ITERS, KAPPA, SWEEPS
from stabfill_oracle import _bilinear
from track_oracle import step

F32 = np.float32
THREADS, PER_THREAD = 256, 4


def _step(pull, test, Hs, Ws, s, a1, a2):
    """One step of every frame pixel through pull tested by test: (ok [N] bool, ox, oy [N] fp32 frame positions)."""
    Hn, Wn = pull.shape[:2]
    ys, xs = (a.reshape(-1) for a in np.mgrid[0:Hs, 0:Ws])
    px, py = _remap(xs, Wn / Ws, Wn), _remap(ys, Hn / Hs, Hn)
    qx, qy, st = step(pull, test, px, py, s, a1, a2)
    ok = st == 0
    ox = np.where(ok, _remap(np.where(ok, qx, 0), Ws / Wn, Ws), F32(0)).astype(F32)
    oy = np.where(ok, _remap(np.where(ok, qy, 0), Hs / Hn, Hs), F32(0)).astype(F32)
    return ok, ox, oy


def tcons_terms(frame, prev_frame, processed, prev_out, fw, bw, strength, s=1.0, a1=0.01, a2=0.5):
    """rb_tcons_terms: [Hs,Ws,3] uint8 frames (prev_frame None: no previous frame), fw / bw [Hn,Wn,2] fp32 the pair
    (t-1, t) -> (c [Hs,Ws] fp32, r [Hs,Ws,3] fp32, status [Hs,Ws] uint8)."""
    Hs, Ws = processed.shape[:2]
    N = Hs * Ws
    lw = np.zeros(N, F32)
    ro = np.zeros((N, 3), F32)
    status = np.full(N, 3, np.uint8)
    if prev_frame is not None:
        ok, ox, oy = _step(bw, fw, Hs, Ws, s, a1, a2)
        status[:] = 1
        idx = np.flatnonzero(ok)
        It = frame.reshape(N, 3)[idx].astype(F32)
        e = (It - _bilinear(prev_frame, ox[idx], oy[idx])).astype(F32)
        d = np.zeros(len(idx), F32)
        for ch in range(3):
            d = (d + (e[:, ch] * e[:, ch]).astype(F32)).astype(F32)
        d = (d / F32(3)).astype(F32)
        x = (d / (F32(KAPPA) * F32(KAPPA))).astype(F32)
        used = x < 1
        om = (F32(1) - x).astype(F32)
        w = np.where(used, (om * om).astype(F32), F32(0)).astype(F32)
        status[idx] = np.where(used, 0, 2).astype(np.uint8)
        lw[idx] = (F32(strength) * w).astype(F32)
        diff = (_bilinear(prev_out, ox[idx], oy[idx]) - processed.reshape(N, 3)[idx].astype(F32)).astype(F32)
        ro[idx] = np.where(used[:, None], diff, F32(0))
    c = (lw + F32(EPS)).astype(F32)
    r = np.where((status == 0)[:, None], (lw[:, None] * ro).astype(F32), F32(0)).astype(F32)
    return c.reshape(Hs, Ws), r.reshape(Hs, Ws, 3), status.reshape(Hs, Ws)


# ---- rb_screened_poisson ----

def _nbsum(e, f):
    """s = f + e_up + e_down + e_left + e_right (+0 outside) and the neighbour count n, as float32."""
    s = f.copy() if f is not None else np.zeros_like(e)
    n = np.zeros(e.shape[:2], F32)
    for sh, ok in _nbrs(e):
        s = (s + sh).astype(F32)
        n = (n + ok.astype(F32)).astype(F32)
    return s, n


def _resid(c, f, e):
    s, n = _nbsum(e, f)
    return (s - ((n[..., None] * e).astype(F32) + (c[..., None] * e).astype(F32)).astype(F32)).astype(F32)


def _sweeps(c, f, e):
    col = _colours(*c.shape)
    for _ in range(SWEEPS):
        for colour in (0, 1):
            s, n = _nbsum(e, f)
            diag = (c + n).astype(F32)
            e = np.where((col == colour)[..., None], (s / diag[..., None]).astype(F32), e)
    return e


def _restrict(a, h, w):
    out = np.zeros((h, w) + a.shape[2:], F32)
    for t, _ in _children(a, h, w, 0):
        out = (out + t).astype(F32)
    return out


def vcycle(cs, levels, f0):
    """The preconditioner V(f0) on the pyramid cs of c: from e = 0, down and up."""
    es, fs = [np.zeros_like(f0)], [f0]
    for l in range(len(levels) - 1):
        es[l] = _sweeps(cs[l], fs[l], es[l])
        h, w = levels[l + 1]
        fs.append(_restrict(_resid(cs[l], fs[l], es[l]), h, w))
        es.append(np.zeros((h, w, 3), F32))
    es[-1] = _sweeps(cs[-1], fs[-1], es[-1])
    for l in range(len(levels) - 2, -1, -1):
        es[l] = (es[l] + _prolong(es[l + 1], *levels[l])).astype(F32)
        es[l] = _sweeps(cs[l], fs[l], es[l])
    return es[0]


def _tree(v):
    """The block tree s[t] += s[t + h], h = 128, ..., 1 over axis 1 of v [n,256,3]."""
    v = v.copy()
    h = THREADS // 2
    while h:
        v[:, :h] = v[:, :h] + v[:, h:2 * h]
        h //= 2
    return v[:, 0]


def dot(a, b):
    """<a, b> per channel of [H,W,3] fp32 fields in fp64, in rb_screened_poisson's reduction order: [3] fp64."""
    p = a.reshape(-1, 3).astype(np.float64) * b.reshape(-1, 3).astype(np.float64)
    chunk = THREADS * PER_THREAD
    nb = -(-len(p) // chunk)
    pad = np.zeros((nb * chunk, 3))
    pad[:len(p)] = p
    pad = pad.reshape(nb, PER_THREAD, THREADS, 3)
    v = np.zeros((nb, THREADS, 3))
    for k in range(PER_THREAD):
        v = v + pad[:, k]
    part = _tree(v)  # [nb,3]
    rounds = -(-nb // THREADS)
    pp = np.zeros((rounds * THREADS, 3))
    pp[:nb] = part
    pp = pp.reshape(rounds, THREADS, 3)
    v = np.zeros((1, THREADS, 3))
    for k in range(rounds):
        v = v + pp[k][None]
    return _tree(v)[0]


def _ratio(num, den):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, num / np.where(den > 0, den, 1.0), 0.0).astype(F32)


def screened_poisson(c, r):
    """rb_screened_poisson: c [H,W] fp32, r [H,W,3] fp32 -> D [H,W,3] fp32."""
    c, r = np.asarray(c, F32), np.asarray(r, F32)
    levels = fill_levels(*c.shape)
    cs = [c]
    for h, w in levels[1:]:
        cs.append(_restrict(cs[-1], h, w))
    x = np.zeros_like(r)
    res = r.copy()
    z = vcycle(cs, levels, res)
    p = z.copy()
    rho = dot(res, z)
    for it in range(ITERS):
        q = (-_resid(c, None, p)).astype(F32)
        alpha = _ratio(rho, dot(p, q))
        x = (x + (alpha * p).astype(F32)).astype(F32)
        new = (res - (alpha * q).astype(F32)).astype(F32)
        d = (new - res).astype(F32)
        res = new
        if it == ITERS - 1:
            break
        z = vcycle(cs, levels, res)
        beta = _ratio(dot(z, d), rho)
        rho = dot(res, z)
        p = (z + (beta * p).astype(F32)).astype(F32)
    return x


def screened_poisson_f64(c, r):
    """The fp64 scipy.sparse solution of the same system: [H,W,3] fp64."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    H, W = c.shape
    idx = np.arange(H * W).reshape(H, W)
    rows, cols = [], []
    n = np.zeros((H, W))
    for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        y0, y1, x0, x1 = max(0, -dy), min(H, H - dy), max(0, -dx), min(W, W - dx)
        rows.append(idx[y0:y1, x0:x1].ravel())
        cols.append(idx[y0 + dy:y1 + dy, x0 + dx:x1 + dx].ravel())
        n[y0:y1, x0:x1] += 1
    off = sum(len(a) for a in rows)
    A = sp.csc_matrix((np.concatenate([-np.ones(off), (np.asarray(c, np.float64) + n).ravel()]),
                       (np.concatenate(rows + [idx.ravel()]), np.concatenate(cols + [idx.ravel()]))),
                      shape=(H * W, H * W))
    lu = spla.splu(A)
    return np.stack([lu.solve(np.asarray(r[..., k], np.float64).ravel()).reshape(H, W) for k in range(3)], -1)


def finish(processed, D):
    """O = clamp(rint(P + D), 0, 255) as uint8."""
    return np.clip(np.rint((processed.astype(F32) + D).astype(F32)), 0, 255).astype(np.uint8)


def consistent(frames, processed, fw, bw, strength, cuts=(), s=1.0, a1=0.01, a2=0.5):
    """The whole causal pass: frames, processed [F,Hs,Ws,3] uint8, fw / bw [F-1,Hn,Wn,2] -> (out, status)."""
    out, status = np.empty_like(processed), np.empty(processed.shape[:3], np.uint8)
    for t in range(len(frames)):
        restart = t == 0 or (t - 1) in set(cuts)
        if restart:
            out[t], status[t] = processed[t], 3
            continue
        c, r, st = tcons_terms(frames[t], frames[t - 1], processed[t], out[t - 1], fw[t - 1], bw[t - 1], strength, s,
                               a1, a2)
        out[t], status[t] = finish(processed[t], screened_poisson(c, r)), st
    return out, status


# ---- rb_warp_error ----

def warp_error_terms(video, fw, bw, s=1.0, a1=0.01, a2=0.5):
    """Per pair k and pixel of frame k: (e [T,Hs,Ws] fp32, valid [T,Hs,Ws] bool)."""
    T = len(fw)
    Hs, Ws = video.shape[1:3]
    N = Hs * Ws
    es, valid = np.zeros((T, N), F32), np.zeros((T, N), bool)
    for k in range(T):
        ok, ox, oy = _step(fw[k], bw[k], Hs, Ws, s, a1, a2)
        idx = np.flatnonzero(ok)
        dif = (video[k].reshape(N, 3)[idx].astype(F32) - _bilinear(video[k + 1], ox[idx], oy[idx])).astype(F32)
        e = np.zeros(len(idx), F32)
        for ch in range(3):
            e = (e + (dif[:, ch] * dif[:, ch]).astype(F32)).astype(F32)
        es[k, idx], valid[k] = e, ok
    return es.reshape(T, Hs, Ws), valid.reshape(T, Hs, Ws)


def warp_error_sums(video, fw, bw, s=1.0, a1=0.01, a2=0.5):
    """[T,2] fp64 (sum e, count) per pair."""
    e, valid = warp_error_terms(video, fw, bw, s, a1, a2)
    return np.stack([np.where(valid, e.astype(np.float64), 0).sum((1, 2)), valid.sum((1, 2)).astype(np.float64)], 1)
