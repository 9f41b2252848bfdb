"""numpy restatements of F24 (rb_masked_fill: the membrane fill, coarse to fine with red-black Gauss-Seidel) and F25
(rb_inpaint_masks: the hole masks at the frames' size and on the network grid; rb_inpaint_propagate: the temporal fill),
bit for bit: every fp32 operation is a numpy float32 operation, rounded on its own.  Also the fp64 sparse Laplace
solution the fill is held to, and the renderer of the exact-recovery clip."""
import numpy as np

from raft_b200.inpaint import FILL_CYCLES, FILL_INIT_SWEEPS, FILL_SMOOTH, fill_levels

F32 = np.float32


def _mean(vals, present):
    """Per pixel the mean of the present values, rb_masked_fill's rounded mean: s = 0 + v_0 + v_1 + ... (present ones,
    in order, each sum rounded), s / n, clamped by comparisons into [min, max] of the present values.  vals: list of
    [...,C] float32 arrays, present: list of [...] bool.  Returns (mean [...,C], n [...])."""
    s = np.zeros_like(vals[0], dtype=F32)
    n = np.zeros(present[0].shape, dtype=np.int32)
    lo = np.zeros_like(s)
    hi = np.zeros_like(s)
    for v, p in zip(vals, present):
        pc = p[..., None]
        first = pc & (n[..., None] == 0)
        lo = np.where(first | (pc & (v < lo)), v, lo)
        hi = np.where(first | (pc & (v > hi)), v, hi)
        s = np.where(pc, (s + v).astype(F32), s)
        n += p
    with np.errstate(invalid="ignore", divide="ignore"):
        m = (s / np.maximum(n, 1)[..., None].astype(F32)).astype(F32)
    m = np.where(m < lo, lo, m)
    m = np.where(m > hi, hi, m)
    return m, n


def _children(a, h, w, fill):
    """The <= 4 children of each pixel of an h x w level in tap order (2i,2j), (2i,2j+1), (2i+1,2j), (2i+1,2j+1); a
    child outside the finer level is `fill` and absent."""
    out = []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        t = np.full((h, w) + a.shape[2:], fill, dtype=a.dtype)
        ok = np.zeros((h, w), bool)
        sub = a[dy::2, dx::2]
        t[:sub.shape[0], :sub.shape[1]] = sub
        ok[:sub.shape[0], :sub.shape[1]] = True
        out.append((t, ok))
    return out


def _nbrs(v):
    """The neighbours up, down, left, right of every pixel of v [H,W,...] and whether each lies in the image."""
    H, W = v.shape[:2]
    out = []
    for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        sh = np.zeros_like(v)
        ok = np.zeros((H, W), bool)
        ys, yd = (slice(0, H + dy), slice(-dy, H)) if dy < 0 else (slice(dy, H), slice(0, H - dy))
        xs, xd = (slice(0, W + dx), slice(-dx, W)) if dx < 0 else (slice(dx, W), slice(0, W - dx))
        sh[yd, xd] = v[ys, xs]
        ok[yd, xd] = True
        out.append((sh, ok))
    return out


def _colours(H, W):
    yy, xx = np.mgrid[0:H, 0:W]
    return (yy + xx) & 1


def _dirichlet(v, hole, count):
    """count red-black Gauss-Seidel sweeps of the membrane equation on the hole pixels of v [H,W,C] (the others fixed):
    red ((x + y) even) then black; a hole pixel becomes the rounded mean of its in-image neighbours (_mean)."""
    col = _colours(*hole.shape)
    for _ in range(count):
        for c in (0, 1):
            nb = _nbrs(v)
            m, n = _mean([a for a, _ in nb], [ok for _, ok in nb])
            v = np.where((hole & (col == c) & (n > 0))[..., None], m, v)
    return v


def _sum_nb(v, f):
    """s = f + the in-image neighbours up, down, left, right (each sum rounded) and their count n."""
    s = f.copy()
    n = np.zeros(v.shape[:2], np.int32)
    for sh, ok in _nbrs(v):
        s = np.where(ok[..., None], (s + sh).astype(F32), s)
        n += ok
    return s, n


def _correct(e, f, hole, count):
    """count red-black sweeps of the correction equation n e_p - sum e_nb = f_p on the hole pixels: e_p = s / n."""
    col = _colours(*hole.shape)
    for _ in range(count):
        for c in (0, 1):
            s, n = _sum_nb(e, f)
            e = np.where((hole & (col == c) & (n > 0))[..., None],
                         (s / np.maximum(n, 1)[..., None].astype(F32)).astype(F32), e)
    return e


def _residual_down(e, f, hole):
    """The next level's right-hand side: per coarse pixel the sum, in tap order from 0, of its children's residuals
    s - n e (s, n of _sum_nb; 0 off the hole)."""
    s, n = _sum_nb(e, f)
    r = np.where(hole[..., None], (s - (n[..., None].astype(F32) * e).astype(F32)).astype(F32), F32(0))
    h, w = -(-hole.shape[0] // 2), -(-hole.shape[1] // 2)
    out = np.zeros((h, w, e.shape[2]), F32)
    for t, _ in _children(r, h, w, 0):
        out = (out + t).astype(F32)
    return out


def _prolong(e, H, W):
    """The bilinear (cell-centred) value of the coarse correction e at every pixel of the H x W level: weights 1/4 and
    3/4 per axis, taps clamped into the coarse level, ((wx0 e00 + wx1 e01) wy0) + ((wx0 e10 + wx1 e11) wy1)."""
    h, w = e.shape[:2]

    def taps(z, n):
        i = z // 2
        even = z % 2 == 0
        a = np.where(even, np.maximum(i - 1, 0), i)
        b = np.where(even, i, np.minimum(i + 1, n - 1))
        return a, b, np.where(even, F32(0.25), F32(0.75)).astype(F32), np.where(even, F32(0.75), F32(0.25)).astype(F32)

    ya, yb, wya, wyb = taps(np.arange(H), h)
    xa, xb, wxa, wxb = taps(np.arange(W), w)
    wxa, wxb, wya, wyb = wxa[None, :, None], wxb[None, :, None], wya[:, None, None], wyb[:, None, None]
    t0 = ((wxa * e[ya][:, xa]).astype(F32) + (wxb * e[ya][:, xb]).astype(F32)).astype(F32)
    t1 = ((wxa * e[yb][:, xa]).astype(F32) + (wxb * e[yb][:, xb]).astype(F32)).astype(F32)
    return ((t0 * wya).astype(F32) + (t1 * wyb).astype(F32)).astype(F32)


def masked_fill(values, hole):
    """rb_masked_fill of one field: values [H,W,C] float32, hole [H,W] (non-zero = hole).  Returns (filled [H,W,C]
    float32, flag): flag 1 when the field has no known pixel (it is then all zeros)."""
    u = np.array(values, dtype=F32, copy=True)
    hole = np.asarray(hole) != 0
    H, W, C = u.shape
    if hole.all():
        return np.zeros_like(u), 1
    lo, hi = u[~hole].min(0), u[~hole].max(0)
    sizes = fill_levels(H, W)
    # the initial guess: known-any pyramid of the values, coarsest to finest, nearest prolongation and Dirichlet sweeps
    vals, ihole, chole = [u], [hole], [hole]
    for h, w in sizes[1:]:
        kids = _children(vals[-1], h, w, 0)
        known = _children(~ihole[-1], h, w, False)
        m, n = _mean([t for t, _ in kids], [k & ok for (k, ok) in known])
        vals.append(np.where((n > 0)[..., None], m, F32(0)))
        ihole.append(n == 0)
        chole.append(np.logical_and.reduce([c | ~ok for c, ok in _children(chole[-1], h, w, True)]))
    for lv in range(len(sizes) - 2, -1, -1):
        h, w = sizes[lv]
        up = vals[lv + 1].repeat(2, 0).repeat(2, 1)[:h, :w]
        vals[lv] = _dirichlet(np.where(ihole[lv][..., None], up, vals[lv]), ihole[lv], FILL_INIT_SWEEPS)
    u = vals[0]

    def vcycle(lv, f):  # the correction of level lv >= 1 from its right-hand side f
        e = np.zeros_like(f)
        e = _correct(e, f, chole[lv], FILL_SMOOTH)
        if lv + 1 < len(sizes):
            ec = vcycle(lv + 1, _residual_down(e, f, chole[lv]))
            e = np.where(chole[lv][..., None], (e + _prolong(ec, *sizes[lv])).astype(F32), e)
        return _correct(e, f, chole[lv], FILL_SMOOTH)

    zero = np.zeros_like(u)
    for _ in range(FILL_CYCLES if len(sizes) > 1 else 0):
        ec = vcycle(1, _residual_down(u, zero, hole))
        c = (u + _prolong(ec, H, W)).astype(F32)
        c = np.where(c < lo, lo, c)
        c = np.where(c > hi, hi, c)
        u = _dirichlet(np.where(hole[..., None], c, u), hole, FILL_SMOOTH)
    return u, 0


def laplace_fp64(values, hole):
    """The exact fp64 membrane fill: the 4-neighbour discrete Laplace equation on the hole pixels, the known pixels as
    Dirichlet data, neighbours outside the image left out (scipy.sparse.linalg.spsolve)."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spl
    v = np.asarray(values, dtype=np.float64).copy()
    H, W, C = v.shape
    hole = np.asarray(hole) != 0
    idx = -np.ones((H, W), np.int64)
    ys, xs = np.nonzero(hole)
    n = len(ys)
    idx[ys, xs] = np.arange(n)
    rows, cols, data = [], [], []
    rhs = np.zeros((n, C))
    deg = np.zeros(n)
    for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        ny, nx = ys + dy, xs + dx
        ok = (ny >= 0) & (ny < H) & (nx >= 0) & (nx < W)
        deg += ok
        k = np.flatnonzero(ok)
        nb = idx[ny[k], nx[k]]
        unk = nb >= 0
        rows += [k[unk]]
        cols += [nb[unk]]
        data += [-np.ones(unk.sum())]
        rhs[k[~unk]] += v[ny[k[~unk]], nx[k[~unk]]]
    A = sp.csr_matrix((np.concatenate(data + [deg]), (np.concatenate(rows + [np.arange(n)]),
                                                       np.concatenate(cols + [np.arange(n)]))), shape=(n, n))
    sol = spl.spsolve(A.tocsc(), rhs)
    v[ys, xs] = sol.reshape(n, C)
    return v


def inpaint_masks(masks, select, dilate, Hn, Wn):
    """rb_inpaint_masks: masks [F,Hs,Ws] uint8, select [256] -> (hole [F,Hs,Ws], hole_net [F,Hn,Wn]) uint8 0 / 1."""
    from scipy.ndimage import maximum_filter
    sel = np.asarray(select)[np.asarray(masks)] != 0
    F, Hs, Ws = sel.shape
    size = (1, 2 * dilate + 1, 2 * dilate + 1)
    hole = maximum_filter(sel.astype(np.uint8), size=size, mode="constant", cval=0) if dilate else sel.astype(np.uint8)
    iy = ((2 * np.arange(Hs, dtype=np.int64) + 1) * Hn) // (2 * Hs)
    ix = ((2 * np.arange(Ws, dtype=np.int64) + 1) * Wn) // (2 * Ws)
    net = np.zeros((F, Hn, Wn), np.uint8)
    hit = np.zeros((Hn, Wn), bool)
    hit[np.ix_(iy, ix)] = True
    np.maximum.at(net, (slice(None), iy[:, None], ix[None, :]), hole)
    # rows / columns no frame pixel maps to take the frame pixel holding their centre
    cy = ((2 * np.arange(Hn, dtype=np.int64) + 1) * Hs) // (2 * Hn)
    cx = ((2 * np.arange(Wn, dtype=np.int64) + 1) * Ws) // (2 * Wn)
    ry = np.zeros(Hn, bool)
    ry[iy] = True
    rx = np.zeros(Wn, bool)
    rx[ix] = True
    for i in range(Hn):
        for j in range(Wn):
            if ry[i] and rx[j]:
                continue
            ys = [cy[i]] if not ry[i] else np.flatnonzero(iy == i)
            xs = [cx[j]] if not rx[j] else np.flatnonzero(ix == j)
            net[:, i, j] = hole[:, ys][:, :, xs].reshape(F, -1).max(1)
    return hole, net


def _remap(x, r, n):
    """fl32((x + 0.5) r - 0.5) in fp64, clamped into [0, n - 1] (track_queries / tracks_to_frames)."""
    v = ((np.asarray(x, np.float64) + 0.5) * r - 0.5).astype(F32)
    return np.clip(v, F32(0), F32(n - 1))


def _side(frames, hole, fw, bw, t, direction, n, px, py, s, a1, a2):
    """One side of the hole pixels at network positions (px, py) of frame t: (distance [N] int, colour [N,3] fp32)."""
    from track_oracle import step
    F, Hs, Ws, _ = frames.shape
    Hn, Wn = fw.shape[1:3]
    N = len(px)
    dist = np.zeros(N, np.int64)
    col = np.zeros((N, 3), F32)
    live = np.arange(N)
    for k in range(1, n + 1):
        if not len(live):
            break
        pair = t + k - 1 if direction > 0 else t - k
        pull, test = (fw[pair], bw[pair]) if direction > 0 else (bw[pair], fw[pair])
        qx, qy, st = step(pull, test, px[live], py[live], s, a1, a2)
        keep = st == 0
        live, px_l, py_l = live[keep], qx[keep], qy[keep]
        px[live], py[live] = px_l, py_l
        fr = t + direction * k
        ox, oy = _remap(px_l, Ws / Wn, Ws), _remap(py_l, Hs / Hn, Hs)
        x0, y0 = np.floor(ox).astype(np.int64), np.floor(oy).astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, Ws - 1), np.minimum(y0 + 1, Hs - 1)
        h = hole[fr]
        vis = (h[y0, x0] | h[y0, x1] | h[y1, x0] | h[y1, x1]) == 0
        if vis.any():
            ax, ay = (ox - x0.astype(F32)).astype(F32), (oy - y0.astype(F32)).astype(F32)
            cx, cy = (F32(1) - ax).astype(F32), (F32(1) - ay).astype(F32)
            img = frames[fr].astype(F32)
            v = vis
            c = [img[y0[v], x0[v]], img[y0[v], x1[v]], img[y1[v], x0[v]], img[y1[v], x1[v]]]
            cxv, axv, cyv, ayv = cx[v, None], ax[v, None], cy[v, None], ay[v, None]
            t0 = (cxv * c[0]).astype(F32) + (axv * c[1]).astype(F32)
            t1 = (cxv * c[2]).astype(F32) + (axv * c[3]).astype(F32)
            col[live[v]] = ((t0.astype(F32) * cyv).astype(F32) + (t1.astype(F32) * ayv).astype(F32)).astype(F32)
            dist[live[v]] = k
            live = live[~v]
    return dist, col


def inpaint_propagate(frames, hole, fw, bw, rows, s=1.0, a1=0.01, a2=0.5):
    """rb_inpaint_propagate: frames [F,Hs,Ws,3] uint8, hole [F,Hs,Ws], fw / bw [F-1,Hn,Wn,2] fp32, rows [n,3] ->
    (colour [n,Hs,Ws,3] fp32, status [n,Hs,Ws] uint8)."""
    frames, hole = np.asarray(frames), np.asarray(hole)
    F, Hs, Ws, _ = frames.shape
    Hn, Wn = fw.shape[1:3]
    colour = np.zeros((len(rows), Hs, Ws, 3), F32)
    status = np.zeros((len(rows), Hs, Ws), np.uint8)
    for r, (t, nf, nb) in enumerate(np.asarray(rows).tolist()):
        colour[r] = frames[t].astype(F32)
        ys, xs = np.nonzero(hole[t])
        px, py = _remap(xs, Wn / Ws, Wn), _remap(ys, Hn / Hs, Hn)
        df, cf = _side(frames, hole, fw, bw, t, 1, min(nf, F - 1 - t), px.copy(), py.copy(), s, a1, a2)
        db, cb = _side(frames, hole, fw, bw, t, -1, min(nb, t), px.copy(), py.copy(), s, a1, a2)
        both = (df > 0) & (db > 0)
        with np.errstate(invalid="ignore", divide="ignore"):
            blend = (((db[:, None].astype(F32) * cf).astype(F32) + (df[:, None].astype(F32) * cb).astype(F32)).astype(F32)
                     / (df + db)[:, None].astype(F32)).astype(F32)
        c = np.where(both[:, None], blend, np.where((df > 0)[:, None], cf, np.where((db > 0)[:, None], cb, F32(0))))
        colour[r, ys, xs] = c
        status[r, ys, xs] = np.where(both, 1, np.where((df > 0) | (db > 0), 2, 3))
    return colour, status


def inpaint(frames, masks, fw, bw, rows, select, dilate, s=1.0, a1=0.01, a2=0.5):
    """The whole of RaftEngine.inpaint after the flow pass: masks, flow completion, temporal and spatial fill, rounding.
    Returns (frames uint8, status)."""
    F = frames.shape[0]
    Hn, Wn = fw.shape[1:3]
    hole, net = inpaint_masks(masks, select, dilate, Hn, Wn)
    cfw = np.stack([masked_fill(fw[k], net[k])[0] for k in range(F - 1)])
    cbw = np.stack([masked_fill(bw[k], net[k + 1])[0] for k in range(F - 1)])
    colour, status = inpaint_propagate(frames, hole, cfw, cbw, rows, s, a1, a2)
    out = np.stack([masked_fill(colour[r], status[r] == 3)[0] for r in range(len(rows))])
    return np.clip(np.rint(out), 0, 255).astype(np.uint8), status
