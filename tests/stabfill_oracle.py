"""numpy restatement of F26, bit for bit: the flows extended past the frame edge (rb_flow_extend_residual, rb_masked_fill,
rb_flow_extend_finish) and rb_frames_warp_affine_fill -- every fp32 / fp64 operation a numpy operation of that type,
rounded on its own.  It reuses the masked fill of tests/inpaint_oracle.py, the tracker's step of tests/track_oracle.py and
the similarity flow of tests/stabilize_oracle.py.  Also the analytic texture clip of the geometry tests."""
import math

import numpy as np

from inpaint_oracle import masked_fill
from track_oracle import step

F32 = np.float32


def global_flow(M, x, y, hw, net_hw, flow_scale=1.0):
    """stabilize_oracle.similarity_flow's formula at network positions x, y (fp64 arrays, anywhere): (u, v) fp32."""
    Hs, Ws = hw
    Hn, Wn = net_hw
    sx, sy = Ws / Wn, Hs / Hn
    px = (x + 0.5) * sx - 0.5 - 0.5 * (Ws - 1)
    py = (y + 0.5) * sy - 0.5 - 0.5 * (Hs - 1)
    a, b, tx, ty = M
    u = (a * px - b * py + tx - px) / sx / flow_scale
    v = (b * px + a * py + ty - py) / sy / flow_scale
    return u.astype(F32), v.astype(F32)


def inverse(M):
    """The similarity (a, b, tx, ty) of M^-1, in fp64 as networks.utils.extend_flows computes it."""
    from raft_b200.stabilize import motion_matrix
    i = np.linalg.inv(motion_matrix(np.asarray(M, np.float64)[None]))[0]
    return i[0, 0], i[1, 0], i[0, 2], i[1, 2]


def extend(flow, M, hw, margin, flow_scale=1.0):
    """One field: flow [Hn,Wn,2] fp32 and its similarity M extended by margin = (my, mx) -> ext [Hc,Wc,2] fp32, with the
    residual and hole that rb_masked_fill takes."""
    Hn, Wn, _ = flow.shape
    my, mx = margin
    Hc, Wc = Hn + 2 * my, Wn + 2 * mx
    y, x = np.meshgrid(np.arange(Hc, dtype=np.float64) - my, np.arange(Wc, dtype=np.float64) - mx, indexing="ij")
    gu, gv = global_flow(M, x, y, hw, (Hn, Wn), flow_scale)
    g = np.stack([gu, gv], -1)
    hole = np.ones((Hc, Wc), np.uint8)
    hole[my:my + Hn, mx:mx + Wn] = 0
    r = np.zeros((Hc, Wc, 2), F32)
    r[my:my + Hn, mx:mx + Wn] = flow - g[my:my + Hn, mx:mx + Wn]
    if my or mx:
        r = masked_fill(r, hole)[0]
    ext = (r + g).astype(F32)
    ext[my:my + Hn, mx:mx + Wn] = flow
    return ext


def extend_flows(fw, bw, motions, hw, margin, flow_scale=1.0):
    """networks.utils.extend_flows: fw, bw [T,Hn,Wn,2], motions [T,4] -> (ext_fw, ext_bw)."""
    efw = np.stack([extend(fw[k], motions[k], hw, margin, flow_scale) for k in range(len(fw))])
    ebw = np.stack([extend(bw[k], inverse(motions[k]), hw, margin, flow_scale) for k in range(len(bw))])
    return efw, ebw


def _bilinear(img, fx, fy):
    """fb_sample.cuh's bilinear sample of img [H,W,3] uint8 at (fx, fy) fp32 inside the frame: [N,3] fp32."""
    H, W = img.shape[:2]
    x0, y0 = np.floor(fx).astype(np.int64), np.floor(fy).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = (fx - x0.astype(F32)).astype(F32)[:, None], (fy - y0.astype(F32)).astype(F32)[:, None]
    cx, cy = F32(1) - ax, F32(1) - ay
    im = img.astype(F32)
    t0 = cx * im[y0, x0] + ax * im[y0, x1]
    t1 = cx * im[y1, x0] + ax * im[y1, x1]
    return (t0 * cy + t1 * ay).astype(F32)


def _inside(x, y, H, W):
    with np.errstate(invalid="ignore"):
        return (x >= 0) & (x <= F32(W - 1)) & (y >= 0) & (y <= F32(H - 1))


def _side(frames, efw, ebw, t, direction, n, px, py, margin, net_hw, s, a1, a2):
    """One side of the sources at canvas positions (px, py) fp32 of frame t: (distance [N], colour [N,3] fp32)."""
    F, Hs, Ws, _ = frames.shape
    Hn, Wn = net_hw
    my, mx = margin
    N = len(px)
    dist = np.zeros(N, np.int64)
    col = np.zeros((N, 3), F32)
    live = np.arange(N)
    for k in range(1, n + 1):
        if not len(live):
            break
        pair = t + k - 1 if direction > 0 else t - k
        pull, test = (efw[pair], ebw[pair]) if direction > 0 else (ebw[pair], efw[pair])
        qx, qy, st = step(pull, test, px, py, s, a1, a2)
        keep = st == 0
        live, px, py = live[keep], qx[keep], qy[keep]
        ox = (((px.astype(np.float64) - mx) + 0.5) * (Ws / Wn) - 0.5).astype(F32)
        oy = (((py.astype(np.float64) - my) + 0.5) * (Hs / Hn) - 0.5).astype(F32)
        vis = _inside(ox, oy, Hs, Ws)
        if vis.any():
            col[live[vis]] = _bilinear(frames[t + direction * k], ox[vis], oy[vis])
            dist[live[vis]] = k
        live, px, py = live[~vis], px[~vis], py[~vis]
    return dist, col


def warp_fill(frames, efw, ebw, net_hw, margin, A, rows, s=1.0, a1=0.01, a2=0.5):
    """rb_frames_warp_affine_fill: frames [F,Hs,Ws,3] uint8, ext flows [F-1,Hc,Wc,2], A [n,2,3], rows [n,3] ->
    (colour [n,Hs,Ws,3] fp32, status [n,Hs,Ws] uint8)."""
    frames = np.asarray(frames)
    F, Hs, Ws, _ = frames.shape
    Hn, Wn = net_hw
    my, mx = margin
    n_rows = len(rows)
    colour = np.zeros((n_rows, Hs, Ws, 3), F32)
    status = np.full((n_rows, Hs, Ws), 3, np.uint8)
    y, x = np.meshgrid(np.arange(Hs, dtype=np.float64), np.arange(Ws, dtype=np.float64), indexing="ij")
    x, y = x.reshape(-1), y.reshape(-1)
    for r, (t, nf, nb) in enumerate(np.asarray(rows).tolist()):
        if not 0 <= t < F:
            continue
        m = np.asarray(A[r], np.float64)
        sx = (m[0, 0] * x + m[0, 1] * y) + m[0, 2]
        sy = (m[1, 0] * x + m[1, 1] * y) + m[1, 2]
        fx, fy = sx.astype(F32), sy.astype(F32)
        ins = _inside(fx, fy, Hs, Ws) | np.isnan(fx) | np.isnan(fy)
        c = np.zeros((Hs * Ws, 3), F32)
        st = np.full(Hs * Ws, 3, np.uint8)
        i = np.flatnonzero(ins)
        cfx = np.minimum(np.maximum(np.nan_to_num(fx[i], nan=0.0), F32(0)), F32(Ws - 1))
        cfy = np.minimum(np.maximum(np.nan_to_num(fy[i], nan=0.0), F32(0)), F32(Hs - 1))
        c[i] = _bilinear(frames[t], cfx, cfy)
        st[i] = 0
        o = np.flatnonzero(~ins)
        px = (((sx[o] + 0.5) * (Wn / Ws) - 0.5) + mx).astype(F32)
        py = (((sy[o] + 0.5) * (Hn / Hs) - 0.5) + my).astype(F32)
        df, cf = _side(frames, efw, ebw, t, 1, min(max(nf, 0), F - 1 - t), px, py, margin, net_hw, s, a1, a2)
        db, cb = _side(frames, efw, ebw, t, -1, min(max(nb, 0), t), px, py, margin, net_hw, s, a1, a2)
        both = (df > 0) & (db > 0)
        with np.errstate(invalid="ignore", divide="ignore"):
            blend = (((db[:, None].astype(F32) * cf).astype(F32) + (df[:, None].astype(F32) * cb).astype(F32)).astype(F32)
                     / (df + db)[:, None].astype(F32)).astype(F32)
        c[o] = np.where(both[:, None], blend, np.where((df > 0)[:, None], cf, np.where((db > 0)[:, None], cb, F32(0))))
        st[o] = np.where(both, 1, np.where((df > 0) | (db > 0), 2, 3))
        colour[r], status[r] = c.reshape(Hs, Ws, 3), st.reshape(Hs, Ws)
    return colour, status


def finish(colour, status):
    """raft_b200.inpaint.finish_frames: the spatial fill of status 3, rint and the clamp to bytes."""
    out = np.stack([masked_fill(colour[r], status[r] == 3)[0] for r in range(len(colour))])
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


# ---- the analytic texture clip: frame t shows the texture at G_t p (p centred frame pixels) ----

def texture(X, Y):
    """A smooth texture of the plane, in [0, 255]."""
    return (128 + 45 * np.sin(0.23 * X + 0.11 * Y) + 35 * np.cos(0.19 * Y - 0.07 * X)
            + 20 * np.sin(0.05 * X * np.cos(0.03 * Y) + 0.3))


def jittered_path(F, seed, pan=(1.5, 0.0), jitter=(2.0, 2.0), rot=0.01, zoom=0.01):
    """G [F,3,3] frame -> texture (centred) along a pan of pan = (x, y) pixels per frame with jitter = (x, y) pixels of
    translation jitter, rot radians of rotation jitter and zoom of zoom jitter, and the pair motions
    [F-1,4] (a, b, tx, ty) of M_k = G_(k+1)^-1 G_k."""
    rng = np.random.default_rng(seed)
    t = np.arange(F)
    th = (0.002 * t + rng.normal(0, rot, F)) if rot else np.zeros(F)
    sc = (1 + rng.normal(0, zoom, F)) if zoom else np.ones(F)
    tx, ty = pan[0] * t + rng.normal(0, jitter[0], F), pan[1] * t + rng.normal(0, jitter[1], F)
    G = np.stack([np.array([[s * math.cos(a), -s * math.sin(a), x], [s * math.sin(a), s * math.cos(a), y], [0, 0, 1]])
                  for s, a, x, y in zip(sc, th, tx, ty)])
    M = np.stack([np.linalg.inv(G[k + 1]) @ G[k] for k in range(F - 1)])
    return G, np.stack([M[:, 0, 0], M[:, 1, 0], M[:, 0, 2], M[:, 1, 2]], 1)


def render(G, hw):
    """The clip [F,Hs,Ws,3] uint8 of the path G: pixel p of frame t is the texture at G_t (p - centre)."""
    Hs, Ws = hw
    y, x = np.meshgrid(np.arange(Hs) - 0.5 * (Hs - 1), np.arange(Ws) - 0.5 * (Ws - 1), indexing="ij")
    out = []
    for g in G:
        v = texture(g[0, 0] * x + g[0, 1] * y + g[0, 2], g[1, 0] * x + g[1, 1] * y + g[1, 2])
        out.append(np.repeat(np.clip(np.rint(v), 0, 255).astype(np.uint8)[..., None], 3, -1))
    return np.stack(out)


def true_view(G, A, hw):
    """The full-frame stabilized clip [F,Hs,Ws] fp64 the transforms A [F,2,3] ask for: output pixel o of frame t shows
    the texture at G_t (A_t o - centre), wherever that source lies."""
    Hs, Ws = hw
    y, x = np.meshgrid(np.arange(Hs, dtype=np.float64), np.arange(Ws, dtype=np.float64), indexing="ij")
    out = []
    for g, a in zip(G, A):
        sx = a[0, 0] * x + a[0, 1] * y + a[0, 2] - 0.5 * (Ws - 1)
        sy = a[1, 0] * x + a[1, 1] * y + a[1, 2] - 0.5 * (Hs - 1)
        out.append(texture(g[0, 0] * sx + g[0, 1] * sy + g[0, 2], g[1, 0] * sx + g[1, 1] * sy + g[1, 2]))
    return np.stack(out)
