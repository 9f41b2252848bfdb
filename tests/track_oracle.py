"""numpy restatement of the point tracker rb_track_points (csrc/track.cu) and of RaftEngine.track's coordinate map, for
the tests.

track is fp32 in the kernel's operation order -- every operation rounded on its own, left to right, no FMA -- so the
kernel must reproduce it bit for bit; track(..., dt=np.float64) is the same formula in fp64, the reference for the fp32
rounding.  The step is tests/fb_oracle.py's check moved from a pixel to a point.  Status: 0 consistent, 1 inconsistent
(occluded), 2 left the frame, 3 before the query frame.
"""
from __future__ import annotations

import numpy as np

CONSISTENT, OCCLUDED, LEFT, BEFORE = 0, 1, 2, 3


def _inside(qx, qy, H, W, dt):
    with np.errstate(invalid="ignore"):
        return (qx >= 0) & (qx <= dt(W - 1)) & (qy >= 0) & (qy <= dt(H - 1))  # NaN -> outside


def _sample(field, qx, qy, s, dt):
    """s times the bilinear sample of the [H,W,2] field at the points (qx, qy), all inside the frame."""
    H, W = field.shape[:2]
    one = dt(1)
    fx0, fy0 = np.floor(qx), np.floor(qy)
    x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = qx - fx0, qy - fy0
    cx, cy = one - ax, one - ay

    def bilerp(c):
        v = field[..., c]
        t0 = cx * v[y0, x0] + ax * v[y0, x1]
        t1 = cx * v[y1, x0] + ax * v[y1, x1]
        return t0 * cy + t1 * ay

    return s * bilerp(0), s * bilerp(1)


def step(fw, bw, px, py, s, a1, a2, dt=np.float32):
    """One step k -> k+1 of points (px, py) through the [H,W,2] flows fw = flow_fw[k], bw = flow_bw[k]
    -> (qx, qy, status); a start outside the frame leaves it (status 2, NaN)."""
    H, W = fw.shape[:2]
    s, a1, a2 = dt(s), dt(a1), dt(a2)
    n = len(px)
    qx, qy = np.full(n, np.nan, dt), np.full(n, np.nan, dt)
    st = np.full(n, LEFT, np.uint8)
    ok = np.flatnonzero(_inside(px, py, H, W, dt))
    with np.errstate(invalid="ignore", over="ignore"):
        fx, fy = _sample(fw, px[ok], py[ok], s, dt)
        tx, ty = px[ok] + fx, py[ok] + fy
        inside = _inside(tx, ty, H, W, dt)
        ok, fx, fy, tx, ty = ok[inside], fx[inside], fy[inside], tx[inside], ty[inside]
        bx, by = _sample(bw, tx, ty, s, dt)
        ex, ey = fx + bx, fy + by
        d = ex * ex + ey * ey
        m = a1 * (((fx * fx + fy * fy) + bx * bx) + by * by) + a2
    st[ok] = (d > m).astype(np.uint8)
    qx[ok], qy[ok] = tx, ty
    return qx, qy, st


def track(flow_fw, flow_bw, qframe, qpos, first_frame=0, n_steps=None, flow_scale=1.0, alpha1=0.01, alpha2=0.5,
          state=None, dt=np.float32):
    """rb_track_points: flows [T,H,W,2], qframe [N], qpos [N,2], the carried state (pos [N,2], state [N]) or None ->
    (tracks [n_steps+1,N,2], status [n_steps+1,N] uint8, (pos, state) after the last row)."""
    fw, bw = np.asarray(flow_fw, dtype=dt), np.asarray(flow_bw, dtype=dt)
    T = fw.shape[0]
    n_steps = T if n_steps is None else int(n_steps)
    q0 = np.asarray(qframe, dtype=np.int64) - int(first_frame)
    qpos = np.asarray(qpos, dtype=dt)
    N = len(q0)
    px, py = np.full(N, np.nan, dt), np.full(N, np.nan, dt)
    st = np.full(N, BEFORE, np.uint8)
    if state is not None:
        carried = q0 < 0
        pos, sst = np.asarray(state[0], dtype=dt), np.asarray(state[1], dtype=np.uint8)
        px[carried], py[carried], st[carried] = pos[carried, 0], pos[carried, 1], sst[carried]
    tracks = np.empty((n_steps + 1, N, 2), dt)
    status = np.empty((n_steps + 1, N), np.uint8)
    for j in range(n_steps + 1):
        moving = np.flatnonzero((j > 0) & (j > q0) & (st <= OCCLUDED))
        if len(moving):
            px[moving], py[moving], st[moving] = step(fw[j - 1], bw[j - 1], px[moving], py[moving], flow_scale, alpha1,
                                                      alpha2, dt)
        before, at = j < q0, j == q0
        px[before], py[before], st[before] = np.nan, np.nan, BEFORE
        px[at], py[at], st[at] = qpos[at, 0], qpos[at, 1], CONSISTENT
        tracks[j, :, 0], tracks[j, :, 1], status[j] = px, py, st
    return tracks, status, (tracks[-1].copy(), status[-1].copy())


def track_passes(flow_fw, flow_bw, qframe, qpos, bounds, **kw):
    """The chunked form: the clip's pairs split at the frame indices `bounds` (0 = b_0 < b_1 < ... < b_m = T), one call
    per chunk with the state carried, the rows stitched (row 0 of a later chunk repeats the last row before it)."""
    state, tracks, status = None, [], []
    for a, b in zip(bounds, bounds[1:]):
        t, s, state = track(flow_fw[a:b], flow_bw[a:b], qframe, qpos, first_frame=a, state=state, **kw)
        tracks.append(t if a == 0 else t[1:])
        status.append(s if a == 0 else s[1:])
    return np.concatenate(tracks), np.concatenate(status)


def to_network(xy, src_hw, net_hw):
    """Query positions [N,2] in Hs x Ws frame pixels -> the Hn x Wn network grid: (x + 0.5) Wn / Ws - 0.5 in fp64, rounded
    once to fp32 and clamped into [0, Wn - 1] x [0, Hn - 1]."""
    xy = np.asarray(xy, dtype=np.float64)
    (Hs, Ws), (Hn, Wn) = src_hw, net_hw
    x = np.clip(np.float32((xy[:, 0] + 0.5) * (Wn / Ws) - 0.5), np.float32(0), np.float32(Wn - 1))
    y = np.clip(np.float32((xy[:, 1] + 0.5) * (Hn / Hs) - 0.5), np.float32(0), np.float32(Hn - 1))
    return np.stack([x, y], axis=-1)


def from_network(xy, src_hw, net_hw):
    """Tracks [...,2] fp32 on the network grid -> frame pixels, the inverse map in fp64 rounded once to fp32."""
    xy = np.asarray(xy, dtype=np.float64)
    (Hs, Ws), (Hn, Wn) = src_hw, net_hw
    return ((xy + 0.5) * np.array([Ws / Wn, Hs / Hn]) - 0.5).astype(np.float32)


def same_bits(a, b):
    """Equal shapes and bits (NaN equals NaN of the same payload)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), np.asarray(b, dtype=np.float32).view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)
