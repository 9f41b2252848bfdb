"""numpy restatement of rb_track_points_backward (csrc/track.cu), for the tests.

track_backward is fp32 in the kernel's operation order (track_oracle.step with the flows' roles swapped), so the kernel
must reproduce it bit for bit; dt=np.float64 is the same formula in fp64.  Rows after a query's frame are not stored:
given tracks / status (e.g. track_oracle.track's) it completes copies of them, otherwise it starts from NaN / 3.
"""
from __future__ import annotations

import numpy as np

from track_oracle import BEFORE, CONSISTENT, OCCLUDED, step


def track_backward(flow_fw, flow_bw, qframe, qpos, tracks=None, status=None, first_frame=0, n_steps=None,
                   flow_scale=1.0, alpha1=0.01, alpha2=0.5, state=None, dt=np.float32):
    """rb_track_points_backward: flows [T,H,W,2], qframe [N], qpos [N,2], tracks [n_steps+1,N,2] / status
    [n_steps+1,N] to complete (None: NaN / 3), the carried state (pos [N,2], state [N]) or None -> (tracks, status,
    (pos, state)); pos / state are row 0 for queries with qframe >= first_frame and the carried ones otherwise."""
    fw, bw = np.asarray(flow_fw, dtype=dt), np.asarray(flow_bw, dtype=dt)
    T = fw.shape[0]
    n_steps = T if n_steps is None else int(n_steps)
    q0 = np.asarray(qframe, dtype=np.int64) - int(first_frame)
    qpos = np.asarray(qpos, dtype=dt)
    N = len(q0)
    tracks = np.full((n_steps + 1, N, 2), np.nan, dt) if tracks is None else np.array(tracks, dtype=dt)
    status = np.full((n_steps + 1, N), BEFORE, np.uint8) if status is None else np.array(status, dtype=np.uint8)
    px, py = np.full(N, np.nan, dt), np.full(N, np.nan, dt)
    st = np.full(N, BEFORE, np.uint8)
    if state is None:
        state = (np.full((N, 2), np.nan, dt), np.full(N, BEFORE, np.uint8))
    pos, sst = np.array(state[0], dtype=dt), np.array(state[1], dtype=np.uint8)
    later = q0 > n_steps
    px[later], py[later], st[later] = pos[later, 0], pos[later, 1], sst[later]
    for j in range(n_steps, -1, -1):
        moving = np.flatnonzero((j < n_steps) & (j < q0) & (st <= OCCLUDED))
        if len(moving):  # step j+1 -> j: flow_bw[j] moves the point, flow_fw[j] checks it
            px[moving], py[moving], st[moving] = step(bw[j], fw[j], px[moving], py[moving], flow_scale, alpha1,
                                                      alpha2, dt)
        at = j == q0
        px[at], py[at], st[at] = qpos[at, 0], qpos[at, 1], CONSISTENT
        rows = j <= q0
        tracks[j, rows, 0], tracks[j, rows, 1], status[j, rows] = px[rows], py[rows], st[rows]
    done = q0 >= 0
    pos[done, 0], pos[done, 1], sst[done] = tracks[0, done, 0], tracks[0, done, 1], status[0, done]
    return tracks, status, (pos, sst)


def reversed_clip(flow_fw, flow_bw):
    """The clip played backward: fw'[k] = flow_bw[T-1-k], bw'[k] = flow_fw[T-1-k]."""
    return np.ascontiguousarray(flow_bw[::-1]), np.ascontiguousarray(flow_fw[::-1])


def track_backward_passes(flow_fw, flow_bw, qframe, qpos, bounds, tracks=None, status=None, **kw):
    """The chunked reverse sweep: the clip's pairs split at the frame indices `bounds` (0 = b_0 < ... < b_m = T), one
    call per chunk from the last to the first with the state carried, each completing its rows of (copies of) tracks /
    status [T+1,N,...].  Row b_i is shared by two chunks; the later chunk's call writes it first, the earlier one rewrites
    the same values."""
    T = np.shape(flow_fw)[0]
    N = len(qframe)
    tracks = np.full((T + 1, N, 2), np.nan, np.float32) if tracks is None else np.array(tracks)
    status = np.full((T + 1, N), BEFORE, np.uint8) if status is None else np.array(status)
    state = None
    for a, b in reversed(list(zip(bounds, bounds[1:]))):
        t, s, state = track_backward(flow_fw[a:b], flow_bw[a:b], qframe, qpos, tracks[a:b + 1], status[a:b + 1],
                                     first_frame=a, state=state, **kw)
        tracks[a:b + 1], status[a:b + 1] = t, s
    return tracks, status
