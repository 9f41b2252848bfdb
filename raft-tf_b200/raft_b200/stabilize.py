"""Video stabilization on the host: the camera path of a clip from the per-pair motions of rb_global_motion
(networks.utils.global_motion), its Gaussian smoothing per shot, one zoom per shot that keeps the frame borders out of
view, and the per-frame warps that rb_frames_warp_affine (networks.utils.warp_frames) applies.  Everything is fp64
numpy; the clip's F x 4 motion parameters are all it reads.

Coordinates are the frames' own pixels centred on the frame centre ((W-1)/2, (H-1)/2).  A motion M_k = [[a, -b, tx],
[b, a, ty]] maps frame k to frame k + 1.  Per shot (the frames between two scene cuts) the camera path is C = I at the
shot's first frame and C_(k+1) = M_k C_k, so a shot never depends on the frames before it.  Its parameters log s, theta
(unwrapped along the shot), tx and ty are smoothed with a Gaussian of sigma frames, reflected oddly about each end of the
shot (a value j frames beyond end e is 2 p_e minus the value j frames inside), so a constant-velocity pan and a still
camera are left as they are.  Frame t's correction is A_t = C_t S_t^-1 Z^-1: S_t the smoothed path and Z one zoom about
the centre per shot, the smallest z >= 1 that keeps the four output corners inside the source frame at every frame of the
shot (in closed form: the condition is linear in 1 / z), capped at max_zoom (past the cap the border replicates).

The defaults below were chosen against synthetic flows (tests/test_stabilize.py's recovery cases); they are not
validated on real footage.
"""
from __future__ import annotations

import math

import numpy as np

# rb_global_motion's robust fit: reweighting rounds after the plain least-squares round, the Cauchy scale in network
# pixels, and the smallest fraction of consistent pixels (occ == 0) below which a pair is unreliable (identity)
MOTION_ROUNDS = 8
MOTION_CAUCHY = 0.1
MOTION_MIN_WEIGHT = 0.05
# the largest zoom per shot; a shot that needs more keeps this zoom and replicates the border where the frame runs out
DEFAULT_MAX_ZOOM = 1.25
# how far (pixels) a corner may land outside the frame and still count as inside: fp64 rounding of the path
ZOOM_SLACK = 1e-9
# full-frame stabilization (fill=True): the largest canvas margin per side as a fraction of the network grid, and the
# network pixels added to the farthest source for the bilinear taps; the cap is not tuned
FILL_MARGIN_CAP = 0.5
FILL_MARGIN_TAPS = 2


def check_sigma(sigma, what="stabilize"):
    """The smoothing width in frames as a float: finite and > 0.  Anything else raises ValueError."""
    try:
        s = float(sigma)
    except (TypeError, ValueError):
        s = None
    if s is None or not (math.isfinite(s) and s > 0):
        raise ValueError(f"{what}: sigma must be a finite number of frames > 0 (got {sigma!r})")
    return s


def check_max_zoom(max_zoom, what="stabilize"):
    """The zoom cap as a float: finite and >= 1.  Anything else raises ValueError."""
    try:
        z = float(max_zoom)
    except (TypeError, ValueError):
        z = None
    if z is None or not (math.isfinite(z) and z >= 1.0):
        raise ValueError(f"{what}: max_zoom must be a finite number >= 1 (got {max_zoom!r})")
    return z


def shots(F, cuts=()):
    """The shots of F frames split at the cut pairs (pair k: between frames k and k + 1): a list of (first, last) frame
    indices, inclusive."""
    out, s = [], 0
    for k in sorted(set(int(c) for c in cuts)):
        out.append((s, k))
        s = k + 1
    out.append((s, int(F) - 1))
    return out


def motion_matrix(m):
    """[...,4] (a, b, tx, ty) -> [...,3,3] similarity matrices [[a, -b, tx], [b, a, ty], [0, 0, 1]]."""
    m = np.asarray(m, dtype=np.float64)
    a, b, tx, ty = np.moveaxis(m, -1, 0)
    out = np.zeros(m.shape[:-1] + (3, 3))
    out[..., 0, 0], out[..., 0, 1], out[..., 0, 2] = a, -b, tx
    out[..., 1, 0], out[..., 1, 1], out[..., 1, 2] = b, a, ty
    out[..., 2, 2] = 1.0
    return out


def camera_path(motions, cuts=()):
    """The camera path [F,3,3] of F - 1 motions (F x 4 rows (a, b, tx, ty), pair k: frame k -> k + 1): C = I at the first
    frame of every shot and C_(k+1) = M_k C_k inside it."""
    M = motion_matrix(motions)
    F = len(M) + 1
    C = np.empty((F, 3, 3))
    for s, e in shots(F, cuts):
        C[s] = np.eye(3)
        for k in range(s, e):
            C[k + 1] = M[k] @ C[k]
    return C


def path_params(C, cuts=()):
    """The [F,4] parameters (log s, theta, tx, ty) of a path of similarities, theta unwrapped along each shot."""
    a, b = C[:, 0, 0], C[:, 1, 0]
    p = np.stack([np.log(np.hypot(a, b)), np.arctan2(b, a), C[:, 0, 2], C[:, 1, 2]], axis=1)
    for s, e in shots(len(C), cuts):
        p[s:e + 1, 1] = np.unwrap(p[s:e + 1, 1])
    return p


def params_matrix(p):
    """[...,4] (log s, theta, tx, ty) -> [...,3,3] similarity matrices."""
    p = np.asarray(p, dtype=np.float64)
    s = np.exp(p[..., 0])
    return motion_matrix(np.stack([s * np.cos(p[..., 1]), s * np.sin(p[..., 1]), p[..., 2], p[..., 3]], axis=-1))


def smooth(p, sigma, cuts=()):
    """Each column of p [F,n] smoothed per shot by a Gaussian of sigma frames over a radius R = min(ceil(3 sigma), L - 1)
    for a shot of L frames, normalised over -R..R, with odd reflection about the shot's ends: index e + j reads
    2 p_e - p_(e-j) and s - j reads 2 p_s - p_(s+j).  A linear run stays as it is."""
    p = np.asarray(p, dtype=np.float64)
    out = np.empty_like(p)
    for s, e in shots(len(p), cuts):
        L = e - s + 1
        R = min(int(math.ceil(3.0 * sigma)), L - 1)
        seg = p[s:e + 1]
        if R == 0:
            out[s:e + 1] = seg
            continue
        j = np.arange(1, R + 1)
        ext = np.concatenate([2 * seg[0] - seg[j][::-1], seg, 2 * seg[-1] - seg[L - 1 - j]])
        k = np.arange(-R, R + 1, dtype=np.float64)
        w = np.exp(-0.5 * (k / sigma) ** 2)
        w /= w.sum()
        out[s:e + 1] = sum(w[i] * ext[i:i + L] for i in range(2 * R + 1))
    return out


def shot_zoom(B, hw, max_zoom):
    """The zoom of one shot: the smallest z >= 1 for which the four output corners c of an H x W frame land inside the
    source frame, B_t (c / z) in [-(W-1)/2, (W-1)/2] x [-(H-1)/2, (H-1)/2], for every B_t [n,3,3] of the shot.  With u =
    1 / z each condition is lo <= u m + d <= hi, linear in u, so the feasible u form one interval; z = 1 / its largest u
    in (0, 1].  A corner may overshoot by ZOOM_SLACK pixels, so the rounding of a path that needs no zoom gives z = 1.
    Returns (z, capped): z = max_zoom and capped True where that z exceeds max_zoom or no u is feasible."""
    H, W = hw
    hx, hy = 0.5 * (W - 1), 0.5 * (H - 1)
    corners = np.array([[-hx, -hy], [hx, -hy], [-hx, hy], [hx, hy]])
    m = np.einsum("nij,cj->nci", B[:, :2, :2], corners)  # [n,4,2]: the linear part at each corner
    d = np.broadcast_to(B[:, None, :2, 2], m.shape)
    h = np.broadcast_to(np.array([hx, hy]) + ZOOM_SLACK, m.shape)
    u_hi, u_lo = 1.0, 0.0
    # u m + d <= h and -(u m + d) <= h, each as u c <= r
    for c, r in ((m, h - d), (-m, h + d)):
        pos, neg, zero = c > 0, c < 0, c == 0
        if pos.any():
            u_hi = min(u_hi, float((r[pos] / c[pos]).min()))
        if neg.any():
            u_lo = max(u_lo, float((r[neg] / c[neg]).max()))
        if zero.any() and (r[zero] < 0).any():
            return float(max_zoom), True
    if u_hi <= 0 or u_hi < u_lo or 1.0 / u_hi > max_zoom:
        return float(max_zoom), True
    return 1.0 / u_hi, False


def centred_to_pixels(A, hw):
    """[...,3,3] maps in centred pixels -> [...,2,3] maps in the frames' own (uncentred) pixels: x -> A (x - c) + c."""
    H, W = hw
    T = np.eye(3)
    T[0, 2], T[1, 2] = 0.5 * (W - 1), 0.5 * (H - 1)
    Ti = np.eye(3)
    Ti[0, 2], Ti[1, 2] = -T[0, 2], -T[1, 2]
    return (T @ A @ Ti)[..., :2, :]


def camera_transforms(motions, hw, sigma, cuts=(), max_zoom=DEFAULT_MAX_ZOOM):
    """The stabilizing warps of a clip of F frames of size hw = (H, W) from its F - 1 motions [F-1,4] (rb_global_motion's
    params; the identity for unreliable and cut pairs): per shot the camera path, its smoothing with sigma frames and the
    shot's zoom.  Returns (transforms [F,2,3] fp64, each mapping an output pixel to its source position in the frame's
    own pixels, as rb_frames_warp_affine takes them; zooms, one per shot; capped, the indices of the shots whose zoom hit
    max_zoom).  motions that are not an [F-1,4] array with F >= 2, or cuts that are not pair indices in [0, F - 1),
    raise ValueError."""
    from .video import check_cuts
    sigma = check_sigma(sigma)
    max_zoom = check_max_zoom(max_zoom)
    motions = np.asarray(motions, dtype=np.float64)
    if motions.ndim != 2 or motions.shape[1] != 4 or len(motions) < 1:
        raise ValueError(f"stabilize: motions must be an [F-1,4] array with F >= 2 (got {list(motions.shape)})")
    F = len(motions) + 1
    cuts = check_cuts(cuts, F, "stabilize")
    C = camera_path(motions, cuts)
    S = params_matrix(smooth(path_params(C, cuts), sigma, cuts))
    B = C @ np.linalg.inv(S)
    A = np.empty((F, 3, 3))
    zooms, capped = [], []
    for i, (s, e) in enumerate(shots(F, cuts)):
        z, cap = shot_zoom(B[s:e + 1], hw, max_zoom)
        zooms.append(z)
        if cap:
            capped.append(i)
        A[s:e + 1] = B[s:e + 1] @ np.diag([1.0 / z, 1.0 / z, 1.0])
    return centred_to_pixels(A, hw), zooms, capped


def fill_margin(transforms, frame_hw, net_hw):
    """The canvas margin (my, mx) in network pixels per side that full-frame stabilization extends the flows by, for the
    transforms [F,2,3] of a whole clip of frame_hw = (Hs, Ws) frames and an (Hn, Wn) network grid.  (0, 0) when every
    source (rb_frames_warp_affine's fp64 position) lies in [0, Ws-1] x [0, Hs-1]: nothing is filled.  Otherwise per axis
    the largest distance by which a source's network position (the pixel-centre rule, (s + 0.5) Wn / Ws - 0.5) falls
    outside the grid [0, Wn-1], rounded up, plus FILL_MARGIN_TAPS for the bilinear taps, capped at FILL_MARGIN_CAP of the
    grid (a source beyond the canvas is filled spatially).  The sources are affine in the output pixel, so the farthest
    lie under the four output corners; the frame's own edge pixels map up to half a network pixel outside the grid when
    the frames are larger than it, so both axes get a margin once any source leaves the frame.  Non-finite transform
    entries are ignored."""
    A = np.asarray(transforms, dtype=np.float64)
    Hs, Ws = (int(v) for v in frame_hw)
    Hn, Wn = (int(v) for v in net_hw)
    if A.ndim != 3 or A.shape[1:] != (2, 3):
        raise ValueError(f"fill_margin: transforms must be [F,2,3] (got {list(A.shape)})")
    x = np.array([0.0, Ws - 1, 0.0, Ws - 1])
    y = np.array([0.0, 0.0, Hs - 1, Hs - 1])
    src, leaves = [], False
    for row, n_src in ((1, Hs), (0, Ws)):
        s = (A[:, row, 0, None] * x + A[:, row, 1, None] * y) + A[:, row, 2, None]
        s = s[np.isfinite(s)]
        leaves = leaves or bool(((s < 0) | (s > n_src - 1)).any())
        src.append(np.concatenate([s, [0.0, n_src - 1.0]]))  # the frame's own edges too
    if not leaves:
        return 0, 0
    out = []
    for s, n_src, n_net in ((src[0], Hs, Hn), (src[1], Ws, Wn)):
        p = (s + 0.5) * (n_net / n_src) - 0.5
        over = max(0.0, float((-p).max()), float((p - (n_net - 1)).max()))
        out.append(min(math.ceil(over) + FILL_MARGIN_TAPS, int(FILL_MARGIN_CAP * n_net)))
    return tuple(out)


def fill_motions(motions, cuts=()):
    """The per-pair similarities [F-1,4] the flows are extended with: the motions (rb_global_motion's params, already the
    identity at unreliable pairs) with the identity at the cut pairs."""
    m = np.array(motions, dtype=np.float64)
    m[list(cuts)] = (1.0, 0.0, 0.0, 0.0)
    return m


def fill_warp(frames, ext_fw, ext_bw, net_hw, margin, A, rows, flow_scale):
    """The full-frame stabilized frames of the table's rows (raft_b200.inpaint.inpaint_rows): one
    rb_frames_warp_affine_fill launch on the extended flows (networks.utils.warp_frames_fill, the forward-backward test
    of the occlusion check), A [n,2,3] the rows' transforms, then raft_b200.inpaint.finish_frames -- the spatial fill of
    what no frame saw (status 3) and the rounding.  Status-0 pixels are rb_frames_warp_affine's bytes.  Returns fresh
    (frames [n,Hs,Ws,3] uint8, status [n,Hs,Ws] uint8)."""
    from networks.utils import warp_frames_fill
    from .engine import FB_ALPHA1, FB_ALPHA2
    from .inpaint import finish_frames
    colour, status = warp_frames_fill(frames, ext_fw, ext_bw, net_hw, margin, A, rows, flow_scale=flow_scale,
                                      alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)
    return finish_frames(colour, status), status
