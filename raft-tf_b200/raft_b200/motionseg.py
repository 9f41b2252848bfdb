"""Motion segmentation (F34 / F35): the host-side rules of RaftEngine.segment_motion and video_segment_motion -- the
constants (mirrors of include/raft_b200.h), the argument checks, the per-frame table of how far each side may chain, the
fit of a batch of fields, and the map of a fitted homography from normalised coordinates to the frames' own pixels."""
import math

import numpy as np
import torch

DEFAULT_WINDOW = 3  # frames each side of a pixel's chain may reach (7 frames in all); not tuned on real footage
MAX_WINDOW = 16  # RB_MOTION_SEG_MAX_WINDOW
TAU = 1.0  # RB_MOTION_SEG_TAU: the residual, in network pixels, at which a field's evidence is 1/2; not tuned on real footage

# rb_homography_motion's constants: the weighted DLT sums per round (RB_HOMOGRAPHY_SUMS), and the rounds and the Cauchy
# scale in network pixels of the fit, chosen on synthetic flows only
SUMS = 45
MAX_ROUNDS = 32
ROUNDS = 8
CAUCHY = 0.5

# flags of rb_homography_motion
FIT, SINGULAR, UNRELIABLE = 0, 1, 2


def check_window(window, what="segment_motion"):
    """The temporal window as an int in [0, MAX_WINDOW]: how many frames each side of a pixel's chain may reach.
    Anything else raises ValueError."""
    if isinstance(window, bool) or not isinstance(window, (int, np.integer)) or not 0 <= window <= MAX_WINDOW:
        raise ValueError(f"{what}: window must be an integer in [0, {MAX_WINDOW}] (got {window!r})")
    return int(window)


def check_tau(tau, what="segment_motion"):
    """The residual scale tau in network pixels as a float that stays finite and > 0 in fp32.  Anything else raises
    ValueError."""
    try:
        with np.errstate(over="ignore"):
            t32 = float(np.float32(tau))
        ok = not isinstance(tau, (bool, str)) and math.isfinite(t32) and t32 > 0
    except (TypeError, ValueError, OverflowError):
        ok = False
    if not ok:
        raise ValueError(f"{what}: tau must be a number > 0 (network pixels) (got {tau!r})")
    return float(tau)


def segment_rows(F, window, cuts=()):
    """rb_motion_segment's table for a clip of F frames: raft_b200.inpaint.inpaint_rows(F, window, cuts), so no chain
    crosses a cut; window 0 gives every frame its own evidence only."""
    from .inpaint import inpaint_rows
    rows = inpaint_rows(F, max(check_window(window, "segment_rows"), 1), cuts)
    if window == 0:
        rows[:, 1:] = 0
    return rows


def cut_flags(cuts, pairs, device):
    """rb_motion_evidence's [len(pairs)] uint8 cut flags of the pairs listed (None when no cut is among them)."""
    c = set(cuts)
    flags = [1 if k in c else 0 for k in pairs]
    return torch.tensor(flags, dtype=torch.uint8, device=device) if any(flags) else None


def fit_fields(flow, occ, frame_hw, flow_scale):
    """F22 then F34 on a batch of fields [B,Hn,Wn,2] with their masks [B,Hn,Wn]: returns (H [B,3,3] fp64 normalised,
    flags [B] uint8), each field's bits independent of the batch."""
    from networks.utils import global_motion, homography_motion
    params, _, reliable = global_motion(flow, occ, frame_hw, flow_scale=flow_scale)
    return homography_motion(flow, occ, frame_hw, params, reliable, flow_scale=flow_scale)


def to_pixels(H, frame_hw):
    """Homographies [B,3,3] in rb_homography_motion's normalised coordinates mapped to the frames' own (uncentred)
    pixels, normalised to h33 = 1, in fp64 on the host."""
    Hs, Ws = frame_hw
    L = max(Hs, Ws) / 2.0
    N = np.array([[1 / L, 0, -0.5 * (Ws - 1) / L], [0, 1 / L, -0.5 * (Hs - 1) / L], [0, 0, 1]], np.float64)
    Ni = np.array([[L, 0, 0.5 * (Ws - 1)], [0, L, 0.5 * (Hs - 1)], [0, 0, 1]], np.float64)
    P = Ni @ np.asarray(H, np.float64) @ N
    return P / P[:, 2:3, 2:3]


def segment_frames(evidence, flow_fw, flow_bw, frame_hw, rows, flow_scale):
    """The masks of the table's rows: one rb_motion_segment launch with the forward-backward test of the occlusion
    check.  Returns fresh (mask [n,Hs,Ws] uint8, status [n,Hs,Ws] uint8)."""
    from networks.utils import motion_segment
    from .engine import FB_ALPHA1, FB_ALPHA2
    return motion_segment(evidence, flow_fw, flow_bw, frame_hw, rows, flow_scale=flow_scale, alpha1=FB_ALPHA1,
                          alpha2=FB_ALPHA2)
