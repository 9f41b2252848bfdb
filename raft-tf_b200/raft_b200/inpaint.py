"""Object removal from video (F24 / F25): the host-side rules of RaftEngine.inpaint and video_inpaint -- the fill
solver's pyramid and sweep counts (mirrors of csrc/inpaint.cu), the hole selection table, and the per-frame table of
how far each side of the temporal fill may chain."""
import numpy as np
import torch

DEFAULT_WINDOW = 10  # frames each side may chain; not tuned on real footage
DEFAULT_DILATE = 2  # mask dilation radius in frame pixels; not tuned on real footage

# rb_masked_fill's iteration counts (RB_FILL_* in include/raft_b200.h): red-black Gauss-Seidel sweeps per level of the
# initial guess, V-cycles on the finest level, and smoothing sweeps before and after each level's coarse correction
FILL_INIT_SWEEPS = 4
FILL_CYCLES = 6
FILL_SMOOTH = 3


def fill_levels(H, W):
    """The pyramid of rb_masked_fill: (H, W) halved with ceil until 1 x 1, finest first."""
    levels = [(int(H), int(W))]
    while levels[-1] != (1, 1):
        h, w = levels[-1]
        levels.append((-(-h // 2), -(-w // 2)))
    return levels


def check_window(window, what="inpaint"):
    """The temporal window as an int >= 1: how many frames each side of the temporal fill may chain.  Anything else
    raises ValueError."""
    if isinstance(window, bool) or not isinstance(window, (int, np.integer)) or window < 1:
        raise ValueError(f"{what}: window must be an integer >= 1 (got {window!r})")
    return int(window)


def check_dilate(dilate, what="inpaint"):
    """The mask dilation radius as an int in [0, RB_INPAINT_MAX_DILATE].  Anything else raises ValueError."""
    if isinstance(dilate, bool) or not isinstance(dilate, (int, np.integer)) or not 0 <= dilate <= MAX_DILATE:
        raise ValueError(f"{what}: dilate must be an integer in [0, {MAX_DILATE}] (got {dilate!r})")
    return int(dilate)


MAX_DILATE = 32  # RB_INPAINT_MAX_DILATE


def selection_table(labels=None, what="inpaint"):
    """rb_inpaint_masks' select table, [256] uint8: with labels None every non-zero mask value is a hole, else exactly the
    listed labels (integers in [0, 255], at least one).  Anything else raises ValueError."""
    table = np.zeros(256, np.uint8)
    if labels is None:
        table[1:] = 1
        return table
    try:
        ls = list(labels)
        ok = len(ls) > 0 and all(not isinstance(v, bool) and int(v) == v and 0 <= int(v) <= 255 for v in ls)
    except (TypeError, ValueError):
        ok = False
    if not ok:
        raise ValueError(f"{what}: labels must be a non-empty list of integers in [0, 255] (got {labels!r})")
    table[[int(v) for v in ls]] = 1
    return table


def inpaint_rows(F, window, cuts=()):
    """rb_inpaint_propagate's table for a clip of F frames: [F,3] int32, row t = (t, nf, nb).  nf = the steps the forward
    side may take, min(window, F - 1 - t, c - t) for the first cut pair c >= t; nb = the backward side's, min(window, t,
    t - 1 - c) for the last cut pair c < t (pair c lies between frames c and c + 1), so no side crosses a cut."""
    from .video import check_cuts
    window = check_window(window, "inpaint_rows")
    cuts = np.asarray(check_cuts(cuts, F, "inpaint_rows"), dtype=np.int64)
    t = np.arange(int(F), dtype=np.int64)
    nf = np.minimum(window, F - 1 - t)
    nb = np.minimum(window, t)
    if len(cuts):
        i = np.searchsorted(cuts, t, side="left")  # the first cut >= t
        nf = np.where(i < len(cuts), np.minimum(nf, cuts[np.minimum(i, len(cuts) - 1)] - t), nf)
        nb = np.where(i > 0, np.minimum(nb, t - 1 - cuts[np.maximum(i - 1, 0)]), nb)
    return np.stack([t, nf, nb], axis=1).astype(np.int32)


def complete_flows(flow_fw, flow_bw, hole_net):
    """The consecutive flows [T,Hn,Wn,2] completed inside the holes as one rb_masked_fill batch of 2T fields: flow_fw[k]
    inside frame k's grid hole, flow_bw[k] inside frame k + 1's (hole_net [T+1,Hn,Wn], inpaint_masks').  Returns fresh
    (flow_fw, flow_bw)."""
    from networks.utils import masked_fill
    T = flow_fw.shape[0]
    flows, _ = masked_fill(torch.cat([flow_fw, flow_bw]), torch.cat([hole_net[:T], hole_net[1:T + 1]]))
    return flows[:T], flows[T:]


def fill_frames(frames, hole, flow_fw, flow_bw, rows, flow_scale):
    """The frames of the table's rows with their holes filled: one rb_inpaint_propagate launch (the temporal fill, the
    forward-backward test of the occlusion check), one rb_masked_fill of the colours the temporal fill left (status 3),
    everything else as known data, then rounded half to even (rintf) and clamped to bytes.  Returns fresh (frames
    [n,Hs,Ws,3] uint8, status [n,Hs,Ws] uint8)."""
    from networks.utils import inpaint_propagate
    from .engine import FB_ALPHA1, FB_ALPHA2
    colour, status = inpaint_propagate(frames, hole, flow_fw, flow_bw, rows, flow_scale=flow_scale, alpha1=FB_ALPHA1,
                                       alpha2=FB_ALPHA2)
    return finish_frames(colour, status), status


def finish_frames(colour, status):
    """The bytes of temporally filled frames: one rb_masked_fill of the colours [n,Hs,Ws,3] fp32 where status [n,Hs,Ws]
    is 3 (what no frame saw), every other pixel known data that keeps its bits, then rounded half to even (rintf) and
    clamped to bytes.  Returns fresh frames [n,Hs,Ws,3] uint8."""
    from networks.utils import masked_fill
    colour, _ = masked_fill(colour, status == 3)
    return colour.round_().clamp_(0, 255).to(torch.uint8)
