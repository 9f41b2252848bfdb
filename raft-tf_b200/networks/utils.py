"""Drop-in mirror of the reference's ``networks/utils.py`` on torch CUDA tensors; every function
runs a raft_b200 CUDA kernel through the C ABI (no TF, no CPU fallback).  NHWC like the reference."""
import ctypes

import torch

from raft_b200 import capi


def coords_grid(batch, ht, wd, device=None):
    """utils.py:4-11 -> [b,h,w,2] with channel 0 = x, 1 = y."""
    device = torch.device(device if device is not None else "cuda")
    out = torch.empty(int(batch), int(ht), int(wd), 2, dtype=torch.float32, device=device)
    with torch.cuda.device(out.device):
        capi.check(capi.lib.rb_coords_grid(capi.ptr(out), int(batch), int(ht), int(wd), capi.stream()))
    return out


def bilinear_sampler(img, coords):
    """utils.py:101-103 (tf_grid_sample, :39-99): img [n,H,W,1], coords [n,a,b,2] (x,y pixels)
    -> [n,a,b,1].  Truncation toward zero, index clamping, weights from the clamped x1/y1."""
    n, H, W, c = img.shape
    assert c == 1, "the reference only samples the single-channel correlation volume"
    a, b = coords.shape[1], coords.shape[2]
    img, coords = img.contiguous().float(), coords.contiguous().float()
    out = torch.empty(n, a, b, 1, dtype=torch.float32, device=img.device)
    with torch.cuda.device(img.device):
        capi.check(capi.lib.rb_bilinear_sample(capi.ptr(img), capi.ptr(coords), capi.ptr(out), n, H, W, a * b,
                                               capi.stream()))
    return out


def upflow8(flow):
    """utils.py:105-111: bilinear x8 (align_corners=True) WITHOUT multiplying by 8 (reference quirk)."""
    b, h, w, _ = flow.shape
    coords1 = (flow + coords_grid(b, h, w, flow.device)).contiguous()
    out = torch.empty(b, 8 * h, 8 * w, 2, dtype=torch.float32, device=flow.device)
    with torch.cuda.device(out.device):
        capi.check(capi.lib.rb_upflow8(capi.ptr(coords1), capi.ptr(out), b, h, w, 1.0, capi.stream()))
    return out


def fb_consistency(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5, flow_scale=1.0):
    """Extension (no counterpart in the reference): forward-backward consistency of two [B,H,W,2] flows on the GPU
    (rb_flow_fb_check; Sundaram et al. 2010, UnFlow's alpha1 / alpha2 as defaults).  flow_scale multiplies both flows
    first: 8.0 for raft-small, whose upflow8 output is in 1/8-resolution units.  Returns (occ_fw, occ_bw), [B,H,W]
    uint8: 0 consistent, 1 inconsistent (occluded), 2 the flow leaves the frame."""
    assert flow_fw.shape == flow_bw.shape and flow_fw.dim() == 4 and flow_fw.shape[-1] == 2, (flow_fw.shape, flow_bw.shape)
    assert flow_fw.device == flow_bw.device, (flow_fw.device, flow_bw.device)
    b, H, W, _ = flow_fw.shape
    fw, bw = flow_fw.contiguous().float(), flow_bw.contiguous().float()
    occ_fw = torch.empty(b, H, W, dtype=torch.uint8, device=fw.device)
    occ_bw = torch.empty_like(occ_fw)
    with torch.cuda.device(fw.device):
        capi.check(capi.lib.rb_flow_fb_check(capi.ptr(fw), capi.ptr(bw), capi.ptr(occ_fw), capi.ptr(occ_bw), b, H, W,
                                             float(flow_scale), float(alpha1), float(alpha2), capi.stream()))
    return occ_fw, occ_bw


def _flow_pair(what, flow_fw, flow_bw):
    """(T, H, W) of two matching [T,H,W,2] float32 CUDA flows; anything else raises ValueError."""
    for name, t in (("flow_fw", flow_fw), ("flow_bw", flow_bw)):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dim() == 4 and t.shape[-1] == 2
                and t.dtype == torch.float32):
            raise ValueError(f"{what}: {name} must be a [T,H,W,2] float32 CUDA tensor (got "
                             f"{getattr(t, 'shape', None)} {getattr(t, 'dtype', type(t))})")
    if flow_fw.shape != flow_bw.shape or flow_fw.device != flow_bw.device:
        raise ValueError(f"{what}: flow_fw {tuple(flow_fw.shape)} and flow_bw {tuple(flow_bw.shape)} must match")
    return tuple(flow_fw.shape[:3])


def _track_args(what, flow_fw, flow_bw, qframe, qpos, state):
    """The argument checks of track_points and track_points_backward -> (T, H, W, N, qframe, qpos, state) with the
    queries as contiguous device tensors and state fresh (NaN, 3) when None."""
    T, H, W = _flow_pair(what, flow_fw, flow_bw)
    dev = flow_fw.device
    qframe = torch.as_tensor(qframe).to(device=dev, dtype=torch.int32).contiguous()
    qpos = torch.as_tensor(qpos).to(device=dev, dtype=torch.float32).contiguous()
    N = qframe.shape[0] if qframe.dim() == 1 else -1
    if N < 1 or tuple(qpos.shape) != (N, 2):
        raise ValueError(f"{what}: qframe must be [N] and qpos [N,2], N >= 1 (got {tuple(qframe.shape)} and "
                         f"{tuple(qpos.shape)})")
    if state is None:
        state = (torch.full((N, 2), float("nan"), dtype=torch.float32, device=dev),
                 torch.full((N,), 3, dtype=torch.uint8, device=dev))
    pos, st = state
    if not (tuple(pos.shape) == (N, 2) and pos.dtype == torch.float32 and tuple(st.shape) == (N,)
            and st.dtype == torch.uint8 and pos.device == dev and st.device == dev and pos.is_contiguous()
            and st.is_contiguous()):
        raise ValueError(f"{what}: state must be contiguous (pos [N,2] float32, state [N] uint8) on {dev}")
    return T, H, W, N, qframe, qpos, (pos, st)


def track_points(flow_fw, flow_bw, qframe, qpos, state=None, first_frame=0, n_steps=None, flow_scale=1.0, alpha1=0.01,
                 alpha2=0.5):
    """Extension (point tracking): N query points chained through the consecutive flows of one pass on the GPU
    (rb_track_points).  flow_fw, flow_bw: [T,H,W,2] fp32 CUDA flows in pair order (forward_sequence_bidirectional's);
    the first n_steps pairs (default T) are used.  qframe [N] (integer global frame indices) and qpos [N,2] (x, y in the
    flows' pixels); first_frame is the global index of the flows' frame 0.  state = (pos [N,2] fp32, state [N] uint8)
    CUDA tensors carry the queries from a previous call on the clip (None: fresh ones); they are updated in place.
    flow_scale, alpha1, alpha2 as in fb_consistency.  Returns (tracks [n_steps+1,N,2] fp32, status [n_steps+1,N] uint8,
    state): row j is frame first_frame + j; status 0 consistent, 1 inconsistent (occluded; the track goes on), 2 left
    the frame (NaN from then on), 3 before the query frame (NaN)."""
    T, H, W, N, qframe, qpos, (pos, st) = _track_args("track_points", flow_fw, flow_bw, qframe, qpos, state)
    dev = flow_fw.device
    n_steps = T if n_steps is None else int(n_steps)
    tracks = torch.empty(n_steps + 1, N, 2, dtype=torch.float32, device=dev)
    status = torch.empty(n_steps + 1, N, dtype=torch.uint8, device=dev)
    fw, bw = flow_fw.contiguous(), flow_bw.contiguous()
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_track_points(capi.ptr(fw), capi.ptr(bw), T, H, W, n_steps, float(flow_scale),
                                            float(alpha1), float(alpha2), capi.ptr(qframe), capi.ptr(qpos), N,
                                            int(first_frame), capi.ptr(pos), capi.ptr(st), capi.ptr(tracks),
                                            capi.ptr(status), capi.stream()))
    return tracks, status, (pos, st)


def track_points_backward(flow_fw, flow_bw, qframe, qpos, tracks=None, status=None, state=None, first_frame=0,
                          n_steps=None, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """Extension (point tracking backward in time): the mirror of track_points (rb_track_points_backward), each query
    followed from its frame back to the flows' frame 0.  Arguments as for track_points.  tracks [n_steps+1,N,2] fp32 and
    status [n_steps+1,N] uint8 (contiguous, on the flows' device; e.g. track_points' outputs) are completed in place:
    rows after a query's frame keep what they hold, the row of its frame becomes (qpos, 0) and the rows before it the
    backward track.  Without them they start as NaN / 3.  state carries a reverse sweep of calls from later frames to
    earlier ones: read for a query whose frame lies after the flows' last frame (its row n_steps is the carried state),
    written with row 0 for every query whose frame is at or after first_frame, untouched for the others.  Returns
    (tracks, status, state)."""
    T, H, W, N, qframe, qpos, (pos, st) = _track_args("track_points_backward", flow_fw, flow_bw, qframe, qpos, state)
    dev = flow_fw.device
    n_steps = T if n_steps is None else int(n_steps)
    if tracks is None:
        tracks = torch.full((n_steps + 1, N, 2), float("nan"), dtype=torch.float32, device=dev)
    if status is None:
        status = torch.full((n_steps + 1, N), 3, dtype=torch.uint8, device=dev)
    if not (tuple(tracks.shape) == (n_steps + 1, N, 2) and tracks.dtype == torch.float32 and tracks.device == dev
            and tracks.is_contiguous() and tuple(status.shape) == (n_steps + 1, N) and status.dtype == torch.uint8
            and status.device == dev and status.is_contiguous()):
        raise ValueError(f"track_points_backward: tracks and status must be contiguous [n_steps+1,N,2] float32 and "
                         f"[n_steps+1,N] uint8 on {dev} with n_steps + 1 = {n_steps + 1}, N = {N} (got "
                         f"{tuple(tracks.shape)} {tracks.dtype} and {tuple(status.shape)} {status.dtype})")
    fw, bw = flow_fw.contiguous(), flow_bw.contiguous()
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_track_points_backward(capi.ptr(fw), capi.ptr(bw), T, H, W, n_steps, float(flow_scale),
                                                     float(alpha1), float(alpha2), capi.ptr(qframe), capi.ptr(qpos), N,
                                                     int(first_frame), capi.ptr(pos), capi.ptr(st), capi.ptr(tracks),
                                                     capi.ptr(status), capi.stream()))
    return tracks, status, (pos, st)


def _accumulate(what, fn, flow_fw, flow_bw, acc, status, start, n_steps, flow_scale, alpha1, alpha2):
    """The checks and the call of accumulate_flow / accumulate_flow_backward."""
    T, H, W = _flow_pair(what, flow_fw, flow_bw)
    dev = flow_fw.device
    n_steps = T if n_steps is None else int(n_steps)
    if not (isinstance(acc, torch.Tensor) and isinstance(status, torch.Tensor)
            and tuple(acc.shape) == (n_steps + 1, H, W, 2) and acc.dtype == torch.float32 and acc.device == dev
            and acc.is_contiguous() and tuple(status.shape) == (n_steps + 1, H, W) and status.dtype == torch.uint8
            and status.device == dev and status.is_contiguous()):
        raise ValueError(f"{what}: acc and status must be contiguous [n_steps+1,H,W,2] float32 and [n_steps+1,H,W] uint8 "
                         f"on {dev} with n_steps + 1 = {n_steps + 1}, H x W = {H}x{W} (got "
                         f"{tuple(getattr(acc, 'shape', ()))} and {tuple(getattr(status, 'shape', ()))})")
    fw, bw = flow_fw.contiguous(), flow_bw.contiguous()
    with torch.cuda.device(dev):
        capi.check(fn(capi.ptr(fw), capi.ptr(bw), T, H, W, n_steps, float(flow_scale), float(alpha1), float(alpha2),
                      int(start), capi.ptr(acc), capi.ptr(status), capi.stream()))
    return acc, status


def accumulate_flow(flow_fw, flow_bw, acc, status, start=0, n_steps=None, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """Extension (keyframe label propagation): per pixel of every later frame, the displacement back to the frame of row
    `start`, composed through the consecutive flows of one pass on the GPU (rb_flow_accumulate).  flow_fw, flow_bw:
    [T,H,W,2] fp32 CUDA flows in pair order (forward_sequence_bidirectional's); the first n_steps pairs (default T) are
    used.  acc [n_steps+1,H,W,2] fp32 and status [n_steps+1,H,W] uint8 are written in place: row `start` is the input
    (zeros for the keyframe, or the last row of the previous pass), rows start+1 .. n_steps are written, no other row is
    touched.  Status: 0 consistent at every step back to the keyframe, 1 occluded at some step (the forward-backward test
    of fb_consistency failed), 2 entered through the frame edge at some step.  flow_scale, alpha1, alpha2 as in
    fb_consistency.  Returns (acc, status)."""
    return _accumulate("accumulate_flow", capi.lib.rb_flow_accumulate, flow_fw, flow_bw, acc, status, start, n_steps,
                       flow_scale, alpha1, alpha2)


def accumulate_flow_backward(flow_fw, flow_bw, acc, status, start=0, n_steps=None, flow_scale=1.0, alpha1=0.01,
                             alpha2=0.5):
    """The mirror of accumulate_flow for the frames before the keyframe (rb_flow_accumulate_backward): rows start-1 .. 0
    are written from row `start`, each step r+1 -> r pulling with flow_fw[r] and testing against flow_bw[r]."""
    return _accumulate("accumulate_flow_backward", capi.lib.rb_flow_accumulate_backward, flow_fw, flow_bw, acc, status,
                       start, n_steps, flow_scale, alpha1, alpha2)


def propagate_labels(acc, status, key):
    """Extension (keyframe label propagation): the [Hs,Ws] uint8 CUDA label map `key` of the keyframe carried to every row
    of acc [n,H,W,2] / status [n,H,W] (accumulate_flow's, at the network size) at the key's own size (rb_labels_propagate):
    per output pixel, the displacement resized as resize_flow does, the origin clamped into the key, and the label of the
    largest summed bilinear weight among the origin's four pixels (ties to the smaller label).  Returns fresh (labels
    [n,Hs,Ws] uint8, status [n,Hs,Ws] uint8): status as accumulate_flow's at the network pixel that holds the output pixel's
    centre, 2 where the origin had to be clamped."""
    if not (isinstance(acc, torch.Tensor) and acc.is_cuda and acc.dim() == 4 and acc.shape[-1] == 2
            and acc.dtype == torch.float32):
        raise ValueError(f"propagate_labels: acc must be an [n,H,W,2] float32 CUDA tensor (got "
                         f"{getattr(acc, 'shape', None)} {getattr(acc, 'dtype', type(acc))})")
    n, H, W, _ = acc.shape
    if not (isinstance(status, torch.Tensor) and tuple(status.shape) == (n, H, W) and status.dtype == torch.uint8
            and status.device == acc.device):
        raise ValueError(f"propagate_labels: status must be an [n,H,W] = {[n, H, W]} uint8 tensor on {acc.device}")
    if not (isinstance(key, torch.Tensor) and key.dim() == 2 and key.dtype == torch.uint8 and key.device == acc.device):
        raise ValueError(f"propagate_labels: key must be an [Hs,Ws] uint8 tensor on {acc.device} (got "
                         f"{getattr(key, 'shape', None)} {getattr(key, 'dtype', type(key))})")
    Hs, Ws = key.shape
    a, s, k = acc.contiguous(), status.contiguous(), key.contiguous()
    labels = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=a.device)
    st = torch.empty_like(labels)
    with torch.cuda.device(a.device):
        capi.check(capi.lib.rb_labels_propagate(capi.ptr(a), capi.ptr(s), n, H, W, capi.ptr(k), Hs, Ws,
                                                capi.ptr(labels), capi.ptr(st), capi.stream()))
    return labels, st


def propagate_labels_keys(acc_a, status_a, acc_b, status_b, keys, rows):
    """Extension (several keyframes): the labels of every row voted between the keyframes on either side of it
    (rb_labels_propagate_keys).  acc_a / status_a and acc_b / status_b: [n,H,W,2] fp32 and [n,H,W] uint8 CUDA rows of
    accumulate_flow's forward chain from the key before each row (side A) and accumulate_flow_backward's chain from the
    key after it (side B); keys [m,Hs,Ws] uint8 the keyframes' label maps at the frames' own size; rows [n,4] int32 per
    row (slot_a, slot_b, w_a, w_b): the key index of each side (-1: absent) and, where both are present, their positive
    integer weights (raft_b200.video.keyframe_rows builds it).  Per pixel the present sides with the smallest status vote
    -- one alone with propagate_labels' bits, two over their eight taps with side A's bilinear weights times w_a and side
    B's times w_b.  Returns fresh (labels [n,Hs,Ws] uint8, status [n,Hs,Ws] uint8): the smallest status of the voters,
    3 (label 0) where no side is present.  Bad shapes or a bad table raise ValueError before the upload."""
    if not (isinstance(acc_a, torch.Tensor) and acc_a.is_cuda and acc_a.dim() == 4 and acc_a.shape[-1] == 2
            and acc_a.dtype == torch.float32):
        raise ValueError(f"propagate_labels_keys: acc_a must be an [n,H,W,2] float32 CUDA tensor (got "
                         f"{getattr(acc_a, 'shape', None)} {getattr(acc_a, 'dtype', type(acc_a))})")
    n, H, W, _ = acc_a.shape
    dev = acc_a.device
    if not (isinstance(acc_b, torch.Tensor) and acc_b.shape == acc_a.shape and acc_b.dtype == torch.float32
            and acc_b.device == dev):
        raise ValueError(f"propagate_labels_keys: acc_b must be an [n,H,W,2] = {[n, H, W, 2]} float32 tensor on {dev}")
    for name, t in (("status_a", status_a), ("status_b", status_b)):
        if not (isinstance(t, torch.Tensor) and tuple(t.shape) == (n, H, W) and t.dtype == torch.uint8
                and t.device == dev):
            raise ValueError(f"propagate_labels_keys: {name} must be an [n,H,W] = {[n, H, W]} uint8 tensor on {dev}")
    if not (isinstance(keys, torch.Tensor) and keys.dim() == 3 and keys.shape[0] >= 1 and keys.dtype == torch.uint8
            and keys.device == dev):
        raise ValueError(f"propagate_labels_keys: keys must be an [m,Hs,Ws] uint8 tensor on {dev} (got "
                         f"{getattr(keys, 'shape', None)} {getattr(keys, 'dtype', type(keys))})")
    m, Hs, Ws = keys.shape
    table = torch.as_tensor(rows).cpu()
    if not (tuple(table.shape) == (n, 4) and not table.is_floating_point() and not table.is_complex()):
        raise ValueError(f"propagate_labels_keys: rows must be an [n,4] = {[n, 4]} integer table (got "
                         f"{list(table.shape)} {table.dtype})")
    table = table.to(torch.int64)
    sa, sb, wa, wb = table.unbind(1)
    if not (((sa >= -1) & (sa < m)).all() and ((sb >= -1) & (sb < m)).all()):
        raise ValueError(f"propagate_labels_keys: the slots must be key indices in [0, {m}) or -1 (absent)")
    both = (sa >= 0) & (sb >= 0)
    if not (((wa > 0) & (wa < 1 << 24) & (wb > 0) & (wb < 1 << 24)) | ~both).all():
        raise ValueError("propagate_labels_keys: where both sides are present, the weights must be integers in [1, 2^24)")
    table = table.to(device=dev, dtype=torch.int32).contiguous()
    aa, a_s, ab, b_s, k = (t.contiguous() for t in (acc_a, status_a, acc_b, status_b, keys))
    labels = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=dev)
    st = torch.empty_like(labels)
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_labels_propagate_keys(capi.ptr(aa), capi.ptr(a_s), capi.ptr(ab), capi.ptr(b_s),
                                                     capi.ptr(table), n, H, W, capi.ptr(k), m, Hs, Ws,
                                                     capi.ptr(labels), capi.ptr(st), capi.stream()))
    return labels, st


LABEL_STATS = ("intersection", "union", "boundary_pred", "boundary_gt", "matched_pred", "matched_gt")  # RB_LABEL_STATS


def label_metrics(pred, gt, n_objects, bound_pix=None):
    """Extension (DAVIS-2017's J and F): the integer counts of [n,H,W] uint8 CUDA label maps pred against gt for the
    objects 1..n_objects (rb_label_metrics).  Returns a fresh [n, n_objects, 6] int64 tensor (LABEL_STATS): |P and G|,
    |P or G|, the boundary pixels of P and of G (davis2017-evaluation's _seg2bmap), and those of each with a boundary
    pixel of the other within a disk of radius bound_pix (default ceil(0.008 hypot(H, W)), DAVIS's; 1 to 32).  Wrong
    shapes or dtypes raise ValueError."""
    for name, t in (("pred", pred), ("gt", gt)):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dim() == 3 and t.dtype == torch.uint8):
            raise ValueError(f"label_metrics: {name} must be an [n,H,W] uint8 CUDA tensor (got "
                             f"{getattr(t, 'shape', None)} {getattr(t, 'dtype', type(t))})")
    if pred.shape != gt.shape or pred.device != gt.device:
        raise ValueError(f"label_metrics: pred {tuple(pred.shape)} and gt {tuple(gt.shape)} must match")
    n, H, W = pred.shape
    if bound_pix is None:
        bound_pix = davis_bound_pix(H, W)
    p, g = pred.contiguous(), gt.contiguous()
    counts = torch.empty(n, int(n_objects), len(LABEL_STATS), dtype=torch.int64, device=p.device)
    with torch.cuda.device(p.device):
        capi.check(capi.lib.rb_label_metrics(capi.ptr(p), capi.ptr(g), n, H, W, int(n_objects), int(bound_pix),
                                             capi.ptr(counts), capi.stream()))
    return counts


def davis_bound_pix(H, W):
    """davis2017-evaluation's f_measure radius: ceil(0.008 * hypot(H, W)) (8 at 480x854, 18 at 1080x1920)."""
    import math
    return int(math.ceil(0.008 * math.hypot(H, W)))


FLOW_STATS = ("n", "sum_epe", "lt1", "lt3", "lt5", "outliers")  # the columns of flow_metrics' stats (RB_FLOW_STATS)


def flow_metrics(flow, gt, valid=None, flow_scale=1.0, return_epe=False):
    """Extension (upstream RAFT's evaluate.py): end-point-error statistics of [B,H,W,2] CUDA flows against ground truth gt
    (rb_flow_metrics).  valid: optional [B,H,W] mask, nonzero = the pixel counts.  flow_scale multiplies the flow first: 8.0
    for raft-small in the reference semantics, whose upflow8 output is in 1/8-resolution units.  Returns the [B,6] fp64
    stats {n, sum of EPE, #(EPE < 1), #(EPE < 3), #(EPE < 5), #KITTI outliers (EPE > 3 and EPE / |gt| > 0.05)} over the
    counted pixels (FLOW_STATS), and with return_epe also the [B,H,W] fp32 per-pixel EPE (every pixel)."""
    assert flow.shape == gt.shape and flow.dim() == 4 and flow.shape[-1] == 2, (flow.shape, gt.shape)
    assert flow.device == gt.device, (flow.device, gt.device)
    B, H, W, _ = flow.shape
    f, g = flow.contiguous().float(), gt.contiguous().float()
    if valid is not None:
        assert tuple(valid.shape) == (B, H, W) and valid.device == f.device, (valid.shape, valid.device)
        valid = valid.contiguous().to(torch.uint8)
    stats = torch.empty(B, len(FLOW_STATS), dtype=torch.float64, device=f.device)
    epe = torch.empty(B, H, W, dtype=torch.float32, device=f.device) if return_epe else None
    with torch.cuda.device(f.device):
        nbytes = capi.size_query(capi.lib.rb_flow_metrics_workspace_bytes, B, H, W)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=f.device)
        capi.check(capi.lib.rb_flow_metrics(capi.ptr(f), float(flow_scale), capi.ptr(g), capi.ptr(valid), B, H, W,
                                            capi.ptr(epe), capi.ptr(stats), capi.ptr(ws), nbytes, capi.stream()))
    return (stats, epe) if return_epe else stats


FRAME_STATS = ("sse", "ssim")  # the columns of frame_metrics' stats (RB_FRAME_STATS)


def frame_metrics(pred, gt):
    """Extension (the Vimeo-90K triplet protocol): SSE and SSIM of [B,H,W,3] CUDA frames pred (fp32 in [0,1], what
    interpolate returns, or uint8) against uint8 ground truth gt (rb_frame_metrics), H and W >= 11.  An fp32 pred is first
    quantised as infer_raft.py --interpolate writes its PNGs (np.clip(np.rint(fl32(255 * x)), 0, 255); NaN -> 0).  Returns a
    fresh [B,2] fp64 tensor {sse, ssim} (FRAME_STATS): the exact sum of squared 8-bit errors, and skimage's
    structural_similarity(gaussian_weights=True, sigma=1.5, use_sample_covariance=False, data_range=255) averaged over the
    3 channels.  PSNR = 10 * log10(255^2 * 3HW / sse) (inf when sse = 0).  Wrong shapes or dtypes raise ValueError."""
    for name, t, dtypes in (("pred", pred, (torch.float32, torch.uint8)), ("gt", gt, (torch.uint8,))):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dim() == 4 and t.shape[-1] == 3 and t.dtype in dtypes):
            raise ValueError(f"frame_metrics: {name} must be a [B,H,W,3] {' or '.join(str(d) for d in dtypes)} CUDA "
                             f"tensor (got {getattr(t, 'shape', None)} {getattr(t, 'dtype', type(t))})")
    if pred.shape != gt.shape or pred.device != gt.device:
        raise ValueError(f"frame_metrics: pred {tuple(pred.shape)} on {pred.device} and gt {tuple(gt.shape)} on "
                         f"{gt.device} must match")
    B, H, W, _ = pred.shape
    if H < 11 or W < 11:
        raise ValueError(f"frame_metrics: frames of {H}x{W} are smaller than the 11x11 SSIM window")
    p, g = pred.contiguous(), gt.contiguous()
    stats = torch.empty(B, len(FRAME_STATS), dtype=torch.float64, device=p.device)
    with torch.cuda.device(p.device):
        nbytes = capi.size_query(capi.lib.rb_frame_metrics_workspace_bytes, B, H, W)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=p.device)
        capi.check(capi.lib.rb_frame_metrics(capi.ptr(p), int(p.dtype == torch.uint8), capi.ptr(g), B, H, W,
                                             capi.ptr(stats), capi.ptr(ws), nbytes, capi.stream()))
    return stats


SCENE_BINS = 512  # RB_SCENE_BINS: 8 levels per channel


def scene_cut_scores(frames, return_hist=False):
    """Extension (scene cuts of a video): the [N-1] fp32 scores of [N,H,W,3] uint8 CUDA frames (N >= 2, any channel
    order), scores[k] = 1 - the intersection of the joint colour histograms of frames k and k + 1 (8 levels per channel,
    bin (c0 >> 5) 64 + (c1 >> 5) 8 + (c2 >> 5)) over H W, rounded once to fp32: 0 for frames with one histogram, 1 for
    frames that share no bin (rb_scene_cut_scores; exact).  With return_hist also the [N,512] int32 histograms.  Wrong
    shapes or dtypes raise ValueError."""
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dim() == 4 and frames.shape[-1] == 3
            and frames.dtype == torch.uint8 and frames.shape[0] >= 2):
        raise ValueError(f"scene_cut_scores: frames must be a [N,H,W,3] uint8 CUDA tensor with N >= 2 (got "
                         f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
    f = frames.contiguous()
    N, H, W, _ = f.shape
    hist = torch.empty(N, SCENE_BINS, dtype=torch.int32, device=f.device)
    scores = torch.empty(N - 1, dtype=torch.float32, device=f.device)
    with torch.cuda.device(f.device):
        capi.check(capi.lib.rb_scene_cut_scores(capi.ptr(f), N, H, W, capi.ptr(hist), capi.ptr(scores), capi.stream()))
    return (scores, hist) if return_hist else scores


def forward_interpolate(flow):
    """Extension (upstream RAFT's core/utils/utils.py forward_interpolate, on the GPU): every grid point of the [B,h,w,2]
    fp32 CUDA flow takes the flow of the nearest source pixel x + flow(x) that lands strictly inside the grid, per
    sample (rb_flow_forward_interpolate; equal distances go to the lower source index, a sample without such a source
    gives zeros).  Returns a fresh [B,h,w,2] tensor: the flow_init of the next frame pair from this pair's flow_low."""
    if not (isinstance(flow, torch.Tensor) and flow.is_cuda and flow.dim() == 4 and flow.shape[-1] == 2
            and flow.dtype == torch.float32):
        raise ValueError(f"forward_interpolate: flow must be a [B,h,w,2] float32 CUDA tensor (got "
                         f"{getattr(flow, 'shape', None)} {getattr(flow, 'dtype', type(flow))})")
    f = flow.contiguous()
    B, h, w, _ = f.shape
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        nbytes = capi.size_query(capi.lib.rb_flow_forward_interpolate_workspace_bytes, B, h, w)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=f.device)
        capi.check(capi.lib.rb_flow_forward_interpolate(capi.ptr(f), capi.ptr(out), B, h, w, capi.ptr(ws), nbytes,
                                                        capi.stream()))
    return out


def flow_to_color(flow, clip_flow=None, convert_to_bgr=False):
    """flow_utils.flow_to_color (the reference's flow_utils.py:95-121) on a batch of CUDA flows (rb_flow_to_color): each
    [H,W,2] sample of the [B,H,W,2] fp32 flow coloured by the Middlebury wheel, normalised by its own maximum radius.
    Returns a fresh [B,H,W,3] uint8 tensor, RGB or BGR with convert_to_bgr.  Equal to the host function wherever numpy's
    float32 arctan2 is correctly rounded; the kernel rounds the fp64 atan2 to fp32 instead (DESIGN §4)."""
    if not (isinstance(flow, torch.Tensor) and flow.is_cuda and flow.dim() == 4 and flow.shape[-1] == 2
            and flow.dtype == torch.float32):
        raise ValueError(f"flow_to_color: flow must be a [B,H,W,2] float32 CUDA tensor (got "
                         f"{getattr(flow, 'shape', None)} {getattr(flow, 'dtype', type(flow))})")
    f = flow.contiguous()
    B, H, W, _ = f.shape
    out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=f.device)
    clip = clip_flow is not None
    with torch.cuda.device(f.device):
        nbytes = capi.size_query(capi.lib.rb_flow_to_color_workspace_bytes, B, H, W)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=f.device)
        capi.check(capi.lib.rb_flow_to_color(capi.ptr(f), B, H, W, int(clip), float(clip_flow) if clip else 0.0,
                                             int(bool(convert_to_bgr)), capi.ptr(out), capi.ptr(ws), nbytes,
                                             capi.stream()))
    return out


def reverse_flow(flow, time_step=1.0, bg=None, im0=None):
    """The reference's flow_utils.py:166 reverse_flow_avg_skip_static on a batch of CUDA flows (rb_flow_reverse, bit for
    bit): projects the [B,H,W,2] flow 0 -> 1 to time `time_step` and returns the flow from there back to frame 0.
    bg, im0: optional [B,H,W,C] images (both or neither); pixels where every channel differs by < 10 are static and
    skipped (uint8 pairs compare the wrapped uint8 difference, as numpy does; any other pair is compared in fp32).
    Returns (flow_t [B,H,W,2] fp32, empty, multi, static, empty_eroded), the last four [B,H,W] uint8: no source
    landed, more than one landed, the static mask, and empty eroded by a 5x5 window.  Empty pixels hold the mean of their
    nearest non-empty neighbours up, down, left and right.  A NaN flow is skipped (the reference raises on it)."""
    assert flow.dim() == 4 and flow.shape[-1] == 2, flow.shape
    if (bg is None) != (im0 is None):
        raise ValueError("reverse_flow: pass both bg and im0, or neither")
    B, H, W, _ = flow.shape
    f = flow.contiguous().float()
    u8, C = 0, 0
    if bg is not None:
        assert bg.shape == im0.shape and bg.dim() == 4 and tuple(bg.shape[:3]) == (B, H, W), (bg.shape, im0.shape)
        if bg.dtype == torch.uint8 and im0.dtype == torch.uint8:
            u8 = 1
        else:  # numpy promotes a uint8 / float32 pair to float32; the values are exact
            bg, im0 = bg.float(), im0.float()
        bg, im0, C = bg.contiguous(), im0.contiguous(), bg.shape[-1]
    out = torch.empty_like(f)
    empty, multi, static, eroded = (torch.empty(B, H, W, dtype=torch.uint8, device=f.device) for _ in range(4))
    with torch.cuda.device(f.device):
        nbytes = capi.size_query(capi.lib.rb_flow_reverse_workspace_bytes, B, H, W)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=f.device)
        capi.check(capi.lib.rb_flow_reverse(capi.ptr(f), capi.ptr(bg), capi.ptr(im0), u8, C, float(time_step),
                                            capi.ptr(out), capi.ptr(empty), capi.ptr(multi), capi.ptr(eroded),
                                            capi.ptr(static), B, H, W, capi.ptr(ws), nbytes, capi.stream()))
    return out, empty, multi, static, eroded


def synthesize(frame0, frame1, flow_t0, flow_t1, empty0, empty1, t):
    """Extension: the frame at time t in [0, 1] between [B,H,W,3] frames frame0 and frame1 (rb_frame_synthesize):
    each frame sampled bilinearly at p + flow_tk(p) (the flows from time t to frame k, e.g. reverse_flow(flow_01, t) and
    reverse_flow(flow_10, 1 - t)) and blended with weights 1 - t and t, a frame whose flow is empty at p weighted 0
    (unless both are).  t = 0 gives frame0 and t = 1 gives frame1 exactly.  -> [B,H,W,3] fp32."""
    t = float(t)
    if not 0.0 <= t <= 1.0:
        raise ValueError(f"synthesize: t must be in [0, 1] (got {t})")
    assert frame0.shape == frame1.shape and frame0.dim() == 4 and frame0.shape[-1] == 3, (frame0.shape, frame1.shape)
    B, H, W, _ = frame0.shape
    assert flow_t0.shape == flow_t1.shape == (B, H, W, 2) and empty0.shape == empty1.shape == (B, H, W)
    frames = torch.cat([frame0, frame1]).float().contiguous()
    f0, f1 = flow_t0.contiguous().float(), flow_t1.contiguous().float()
    e0, e1 = empty0.contiguous().to(torch.uint8), empty1.contiguous().to(torch.uint8)
    out = torch.empty(B, H, W, 3, dtype=torch.float32, device=frames.device)
    with torch.cuda.device(out.device):
        capi.check(capi.lib.rb_frame_synthesize(capi.ptr(frames), H, W, 0, 0, capi.ptr(f0), capi.ptr(f1), capi.ptr(e0),
                                                capi.ptr(e1), t, capi.ptr(out), B, H, W, capi.stream()))
    return out


def synthesize_resized(frame0, frame1, flow_t0, flow_t1, empty0, empty1, t, uint8=False, bgr=False):
    """Extension: synthesize at the frames' own size from flows at the network size (rb_frame_synthesize_pairs_resized).
    frame0, frame1: [B,Hs,Ws,3] CUDA frames, uint8 (divided by 255 like rb_frames_prepare) or fp32; flow_t0, flow_t1
    [B,H,W,2] and empty0, empty1 [B,H,W] at the network size (e.g. reverse_flow of the flows the network estimated).
    Each flow is resized to Hs x Ws as resize_flow does and each mask taken at the network pixel that holds the output
    pixel's centre, then blended as synthesize does, bit for bit, without those Hs x Ws intermediates.  -> [B,Hs,Ws,3]
    fp32, or with uint8 quantised as infer_raft.py writes PNGs (bgr: channels reversed)."""
    t = float(t)
    if not 0.0 <= t <= 1.0:
        raise ValueError(f"synthesize_resized: t must be in [0, 1] (got {t})")
    if bgr and not uint8:
        raise ValueError("synthesize_resized: bgr swaps the channels of uint8 output; pass uint8=True")
    assert frame0.shape == frame1.shape and frame0.dim() == 4 and frame0.shape[-1] == 3, (frame0.shape, frame1.shape)
    assert frame0.dtype == frame1.dtype and frame0.dtype in (torch.uint8, torch.float32), (frame0.dtype, frame1.dtype)
    B, Hs, Ws, _ = frame0.shape
    H, W = flow_t0.shape[1:3]
    assert flow_t0.shape == flow_t1.shape == (B, H, W, 2) and empty0.shape == empty1.shape == (B, H, W)
    i0, i1 = frame0.contiguous(), frame1.contiguous()
    f0, f1 = flow_t0.contiguous().float(), flow_t1.contiguous().float()
    e0, e1 = empty0.contiguous().to(torch.uint8), empty1.contiguous().to(torch.uint8)
    out = torch.empty(1, B, Hs, Ws, 3, dtype=torch.uint8 if uint8 else torch.float32, device=i0.device)
    ts = (ctypes.c_float * 1)(t)
    with torch.cuda.device(out.device):
        capi.check(capi.lib.rb_frame_synthesize_pairs_resized(
            capi.ptr(i0), capi.ptr(i1), int(i0.dtype == torch.uint8), Hs, Ws, capi.ptr(f0), capi.ptr(f1), capi.ptr(e0),
            capi.ptr(e1), H, W, ts, 1, capi.ptr(out), int(uint8), int(bgr), B, capi.stream()))
    return out[0]


def resize_frames(frames, size, pad=(0, 0, 0, 0)):
    """The reference's cv2.resize of frames to size = (Ho, Wo) (test_dataflow.py:85-87), bit for bit, on [B,H,W,3]
    CUDA frames: uint8 (then divided by 255 like test_dataflow.py:96-97) or fp32 -> [B,Ho,Wo,3] fp32, replicate-padded
    by pad = (top, bottom, left, right) (rb_frames_resize)."""
    assert frames.dim() == 4 and frames.shape[-1] == 3 and frames.dtype in (torch.uint8, torch.float32), frames.shape
    frames = frames.contiguous()
    B, H, W, _ = frames.shape
    Ho, Wo = int(size[0]), int(size[1])
    t, b, l, r = (int(p) for p in pad)
    out = torch.empty(B, Ho + t + b, Wo + l + r, 3, dtype=torch.float32, device=frames.device)
    with torch.cuda.device(frames.device):
        capi.check(capi.lib.rb_frames_resize(capi.ptr(frames), int(frames.dtype == torch.uint8), capi.ptr(out), B, H, W,
                                             Ho, Wo, t, b, l, r, capi.stream()))
    return out


def resize_flow(flow, size):
    """The reference's flow_utils.resize_flow (flow_utils.py:277-284) on [B,H,W,2] fp32 CUDA flows: both channels
    resized to size = (Ho, Wo) like cv2.resize, u scaled by Wo / W and v by Ho / H -> [B,Ho,Wo,2] (rb_flow_resize)."""
    assert flow.dim() == 4 and flow.shape[-1] == 2 and flow.dtype == torch.float32, (flow.shape, flow.dtype)
    flow = flow.contiguous()
    B, H, W, _ = flow.shape
    Ho, Wo = int(size[0]), int(size[1])
    out = torch.empty(B, Ho, Wo, 2, dtype=torch.float32, device=flow.device)
    with torch.cuda.device(flow.device):
        capi.check(capi.lib.rb_flow_resize(capi.ptr(flow), capi.ptr(out), B, H, W, Ho, Wo, capi.stream()))
    return out


MOTION_SUMS = 8  # RB_MOTION_SUMS


def global_motion(flow_fw, occ_fw, frame_hw, flow_scale=1.0, rounds=None, cauchy_c=None, min_weight=None,
                  return_sums=False):
    """Extension (video stabilization): the camera motion of B frame pairs, a similarity M = [[a, -b, tx], [b, a, ty]]
    from frame k to frame k + 1 fitted robustly to each pair's flow on the GPU (rb_global_motion).  flow_fw [B,Hn,Wn,2]
    fp32 CUDA flows on the network grid (forward_sequence_bidirectional's) and occ_fw [B,Hn,Wn] uint8 their
    forward-backward masks (only pixels with 0 count); frame_hw = (Hs, Ws), the frames' own size, in whose pixels,
    centred on the frame centre, the similarity is expressed.  flow_scale as in fb_consistency.  A plain least-squares
    round, then `rounds` Cauchy reweighting rounds of scale cauchy_c network pixels, all on the device (defaults:
    raft_b200.stabilize's MOTION_ROUNDS, MOTION_CAUCHY, MOTION_MIN_WEIGHT, chosen on synthetic flows only).  Returns
    fresh (params [B,4] fp64 (a, b, tx, ty), weight [B] fp64, the fraction of consistent pixels, reliable [B] bool);
    an unreliable pair (weight below min_weight, or a singular fit) has the identity.  With return_sums also the [B,8]
    fp64 weighted sums of the last round (MOTION_SUMS in rb_global_motion's order).  Wrong shapes or dtypes raise
    ValueError."""
    from raft_b200.stabilize import MOTION_CAUCHY, MOTION_MIN_WEIGHT, MOTION_ROUNDS
    if not (isinstance(flow_fw, torch.Tensor) and flow_fw.is_cuda and flow_fw.dim() == 4 and flow_fw.shape[-1] == 2
            and flow_fw.dtype == torch.float32):
        raise ValueError(f"global_motion: flow_fw must be a [B,Hn,Wn,2] float32 CUDA tensor (got "
                         f"{getattr(flow_fw, 'shape', None)} {getattr(flow_fw, 'dtype', type(flow_fw))})")
    B, Hn, Wn, _ = flow_fw.shape
    dev = flow_fw.device
    if not (isinstance(occ_fw, torch.Tensor) and tuple(occ_fw.shape) == (B, Hn, Wn) and occ_fw.dtype == torch.uint8
            and occ_fw.device == dev):
        raise ValueError(f"global_motion: occ_fw must be a [B,Hn,Wn] = {[B, Hn, Wn]} uint8 tensor on {dev}")
    try:
        Hs, Ws = (int(v) for v in frame_hw)
    except (TypeError, ValueError):
        raise ValueError(f"global_motion: frame_hw must be (Hs, Ws) (got {frame_hw!r})") from None
    if Hs < 1 or Ws < 1:
        raise ValueError(f"global_motion: frame_hw must be positive (got {frame_hw!r})")
    rounds = MOTION_ROUNDS if rounds is None else int(rounds)
    cauchy_c = MOTION_CAUCHY if cauchy_c is None else float(cauchy_c)
    min_weight = MOTION_MIN_WEIGHT if min_weight is None else float(min_weight)
    f, o = flow_fw.contiguous(), occ_fw.contiguous()
    params = torch.empty(B, 4, dtype=torch.float64, device=dev)
    weight = torch.empty(B, dtype=torch.float64, device=dev)
    flags = torch.empty(B, dtype=torch.uint8, device=dev)
    sums = torch.empty(B, MOTION_SUMS, dtype=torch.float64, device=dev) if return_sums else None
    with torch.cuda.device(dev):
        nbytes = capi.size_query(capi.lib.rb_global_motion_workspace_bytes, B, Hn, Wn)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        capi.check(capi.lib.rb_global_motion(capi.ptr(f), capi.ptr(o), B, Hn, Wn, Hs, Ws, float(flow_scale), rounds,
                                             cauchy_c, min_weight, capi.ptr(params), capi.ptr(weight), capi.ptr(flags),
                                             capi.ptr(sums), capi.ptr(ws), nbytes, capi.stream()))
    out = (params, weight, flags == 0)
    return out + (sums,) if return_sums else out


def homography_motion(flow_fw, occ_fw, frame_hw, params, reliable, flow_scale=1.0, rounds=None, cauchy_c=None,
                      return_sums=False):
    """Extension (motion segmentation): the camera homography of B fields fitted robustly to their flows on the GPU
    (rb_homography_motion, include/raft_b200.h F34), started from global_motion's similarities.  flow_fw [B,Hn,Wn,2]
    fp32 CUDA fields (forward or backward), occ_fw [B,Hn,Wn] uint8 their forward-backward masks, frame_hw = (Hs, Ws);
    params [B,4] fp64 and reliable [B] bool are global_motion's.  `rounds` iteratively reweighted DLT rounds with Cauchy
    scale cauchy_c network pixels (defaults: raft_b200.motionseg's ROUNDS, CAUCHY).  Returns fresh (H [B,3,3] fp64 in
    the normalised centred coordinates of F34, flags [B] uint8: 0 fitted, 1 singular (the similarity kept), 2 the
    similarity was unreliable (the identity)); with return_sums also the last round's [B,45] fp64 sums.  Wrong shapes or
    dtypes raise ValueError."""
    from raft_b200.motionseg import CAUCHY, ROUNDS, SUMS
    if not (isinstance(flow_fw, torch.Tensor) and flow_fw.is_cuda and flow_fw.dim() == 4 and flow_fw.shape[-1] == 2
            and flow_fw.dtype == torch.float32):
        raise ValueError(f"homography_motion: flow_fw must be a [B,Hn,Wn,2] float32 CUDA tensor (got "
                         f"{getattr(flow_fw, 'shape', None)} {getattr(flow_fw, 'dtype', type(flow_fw))})")
    B, Hn, Wn, _ = flow_fw.shape
    dev = flow_fw.device
    if not (isinstance(occ_fw, torch.Tensor) and tuple(occ_fw.shape) == (B, Hn, Wn) and occ_fw.dtype == torch.uint8
            and occ_fw.device == dev):
        raise ValueError(f"homography_motion: occ_fw must be a [B,Hn,Wn] = {[B, Hn, Wn]} uint8 tensor on {dev}")
    if not (isinstance(params, torch.Tensor) and tuple(params.shape) == (B, 4) and params.dtype == torch.float64
            and params.device == dev and isinstance(reliable, torch.Tensor) and tuple(reliable.shape) == (B,)
            and reliable.dtype == torch.bool and reliable.device == dev):
        raise ValueError(f"homography_motion: params and reliable must be global_motion's [B,4] float64 and [B] bool "
                         f"tensors on {dev}")
    try:
        Hs, Ws = (int(v) for v in frame_hw)
    except (TypeError, ValueError):
        raise ValueError(f"homography_motion: frame_hw must be (Hs, Ws) (got {frame_hw!r})") from None
    if Hs < 1 or Ws < 1:
        raise ValueError(f"homography_motion: frame_hw must be positive (got {frame_hw!r})")
    rounds = ROUNDS if rounds is None else int(rounds)
    cauchy_c = CAUCHY if cauchy_c is None else float(cauchy_c)
    f, o, p = flow_fw.contiguous(), occ_fw.contiguous(), params.contiguous()
    sim_flags = (~reliable).to(torch.uint8)
    H = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
    flags = torch.empty(B, dtype=torch.uint8, device=dev)
    sums = torch.empty(B, SUMS, dtype=torch.float64, device=dev) if return_sums else None
    with torch.cuda.device(dev):
        nbytes = capi.size_query(capi.lib.rb_homography_motion_workspace_bytes, B, Hn, Wn)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        capi.check(capi.lib.rb_homography_motion(capi.ptr(f), capi.ptr(o), B, Hn, Wn, Hs, Ws, float(flow_scale),
                                                 capi.ptr(p), capi.ptr(sim_flags), rounds, cauchy_c, capi.ptr(H),
                                                 capi.ptr(flags), capi.ptr(sums), capi.ptr(ws), nbytes, capi.stream()))
    return (H, flags, sums) if return_sums else (H, flags)


def motion_evidence(flow_fw, flow_bw, occ_fw, occ_bw, H, flags, frame_hw, cuts=None, flow_scale=1.0, tau=None):
    """Extension (motion segmentation): the per-frame evidence of motion that departs from the camera's
    (rb_motion_evidence, F35).  flow_fw, flow_bw [T,Hn,Wn,2] float32 consecutive flows and occ_fw, occ_bw [T,Hn,Wn] uint8
    their masks; H [2T,3,3] fp64 and flags [2T] uint8 homography_motion's fit of the 2T fields cat(flow_fw, flow_bw);
    frame_hw = (Hs, Ws); cuts None or a [T] uint8 CUDA tensor, non-zero for a scene-cut pair; tau in network pixels
    (default raft_b200.motionseg.TAU).  Returns a fresh [T+1,Hn,Wn,2] float32 tensor of (N, C): the sum of
    r^2 / (r^2 + tau^2) over the frame's usable fields and their count.  Bad arguments raise ValueError."""
    from raft_b200.motionseg import TAU, check_tau
    T, Hn, Wn = _flow_pair("motion_evidence", flow_fw, flow_bw)
    dev = flow_fw.device
    for name, t in (("occ_fw", occ_fw), ("occ_bw", occ_bw)):
        if not (isinstance(t, torch.Tensor) and tuple(t.shape) == (T, Hn, Wn) and t.dtype == torch.uint8
                and t.device == dev):
            raise ValueError(f"motion_evidence: {name} must be a [T,Hn,Wn] = {[T, Hn, Wn]} uint8 tensor on {dev}")
    if not (isinstance(H, torch.Tensor) and tuple(H.shape) == (2 * T, 3, 3) and H.dtype == torch.float64
            and H.device == dev and isinstance(flags, torch.Tensor) and tuple(flags.shape) == (2 * T,)
            and flags.dtype == torch.uint8 and flags.device == dev):
        raise ValueError(f"motion_evidence: H and flags must be [2T,3,3] = {[2 * T, 3, 3]} float64 and [2T] uint8 "
                         f"tensors on {dev}")
    if cuts is not None and not (isinstance(cuts, torch.Tensor) and tuple(cuts.shape) == (T,)
                                 and cuts.dtype == torch.uint8 and cuts.device == dev):
        raise ValueError(f"motion_evidence: cuts must be None or a [T] = [{T}] uint8 tensor on {dev}")
    try:
        Hs, Ws = (int(v) for v in frame_hw)
    except (TypeError, ValueError):
        raise ValueError(f"motion_evidence: frame_hw must be (Hs, Ws) (got {frame_hw!r})") from None
    tau = check_tau(TAU if tau is None else tau, "motion_evidence")
    fw, bw, of, ob = flow_fw.contiguous(), flow_bw.contiguous(), occ_fw.contiguous(), occ_bw.contiguous()
    h, fl, c = H.contiguous(), flags.contiguous(), None if cuts is None else cuts.contiguous()
    ev = torch.empty(T + 1, Hn, Wn, 2, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_motion_evidence(capi.ptr(fw), capi.ptr(bw), capi.ptr(of), capi.ptr(ob), capi.ptr(h),
                                               capi.ptr(fl), capi.ptr(c), T, Hn, Wn, Hs, Ws, float(flow_scale),
                                               float(tau), capi.ptr(ev), capi.stream()))
    return ev


def motion_segment(evidence, flow_fw, flow_bw, frame_hw, rows, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """Extension (motion segmentation): the binary moving-object masks of F frames at their own size frame_hw = (Hs, Ws)
    (rb_motion_segment, F35).  evidence [F,Hn,Wn,2] float32 (motion_evidence's); flow_fw, flow_bw [F-1,Hn,Wn,2] float32
    consecutive flows; rows [n,3] integer table (t, nf, nb) (raft_b200.motionseg.segment_rows).  Each pixel adds the
    evidence of its own frame and of every frame its chain reaches through the forward-backward test of fb_consistency.
    Returns fresh (mask [n,Hs,Ws] uint8 0 / 1, status [n,Hs,Ws] uint8: 1 where no evidence reached the pixel).  Bad
    shapes or a bad table raise ValueError."""
    if not (isinstance(evidence, torch.Tensor) and evidence.is_cuda and evidence.dim() == 4 and evidence.shape[-1] == 2
            and evidence.dtype == torch.float32):
        raise ValueError(f"motion_segment: evidence must be an [F,Hn,Wn,2] float32 CUDA tensor (got "
                         f"{getattr(evidence, 'shape', None)} {getattr(evidence, 'dtype', type(evidence))})")
    F, Hn, Wn, _ = evidence.shape
    dev = evidence.device
    T, fh, fwd = _flow_pair("motion_segment", flow_fw, flow_bw)
    if (T, fh, fwd) != (F - 1, Hn, Wn) or flow_fw.device != dev:
        raise ValueError(f"motion_segment: {F} evidence maps need [F-1,Hn,Wn,2] = [{F - 1},{Hn},{Wn},2] flows on {dev} "
                         f"(got {tuple(flow_fw.shape)})")
    try:
        Hs, Ws = (int(v) for v in frame_hw)
    except (TypeError, ValueError):
        raise ValueError(f"motion_segment: frame_hw must be (Hs, Ws) (got {frame_hw!r})") from None
    if Hs < 1 or Ws < 1:
        raise ValueError(f"motion_segment: frame_hw must be positive (got {frame_hw!r})")
    table = _rows_table("motion_segment", rows, F, dev)
    n = table.shape[0]
    ev, fw, bw = evidence.contiguous(), flow_fw.contiguous(), flow_bw.contiguous()
    mask = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=dev)
    status = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_motion_segment(capi.ptr(ev), F, Hn, Wn, capi.ptr(fw), capi.ptr(bw), Hs, Ws,
                                              float(flow_scale), float(alpha1), float(alpha2), capi.ptr(table), n,
                                              capi.ptr(mask), capi.ptr(status), capi.stream()))
    return mask, status


def warp_frames(frames, A):
    """Extension (video stabilization): every frame of [F,H,W,C] uint8 CUDA frames (C in 1..4, any channel order) warped
    by its [2,3] matrix of A [F,2,3] (fp64, host or device), which maps an output pixel (x, y) to its source position in
    the frame's own pixels (rb_frames_warp_affine): the position in fp64, rounded once to fp32, clamped into the frame
    (the border replicates), sampled bilinearly and rounded to bytes.  The identity returns the frames byte for byte.
    Returns a fresh [F,H,W,C] uint8 tensor.  Wrong shapes or dtypes raise ValueError."""
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dim() == 4 and frames.dtype == torch.uint8
            and 1 <= frames.shape[-1] <= 4):
        raise ValueError(f"warp_frames: frames must be an [F,H,W,C] uint8 CUDA tensor with C in 1..4 (got "
                         f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
    F, H, W, C = frames.shape
    m = torch.as_tensor(A)
    if not (tuple(m.shape) == (F, 2, 3) and m.is_floating_point()):
        raise ValueError(f"warp_frames: A must be an [F,2,3] = {[F, 2, 3]} float array (got {list(m.shape)} {m.dtype})")
    m = m.to(device=frames.device, dtype=torch.float64).contiguous()
    f = frames.contiguous()
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        capi.check(capi.lib.rb_frames_warp_affine(capi.ptr(f), capi.ptr(m), F, H, W, C, capi.ptr(out), capi.stream()))
    return out


def masked_fill(values, hole):
    """Extension (object removal): the membrane (Laplace) fill of [B,H,W,C] float32 CUDA fields (C = 2 flows or 3
    colours) inside the holes of [B,H,W] uint8 (or bool) masks, non-zero = unknown (rb_masked_fill: a coarse-to-fine
    initial guess and multigrid V-cycles of red-black Gauss-Seidel, include/raft_b200.h F24).  The known pixels keep
    their bits, every filled value lies within the field's known [min, max] per channel, and a field's bits depend
    neither on B nor on its place in the batch.  Returns fresh (filled [B,H,W,C] float32, empty [B] bool): empty marks a
    field without a known pixel, filled with zeros.  Wrong shapes or dtypes raise ValueError."""
    if not (isinstance(values, torch.Tensor) and values.is_cuda and values.dim() == 4 and values.shape[-1] in (2, 3)
            and values.dtype == torch.float32):
        raise ValueError(f"masked_fill: values must be a [B,H,W,C] float32 CUDA tensor with C in (2, 3) (got "
                         f"{getattr(values, 'shape', None)} {getattr(values, 'dtype', type(values))})")
    B, H, W, C = values.shape
    if not (isinstance(hole, torch.Tensor) and tuple(hole.shape) == (B, H, W) and hole.dtype in (torch.uint8, torch.bool)
            and hole.device == values.device):
        raise ValueError(f"masked_fill: hole must be a [B,H,W] = {[B, H, W]} uint8 or bool tensor on {values.device}")
    dev = values.device
    out = values.clone(memory_format=torch.contiguous_format)
    h = hole.contiguous().view(torch.uint8)
    flags = torch.empty(B, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        nbytes = capi.size_query(capi.lib.rb_masked_fill_workspace_bytes, B, H, W, C)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        capi.check(capi.lib.rb_masked_fill(capi.ptr(out), capi.ptr(h), B, H, W, C, capi.ptr(flags), capi.ptr(ws), nbytes,
                                           capi.stream()))
    return out, flags != 0


def inpaint_masks(masks, net_hw, dilate=2, labels=None):
    """Extension (object removal): the holes of [F,Hs,Ws] uint8 CUDA label maps (rb_inpaint_masks).  A pixel is removed
    when its value is non-zero, or with labels when it is one of them; the removed pixels are dilated by the
    (2 dilate + 1)^2 square.  Returns fresh (hole [F,Hs,Ws] uint8 0 / 1, hole_net [F,Hn,Wn] uint8): hole_net[i, j] is 1
    when any frame pixel whose centre maps into network pixel (i, j) of net_hw = (Hn, Wn) is a hole (the pixel holding
    its centre when none maps into it).  Bad arguments raise ValueError."""
    from raft_b200.inpaint import check_dilate, selection_table
    if not (isinstance(masks, torch.Tensor) and masks.is_cuda and masks.dim() == 3 and masks.dtype == torch.uint8):
        raise ValueError(f"inpaint_masks: masks must be an [F,Hs,Ws] uint8 CUDA tensor (got "
                         f"{getattr(masks, 'shape', None)} {getattr(masks, 'dtype', type(masks))})")
    dilate = check_dilate(dilate, "inpaint_masks")
    try:
        Hn, Wn = (int(v) for v in net_hw)
    except (TypeError, ValueError):
        raise ValueError(f"inpaint_masks: net_hw must be (Hn, Wn) (got {net_hw!r})") from None
    if Hn < 1 or Wn < 1:
        raise ValueError(f"inpaint_masks: net_hw must be positive (got {net_hw!r})")
    dev = masks.device
    m = masks.contiguous()
    F, Hs, Ws = m.shape
    select = torch.from_numpy(selection_table(labels, "inpaint_masks")).to(dev)
    hole = torch.empty(F, Hs, Ws, dtype=torch.uint8, device=dev)
    hole_net = torch.empty(F, Hn, Wn, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_inpaint_masks(capi.ptr(m), capi.ptr(select), F, Hs, Ws, dilate, Hn, Wn, capi.ptr(hole),
                                             capi.ptr(hole_net), capi.stream()))
    return hole, hole_net


def inpaint_propagate(frames, hole, flow_fw, flow_bw, rows, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """Extension (object removal): the temporal fill of the holes of F frames from the nearest frames that see behind
    them (rb_inpaint_propagate).  frames [F,Hs,Ws,3] uint8 and hole [F,Hs,Ws] uint8 CUDA tensors (inpaint_masks' hole);
    flow_fw, flow_bw [F-1,Hn,Wn,2] float32 consecutive flows completed inside the holes (masked_fill); rows [n,3] integer
    table (t, nf, nb) (raft_b200.inpaint.inpaint_rows): the frame of each output row and how many steps each side may
    chain.  Each side follows the flows with the forward-backward test of fb_consistency at every step and stops at the
    first frame where the four taps of its position are all visible; two sides blend weighted toward the nearer frame.
    Returns fresh (colour [n,Hs,Ws,3] float32, status [n,Hs,Ws] uint8): status 0 not a hole (the frame's bytes), 1
    filled from both sides, 2 from one, 3 from none (colour 0).  Bad shapes or a bad table raise ValueError."""
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dim() == 4 and frames.shape[-1] == 3
            and frames.dtype == torch.uint8):
        raise ValueError(f"inpaint_propagate: frames must be an [F,Hs,Ws,3] uint8 CUDA tensor (got "
                         f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
    F, Hs, Ws, _ = frames.shape
    dev = frames.device
    if not (isinstance(hole, torch.Tensor) and tuple(hole.shape) == (F, Hs, Ws) and hole.dtype == torch.uint8
            and hole.device == dev):
        raise ValueError(f"inpaint_propagate: hole must be an [F,Hs,Ws] = {[F, Hs, Ws]} uint8 tensor on {dev}")
    T, Hn, Wn = _flow_pair("inpaint_propagate", flow_fw, flow_bw)
    if T != F - 1 or flow_fw.device != dev:
        raise ValueError(f"inpaint_propagate: {F} frames need [F-1,Hn,Wn,2] = [{F - 1},Hn,Wn,2] flows on {dev} (got "
                         f"{tuple(flow_fw.shape)})")
    table = _rows_table("inpaint_propagate", rows, F, dev)
    n = table.shape[0]
    f, h, fw, bw = frames.contiguous(), hole.contiguous(), flow_fw.contiguous(), flow_bw.contiguous()
    colour = torch.empty(n, Hs, Ws, 3, dtype=torch.float32, device=dev)
    status = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_inpaint_propagate(capi.ptr(f), capi.ptr(h), F, Hs, Ws, capi.ptr(fw), capi.ptr(bw), Hn, Wn,
                                                 float(flow_scale), float(alpha1), float(alpha2), capi.ptr(table), n,
                                                 capi.ptr(colour), capi.ptr(status), capi.stream()))
    return colour, status


def _rows_table(what, rows, F, dev):
    """An [n,3] integer (t, nf, nb) table checked against F frames, as int32 on dev."""
    table = torch.as_tensor(rows).cpu()
    if not (table.dim() == 2 and table.shape[0] >= 1 and table.shape[1] == 3 and not table.is_floating_point()
            and not table.is_complex()):
        raise ValueError(f"{what}: rows must be an [n,3] integer table (got {list(table.shape)} {table.dtype})")
    t, nf, nb = table.to(torch.int64).unbind(1)
    if not (((t >= 0) & (t < F) & (nf >= 0) & (t + nf <= F - 1) & (nb >= 0) & (nb <= t)).all()):
        raise ValueError(f"{what}: each row (t, nf, nb) needs t in [0, {F}), 0 <= nf <= F-1-t and 0 <= nb <= t")
    return table.to(device=dev, dtype=torch.int32).contiguous()


def denoise_merge(frames, flow_fw, flow_bw, rows, sigma, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """Extension (video denoising): each pixel of F frames merged with its patch matches along the chained flows
    (rb_denoise_merge).  frames [F,Hs,Ws,3] uint8 CUDA tensor; flow_fw, flow_bw [F-1,Hn,Wn,2] float32 consecutive flows;
    rows [n,3] integer table (t, nf, nb) (raft_b200.inpaint.inpaint_rows): the frame of each output row and how many
    steps each side may chain (at most raft_b200.denoise.MAX_WINDOW count); sigma > 0 the noise's standard deviation in
    grey levels.  Each side follows the flows with the forward-backward test of fb_consistency at every step and stops
    at the first step that fails; every frame reached is a match.  Returns fresh (frames [n,Hs,Ws,3] uint8, support
    [n,Hs,Ws] uint8: the matched frames of both sides).  Bad shapes, a bad table or a bad sigma raise ValueError."""
    import math
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dim() == 4 and frames.shape[-1] == 3
            and frames.dtype == torch.uint8):
        raise ValueError(f"denoise_merge: frames must be an [F,Hs,Ws,3] uint8 CUDA tensor (got "
                         f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
    F, Hs, Ws, _ = frames.shape
    dev = frames.device
    T, Hn, Wn = _flow_pair("denoise_merge", flow_fw, flow_bw)
    if T != F - 1 or flow_fw.device != dev:
        raise ValueError(f"denoise_merge: {F} frames need [F-1,Hn,Wn,2] = [{F - 1},Hn,Wn,2] flows on {dev} (got "
                         f"{tuple(flow_fw.shape)})")
    try:
        sigma = float(sigma)
    except (TypeError, ValueError):
        sigma = float("nan")
    if not (math.isfinite(sigma) and sigma > 0):
        raise ValueError("denoise_merge: sigma must be a finite number > 0")
    table = _rows_table("denoise_merge", rows, F, dev)
    n = table.shape[0]
    f, fw, bw = frames.contiguous(), flow_fw.contiguous(), flow_bw.contiguous()
    out = torch.empty(n, Hs, Ws, 3, dtype=torch.uint8, device=dev)
    support = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_denoise_merge(capi.ptr(f), F, Hs, Ws, capi.ptr(fw), capi.ptr(bw), Hn, Wn,
                                             float(flow_scale), float(alpha1), float(alpha2), capi.ptr(table), n,
                                             sigma, capi.ptr(out), capi.ptr(support), capi.stream()))
    return out, support


def noise_sums(frames):
    """Extension (video denoising): rb_noise_sums of [N,H,W,3] uint8 CUDA frames (H, W >= 3) -- the [N,3] int64 sums of
    |I * M| over the interior pixels per frame and channel, M Immerkaer's mask [[1,-2,1],[-2,4,-2],[1,-2,1]]."""
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dim() == 4 and frames.shape[-1] == 3
            and frames.dtype == torch.uint8 and frames.shape[0] >= 1 and min(frames.shape[1:3]) >= 3):
        raise ValueError(f"noise_sums: frames must be an [N,H,W,3] uint8 CUDA tensor with N >= 1 and H, W >= 3 (got "
                         f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
    N, H, W, _ = frames.shape
    f = frames.contiguous()
    sums = torch.empty(N, 3, dtype=torch.int64, device=f.device)
    with torch.cuda.device(f.device):
        capi.check(capi.lib.rb_noise_sums(capi.ptr(f), N, H, W, capi.ptr(sums), capi.stream()))
    return sums


def noise_sigma(frames):
    """Extension (video denoising): Immerkaer's estimate ("Fast noise variance estimation", CVIU 1996) of the
    standard deviation of additive white noise in [N,H,W,3] uint8 CUDA frames, in grey levels: sqrt(pi/2) S /
    (6 (H-2)(W-2)) per frame and channel from noise_sums, averaged over both.  Exactly 0 on frames that are locally
    linear (flat frames, ramps)."""
    from raft_b200.denoise import sigma_from_sums
    sums = noise_sums(frames)
    return sigma_from_sums(sums.cpu().numpy(), frames.shape[1], frames.shape[2])


def _margin(what, margin):
    try:
        my, mx = (int(v) for v in margin)
    except (TypeError, ValueError):
        raise ValueError(f"{what}: margin must be (my, mx) (got {margin!r})") from None
    if my < 0 or mx < 0:
        raise ValueError(f"{what}: margin must be >= 0 (got {margin!r})")
    return my, mx


def _hw(what, name, hw):
    try:
        h, w = (int(v) for v in hw)
    except (TypeError, ValueError):
        raise ValueError(f"{what}: {name} must be (H, W) (got {hw!r})") from None
    if h < 1 or w < 1:
        raise ValueError(f"{what}: {name} must be positive (got {hw!r})")
    return h, w


def extend_flows(flow_fw, flow_bw, motions, frame_hw, margin, flow_scale=1.0):
    """Extension (full-frame stabilization): the consecutive flows [T,Hn,Wn,2] float32 CUDA tensors extended by margin =
    (my, mx) network pixels per side onto the canvas [T,Hn+2my,Wn+2mx,2] (include/raft_b200.h F26).  motions [T,4] fp64
    (host or device): each pair's similarity (a, b, tx, ty) in the centred pixels of frame_hw = (Hs, Ws), as
    raft_b200.stabilize.camera_transforms takes them (the identity at cuts and unreliable pairs); the backward flow uses
    its inverse, computed here in fp64.  The residual after the global motion is filled over the band by rb_masked_fill,
    all 2T canvases in one batch, and the global motion added back; inside the grid the flows keep their bits.  Returns
    fresh (ext_fw, ext_bw).  Wrong shapes or dtypes raise ValueError."""
    import numpy as np
    from raft_b200.stabilize import motion_matrix
    T, Hn, Wn = _flow_pair("extend_flows", flow_fw, flow_bw)
    Hs, Ws = _hw("extend_flows", "frame_hw", frame_hw)
    my, mx = _margin("extend_flows", margin)
    m = torch.as_tensor(motions).cpu().to(torch.float64).numpy()
    if m.shape != (T, 4):
        raise ValueError(f"extend_flows: motions must be [T,4] = [{T},4] (got {list(m.shape)})")
    inv = np.linalg.inv(motion_matrix(m))
    both = np.concatenate([m, np.stack([inv[:, 0, 0], inv[:, 1, 0], inv[:, 0, 2], inv[:, 1, 2]], 1)])
    dev = flow_fw.device
    flows = torch.cat([flow_fw, flow_bw]).contiguous()
    mot = torch.from_numpy(both).to(dev)
    Hc, Wc = Hn + 2 * my, Wn + 2 * mx
    resid = torch.empty(2 * T, Hc, Wc, 2, dtype=torch.float32, device=dev)
    hole = torch.empty(2 * T, Hc, Wc, dtype=torch.uint8, device=dev)
    args = (capi.ptr(flows), capi.ptr(mot), 2 * T, Hn, Wn, Hs, Ws, my, mx, float(flow_scale))
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_flow_extend_residual(*args, capi.ptr(resid), capi.ptr(hole), capi.stream()))
        if my or mx:  # without a band there is nothing to fill, and the fill would leave every known value as it is
            resid, _ = masked_fill(resid, hole)
        capi.check(capi.lib.rb_flow_extend_finish(*args, capi.ptr(resid), capi.ptr(resid), capi.stream()))
    return resid[:T], resid[T:]


def warp_frames_fill(frames, ext_fw, ext_bw, net_hw, margin, A, rows, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """Extension (full-frame stabilization): rb_frames_warp_affine_fill (include/raft_b200.h F26).  frames [F,Hs,Ws,3]
    uint8 CUDA; ext_fw, ext_bw [F-1,Hc,Wc,2] float32 (extend_flows' canvases of the net_hw = (Hn, Wn) grid with margin
    (my, mx)); A [n,2,3] float (host or device), row r's warp as warp_frames takes it; rows [n,3] integer table (t, nf,
    nb) (raft_b200.inpaint.inpaint_rows).  A pixel whose source lies in frame t gets warp_frames' value before rounding
    (status 0); any other follows the extended flows up to nf frames forward and nb back, with the forward-backward test
    of fb_consistency at every step, to the first frame that holds it: status 1 both sides (blended toward the nearer
    frame), 2 one side, 3 none (colour 0).  Returns fresh (colour [n,Hs,Ws,3] float32, status [n,Hs,Ws] uint8).  Bad
    shapes or a bad table raise ValueError."""
    if not (isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dim() == 4 and frames.shape[-1] == 3
            and frames.dtype == torch.uint8):
        raise ValueError(f"warp_frames_fill: frames must be an [F,Hs,Ws,3] uint8 CUDA tensor (got "
                         f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
    F, Hs, Ws, _ = frames.shape
    dev = frames.device
    Hn, Wn = _hw("warp_frames_fill", "net_hw", net_hw)
    my, mx = _margin("warp_frames_fill", margin)
    T, Hc, Wc = _flow_pair("warp_frames_fill", ext_fw, ext_bw)
    if T != F - 1 or (Hc, Wc) != (Hn + 2 * my, Wn + 2 * mx) or ext_fw.device != dev:
        raise ValueError(f"warp_frames_fill: {F} frames need [F-1,Hn+2my,Wn+2mx,2] = [{F - 1},{Hn + 2 * my},"
                         f"{Wn + 2 * mx},2] flows on {dev} (got {tuple(ext_fw.shape)})")
    table = torch.as_tensor(rows).cpu()
    if not (table.dim() == 2 and table.shape[0] >= 1 and table.shape[1] == 3 and not table.is_floating_point()
            and not table.is_complex()):
        raise ValueError(f"warp_frames_fill: rows must be an [n,3] integer table (got {list(table.shape)} {table.dtype})")
    t, nf, nb = table.to(torch.int64).unbind(1)
    if not (((t >= 0) & (t < F) & (nf >= 0) & (t + nf <= F - 1) & (nb >= 0) & (nb <= t)).all()):
        raise ValueError(f"warp_frames_fill: each row (t, nf, nb) needs t in [0, {F}), 0 <= nf <= F-1-t and 0 <= nb <= t")
    n = table.shape[0]
    m = torch.as_tensor(A)
    if not (tuple(m.shape) == (n, 2, 3) and m.is_floating_point()):
        raise ValueError(f"warp_frames_fill: A must be an [n,2,3] = {[n, 2, 3]} float array (got {list(m.shape)} "
                         f"{m.dtype})")
    m = m.to(device=dev, dtype=torch.float64).contiguous()
    table = table.to(device=dev, dtype=torch.int32).contiguous()
    f, fw, bw = frames.contiguous(), ext_fw.contiguous(), ext_bw.contiguous()
    colour = torch.empty(n, Hs, Ws, 3, dtype=torch.float32, device=dev)
    status = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_frames_warp_affine_fill(capi.ptr(f), F, Hs, Ws, capi.ptr(fw), capi.ptr(bw), Hn, Wn, my, mx,
                                                       float(flow_scale), float(alpha1), float(alpha2), capi.ptr(m),
                                                       capi.ptr(table), n, capi.ptr(colour), capi.ptr(status),
                                                       capi.stream()))
    return colour, status


def _frame_u8(what, name, x, shape=None, dev=None):
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dim() == 3 and x.shape[-1] == 3 and x.dtype == torch.uint8
            and (shape is None or tuple(x.shape) == tuple(shape)) and (dev is None or x.device == dev)):
        raise ValueError(f"{what}: {name} must be an [Hs,Ws,3] uint8 CUDA tensor"
                         + ("" if shape is None else f" of shape {list(shape)} on {dev}") + f" (got "
                         f"{getattr(x, 'shape', None)} {getattr(x, 'dtype', type(x))})")
    return x.contiguous()


def tcons_terms(frame, prev_frame, processed, prev_out, flow_fw, flow_bw, strength, flow_scale=1.0, alpha1=0.01,
                alpha2=0.5):
    """Extension (temporal consistency): frame t's temporal term (rb_tcons_terms).  frame, prev_frame (the originals
    I_t, I_(t-1)), processed (P_t) and prev_out (O_(t-1)): [Hs,Ws,3] uint8 CUDA tensors; flow_fw, flow_bw [Hn,Wn,2]
    float32 the pair (t-1, t); strength > 0.  Each pixel takes one backward step through the flows with the
    forward-backward test of fb_consistency, and the originals' colour difference at its target weighs the pull toward
    the previous output (Tukey's biweight, cut-off raft_b200.temporal.KAPPA).  prev_frame None: no previous frame
    (prev_out and the flows are ignored).  Returns fresh (c [Hs,Ws] float32, r [Hs,Ws,3] float32, status [Hs,Ws]
    uint8: 0 used, 1 step failed, 2 rejected by the colour check, 3 no previous frame).  Bad arguments raise
    ValueError."""
    from raft_b200.temporal import check_strength
    P = _frame_u8("tcons_terms", "processed", processed)
    dev, (Hs, Ws) = P.device, P.shape[:2]
    strength = check_strength(strength, "tcons_terms")
    c = torch.empty(Hs, Ws, dtype=torch.float32, device=dev)
    r = torch.empty(Hs, Ws, 3, dtype=torch.float32, device=dev)
    status = torch.empty(Hs, Ws, dtype=torch.uint8, device=dev)
    if prev_frame is None:
        ptrs, Hn, Wn = (None, None, P, None, None, None), 1, 1
    else:
        I = _frame_u8("tcons_terms", "frame", frame, P.shape, dev)
        Ip = _frame_u8("tcons_terms", "prev_frame", prev_frame, P.shape, dev)
        Op = _frame_u8("tcons_terms", "prev_out", prev_out, P.shape, dev)
        if not all(isinstance(f, torch.Tensor) and f.dim() == 3 for f in (flow_fw, flow_bw)):
            raise ValueError("tcons_terms: flow_fw and flow_bw must be [Hn,Wn,2] float32 CUDA tensors")
        _, Hn, Wn = _flow_pair("tcons_terms", flow_fw[None], flow_bw[None])
        if flow_fw.device != dev:
            raise ValueError(f"tcons_terms: the flows must be on {dev}")
        ptrs = (I, Ip, P, Op, flow_fw.contiguous(), flow_bw.contiguous())
    with torch.cuda.device(dev):
        capi.check(capi.lib.rb_tcons_terms(*(None if t is None else capi.ptr(t) for t in ptrs[:4]), Hs, Ws,
                                           *(None if t is None else capi.ptr(t) for t in ptrs[4:]), Hn, Wn,
                                           float(flow_scale), float(alpha1), float(alpha2), strength, capi.ptr(c),
                                           capi.ptr(r), capi.ptr(status), capi.stream()))
    return c, r, status


def screened_poisson(c, r, workspace=None):
    """Extension (temporal consistency): the correction D [H,W,3] float32 that solves (c_p + n_p) D_p - sum of the
    in-image 4-neighbours' D = r_p per channel (rb_screened_poisson: flexible conjugate gradients preconditioned by a
    multigrid V-cycle of red-black Gauss-Seidel, include/raft_b200.h F30).  c [H,W] float32 > 0 and r [H,W,3] float32
    CUDA tensors; workspace an optional uint8 CUDA buffer of at least rb_screened_poisson_workspace_bytes.  r = 0 gives
    D = 0 bit for bit.  Bad shapes or dtypes raise ValueError."""
    if not (isinstance(c, torch.Tensor) and c.is_cuda and c.dim() == 2 and c.dtype == torch.float32):
        raise ValueError(f"screened_poisson: c must be an [H,W] float32 CUDA tensor (got {getattr(c, 'shape', None)} "
                         f"{getattr(c, 'dtype', type(c))})")
    H, W = c.shape
    if not (isinstance(r, torch.Tensor) and tuple(r.shape) == (H, W, 3) and r.dtype == torch.float32
            and r.device == c.device):
        raise ValueError(f"screened_poisson: r must be an [H,W,3] = {[H, W, 3]} float32 tensor on {c.device}")
    dev = c.device
    cc, rr = c.contiguous(), r.contiguous()
    D = torch.empty(H, W, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        nbytes = capi.size_query(capi.lib.rb_screened_poisson_workspace_bytes, H, W)
        if workspace is None or workspace.numel() < nbytes or workspace.device != dev:
            workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        capi.check(capi.lib.rb_screened_poisson(capi.ptr(cc), capi.ptr(rr), H, W, capi.ptr(D), capi.ptr(workspace),
                                                workspace.numel(), capi.stream()))
    return D


def warp_error(video, flow_fw, flow_bw, flow_scale=1.0, alpha1=0.01, alpha2=0.5):
    """Extension (temporal consistency): Lai et al.'s warping-error sums (rb_warp_error) of [F,Hs,Ws,3] uint8 CUDA
    frames V aligned with the frames that flow_fw, flow_bw [F-1,Hn,Wn,2] float32 were computed on: per pair k, the sum
    over the pixels of frame k whose forward step passes the forward-backward test of sum_c (V_k(p) - V_(k+1)(o))^2 in
    grey levels, and their count.  Returns a fresh [F-1,2] float64 CUDA tensor (raft_b200.temporal.pair_errors forms
    E_warp).  Bad shapes raise ValueError."""
    if not (isinstance(video, torch.Tensor) and video.is_cuda and video.dim() == 4 and video.shape[-1] == 3
            and video.dtype == torch.uint8 and video.shape[0] >= 2):
        raise ValueError(f"warp_error: video must be an [F,Hs,Ws,3] uint8 CUDA tensor with F >= 2 (got "
                         f"{getattr(video, 'shape', None)} {getattr(video, 'dtype', type(video))})")
    F, Hs, Ws, _ = video.shape
    dev = video.device
    T, Hn, Wn = _flow_pair("warp_error", flow_fw, flow_bw)
    if T != F - 1 or flow_fw.device != dev:
        raise ValueError(f"warp_error: {F} frames need [F-1,Hn,Wn,2] = [{F - 1},Hn,Wn,2] flows on {dev} (got "
                         f"{tuple(flow_fw.shape)})")
    v, fw, bw = video.contiguous(), flow_fw.contiguous(), flow_bw.contiguous()
    sums = torch.empty(F - 1, 2, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        nbytes = capi.size_query(capi.lib.rb_warp_error_workspace_bytes, F, Hs, Ws)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        capi.check(capi.lib.rb_warp_error(capi.ptr(v), F, Hs, Ws, capi.ptr(fw), capi.ptr(bw), Hn, Wn, float(flow_scale),
                                          float(alpha1), float(alpha2), capi.ptr(sums), capi.ptr(ws), nbytes,
                                          capi.stream()))
    return sums
