"""F17: TAP-Vid point-tracking evaluation (Doersch et al. 2022) of the chained-flow tracker (RaftEngine.track's kernels).

    from raft_b200.evaluate import evaluate
    res = evaluate(RAFT(None, args).load("raft-things.npz"), "tapvid_davis.pkl", "tapvid", query_mode="strided")

Data: a .pkl file, or a directory of *.pkl shards (Kinetics) read in sorted order.  Each pickle holds a dict name ->
entry (DAVIS) or a list of entries (RGB-Stacking, Kinetics; entry i of shard <stem>.pkl is named <stem>/<i>).  An entry
has `video` ([F,H,W,3] uint8 RGB, or a sequence of encoded images that cv2.imdecode reads), `points` ([N,F,2] (x, y)
normalised to [0, 1]: (0, 0) is the top-left corner of the top-left pixel, (1, 1) the bottom-right corner of the
bottom-right pixel) and `occluded` ([N,F] bool).  pickle.load runs code the file names: that is the dataset's own format,
so read only files from a source you trust.

Protocol: frames run at TAP-Vid's 256 x 256 (the engine's cv2-exact GPU resize), 20 iterations.  Ground truth in pixels
is points * 256 - 0.5, the tracker's pixel-centre convention; a query starts at its ground truth clamped into
[0, 255]^2.  Query modes: 'first' -- one query per track at its first visible frame (tracks never visible are dropped);
'strided' -- a query for every track visible at frame t, for t = 0, 5, 10, ... < F, ordered by t, then by track.  Each
query is scored against its track's whole row.  A video's flows come from interp_schedule(F, batch) passes of
forward_sequence_bidirectional(check=False), kept on the GPU ([F-1,256,256,2] per direction, 0.5 MB per pair and
direction); then one rb_track_points launch tracks every query to the last frame and, in 'strided' mode, one
rb_track_points_backward launch to frame 0.  A point is predicted occluded where its status is not 0.  Every kernel is
batch-invariant, so the predictions are the same bits for every batch.

Metrics (TAP-Vid's definitions).  E = the evaluated (query, frame) entries: the frames after the query frame ('first') or
every frame but the query frame ('strided').  V = visible in the ground truth, P = predicted visible, and w_d = |pred -
gt|^2 < d^2 (NaN counts as false), d in {1, 2, 4, 8, 16} pixels at 256 x 256.  Sums run over E:

    occlusion accuracy  OA  = sum[(not P) == (not V)] / |E|
    points within d     δ_d = sum(w_d and V) / sum(V)
    Jaccard at d        J_d = sum(w_d and V and P) / (sum(V) + sum(P and (not V or not w_d)))

average_jaccard (AJ) is the mean of J_d over d and average_pts_within_thresh (δ_avg) the mean of δ_d.  Each metric is
computed per video in fp64 from integer counts, then averaged over the videos; a video whose denominator is zero has
NaN there and stays out of that mean (n_scored counts the videos in each mean).
"""
from __future__ import annotations

import glob
import os
import pickle
from collections import namedtuple

import numpy as np
import torch

from .evaluate import QUERY_MODES

SIZE = (256, 256)  # TAP-Vid's evaluation resolution
THRESHOLDS = (1, 2, 4, 8, 16)  # pixels at SIZE
STRIDE = 5  # the query frames of 'strided' mode
SUMMARY = ("average_jaccard", "average_pts_within_thresh", "occlusion_accuracy")

Video = namedtuple("Video", "name frames points occluded")


# ---- reading ---------------------------------------------------------------------------------------------------------
def tapvid_files(path):
    """The pickles of `path`: the file itself, or a directory's *.pkl in sorted order.  Nothing there raises
    FileNotFoundError."""
    path = os.fspath(path)
    if os.path.isdir(path):
        files = sorted(glob.glob(os.path.join(path, "*.pkl")))
        if not files:
            raise FileNotFoundError(f"TAP-Vid: no *.pkl shards in {path}")
        return files
    if not os.path.isfile(path):
        raise FileNotFoundError(f"TAP-Vid: no file or directory {path}")
    return [path]


def _frames(name, video):
    """[F,H,W,3] uint8 RGB from an entry's video: the array itself, or each encoded image decoded (BGR -> RGB)."""
    import cv2
    if isinstance(video, np.ndarray) and video.dtype != object:
        if video.dtype != np.uint8 or video.ndim != 4 or video.shape[-1] != 3:
            raise ValueError(f"TAP-Vid: video {name}: frames must be [F,H,W,3] uint8 (got {video.shape} {video.dtype})")
        return video
    try:
        frames = []
        for i, b in enumerate(video):
            img = cv2.imdecode(np.frombuffer(bytes(b), dtype=np.uint8), cv2.IMREAD_COLOR)
            if img is None:
                raise ValueError(f"TAP-Vid: video {name}: frame {i} is not an image cv2 can decode")
            if frames and img.shape != frames[0].shape:
                raise ValueError(f"TAP-Vid: video {name}: frame {i} is {img.shape[:2]}, frame 0 {frames[0].shape[:2]}")
            frames.append(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    except TypeError:
        raise ValueError(f"TAP-Vid: video {name}: `video` must be a [F,H,W,3] uint8 array or a sequence of encoded "
                         f"images (got {type(video).__name__})") from None
    if not frames:
        raise ValueError(f"TAP-Vid: video {name} has no frames")
    return np.stack(frames)


def check_entry(name, entry):
    """One entry as a Video(name, frames [F,H,W,3] uint8 RGB, points [N,F,2] fp64, occluded [N,F] bool); a missing
    field, a wrong shape, F < 2 or a frame-count mismatch raises ValueError naming the video."""
    if not isinstance(entry, dict) or any(k not in entry for k in ("video", "points", "occluded")):
        raise ValueError(f"TAP-Vid: video {name}: an entry is a dict with `video`, `points` and `occluded`")
    frames = _frames(name, entry["video"])
    points = np.asarray(entry["points"], dtype=np.float64)
    occluded = np.asarray(entry["occluded"])
    F = len(frames)
    if F < 2:
        raise ValueError(f"TAP-Vid: video {name} has {F} frame; tracking needs two at least")
    if points.ndim != 3 or points.shape[2] != 2:
        raise ValueError(f"TAP-Vid: video {name}: points must be [N,F,2] (got {points.shape})")
    if occluded.shape != points.shape[:2]:
        raise ValueError(f"TAP-Vid: video {name}: occluded must be [N,F] = {list(points.shape[:2])} (got "
                         f"{list(occluded.shape)})")
    if points.shape[1] != F:
        raise ValueError(f"TAP-Vid: video {name}: points cover {points.shape[1]} frames, the video has {F}")
    return Video(name, frames, points, occluded.astype(bool))


def read_tapvid(path):
    """The videos of tapvid_files(path), one at a time (a shard is loaded when its first video is due), each checked by
    check_entry.  A pickle that holds neither a dict nor a list raises ValueError."""
    for f in tapvid_files(path):
        with open(f, "rb") as fh:
            data = pickle.load(fh)  # runs code from the file: TAP-Vid's own format, read trusted files only
        if isinstance(data, dict):
            items = list(data.items())
        elif isinstance(data, (list, tuple)):
            stem = os.path.splitext(os.path.basename(f))[0]
            items = [(f"{stem}/{i}", e) for i, e in enumerate(data)]
        else:
            raise ValueError(f"TAP-Vid: {f} holds a {type(data).__name__}; expected a dict name -> entry or a list of "
                             "entries")
        for name, entry in items:
            yield check_entry(str(name), entry)


# ---- queries and ground truth ----------------------------------------------------------------------------------------
def to_pixels(points, size=SIZE):
    """Normalised (x, y) -> pixels of an H x W = size frame in the tracker's pixel-centre convention, in fp64: x W - 0.5,
    y H - 0.5."""
    return np.asarray(points, dtype=np.float64) * np.array([size[1], size[0]], dtype=np.float64) - 0.5


def sample_queries(occluded, mode):
    """The queries of one video's [N,F] occlusion mask -> (track [Q], frame [Q]) int64.  'first': each track with a
    visible frame, at its first one, in track order.  'strided': every track visible at t, for t = 0, STRIDE, 2 STRIDE,
    ... < F, ordered by t, then by track."""
    occluded = np.asarray(occluded, dtype=bool)
    visible = ~occluded
    if mode == "first":
        track = np.flatnonzero(visible.any(axis=1))
        return track, visible[track].argmax(axis=1).astype(np.int64)
    if mode == "strided":
        ts = np.arange(0, occluded.shape[1], STRIDE)
        t, track = np.nonzero(visible[:, ts].T)
        return track.astype(np.int64), ts[t].astype(np.int64)
    raise ValueError(f"TAP-Vid: query_mode must be one of {QUERY_MODES} (got {mode!r})")


def query_inputs(points, track, frame, size=SIZE):
    """The kernel inputs of the queries (track, frame): (qframe [Q] int32, qpos [Q,2] fp32), qpos the ground truth in
    pixels (to_pixels) clamped into [0, W - 1] x [0, H - 1] and rounded once to fp32."""
    gt = to_pixels(points, size)[track, frame]
    hi = np.array([size[1] - 1, size[0] - 1], dtype=np.float64)
    return frame.astype(np.int32), np.clip(gt, 0.0, hi).astype(np.float32)


# ---- metrics --------------------------------------------------------------------------------------------------------
def video_counts(pred, pred_occluded, gt, gt_occluded, qframe, mode):
    """The integer counts of one video's Q queries over F frames: pred [Q,F,2] (any float; NaN allowed), pred_occluded
    [Q,F] bool, gt [Q,F,2] pixels and gt_occluded [Q,F] bool of each query's track, qframe [Q].  Returns {"evaluated":
    |E|, "occlusion_correct", "visible": sum(V), and per d "within_<d>": sum(w_d and V), "true_pos_<d>", "false_pos_<d>"}
    as Python ints."""
    Q, F = np.shape(gt_occluded)
    t = np.arange(F)[None, :]
    q = np.asarray(qframe, dtype=np.int64)[:, None]
    E = (t > q) if mode == "first" else (t != q)
    V, P = ~np.asarray(gt_occluded, bool), ~np.asarray(pred_occluded, bool)
    d2 = np.sum((np.asarray(pred, np.float64) - np.asarray(gt, np.float64)) ** 2, axis=-1)
    c = {"evaluated": int(E.sum()), "occlusion_correct": int((E & (P == V)).sum()), "visible": int((E & V).sum())}
    for d in THRESHOLDS:
        with np.errstate(invalid="ignore"):
            w = d2 < d * d  # NaN -> False
        c[f"within_{d}"] = int((E & w & V).sum())
        c[f"true_pos_{d}"] = int((E & w & V & P).sum())
        c[f"false_pos_{d}"] = int((E & P & (~V | ~w)).sum())
    return c


def _ratio(a, b):
    return float(a) / float(b) if b else float("nan")


def video_metrics(c):
    """The metrics of one video's counts (video_counts) in fp64: occlusion_accuracy, pts_within_<d>, jaccard_<d>,
    average_pts_within_thresh, average_jaccard; NaN where the denominator is zero."""
    m = {"occlusion_accuracy": _ratio(c["occlusion_correct"], c["evaluated"])}
    for d in THRESHOLDS:
        m[f"pts_within_{d}"] = _ratio(c[f"within_{d}"], c["visible"])
        m[f"jaccard_{d}"] = _ratio(c[f"true_pos_{d}"], c["visible"] + c[f"false_pos_{d}"])
    m["average_pts_within_thresh"] = sum(m[f"pts_within_{d}"] for d in THRESHOLDS) / len(THRESHOLDS)
    m["average_jaccard"] = sum(m[f"jaccard_{d}"] for d in THRESHOLDS) / len(THRESHOLDS)
    return m


def aggregate_tapvid(records):
    """The split's means over the per-video records (each with name, n_frames, n_queries and video_metrics' keys): every
    metric averaged over the videos where it is not NaN (NaN when there is none), n_videos, and n_scored = the number of
    videos in each mean."""
    keys = list(SUMMARY) + [f"jaccard_{d}" for d in THRESHOLDS] + [f"pts_within_{d}" for d in THRESHOLDS]
    res, scored = {}, {}
    for k in keys:
        v = np.array([r[k] for r in records], dtype=np.float64)
        ok = ~np.isnan(v)
        res[k] = float(v[ok].mean()) if ok.any() else float("nan")
        scored[k] = int(ok.sum())
    res["n_videos"] = len(records)
    res["n_scored"] = {k: scored[k] for k in SUMMARY}
    res["videos"] = list(records)
    return res


# ---- prediction ------------------------------------------------------------------------------------------------------
def predict_video(engine, frames, qframe, qpos, batch=1, backward=False):
    """The tracker's predictions for one video: frames [F,H,W,3] uint8 in the engine's channel order (numpy or a torch
    tensor), qframe [Q] int32 and qpos [Q,2] fp32 on the engine's network grid.  interp_schedule(F, batch) passes of
    forward_sequence_bidirectional(check=False) fill a device store of the F - 1 flows per direction; then one
    rb_track_points launch over the whole clip and, with backward, one rb_track_points_backward launch on the same
    buffers.  Returns (tracks [F,Q,2] fp32, status [F,Q] uint8) CUDA tensors on the network grid; the same bits for
    every batch."""
    from networks.utils import track_points, track_points_backward
    from .engine import FB_ALPHA1, FB_ALPHA2
    from .video import interp_schedule
    F = len(frames)
    dev = engine.device
    kw = dict(flow_scale=engine.flow_scale, alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)
    with torch.cuda.device(dev):
        clip = torch.as_tensor(np.ascontiguousarray(frames) if isinstance(frames, np.ndarray) else frames).to(dev)
        store = None
        for ps in interp_schedule(F, batch):
            fw, bw, _, _ = engine.forward_sequence_bidirectional(clip[ps.frames], check=False)
            if store is None:
                store = [torch.empty((F - 1,) + tuple(fw.shape[1:]), dtype=torch.float32, device=dev) for _ in range(2)]
            live = [k for k in ps.pairs if k is not None]
            store[0][live[0]:live[-1] + 1].copy_(fw[:len(live)])
            store[1][live[0]:live[-1] + 1].copy_(bw[:len(live)])
        qframe = torch.as_tensor(qframe).to(dev)
        qpos = torch.as_tensor(qpos).to(dev)
        tracks, status, _ = track_points(store[0], store[1], qframe, qpos, **kw)
        if backward:
            track_points_backward(store[0], store[1], qframe, qpos, tracks, status, **kw)
    return tracks, status


def run(engine, path, query_mode="first", batch=1, rgb=False):
    """Every video of read_tapvid(path) through predict_video (frames in RGB with rgb, else BGR) and scored: returns the
    per-video records, in file order, each {name, n_frames, n_queries, **video_metrics}."""
    if query_mode not in QUERY_MODES:
        raise ValueError(f"TAP-Vid: query_mode must be one of {QUERY_MODES} (got {query_mode!r})")
    records = []
    for v in read_tapvid(path):
        track, frame = sample_queries(v.occluded, query_mode)
        F = len(v.frames)
        gt = to_pixels(v.points)[track]
        gt_occ = v.occluded[track]
        if len(track):
            qframe, qpos = query_inputs(v.points, track, frame)
            frames = v.frames if rgb else v.frames[..., ::-1]
            tracks, status = predict_video(engine, frames, qframe, qpos, batch, backward=query_mode == "strided")
            pred = tracks.cpu().numpy().transpose(1, 0, 2)
            pred_occ = status.cpu().numpy().T != 0
        else:
            pred, pred_occ = np.zeros((0, F, 2)), np.zeros((0, F), bool)
        c = video_counts(pred, pred_occ, gt, gt_occ, frame, query_mode)
        records.append({"name": v.name, "n_frames": F, "n_queries": int(len(track)), **video_metrics(c)})
    return records
