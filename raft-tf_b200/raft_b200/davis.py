"""F20: DAVIS-2017 semi-supervised validation of keyframe label propagation (RaftEngine.propagate's kernels).

    from raft_b200.evaluate import evaluate
    res = evaluate(RAFT(None, args).load("raft-things.npz"), "datasets/DAVIS", "davis", masks_out="out/davis_val")

Data: the sequences of <root>/ImageSets/2017/val.txt, frames <root>/JPEGImages/480p/<seq>/*.jpg and annotations
<root>/Annotations/480p/<seq>/*.png (palette PNGs) in sorted order.  Every file, and one annotation per frame with the same
stem, is checked up front.

Protocol: frame 0's annotation is propagated forward through the sequence at the frames' own size, 20 iterations,
'sintel' padding (PROTOCOLS["davis"]).  With keyframe_step N (F21) the annotations of frames 0, N, 2N, ... < F are the
keyframes, each frame votes between the nearest two (RaftEngine.propagate with a list of keys), and the keyframes are
dropped from the scored frames.  The flows come from interp_schedule(F, batch) passes of
forward_sequence_bidirectional(check=False); each pass continues the accumulation from the last row of the one before
(rb_flow_accumulate) and labels its rows (rb_labels_propagate), so the predictions are the same bits for every batch.
The void label 255 of an annotation is background.  With masks_out the predictions of every frame are written in DAVIS's
results layout, <masks_out>/<seq>/<stem>.png in the palette of the sequence's first annotation, for a cross-check with the
official evaluator.

Metrics.  This restates davis2017-evaluation (metrics.py: db_eval_iou, f_measure and _seg2bmap; utils.db_statistics;
evaluation.py: the semi-supervised path) from its published definitions; the public evaluator could not be consulted
while this was written, so a reader who has it should diff these formulas against it.

  objects   o = 1..N, N = the largest label of frame 0's annotation (255 -> 0 first); a ground-truth label that matches
            no object counts as background for every object; no void handling (the semi-supervised path passes none).
  frames    1..F-2 are scored (the evaluator drops the first and the last frame).
  J         |P and G| / |P or G| per frame and object (P = pred == o, G = gt == o), 1 when the union is empty.
  F         boundaries by _seg2bmap: b = (m ^ e) | (m ^ s) | (m ^ se) with e, s, se the right, down and down-right
            neighbours (0 outside the image), the last row m ^ e, the last column m ^ s, the last pixel 0; a boundary
            pixel of P matches when a boundary pixel of G lies within the disk dx^2 + dy^2 <= r^2 (cv2.dilate with
            skimage.morphology.disk(r), pixels outside the image never match), and vice versa;
            r = bound_pix = ceil(0.008 * hypot(H, W)).  precision = matched P / |b(P)|, recall = matched G / |b(G)|,
            with (|b(P)|, |b(G)|) = (0, >0) -> (1, 0), (>0, 0) -> (0, 1), (0, 0) -> (1, 1);
            F = 2 P R / (P + R), 0 when P + R = 0.
  per object, over its per-frame values v (L frames):  M = nanmean(v), O (recall) = nanmean(v > 0.5),
            ids = uint8(round(linspace(1, L, 5) + 1e-10) - 1), bins v[ids[i]:ids[i+1]+1] for i = 0..3,
            D (decay) = nanmean(bin 0) - nanmean(bin 3).
  global    J-Mean, J-Recall, J-Decay, F-Mean, F-Recall, F-Decay = the means over every object of every sequence;
            J&F-Mean = (J-Mean + F-Mean) / 2.

The counts are rb_label_metrics' integers (exact, on the GPU); the ratios and statistics are fp64 on the host.
"""
from __future__ import annotations

import os
import warnings
from collections import namedtuple

import numpy as np
import torch

SUMMARY = ("J&F-Mean", "J-Mean", "J-Recall", "J-Decay", "F-Mean", "F-Recall", "F-Decay")

Sequence = namedtuple("Sequence", "name frames annotations")


# ---- reading ---------------------------------------------------------------------------------------------------------
def davis_sequences(root, split="val"):
    """The sequences of <root>/ImageSets/2017/<split>.txt, each Sequence(name, frame paths, annotation paths) in sorted
    order.  A missing list, directory or annotation, an extra annotation, or a sequence of fewer than two frames raises
    (FileNotFoundError / ValueError) naming it."""
    root = os.fspath(root)
    lst = os.path.join(root, "ImageSets", "2017", f"{split}.txt")
    if not os.path.isfile(lst):
        raise FileNotFoundError(f"DAVIS: no sequence list {lst}")
    with open(lst) as f:
        names = [line.strip() for line in f if line.strip()]
    if not names:
        raise ValueError(f"DAVIS: {lst} lists no sequence")
    seqs = []
    for name in names:
        fdir = os.path.join(root, "JPEGImages", "480p", name)
        adir = os.path.join(root, "Annotations", "480p", name)
        for d in (fdir, adir):
            if not os.path.isdir(d):
                raise FileNotFoundError(f"DAVIS: sequence {name}: no directory {d}")
        frames = sorted(f for f in os.listdir(fdir) if f.endswith(".jpg"))
        annos = sorted(f for f in os.listdir(adir) if f.endswith(".png"))
        if len(frames) < 2:
            raise ValueError(f"DAVIS: sequence {name} has {len(frames)} frames; propagation needs two at least")
        if len(frames) != len(annos):
            raise ValueError(f"DAVIS: sequence {name} has {len(frames)} frames and {len(annos)} annotations")
        for fr, an in zip(frames, annos):
            if os.path.splitext(fr)[0] != os.path.splitext(an)[0]:
                raise ValueError(f"DAVIS: sequence {name}: frame {fr} has no annotation {os.path.splitext(fr)[0]}.png")
        seqs.append(Sequence(name, [os.path.join(fdir, f) for f in frames], [os.path.join(adir, f) for f in annos]))
    return seqs


# ---- metrics --------------------------------------------------------------------------------------------------------
def frame_scores(counts):
    """Per-frame J and F of rb_label_metrics' [n, n_objects, 6] counts -> (J, F), each [n_objects, n] fp64."""
    c = np.asarray(counts, dtype=np.int64)
    inter, union, n_fg, n_gt, fg_match, gt_match = (c[..., k].astype(np.float64) for k in range(6))
    with np.errstate(invalid="ignore", divide="ignore"):
        J = np.where(union == 0, 1.0, inter / union)
        precision = np.where(n_fg == 0, 1.0, fg_match / n_fg)
        recall = np.where(n_gt == 0, 1.0, gt_match / n_gt)
        precision = np.where((n_fg > 0) & (n_gt == 0), 0.0, precision)
        recall = np.where((n_fg == 0) & (n_gt > 0), 0.0, recall)
        s = precision + recall
        F = np.where(s == 0, 0.0, 2 * precision * recall / np.where(s == 0, 1.0, s))
    return J.T, F.T


def db_statistics(v):
    """(M, O, D) of one object's per-frame values, as davis2017-evaluation's utils.db_statistics computes them."""
    v = np.asarray(v, dtype=np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=RuntimeWarning)
        M = np.nanmean(v)
        O = np.nanmean(v > 0.5)
        ids = (np.round(np.linspace(1, len(v), 5) + 1e-10) - 1).astype(np.uint8)
        bins = [v[ids[i]:ids[i + 1] + 1] for i in range(4)]
        D = np.nanmean(bins[0]) - np.nanmean(bins[3])
    return float(M), float(O), float(D)


def aggregate_davis(records):
    """The split's globals over the per-sequence records (each with `objects`, a list of per-object {J-Mean, J-Recall,
    J-Decay, F-Mean, F-Recall, F-Decay}): every statistic's mean over all objects, J&F-Mean, n_sequences, n_objects and the
    records."""
    objs = [o for r in records for o in r["objects"]]
    res = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=RuntimeWarning)
        for k in SUMMARY[1:]:
            res[k] = float(np.mean([o[k] for o in objs])) if objs else float("nan")
    res = {"J&F-Mean": (res["J-Mean"] + res["F-Mean"]) / 2, **res}
    res["n_sequences"] = len(records)
    res["n_objects"] = len(objs)
    res["sequences"] = list(records)
    return res


# ---- prediction ------------------------------------------------------------------------------------------------------
def propagate_clip(engine, frames, key, batch=1, frame=0):
    """The [Hs,Ws] uint8 labels `key` of frame `frame` (or the [m,Hs,Ws] keys of the strictly increasing frames `frame`)
    propagated through frames [F,Hs,Ws,3] uint8 (the engine's channel order, numpy or torch) in interp_schedule(F, batch)
    passes, the accumulation carried from pass to pass on the GPU (raft_b200.video.KeyframeSweep).  Returns (labels
    [F,Hs,Ws] uint8, status [F,Hs,Ws] uint8) CUDA tensors: RaftEngine.propagate(frames, key, frame)'s bits for every
    batch."""
    from .video import KeyframeSweep, check_keyframes, interp_schedule
    F = len(frames)
    K = check_keyframes(frame, F, "DAVIS")
    dev = engine.device
    with torch.cuda.device(dev):
        clip = torch.as_tensor(np.ascontiguousarray(frames) if isinstance(frames, np.ndarray) else frames).to(dev)
        keys = torch.as_tensor(np.ascontiguousarray(key) if isinstance(key, np.ndarray) else key).to(dev)
        keys = keys[None] if keys.dim() == 2 else keys
        labels = torch.empty(F, *keys.shape[1:], dtype=torch.uint8, device=dev)
        status = torch.empty_like(labels)
        sweep = KeyframeSweep(engine, keys, K, F, batch, [], simple=isinstance(frame, (int, np.integer)))
        passes = interp_schedule(F, batch)
        j0 = sweep.first_pass(len(passes))
        for part, step in ((passes[j0:], sweep.forward), (passes[:j0][::-1], sweep.reverse)):
            for ps in part:
                fw, bw, _, _ = engine.forward_sequence_bidirectional(clip[ps.frames], check=False)
                for a, lab, st in step(ps, fw, bw):
                    labels[a:a + len(lab)], status[a:a + len(lab)] = lab, st
    return labels, status


def keyframe_frames(F, step):
    """The keyframes of a clip of F frames annotated every `step` frames: 0, step, 2 step, ... < F."""
    return list(range(0, int(F), int(step)))


def scored_frames(F, keyframes=(0,)):
    """The frames DAVIS scores: 1 .. F - 2 (the evaluator drops the first and the last), minus the keyframes."""
    keys = set(keyframes)
    return [t for t in range(1, F - 1) if t not in keys]


def run(engine, seqs, batch=1, rgb=False, masks_out=None, keyframe_step=None):
    """Every sequence of davis_sequences() through propagate_clip (frames in RGB with rgb, else BGR) and scored by
    rb_label_metrics: returns the per-sequence records, in list order, each {name, n_frames, n_objects, objects: [...]}.
    keyframe_step N propagates the annotations of frames 0, N, 2N, ... < F as keyframes (each frame votes between the
    nearest two) and scores frames 1 .. F-2 minus those keyframes, in order; the objects stay frame 0's (labels above
    them in later keys are propagated, not scored), so numbers compare across steps."""
    from networks.utils import davis_bound_pix, label_metrics
    from .evaluate import _imread
    from .video import read_labels, write_labels
    records = []
    for seq in seqs:
        frames = np.stack([_imread(p, rgb) for p in seq.frames])
        annos = []
        for p in seq.annotations:
            lab, pal = read_labels(p)
            annos.append(lab)
            if len(annos) == 1:
                palette = pal
        gt = np.stack(annos)
        if gt.shape[1:] != frames.shape[1:3]:
            raise ValueError(f"DAVIS: sequence {seq.name}: annotations of {gt.shape[1]}x{gt.shape[2]}, frames of "
                             f"{frames.shape[1]}x{frames.shape[2]}")
        gt[gt == 255] = 0
        n_obj = int(gt[0].max())
        F, H, W = gt.shape
        if keyframe_step is None:
            pred, _ = propagate_clip(engine, frames, gt[0], batch)
            scored = list(range(1, F - 1))
        else:
            K = keyframe_frames(F, keyframe_step)
            pred, _ = propagate_clip(engine, frames, gt[K], batch, frame=K)
            scored = scored_frames(F, K)
        objects = [dict(zip(SUMMARY[1:], (float("nan"),) * 6)) for _ in range(n_obj)]
        if n_obj and scored:
            with torch.cuda.device(engine.device):
                idx = torch.tensor(scored, device=engine.device)
                counts = label_metrics(pred[idx], torch.from_numpy(gt[scored]).to(engine.device), n_obj,
                                       davis_bound_pix(H, W)).cpu().numpy()
            J, Fm = frame_scores(counts)
            for o in range(n_obj):
                jm, jr, jd = db_statistics(J[o])
                fm, fr, fd = db_statistics(Fm[o])
                objects[o] = {"J-Mean": jm, "J-Recall": jr, "J-Decay": jd, "F-Mean": fm, "F-Recall": fr, "F-Decay": fd}
        if masks_out is not None:
            d = os.path.join(os.fspath(masks_out), seq.name)
            os.makedirs(d, exist_ok=True)
            host = pred.cpu().numpy()
            for p, m in zip(seq.annotations, host):
                write_labels(os.path.join(d, os.path.basename(p)), m, palette)
        records.append({"name": seq.name, "n_frames": F, "n_objects": n_obj, "objects": objects})
    return records
