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
def davis_sequences(root, split="val", year="2017"):
    """The sequences of <root>/ImageSets/<year>/<split>.txt, each Sequence(name, frame paths, annotation paths) in sorted
    order (year "2016": DAVIS-2016's list, which ships in the DAVIS-2017 tree).  A missing list, directory or annotation,
    an extra annotation, or a sequence of fewer than two frames raises (FileNotFoundError / ValueError) naming it."""
    root = os.fspath(root)
    lst = os.path.join(root, "ImageSets", year, f"{split}.txt")
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


# ---- video denoising (F27) -------------------------------------------------------------------------------------------
# The video-denoising protocol of DVDnet / FastDVDnet (Tassano et al.) on DAVIS-2017 test-dev, frames only:
#
#     res = evaluate_denoise(RAFT(None, args).load("raft-things.npz"), "datasets/DAVIS", sigma=20)
#
# Noise: additive Gaussian noise of sigma grey levels on every frame of <root>/ImageSets/2017/test-dev.txt's sequences,
# seeded per frame from numpy's PCG64 with (crc32(sequence name), frame index), z drawn as [H,W,3] in RGB order, and the
# noisy frame clip(rint(clean + sigma z), 0, 255) as uint8 -- unlike the published protocol, which feeds unclipped float
# frames, so the numbers are close to published tables but not directly comparable.  The merge uses the true sigma; the
# flow runs at the frames' own size, 20 iterations, 'sintel' padding (PROTOCOLS["davis"]).  Metrics: PSNR and SSIM of the
# uint8 output against the clean frame (rb_frame_metrics), per-frame PSNR averaged within a sequence, then over the
# sequences; the noisy input's alongside.
Clip = namedtuple("Clip", "name frames")


def davis_frames(root, split="test-dev"):
    """The sequences of <root>/ImageSets/2017/<split>.txt, each Clip(name, frame paths) in sorted order -- frames only,
    no annotations.  A missing list or directory, or a sequence of fewer than two frames, raises (FileNotFoundError /
    ValueError) naming it."""
    root = os.fspath(root)
    lst = os.path.join(root, "ImageSets", "2017", f"{split}.txt")
    if not os.path.isfile(lst):
        raise FileNotFoundError(f"DAVIS: no sequence list {lst}")
    with open(lst) as f:
        names = [line.strip() for line in f if line.strip()]
    if not names:
        raise ValueError(f"DAVIS: {lst} lists no sequence")
    clips = []
    for name in names:
        fdir = os.path.join(root, "JPEGImages", "480p", name)
        if not os.path.isdir(fdir):
            raise FileNotFoundError(f"DAVIS: sequence {name}: no directory {fdir}")
        frames = sorted(f for f in os.listdir(fdir) if f.endswith(".jpg"))
        if len(frames) < 2:
            raise ValueError(f"DAVIS: sequence {name} has {len(frames)} frames; denoising needs two at least")
        clips.append(Clip(name, [os.path.join(fdir, f) for f in frames]))
    return clips


def noisy_frame(clean, name, index, sigma):
    """The protocol's noisy copy of frame `index` of sequence `name`: clean [H,W,3] uint8 in RGB order plus sigma z, z
    standard normal [H,W,3] from PCG64 seeded with (crc32(name), index), rounded half to even and clipped to uint8."""
    import zlib
    rng = np.random.Generator(np.random.PCG64([zlib.crc32(name.encode()), int(index)]))
    z = rng.standard_normal(clean.shape)
    return np.clip(np.rint(clean.astype(np.float64) + float(sigma) * z), 0, 255).astype(np.uint8)


def psnr_ssim(stats, H, W):
    """Per-frame (PSNR, SSIM) [n] fp64 of rb_frame_metrics' [n,2] {sse, ssim}: PSNR = 10 log10(255^2 3HW / sse), inf
    when sse = 0."""
    s = np.asarray(stats, np.float64)
    with np.errstate(divide="ignore"):
        psnr = 10.0 * np.log10(255.0 ** 2 * 3 * H * W / s[:, 0])
    return psnr, s[:, 1]


def denoise_clip(engine, frames, sigma, window=None, batch=8):
    """RaftEngine.denoise's bits for frames [F,Hs,Ws,3] uint8 (the engine's channel order, a CUDA tensor) with the flows
    of interp_schedule(F, batch) passes kept on the GPU, so a long sequence needs no single pass over all its pairs.
    Returns (frames [F,Hs,Ws,3] uint8, support [F,Hs,Ws] uint8) CUDA tensors."""
    from .denoise import DEFAULT_WINDOW, check_window, merge_frames
    from .inpaint import inpaint_rows
    from .video import interp_schedule
    F = len(frames)
    window = check_window(DEFAULT_WINDOW if window is None else window, "DAVIS")
    fws, bws = [], []
    for ps in interp_schedule(F, batch):
        fw, bw, _, _ = engine.forward_sequence_bidirectional(frames[ps.frames], check=False)
        n = sum(k is not None for k in ps.pairs)
        fws.append(fw[:n].clone())
        bws.append(bw[:n].clone())
    with torch.cuda.device(engine.device):
        return merge_frames(frames, torch.cat(fws), torch.cat(bws), inpaint_rows(F, window), sigma, engine.flow_scale)


def evaluate_denoise(model, root, sigma, window=None, batch=8, iters=None):
    """Video denoising of a loaded networks.RAFT.RAFT model on a DAVIS-2017 tree's test-dev frames (the protocol above).
    A model with input_size, a sigma that is not a number > 0 ("auto" included: the protocol knows its noise) or a bad
    window raise ValueError before any frame is read.  Returns {"dataset", "split", "sigma", "iters", "pad_mode",
    "window", "PSNR", "SSIM", "noisy_PSNR", "noisy_SSIM", "n_sequences", "sequences": [per-sequence records]}; the same
    for every batch."""
    from networks.utils import frame_metrics
    from .denoise import DEFAULT_WINDOW, check_sigma, check_window
    from .evaluate import PROTOCOLS, _engine, _imread
    if getattr(model, "input_size", None) is not None:
        raise ValueError("evaluate_denoise: frames run at their own size; build the model without input_size")
    if isinstance(sigma, str):
        raise ValueError(f"evaluate_denoise: the protocol adds noise of a known level: sigma must be a number > 0 "
                         f"(got {sigma!r})")
    sigma = check_sigma(sigma, "evaluate_denoise")
    window = check_window(DEFAULT_WINDOW if window is None else window, "evaluate_denoise")
    if int(batch) < 1:
        raise ValueError(f"evaluate_denoise: batch must be >= 1 (got {batch})")
    if model._params is None:
        raise RuntimeError("RAFT.load(<npz>) must be called before evaluate_denoise")
    clips = davis_frames(root)  # every directory checked up front
    n_iters, pad_mode = PROTOCOLS["davis"]
    n_iters = n_iters if iters is None else int(iters)
    engine = _engine(model, n_iters, pad_mode)
    dev = engine.device
    records = []
    for clip in clips:
        clean = np.stack([_imread(p, True) for p in clip.frames])
        noisy = np.stack([noisy_frame(c, clip.name, i, sigma) for i, c in enumerate(clean)])
        if not model.upstream:  # the engine's channel order
            clean, noisy = clean[..., ::-1], noisy[..., ::-1]
        F, H, W, _ = clean.shape
        with torch.cuda.device(dev):
            gt = torch.from_numpy(np.ascontiguousarray(clean)).to(dev)
            inp = torch.from_numpy(np.ascontiguousarray(noisy)).to(dev)
            out, support = denoise_clip(engine, inp, sigma, window, int(batch))
            p_out, s_out = psnr_ssim(frame_metrics(out, gt).cpu().numpy(), H, W)
            p_in, s_in = psnr_ssim(frame_metrics(inp, gt).cpu().numpy(), H, W)
            mean_support = float(support.double().mean().item())
        records.append({"name": clip.name, "n_frames": F, "PSNR": float(p_out.mean()), "SSIM": float(s_out.mean()),
                        "noisy_PSNR": float(p_in.mean()), "noisy_SSIM": float(s_in.mean()), "support": mean_support})
    mean = lambda k: float(np.mean([r[k] for r in records]))  # noqa: E731
    return {"dataset": "davis", "split": "test-dev", "sigma": sigma, "iters": n_iters, "pad_mode": pad_mode,
            "window": window, "PSNR": mean("PSNR"), "SSIM": mean("SSIM"), "noisy_PSNR": mean("noisy_PSNR"),
            "noisy_SSIM": mean("noisy_SSIM"), "n_sequences": len(records), "sequences": records}


def denoise_summary(res):
    """The summary line of evaluate_denoise's result."""
    return (f"Validation DAVIS-2017 denoising (test-dev, sigma {res['sigma']:g}): PSNR: {res['PSNR']:.4f}, SSIM: "
            f"{res['SSIM']:.4f} (noisy: PSNR: {res['noisy_PSNR']:.4f}, SSIM: {res['noisy_SSIM']:.4f})")


# ---- motion segmentation (F34 / F35) ---------------------------------------------------------------------------------
# DAVIS-2016's unsupervised protocol for RaftEngine.segment_motion:
#
#     res = evaluate_motion(RAFT(None, args).load("raft-things.npz"), "datasets/DAVIS")
#
# Data: the sequences of <root>/ImageSets/2016/val.txt (the 20 DAVIS-2016 val sequences, listed in the DAVIS-2017 tree),
# frames JPEGImages/480p, checked up front as davis_sequences does.  The flow runs at the frames' own size, 20
# iterations, 'sintel' padding (PROTOCOLS["davis"]).  Ground truth: the union of the non-zero labels of Annotations/480p,
# the void label 255 counted as background, scored as one object with rb_label_metrics, frame_scores and db_statistics
# on frames 1 .. F-2.
#
# Two caveats before comparing with published tables: the union of the DAVIS-2017 labels stands in for DAVIS-2016's
# binary masks (they are drawn from the same annotations but may differ at object boundaries), and the scored-frame rule
# above is the DAVIS-2017 evaluator's; diff it against the official DAVIS-2016 toolkit first.
def segment_clip(engine, frames, window=None, tau=None, batch=8):
    """RaftEngine.segment_motion's masks for frames [F,Hs,Ws,3] uint8 (the engine's channel order, a CUDA tensor) from
    interp_schedule(F, batch) passes: each pass's 2n fields fitted as one batch and its evidence launched; the frame two
    passes share sums its two halves (each launch starts from +0, so the bits are one launch's).  Returns (masks
    [F,Hs,Ws] uint8, status [F,Hs,Ws] uint8) CUDA tensors, the same for every batch."""
    from networks.utils import motion_evidence
    from .motionseg import DEFAULT_WINDOW, TAU, check_tau, check_window, fit_fields, segment_frames, segment_rows
    from .video import interp_schedule
    F = len(frames)
    window = check_window(DEFAULT_WINDOW if window is None else window, "DAVIS")
    tau = check_tau(TAU if tau is None else tau, "DAVIS")
    hw = tuple(frames.shape[1:3])
    fws, bws, evs = [], [], []
    for ps in interp_schedule(F, batch):
        fw, bw, ofw, obw = engine.forward_sequence_bidirectional(frames[ps.frames], check=True)
        n = sum(k is not None for k in ps.pairs)
        fw, bw, ofw, obw = fw[:n], bw[:n], ofw[:n], obw[:n]
        with torch.cuda.device(engine.device):
            H, flags = fit_fields(torch.cat([fw, bw]), torch.cat([ofw, obw]), hw, engine.flow_scale)
            ev = motion_evidence(fw, bw, ofw, obw, H, flags, hw, None, engine.flow_scale, tau)
        if evs:
            evs[-1][-1].add_(ev[0])
            ev = ev[1:]
        fws.append(fw.clone())
        bws.append(bw.clone())
        evs.append(ev)
    with torch.cuda.device(engine.device):
        return segment_frames(torch.cat(evs), torch.cat(fws), torch.cat(bws), hw, segment_rows(F, window),
                              engine.flow_scale)


def evaluate_motion(model, root, window=None, tau=None, batch=8, iters=None, masks_out=None):
    """Motion segmentation of a loaded networks.RAFT.RAFT model on a DAVIS tree's DAVIS-2016 val sequences (the protocol
    above).  A model with input_size, a bad window or tau raise ValueError before any frame is read.  With masks_out the
    masks of every frame are written in DAVIS's results layout, <masks_out>/<seq>/<stem>.png (labels 0 / 1, palette of
    the sequence's first annotation).  Returns aggregate_davis' dict plus "dataset", "split", "iters", "pad_mode",
    "window" and "tau"; the same for every batch."""
    from networks.utils import davis_bound_pix, label_metrics
    from .evaluate import PROTOCOLS, _engine, _imread
    from .motionseg import DEFAULT_WINDOW, TAU, check_tau, check_window
    from .video import read_labels, write_labels
    if getattr(model, "input_size", None) is not None:
        raise ValueError("evaluate_motion: frames run at their own size; build the model without input_size")
    window = check_window(DEFAULT_WINDOW if window is None else window, "evaluate_motion")
    tau = check_tau(TAU if tau is None else tau, "evaluate_motion")
    if int(batch) < 1:
        raise ValueError(f"evaluate_motion: batch must be >= 1 (got {batch})")
    if model._params is None:
        raise RuntimeError("RAFT.load(<npz>) must be called before evaluate_motion")
    seqs = davis_sequences(root, "val", year="2016")  # every file checked up front
    n_iters, pad_mode = PROTOCOLS["davis"]
    n_iters = n_iters if iters is None else int(iters)
    engine = _engine(model, n_iters, pad_mode)
    dev = engine.device
    records = []
    for seq in seqs:
        frames = np.stack([_imread(p, bool(model.upstream)) for p in seq.frames])
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
        gt = ((gt != 0) & (gt != 255)).astype(np.uint8)
        F, H, W = gt.shape
        scored = list(range(1, F - 1))
        with torch.cuda.device(dev):
            pred, _ = segment_clip(engine, torch.from_numpy(frames).to(dev), window, tau, int(batch))
            obj = dict(zip(SUMMARY[1:], (float("nan"),) * 6))
            if scored:
                idx = torch.tensor(scored, device=dev)
                counts = label_metrics(pred[idx], torch.from_numpy(gt[scored]).to(dev), 1,
                                       davis_bound_pix(H, W)).cpu().numpy()
                J, Fm = frame_scores(counts)
                jm, jr, jd = db_statistics(J[0])
                fm, fr, fd = db_statistics(Fm[0])
                obj = {"J-Mean": jm, "J-Recall": jr, "J-Decay": jd, "F-Mean": fm, "F-Recall": fr, "F-Decay": fd}
            host = pred.cpu().numpy()
        if masks_out is not None:
            d = os.path.join(os.fspath(masks_out), seq.name)
            os.makedirs(d, exist_ok=True)
            for p, m in zip(seq.annotations, host):
                write_labels(os.path.join(d, os.path.basename(p)), m, palette)
        records.append({"name": seq.name, "n_frames": F, "n_objects": 1, "moving": float(host.mean()),
                        "objects": [obj]})
    res = aggregate_davis(records)
    return {"dataset": "davis", "split": "val", "protocol": "DAVIS-2016 unsupervised", "iters": n_iters,
            "pad_mode": pad_mode, "window": window, "tau": tau, **res}


def motion_summary(res):
    """The summary line of evaluate_motion's result."""
    return (f"Validation DAVIS-2016 motion segmentation (val): J&F: {res['J&F-Mean']:.4f}, J: {res['J-Mean']:.4f}, "
            f"F: {res['F-Mean']:.4f}")
