"""F33: the GoPro motion-blur protocol for frame-rate conversion with a shutter (F32).

The GoPro deblurring set (Nah et al., CVPR 2017; layout of GOPRO_Large_all: <root>/<split>/<sequence>/*.png, 240 fps)
made each blurred frame as the mean of consecutive sharp 240 fps frames.  That makes any clip of it ground truth for a
shutter: take every S-th frame as a 240/S fps input, convert it at the same rate with shutter 360 M / S degrees and
density S, and the M samples of input frame c land exactly on the true frames S c - (M - 1)/2 .. S c + (M - 1)/2.
The ground truth is np.rint of the mean of those M uint8 frames; input frames whose window leaves the sequence are not
scored.  PSNR and SSIM come from rb_frame_metrics (networks.utils.frame_metrics), with the sharp input frame's scores
beside them as the no-blur baseline.
"""
from __future__ import annotations

import glob
import os
from fractions import Fraction

import numpy as np

DEFAULT_STRIDE, DEFAULT_BLUR_FRAMES = 8, 7


def check_window(stride, blur_frames):
    """(S, M) as ints: S >= 1, M odd and 1 <= M <= S (the samples of one exposure must not reach the next input frame's
    window).  Anything else raises ValueError."""
    try:
        S, M = int(stride), int(blur_frames)
        ok = S == stride and M == blur_frames and S >= 1 and 1 <= M <= S and M % 2 == 1
    except (TypeError, ValueError, OverflowError):
        ok = False
    if not ok:
        raise ValueError(f"gopro: the stride S must be >= 1 and the blur frames M odd with 1 <= M <= S (got {stride!r}, "
                         f"{blur_frames!r})")
    return S, M


def protocol(stride, blur_frames):
    """The shutter (degrees, a Fraction) and density of the protocol: 360 M / S and S."""
    S, M = check_window(stride, blur_frames)
    return Fraction(360 * M, S), S


def sequences(root, split="test"):
    """[(name, sorted *.png paths)] of <root>/<split>/<sequence>/, sequences in sorted order.  A missing split directory,
    a split without sequences or a sequence without frames raises (FileNotFoundError / ValueError)."""
    d = os.path.join(os.fspath(root), split)
    if not os.path.isdir(d):
        raise FileNotFoundError(f"gopro: no directory {d}")
    names = sorted(n for n in os.listdir(d) if os.path.isdir(os.path.join(d, n)))
    if not names:
        raise ValueError(f"gopro: {d} holds no sequence directories")
    out = []
    for n in names:
        paths = sorted(glob.glob(os.path.join(d, n, "*.png")))
        if not paths:
            raise ValueError(f"gopro: {os.path.join(d, n)} holds no *.png frames")
        out.append((n, paths))
    return out


def scored(n_frames, stride, blur_frames):
    """The input frames c (frame S c of the sequence) whose window S c - (M-1)/2 .. S c + (M-1)/2 lies inside the
    n_frames frames, in order."""
    S, M = check_window(stride, blur_frames)
    h = (M - 1) // 2
    n_in = (n_frames - 1) // S + 1
    return [c for c in range(n_in) if S * c - h >= 0 and S * c + h <= n_frames - 1]


def ground_truth(window):
    """[M,H,W,3] uint8 true frames -> np.rint of their mean (ties to even) as uint8, the average Nah et al. used."""
    return np.rint(np.asarray(window, np.float64).mean(axis=0)).astype(np.uint8)


def evaluate(model, root, split="test", stride=DEFAULT_STRIDE, blur_frames=DEFAULT_BLUR_FRAMES, batch=8):
    """The protocol on every sequence of <root>/<split> with a loaded networks.RAFT.RAFT model running at the frames'
    own size.  Each sequence's inputs run through RaftEngine.expose in interp_schedule()'s passes of batch pairs
    (shutter_schedule() at equal rates; the frames equal model.motion_blur on the whole input clip), and every scored
    frame and its sharp input are scored against the ground truth on the GPU.  Frames go in RGB with model.upstream and
    BGR otherwise, like the CLI; the ground truth is formed in the same channel order.  Returns a dict: dataset,
    split, stride, blur_frames, shutter, density, psnr / ssim (means over all scored frames), sharp_psnr / sharp_ssim,
    frames (the count) and sequences (per-sequence records with the same means)."""
    import torch

    from networks.utils import frame_metrics

    from .evaluate import _imread, psnr
    from .video import exposure, shutter_schedule

    S, M = check_window(stride, blur_frames)
    shutter, density = protocol(S, M)
    _, m = exposure(1, 1, shutter, density)
    seqs = sequences(root, split)
    engine, rgb, dev = model.engine(), bool(model.upstream), model.engine().device
    records, all_stats = [], []
    for name, paths in seqs:
        cs = scored(len(paths), S, M)
        inputs = np.stack([_imread(p, rgb) for p in paths[::S]])
        if len(inputs) < 2 or not cs:
            records.append({"sequence": name, "frames": len(paths), "scored": 0})
            continue
        blurred = {}
        for ps in shutter_schedule(len(inputs), 1, 1, shutter, density, int(batch)):
            if not ps.samples:
                continue
            first = ps.frames[0]
            src = torch.from_numpy(inputs[ps.frames])
            res = engine.expose(src, [(n, i - first, t) for n, i, t in ps.samples], m, ps.opens, ps.closes)
            for r, n in enumerate(ps.closes):
                blurred[n] = res[r]
        h = (M - 1) // 2
        stats = []
        for c in cs:
            gt = torch.from_numpy(ground_truth([_imread(p, rgb) for p in paths[S * c - h:S * c + h + 1]])).to(dev)
            pair = torch.stack([blurred[c], torch.from_numpy(inputs[c]).to(dev)])
            stats.append(frame_metrics(pair, torch.stack([gt, gt])).cpu().numpy())
        st = np.stack(stats)  # [n, 2 (blur | sharp), 2 (sse | ssim)]
        values = inputs[0].size
        p = np.array([[psnr(st[i, k, 0], values) for k in range(2)] for i in range(len(st))])
        records.append({"sequence": name, "frames": len(paths), "scored": len(cs),
                        "psnr": float(p[:, 0].mean()), "ssim": float(st[:, 0, 1].mean()),
                        "sharp_psnr": float(p[:, 1].mean()), "sharp_ssim": float(st[:, 1, 1].mean()),
                        "per_frame": [{"input": c, "frame": S * c, "psnr": float(p[i, 0]), "ssim": float(st[i, 0, 1]),
                                       "sharp_psnr": float(p[i, 1]), "sharp_ssim": float(st[i, 1, 1])}
                                      for i, c in enumerate(cs)]})
        all_stats += [r for r in records[-1]["per_frame"]]
    if not all_stats:
        raise ValueError(f"gopro: no sequence of {os.path.join(os.fspath(root), split)} has a frame whose {M}-frame "
                         f"window fits (stride {S})")
    mean = lambda key: float(np.mean([r[key] for r in all_stats]))  # noqa: E731
    return {"dataset": "gopro", "split": split, "stride": S, "blur_frames": M, "shutter": float(shutter),
            "density": density, "frames": len(all_stats), "psnr": mean("psnr"), "ssim": mean("ssim"),
            "sharp_psnr": mean("sharp_psnr"), "sharp_ssim": mean("sharp_ssim"), "sequences": records}


def summary_line(res):
    return (f"Validation GoPro motion blur ({res['split']}, stride {res['stride']}, {res['blur_frames']} frames): "
            f"PSNR: {res['psnr']:.4f}, SSIM: {res['ssim']:.4f} (sharp: PSNR: {res['sharp_psnr']:.4f}, "
            f"SSIM: {res['sharp_ssim']:.4f})")
