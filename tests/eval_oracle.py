"""Upstream RAFT's evaluation formulas (evaluate.py: validate_sintel, validate_kitti) restated in torch on the CPU, for the
tests of rb_flow_metrics and raft_b200.evaluate.

Per pixel, as upstream writes them on fp32 tensors (each operation rounded on its own):
    epe = torch.sum((flow - flow_gt) ** 2, dim=0).sqrt(),  mag = torch.sum(flow_gt ** 2, dim=0).sqrt(),
    out = (epe > 3.0) & ((epe / mag) > 0.05)   (torch compares an fp32 tensor with a Python float in fp32: 0.05f)
with the flow first multiplied by flow_scale (8 for raft-small in the reference semantics; exact).  Aggregation: Sintel
pools every pixel (np.mean of the concatenated EPE), KITTI averages the per-image means of the valid pixels, and both
take 1px / 3px / 5px and F1 over the pooled pixels.  Sums here are fp64.
"""
from __future__ import annotations

import numpy as np
import torch


def _sqrt(x):
    """IEEE fp32 sqrt, as torch computes it on CUDA where upstream evaluates.  torch's vectorised CPU sqrt is not always
    correctly rounded (it misses by one ulp next to a rounding midpoint); the fp64 sqrt rounded once to fp32 is (53 >= 2 * 24
    + 2 bits, so the double rounding is innocuous)."""
    return torch.sqrt(x.double()).float()


def pixel_terms(flow, gt, flow_scale=1.0):
    """[B,H,W,2] flow and ground truth -> (epe, mag, outlier), each [B,H,W] (fp32, fp32, bool)."""
    flow = torch.as_tensor(np.asarray(flow), dtype=torch.float32)
    gt = torch.as_tensor(np.asarray(gt), dtype=torch.float32)
    d = flow * float(flow_scale) - gt
    epe = _sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1])
    mag = _sqrt(gt[..., 0] * gt[..., 0] + gt[..., 1] * gt[..., 1])
    out = (epe > 3.0) & ((epe / mag) > 0.05)
    return epe, mag, out


def sample_stats(flow, gt, valid=None, flow_scale=1.0):
    """[B,6] fp64 {n, sum epe, #(epe < 1), #(epe < 3), #(epe < 5), #outliers} over the counted pixels of each sample (valid:
    [B,H,W], nonzero counts; None: all); the sum is an fp64 sum of the fp32 EPE."""
    epe, _, out = pixel_terms(flow, gt, flow_scale)
    B = epe.shape[0]
    sel = torch.ones_like(epe, dtype=torch.bool) if valid is None else torch.as_tensor(np.asarray(valid)) != 0
    res = torch.zeros(B, 6, dtype=torch.float64)
    for b in range(B):
        e = epe[b][sel[b]]
        res[b] = torch.tensor([e.numel(), float(e.double().sum()), int((e < 1).sum()), int((e < 3).sum()),
                               int((e < 5).sum()), int(out[b][sel[b]].sum())], dtype=torch.float64)
    return res


def aggregate_pixels(epes, outliers, kitti):
    """Upstream's aggregation from per-image lists of counted-pixel arrays: epes[i] the fp32 EPE, outliers[i] the bools.
    -> dict epe, 1px, 3px, 5px, f1 (fp64)."""
    all_e = np.concatenate([np.asarray(e, dtype=np.float64).ravel() for e in epes])
    all_o = np.concatenate([np.asarray(o, dtype=np.float64).ravel() for o in outliers])
    epe = np.mean([np.mean(np.asarray(e, dtype=np.float64)) for e in epes]) if kitti else np.mean(all_e)
    return {"epe": float(epe), "1px": float(np.mean(all_e < 1)), "3px": float(np.mean(all_e < 3)),
            "5px": float(np.mean(all_e < 5)), "f1": float(100.0 * np.mean(all_o))}


def aggregate_stats(stats, kitti):
    """The same aggregates from per-image stats rows (what raft_b200.evaluate keeps)."""
    s = np.asarray(stats, dtype=np.float64).reshape(-1, 6)
    n = s[:, 0].sum()
    epe = np.mean(s[:, 1] / s[:, 0]) if kitti else s[:, 1].sum() / n
    return {"epe": float(epe), "1px": float(s[:, 2].sum() / n), "3px": float(s[:, 3].sum() / n),
            "5px": float(s[:, 4].sum() / n), "f1": float(100.0 * s[:, 5].sum() / n)}
