"""numpy restatement of davis2017-evaluation's semi-supervised scoring, as that evaluator writes it, for the tests:
db_eval_iou and f_measure (davis2017/metrics.py, with _seg2bmap, cv2.dilate and skimage.morphology.disk's formula),
db_statistics (davis2017/utils.py) and the per-object bookkeeping of davis2017/evaluation.py.  No void pixels: the
semi-supervised path passes none."""
from __future__ import annotations

import math
import warnings

import numpy as np


def db_eval_iou(annotation, segmentation):
    annotation, segmentation = annotation.astype(bool), segmentation.astype(bool)
    inters = np.sum(segmentation & annotation)
    union = np.sum(segmentation | annotation)
    return 1.0 if np.isclose(union, 0) else inters / union


def seg2bmap(seg):
    seg = seg.astype(bool)
    e, s, se = np.zeros_like(seg), np.zeros_like(seg), np.zeros_like(seg)
    e[:, :-1] = seg[:, 1:]
    s[:-1, :] = seg[1:, :]
    se[:-1, :-1] = seg[1:, 1:]
    b = seg ^ e | seg ^ s | seg ^ se
    b[-1, :] = seg[-1, :] ^ e[-1, :]
    b[:, -1] = seg[:, -1] ^ s[:, -1]
    b[-1, -1] = 0
    return b


def disk(r):
    """skimage.morphology.disk(r)."""
    L = np.arange(-r, r + 1)
    X, Y = np.meshgrid(L, L)
    return np.array((X ** 2 + Y ** 2) <= r ** 2, dtype=np.uint8)


def bound_pix(H, W, bound_th=0.008):
    return bound_th if bound_th >= 1 else int(np.ceil(bound_th * np.linalg.norm((H, W))))


def boundary_counts(fg_mask, gt_mask, r):
    """(n_fg, n_gt, fg_match, gt_match) of f_measure: the boundary pixels and those matched within disk(r)."""
    import cv2
    fg_boundary, gt_boundary = seg2bmap(fg_mask), seg2bmap(gt_mask)
    fg_dil = cv2.dilate(fg_boundary.astype(np.uint8), disk(r))
    gt_dil = cv2.dilate(gt_boundary.astype(np.uint8), disk(r))
    return (int(np.sum(fg_boundary)), int(np.sum(gt_boundary)), int(np.sum(fg_boundary * gt_dil)),
            int(np.sum(gt_boundary * fg_dil)))


def f_from_counts(n_fg, n_gt, fg_match, gt_match):
    if n_fg == 0 and n_gt > 0:
        precision, recall = 1, 0
    elif n_fg > 0 and n_gt == 0:
        precision, recall = 0, 1
    elif n_fg == 0 and n_gt == 0:
        precision, recall = 1, 1
    else:
        precision, recall = fg_match / float(n_fg), gt_match / float(n_gt)
    return 0 if precision + recall == 0 else 2 * precision * recall / (precision + recall)


def f_measure(fg_mask, gt_mask, r=None):
    if r is None:
        r = bound_pix(*fg_mask.shape)
    return f_from_counts(*boundary_counts(fg_mask, gt_mask, r))


def counts(pred, gt, n_objects, r):
    """The six counts of rb_label_metrics for [n,H,W] label maps -> [n, n_objects, 6] int64."""
    out = np.zeros((len(pred), n_objects, 6), np.int64)
    for i in range(len(pred)):
        for o in range(1, n_objects + 1):
            P, G = pred[i] == o, gt[i] == o
            n_fg, n_gt, fg_match, gt_match = boundary_counts(P, G, r)
            out[i, o - 1] = (np.sum(P & G), np.sum(P | G), n_fg, n_gt, fg_match, gt_match)
    return out


def db_statistics(per_frame_values):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=RuntimeWarning)
        M = np.nanmean(per_frame_values)
        O = np.nanmean(per_frame_values > 0.5)
    N_bins = 4
    ids = np.round(np.linspace(1, len(per_frame_values), N_bins + 1) + 1e-10) - 1
    ids = ids.astype(np.uint8)
    D_bins = [per_frame_values[ids[i]:ids[i + 1] + 1] for i in range(0, 4)]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", category=RuntimeWarning)
        D = np.nanmean(D_bins[0]) - np.nanmean(D_bins[3])
    return M, O, D


def evaluate_sequences(sequences):
    """sequences: [(gt [F,H,W] uint8, pred [F,H,W] uint8)] -> the global {J&F-Mean, J-Mean, J-Recall, J-Decay, F-Mean,
    F-Recall, F-Decay} of evaluation.py's semi-supervised path (frames 1..F-2, objects 1..max(gt[0]) with 255 -> 0)."""
    J = {"M": [], "R": [], "D": []}
    F = {"M": [], "R": [], "D": []}
    for gt, pred in sequences:
        gt = np.where(gt == 255, 0, gt)
        n_obj = int(gt[0].max())
        gt, pred = gt[1:-1], pred[1:-1]
        for o in range(1, n_obj + 1):
            j = np.array([db_eval_iou(gt[i] == o, pred[i] == o) for i in range(len(gt))], dtype=np.float64)
            f = np.array([f_measure(pred[i] == o, gt[i] == o) for i in range(len(gt))], dtype=np.float64)
            for store, v in ((J, j), (F, f)):
                m, r, d = db_statistics(v)
                store["M"].append(m)
                store["R"].append(r)
                store["D"].append(d)
    res = {"J-Mean": np.mean(J["M"]), "J-Recall": np.mean(J["R"]), "J-Decay": np.mean(J["D"]),
           "F-Mean": np.mean(F["M"]), "F-Recall": np.mean(F["R"]), "F-Decay": np.mean(F["D"])}
    res["J&F-Mean"] = (res["J-Mean"] + res["F-Mean"]) / 2
    return {k: float(v) for k, v in res.items()}


assert math.isclose(bound_pix(480, 854), 8) and bound_pix(1080, 1920) == 18
