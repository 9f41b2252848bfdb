"""TAP-Vid's metrics and query sampling restated as plain loops over (query, frame) entries, written apart from the
vectorised raft_b200.tapvid, for the tests.

metrics(pred, pred_occluded, gt, gt_occluded, qframe, mode) -> the per-video dict of raft_b200.tapvid.video_metrics;
queries(occluded, mode) -> the (track, frame) list of raft_b200.tapvid.sample_queries.
"""
from __future__ import annotations

import math

THRESHOLDS = (1, 2, 4, 8, 16)


def queries(occluded, mode):
    N, F = len(occluded), len(occluded[0])
    out = []
    if mode == "first":
        for n in range(N):
            for t in range(F):
                if not occluded[n][t]:
                    out.append((n, t))
                    break
    else:
        for t in range(0, F, 5):
            for n in range(N):
                if not occluded[n][t]:
                    out.append((n, t))
    return out


def metrics(pred, pred_occluded, gt, gt_occluded, qframe, mode):
    n_eval = n_oa = n_vis = 0
    within = {d: 0 for d in THRESHOLDS}
    tp = {d: 0 for d in THRESHOLDS}
    fp = {d: 0 for d in THRESHOLDS}
    for q in range(len(qframe)):
        for t in range(len(gt_occluded[q])):
            if (mode == "first" and t <= qframe[q]) or (mode == "strided" and t == qframe[q]):
                continue
            n_eval += 1
            visible = not gt_occluded[q][t]
            pred_visible = not pred_occluded[q][t]
            if pred_visible == visible:
                n_oa += 1
            n_vis += visible
            dx = float(pred[q][t][0]) - float(gt[q][t][0])
            dy = float(pred[q][t][1]) - float(gt[q][t][1])
            dist2 = dx * dx + dy * dy
            for d in THRESHOLDS:
                close = (not math.isnan(dist2)) and dist2 < d * d
                if close and visible:
                    within[d] += 1
                    if pred_visible:
                        tp[d] += 1
                if pred_visible and (not visible or not close):
                    fp[d] += 1
    nan = float("nan")
    m = {"occlusion_accuracy": n_oa / n_eval if n_eval else nan}
    for d in THRESHOLDS:
        m[f"pts_within_{d}"] = within[d] / n_vis if n_vis else nan
        m[f"jaccard_{d}"] = tp[d] / (n_vis + fp[d]) if n_vis + fp[d] else nan
    m["average_pts_within_thresh"] = sum(m[f"pts_within_{d}"] for d in THRESHOLDS) / len(THRESHOLDS)
    m["average_jaccard"] = sum(m[f"jaccard_{d}"] for d in THRESHOLDS) / len(THRESHOLDS)
    return m


def same(a, b):
    """Two metric dicts equal key by key (NaN equals NaN)."""
    return a.keys() == b.keys() and all((math.isnan(a[k]) and math.isnan(b[k])) or a[k] == b[k] for k in a)
