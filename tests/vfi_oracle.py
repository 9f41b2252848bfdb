"""The frame metrics of the Vimeo-90K triplet protocol (rb_frame_metrics, include/raft_b200.h F12) restated in numpy /
scipy fp64, for the tests of the kernel and of raft_b200.evaluate's 'vimeo' dataset.

    quantise:  q = np.clip(np.rint(np.float32(255) * x), 0, 255) on fp32 x, the expression infer_raft.py --interpolate
               writes its PNGs with (fl32 product, ties to even), with a NaN made 0 explicitly (numpy's uint8 cast of a
               NaN is undefined);
    SSE:       sum of (q - gt)^2 in int64;
    SSIM:      skimage.metrics.structural_similarity(gt_c, q_c, gaussian_weights=True, sigma=1.5,
               use_sample_covariance=False, data_range=255) per channel, averaged over the 3 channels: the five moments
               by scipy.ndimage.gaussian_filter(sigma=1.5, truncate=3.5, mode='reflect') -- the call skimage makes --
               and the mean of S over the crop [5, H-5) x [5, W-5).

skimage is not available to the test suite, so this restatement is not pinned against skimage itself; it follows
skimage's documented algorithm (structural_similarity with gaussian_weights), and test_vimeo_eval.py pins it against an
independent direct 2-D form of the same window.
"""
from __future__ import annotations

import numpy as np

SIGMA, TRUNCATE, R = 1.5, 3.5, 5  # R = int(TRUNCATE * SIGMA + 0.5): the 11-tap window
C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2


def quantise(x):
    """[..] fp32 in [0,1] -> uint8 as the CLI writes it; NaN -> 0."""
    x = np.asarray(x, dtype=np.float32)
    q = np.clip(np.rint(np.float32(255.0) * x), 0, 255)
    return np.where(np.isnan(q), 0, q).astype(np.uint8)


def as_u8(pred):
    pred = np.asarray(pred)
    return pred if pred.dtype == np.uint8 else quantise(pred)


def sse(pred, gt):
    """Exact int64 sum of squared errors of one [H,W,3] frame (fp32 preds quantised first)."""
    d = as_u8(pred).astype(np.int64) - np.asarray(gt).astype(np.int64)
    return int((d * d).sum())


def ssim_channel(x, y, mode="reflect"):
    """skimage's Gaussian-window SSIM of two [H,W] images (x the reference, y the test image; symmetric anyway)."""
    from scipy.ndimage import gaussian_filter
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    f = lambda a: gaussian_filter(a, sigma=SIGMA, truncate=TRUNCATE, mode=mode)  # noqa: E731
    ux, uy, uxx, uyy, uxy = f(x), f(y), f(x * x), f(y * y), f(x * y)
    vx, vy, vxy = uxx - ux * ux, uyy - uy * uy, uxy - ux * uy
    S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2))
    return float(S[R:-R, R:-R].mean())


def ssim(pred, gt, mode="reflect"):
    """The mean over the 3 channels of ssim_channel(gt_c, pred_c) of one [H,W,3] frame."""
    q, g = as_u8(pred), np.asarray(gt)
    return float(np.mean([ssim_channel(g[..., c], q[..., c], mode) for c in range(3)]))


def frame_stats(pred, gt):
    """[B,2] fp64 {SSE, SSIM} of a batch of [B,H,W,3] frames: what rb_frame_metrics returns."""
    return np.array([[sse(p, g), ssim(p, g)] for p, g in zip(pred, gt)], dtype=np.float64)


def psnr(sse_value, n_values):
    """10 log10(255^2 n / SSE) in fp64; inf for SSE = 0."""
    return float("inf") if sse_value == 0 else float(10.0 * np.log10(255.0 ** 2 * n_values / sse_value))
