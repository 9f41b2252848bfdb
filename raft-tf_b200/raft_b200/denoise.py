"""Video denoising (F27 / F28): the host-side rules of RaftEngine.denoise and video_denoise -- the merge's constants
(mirrors of include/raft_b200.h), the noise level as given or estimated, and the merge of a table's rows.  The per-frame
table of how far each side may chain is raft_b200.inpaint.inpaint_rows'."""
import math

import numpy as np
import torch

DEFAULT_WINDOW = 3  # frames each side may chain (7 frames in all); not tuned on real footage

# rb_denoise_merge's constants (RB_DENOISE_* in include/raft_b200.h): candidates at integer offsets -SEARCH .. SEARCH per
# axis, patches of (2 PATCH + 1)^2 pixels, the longest chain per side, and Tukey's biweight cut-off H sigma above the
# noise floor 2 sigma^2
SEARCH = 1
PATCH = 1
MAX_WINDOW = 16
H = 3.0

ESTIMATE_FRAMES = 8  # sigma="auto" estimates from frames 0 .. min(F, 8) - 1, so it does not depend on the batch


def check_sigma(sigma, what="denoise"):
    """The noise level as "auto" or a float > 0 (the standard deviation in grey levels, 0-255).  Anything else raises
    ValueError."""
    if isinstance(sigma, str):
        if sigma == "auto":
            return sigma
        try:
            sigma = float(sigma)
        except ValueError:
            sigma = None
    if isinstance(sigma, bool) or not isinstance(sigma, (int, float, np.integer, np.floating)) or \
            not (math.isfinite(float(sigma)) and float(sigma) > 0):
        raise ValueError(f"{what}: sigma must be a number > 0 (the noise's standard deviation in grey levels) or "
                         f"\"auto\" (got {sigma!r})")
    return float(sigma)


def check_window(window, what="denoise"):
    """The temporal window as an int in [1, MAX_WINDOW]: how many frames each side of the merge may chain.  Anything else
    raises ValueError."""
    if isinstance(window, bool) or not isinstance(window, (int, np.integer)) or not 1 <= window <= MAX_WINDOW:
        raise ValueError(f"{what}: window must be an integer in [1, {MAX_WINDOW}] (got {window!r})")
    return int(window)


def sigma_from_sums(sums, H, W):
    """Immerkaer's estimate from rb_noise_sums' [N,3] sums of |I * M| over the interior of H x W frames:
    sqrt(pi / 2) S / (6 (H - 2)(W - 2)) per frame and channel, averaged over both, in fp64."""
    s = np.asarray(sums, np.float64)
    return float(np.mean(math.sqrt(math.pi / 2) * s / (6.0 * (H - 2) * (W - 2))))


def estimate_sigma(frames):
    """sigma="auto": the noise estimate (networks.utils.noise_sigma) of frames 0 .. min(F, ESTIMATE_FRAMES) - 1 of
    [F,H,W,3] uint8 CUDA frames."""
    from networks.utils import noise_sigma
    return noise_sigma(frames[:ESTIMATE_FRAMES])


def merge_frames(frames, flow_fw, flow_bw, rows, sigma, flow_scale):
    """The denoised frames of the table's rows: one rb_denoise_merge launch with the forward-backward test of the
    occlusion check.  sigma 0 (an estimate on noise-free frames) returns the rows' frames unchanged with support 0.
    Returns fresh (frames [n,Hs,Ws,3] uint8, support [n,Hs,Ws] uint8)."""
    from networks.utils import denoise_merge
    from .engine import FB_ALPHA1, FB_ALPHA2
    if sigma == 0:
        t = torch.as_tensor(np.asarray(rows)[:, 0], dtype=torch.int64, device=frames.device)
        return frames[t].clone(), torch.zeros(frames.shape[1:3], dtype=torch.uint8,
                                              device=frames.device).expand(len(t), -1, -1).clone()
    return denoise_merge(frames, flow_fw, flow_bw, rows, sigma, flow_scale=flow_scale, alpha1=FB_ALPHA1,
                         alpha2=FB_ALPHA2)
