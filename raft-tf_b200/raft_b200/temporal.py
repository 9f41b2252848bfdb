"""Temporal consistency of per-frame processed video (F29 / F30) and its warping error (F31): the host-side rules of
RaftEngine.consistent / warp_error and video_consistent / video_warp_error -- the constants (mirrors of
include/raft_b200.h), the strength check, one frame's correction (terms -> solve -> round) and E_warp from the per-pair
sums."""
import math

import numpy as np
import torch

# rb_tcons_terms' photometric cut-off in grey levels (Tukey's biweight on the originals' mean squared colour difference)
# and the screening that keeps the solve non-singular; neither is tuned on real footage
KAPPA = 20.0
EPS = 1e-4
# rb_screened_poisson's flexible conjugate-gradient iterations and red-black sweeps per level and V-cycle leg
ITERS = 6
SWEEPS = 2

# per-pixel status of consistent()
USED, STEP_FAILED, REJECTED, NO_PREVIOUS = 0, 1, 2, 3


def check_strength(strength, what="consistent"):
    """The strength lambda as a float whose fp32 value (the kernels') is finite and > 0.  Anything else raises
    ValueError."""
    if isinstance(strength, str):
        try:
            strength = float(strength)
        except ValueError:
            strength = None
    with np.errstate(over="ignore"):
        return _checked_strength(strength, what)


def _checked_strength(strength, what):
    if isinstance(strength, bool) or not isinstance(strength, (int, float, np.integer, np.floating)) or \
            not (math.isfinite(float(strength)) and float(strength) > 0) or \
            not (np.isfinite(np.float32(strength)) and np.float32(strength) > 0):  # the kernels take fp32
        raise ValueError(f"{what}: strength must be a finite number > 0 (got {strength!r})")
    return float(strength)


def cutoff_wavelength(strength):
    """The wavelength in pixels, 2 pi / sqrt(lambda), below which the processed frame's detail keeps its gradients."""
    return 2 * math.pi / math.sqrt(strength)


def consistent_frame(frame, prev_frame, processed, prev_out, flow_fw, flow_bw, strength, flow_scale, workspace=None):
    """Frame t's output: rb_tcons_terms, rb_screened_poisson and O = clamp(rint(P + D), 0, 255), all on the current
    stream without a host synchronisation.  prev_frame None (frame 0, or the first frame after a cut) returns P_t
    byte for byte with status 3.  Returns fresh (out [Hs,Ws,3] uint8, status [Hs,Ws] uint8)."""
    from networks.utils import screened_poisson, tcons_terms
    from .engine import FB_ALPHA1, FB_ALPHA2
    c, r, status = tcons_terms(frame, prev_frame, processed, prev_out, flow_fw, flow_bw, strength,
                               flow_scale=flow_scale, alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)
    if prev_frame is None:
        return processed.clone(), status
    D = screened_poisson(c, r, workspace=workspace)
    return (processed.float() + D).round_().clamp_(0, 255).to(torch.uint8), status


def pair_errors(sums, cuts=()):
    """E_pair = sum e / (255^2 count) per pair from rb_warp_error's [T,2] sums (NaN for a cut pair or a pair with no
    counted pixel) and E_warp, the mean over the other pairs (NaN when none counts).  Returns (E_warp, E_pair [T]
    float64, excluded: the sorted pairs left out)."""
    s = np.asarray(sums, np.float64).reshape(-1, 2)
    cut = set(int(k) for k in cuts)
    e = np.full(len(s), np.nan)
    excluded = []
    for k, (se, n) in enumerate(s):
        if k in cut or n == 0:
            excluded.append(k)
        else:
            e[k] = se / (255.0 ** 2 * n)
    ok = ~np.isnan(e)
    return (float(e[ok].mean()) if ok.any() else float("nan")), e, excluded
