"""Temporal consistency without a GPU: the numpy restatement of rb_tcons_terms / rb_screened_poisson / rb_warp_error
(tests/tcons_oracle.py) against fp64, the closed-form response of the solve, the identities of the method, the quality
on a clip with a known camera path and exact flows, and the refusals of the host checks and the C entries."""
import math

import numpy as np
import pytest

import stabfill_oracle as SF
import stabilize_oracle as SO
import tcons_oracle as TO
from raft_b200 import temporal as T

F32 = np.float32


def _psnr(a, b):
    return 10 * np.log10(255.0 ** 2 / np.mean((a.astype(np.float64) - b) ** 2))


def _system(rng, H, W, lam, kind):
    w = {"ones": np.ones((H, W), F32), "half": np.zeros((H, W), F32), "blobs": (rng.random((H, W)) ** 2).astype(F32),
         "point": np.zeros((H, W), F32)}[kind]
    if kind == "half":
        w[:, :max(1, W // 3)] = 1
    if kind == "blobs":
        w[H // 4:, W // 4:] = 0
    if kind == "point":
        w[0, 0] = 1
    diff = rng.integers(-255, 256, (H, W, 3)).astype(F32)
    lw = (F32(lam) * w).astype(F32)
    return (lw + F32(T.EPS)).astype(F32), (lw[..., None] * diff).astype(F32)


@pytest.mark.parametrize("hw", [(1, 1), (1, 7), (6, 1), (5, 3), (33, 47), (64, 96)])
@pytest.mark.parametrize("lam", [1e-4, 1e-2, 1.0, 10.0])
def test_solve_is_within_a_quarter_grey_level_of_fp64(hw, lam):
    """Measured worst case over these sizes, weights and strengths: 0.029 grey levels."""
    rng = np.random.default_rng(hw[0] * 100 + hw[1])
    for kind in ("ones", "half", "blobs", "point"):
        c, r = _system(rng, *hw, lam, kind)
        err = np.abs(TO.screened_poisson(c, r) - TO.screened_poisson_f64(c, r)).max()
        assert err <= 0.25, (kind, err)


@pytest.mark.parametrize("lam", [1e-3, 1e-2, 0.1, 1.0])
def test_cosine_mode_response(lam):
    """w = 1: a Neumann cosine mode of (O^ - P) is corrected by lambda / (lambda + eps + mu)."""
    H, W = 24, 64
    x = np.arange(W)
    for k in (0, 1, 3, 8):
        mode = np.cos(np.pi * k * (x + 0.5) / W)
        mu = 2 - 2 * math.cos(math.pi * k / W)
        diff = np.broadcast_to((100 * mode)[None, :, None], (H, W, 3)).astype(F32)
        lw = np.full((H, W), F32(lam), F32)
        D = TO.screened_poisson((lw + F32(T.EPS)).astype(F32), (lw[..., None] * diff).astype(F32))
        gain = lam / (lam + T.EPS + mu)
        assert np.abs(D - gain * diff).max() < 0.05, (k, np.abs(D - gain * diff).max())


def test_zero_right_hand_side_gives_zero():
    c = np.full((7, 9), F32(T.EPS), F32)
    c[2:5] = F32(3.0)
    D = TO.screened_poisson(c, np.zeros((7, 9, 3), F32))
    assert np.array_equal(D, np.zeros_like(D))


def _known_clip(seed=0):
    """A pan with rotation, zoom and translation jitter rendered at 48x80 (stabfill_oracle), its exact flows on a 24x40
    grid, P = a tone curve of the clean frames with a seeded per-frame flicker (gain in [0.85, 1.15], per-channel offset
    in +-12, a smooth illumination field of amplitude 10), and the target: the same curve with frame 0's flicker."""
    F, hw, net = 12, (48, 80), (24, 40)
    G, motions = SF.jittered_path(F, seed)
    clean = SF.render(G, hw)
    fw = np.stack([SO.similarity_flow(m, *net, *hw) for m in motions]).astype(F32)
    bw = np.stack([SO.similarity_flow(SF.inverse(m), *net, *hw) for m in motions]).astype(F32)
    rng = np.random.default_rng(200 + seed)
    H, W = hw
    y, x = np.mgrid[0:H, 0:W] / np.array([H, W])[:, None, None]

    def flicker():
        g, off, ph = rng.uniform(0.85, 1.15), rng.uniform(-12, 12, 3), rng.uniform(0, 2 * np.pi, 2)
        return g, off, 10 * np.sin(np.pi * x + ph[0]) * np.cos(0.5 * np.pi * y + ph[1])

    def apply(t, f):
        return np.clip(np.rint(f[0] * t + f[1] + f[2][..., None]), 0, 255).astype(np.uint8)

    fl = [flicker() for _ in range(F)]
    tone = 255 * (clean / 255.0) ** 0.8
    P = np.stack([apply(tone[k], fl[k]) for k in range(F)])
    target = np.stack([apply(tone[k], fl[0]) for k in range(F)])
    return clean, P, target, fw, bw


@pytest.mark.parametrize("lam", [0.01, 0.1])
def test_flicker_is_removed_on_the_known_path(lam):
    """Measured with RB_TCONS_KAPPA = 20: PSNR against the target 25.54 dB for P, 35.59 / 40.35 dB for O at lambda
    0.01 / 0.1; E_warp 0.01151 for P, 4.8e-4 / 9.7e-5 for O (4.5e-5 for the target itself).  No match is rejected by
    the colour check on this clip."""
    clean, P, target, fw, bw = _known_clip()
    O, status = TO.consistent(clean, P, fw, bw, lam)
    assert _psnr(O, target) > _psnr(P, target) + 8.0
    eP = T.pair_errors(TO.warp_error_sums(P, fw, bw))[0]
    eO = T.pair_errors(TO.warp_error_sums(O, fw, bw))[0]
    assert eO < 0.05 * eP, (eO, eP)
    assert (status[0] == 3).all() and not (status[1:] == 3).any() and (status[1:] == 0).mean() > 0.85


def test_identities_cut_and_tiny_strength():
    clean, P, _, fw, bw = _known_clip()
    O, status = TO.consistent(clean, P, fw, bw, 0.1, cuts=(4,))
    assert np.array_equal(O[0], P[0]) and np.array_equal(O[5], P[5]) and (status[5] == 3).all()
    assert not np.array_equal(O[6], P[6])
    tiny, _ = TO.consistent(clean[:3], P[:3], fw[:2], bw[:2], 1e-9)
    assert np.array_equal(tiny, P[:3])
    # flow that fails everywhere: r = 0, so O = P bit for bit
    far = fw[:2] + F32(1000)
    O2, st2 = TO.consistent(clean[:3], P[:3], far, bw[:2], 0.1)
    assert np.array_equal(O2, P[:3]) and (st2[1:] == 1).all()


def test_fine_detail_passes_through():
    """Detail much finer than the cut-off wavelength 2 pi / sqrt(lambda) keeps P's gradients."""
    H, W, lam = 32, 64, 0.01  # cut-off ~63 pixels
    x = np.arange(W)
    detail = (20 * np.cos(np.pi * 48 * (x + 0.5) / W))[None, :, None]  # a Neumann mode of period 2.7 pixels
    diff = np.broadcast_to(detail, (H, W, 3)).astype(F32)
    lw = np.full((H, W), F32(lam), F32)
    D = TO.screened_poisson((lw + F32(T.EPS)).astype(F32), (lw[..., None] * diff).astype(F32))
    assert np.abs(D).max() < 0.25
    assert T.cutoff_wavelength(lam) == pytest.approx(2 * math.pi / 0.1)


def test_warp_error_is_zero_for_an_exact_whole_pixel_translation():
    rng = np.random.default_rng(5)
    big = rng.integers(0, 256, (20, 40, 3), dtype=np.uint8)
    F, H, W = 4, 12, 16
    video = np.stack([big[2:2 + H, 2 * k:2 * k + W] for k in range(F)])  # content moves 2 pixels left per frame
    fw = np.zeros((F - 1, H, W, 2), F32)
    fw[..., 0] = -2
    bw = -fw
    sums = TO.warp_error_sums(video, fw, bw)
    assert (sums[:, 0] == 0).all() and (sums[:, 1] == H * (W - 2)).all()
    e, per, excluded = T.pair_errors(sums, cuts=[1])
    assert e == 0 and np.isnan(per[1]) and excluded == [1]


def test_warp_error_hand_computed():
    """2x2 frames, zero flow: every pixel passes; frame 1 adds 3 to channel 0 of one pixel: e = 9 there."""
    a = np.full((2, 2, 3), 50, np.uint8)
    b = a.copy()
    b[1, 0, 0] = 53
    fw = np.zeros((1, 2, 2, 2), F32)
    sums = TO.warp_error_sums(np.stack([a, b]), fw, fw)
    assert sums.tolist() == [[9.0, 4.0]]
    assert T.pair_errors(sums)[0] == 9.0 / (255 ** 2 * 4)


@pytest.mark.parametrize("bad", [0, -1.0, float("nan"), float("inf"), "x", True, None])
def test_strength_refusals(bad):
    with pytest.raises(ValueError):
        T.check_strength(bad)


def test_header_constants_match():
    import os
    import re
    text = open(os.path.join(os.path.dirname(__file__), "..", "include", "raft_b200.h")).read()
    consts = dict(re.findall(r"#define RB_TCONS_(\w+) ([0-9.e-]+)f?\n", text))
    assert (float(consts["KAPPA"]), float(consts["EPS"]), int(consts["ITERS"]), int(consts["SWEEPS"])) == \
        (T.KAPPA, T.EPS, T.ITERS, T.SWEEPS)


def test_c_entries_refuse_bad_arguments_before_any_cuda_call():
    import ctypes
    from raft_b200 import capi
    lib, fake = capi.lib, 4096
    args = [fake, fake, fake, fake, 8, 8, fake, fake, 4, 4, 1.0, 0.01, 0.5, 0.1, fake, fake, fake, None]
    for i, v, code in ((14, None, -2), (6, None, -2), (4, 0, -1), (8, 0, -1), (10, 0.0, -2), (11, -1.0, -2),
                       (13, 0.0, -2), (13, float("nan"), -2), (13, float("inf"), -2)):
        a = list(args)
        a[i] = v
        assert lib.rb_tcons_terms(*a) == code, (i, v)
    size = ctypes.c_size_t(0)
    assert lib.rb_screened_poisson_workspace_bytes(0, 4, ctypes.byref(size)) == -1
    assert lib.rb_screened_poisson_workspace_bytes(4, 4, ctypes.byref(size)) == 0 and size.value > 0
    assert lib.rb_screened_poisson(fake, fake, 4, 4, fake, fake, size.value - 1, None) == -2
    assert lib.rb_screened_poisson(fake, fake, 4, 4, fake, None, size.value, None) == -2
    assert lib.rb_screened_poisson(fake, fake, 4, 0, fake, fake, size.value, None) == -1
    assert lib.rb_screened_poisson(fake, fake, 4, 4, fake + 0, fake, size.value, None) == -2  # D aliases r
    assert lib.rb_warp_error_workspace_bytes(1, 4, 4, ctypes.byref(size)) == -1
    assert lib.rb_warp_error_workspace_bytes(3, 4, 4, ctypes.byref(size)) == 0
    wargs = [fake, 3, 4, 4, fake, fake, 4, 4, 1.0, 0.01, 0.5, fake, fake, size.value, None]
    for i, v, code in ((0, None, -2), (11, None, -2), (1, 1, -1), (8, -1.0, -2), (10, float("nan"), -2),
                       (13, size.value - 1, -2)):
        a = list(wargs)
        a[i] = v
        assert lib.rb_warp_error(*a) == code, (i, v)


@pytest.mark.parametrize("bad", [1e-50, 1e39])
def test_strength_must_be_finite_and_positive_in_fp32(bad):
    with pytest.raises(ValueError):
        T.check_strength(bad)


def test_solver_refuses_overlapping_buffers():
    import ctypes
    from raft_b200 import capi
    lib, fake = capi.lib, 1 << 20
    size = ctypes.c_size_t(0)
    assert lib.rb_screened_poisson_workspace_bytes(4, 4, ctypes.byref(size)) == 0
    ws = 1 << 30
    assert lib.rb_screened_poisson(fake, fake + 4096, 4, 4, fake + 4096 + 8, ws, size.value, None) == -2  # D inside r
    assert lib.rb_screened_poisson(fake, fake + 4096, 4, 4, fake + 32, ws, size.value, None) == -2  # D over c
    assert lib.rb_screened_poisson(fake, fake + 4096, 4, 4, ws + 64, ws, size.value, None) == -2  # D in the workspace
    assert lib.rb_screened_poisson(fake, fake + 4096, 4, 4, fake + 8192, fake + 4096 + 16, size.value, None) == -2


def _usage_error(argv, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


@pytest.fixture
def dirs(tmp_path):
    import cv2
    a, b, c, d = (tmp_path / n for n in ("a", "b", "c", "d"))
    for x in (a, b, c, d):
        x.mkdir()
    img = np.zeros((12, 16, 3), np.uint8)
    for i in range(4):
        cv2.imwrite(str(a / f"{i}.png"), img)
        cv2.imwrite(str(b / f"{i}.png"), img)
        cv2.imwrite(str(d / f"{i}.png"), img[:-2])
        if i < 3:
            cv2.imwrite(str(c / f"{i}.png"), img)
    return str(a), str(b), str(c), str(d)


@pytest.mark.parametrize("argv,words", [
    (["--consistent", "B"], "needs --consistent-strength"),
    (["--consistent-strength", "0.1"], "goes with --consistent"),
    (["--path", "A", "--consistent", "B", "--consistent-strength", "0"], "L must be"),
    (["--path", "A", "--consistent", "B", "--consistent-strength", "nan"], "L must be"),
    (["--path", "A", "--consistent", "B", "--consistent-strength", "1e-50"], "L must be"),
    (["--consistent", "B", "--consistent-strength", "0.1"], "needs --path"),
    (["--path", "A", "--consistent", "B", "--consistent-strength", "0.1", "--denoise", "20"],
     "cannot be combined with --denoise"),
    (["--path", "A", "--consistent", "B", "--consistent-strength", "0.1", "--warp-error", "B"],
     "cannot be combined with --warp-error"),
    (["--path", "A", "--consistent", "B", "--consistent-strength", "0.1", "--stabilize", "5"],
     "cannot be combined with --stabilize"),
    (["--path", "A", "--warp-error", "B", "--interpolate", "0.5"], "cannot be combined with --interpolate"),
    (["--path", "A", "--warp-error", "B", "--inpaint", "m/"], "cannot be combined with --inpaint"),
    (["--warp-error", "B"], "needs --path"),
    (["--path", "A", "--warp-error", "B", "--scene-cut", "2"], "--scene-cut"),
    (["--path", "A", "--consistent", "C", "--consistent-strength", "0.1"], "must be aligned"),
    (["--path", "A", "--warp-error", "C"], "must be aligned"),
    (["--path", "A", "--warp-error", "D"], "must be aligned"),
    (["--path", "A", "--consistent", "D", "--consistent-strength", "0.1"], "must be aligned"),
])
def test_cli_refusals(argv, words, dirs, capsys):
    names = dict(zip("ABCD", dirs))
    argv = [names.get(v, v) for v in argv]
    assert words in _usage_error(argv, capsys)
