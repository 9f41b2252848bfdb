"""Video denoising without a GPU: the numpy restatement of rb_denoise_merge on a clip with a known camera path and exact
flows (the quality claims), the Immerkaer noise estimate, the DAVIS protocol's noise, the host checks, the CLI's
argument errors and the C entries' RB_ERR_* returns before any CUDA call."""
import ctypes
import math

import numpy as np
import pytest

import denoise_oracle as DO
import stabfill_oracle as SF
import stabilize_oracle as SO
from raft_b200 import denoise as D
from raft_b200.inpaint import inpaint_rows


def _psnr(a, b):
    return 10 * np.log10(255.0 ** 2 / np.mean((a.astype(np.float64) - b) ** 2))


def _known_clip(sigma, seed=0):
    """A pan with rotation, zoom and translation jitter rendered at 48x80 (stabfill_oracle), its exact flows on a 24x40
    grid, and the frames with seeded Gaussian noise of sigma grey levels, rounded and clipped to bytes."""
    F, hw, net = 12, (48, 80), (24, 40)
    G, motions = SF.jittered_path(F, seed)
    clean = SF.render(G, hw)
    fw = np.stack([SO.similarity_flow(m, *net, *hw) for m in motions])
    bw = np.stack([SO.similarity_flow(SF.inverse(m), *net, *hw) for m in motions])
    rng = np.random.default_rng(100 + seed)
    noisy = np.clip(np.rint(clean + sigma * rng.standard_normal(clean.shape)), 0, 255).astype(np.uint8)
    return clean, noisy, fw, bw


@pytest.mark.parametrize("sigma", [10, 25])
def test_temporal_merge_beats_spatial_merge_beats_noisy_input(sigma):
    """Thresholds from a CPU run of the oracle with RB_DENOISE_H = 3 and window 3: PSNR 28.14 / 36.77 / 42.11 dB (noisy /
    spatial only / temporal) at sigma 10 and 20.23 / 29.45 / 35.88 dB at sigma 25."""
    clean, noisy, fw, bw = _known_clip(sigma)
    rows = inpaint_rows(len(clean), 3)
    spatial = rows.copy()
    spatial[:, 1:] = 0
    out, support = DO.denoise_merge(noisy, fw, bw, rows, sigma)
    out0, support0 = DO.denoise_merge(noisy, fw, bw, spatial, sigma)
    p_noisy, p_spatial, p_temporal = _psnr(noisy, clean), _psnr(out0, clean), _psnr(out, clean)
    assert not support0.any()
    assert p_spatial > p_noisy + 5.0, (p_spatial, p_noisy)
    assert p_temporal > p_spatial + 4.0, (p_temporal, p_spatial)


@pytest.mark.parametrize("cuts", [(), (5,)])
def test_support_is_the_full_window_away_from_cuts_and_edges(cuts):
    clean, noisy, fw, bw = _known_clip(10)
    rows = inpaint_rows(len(clean), 3, cuts)
    _, support = DO.denoise_merge(noisy, fw, bw, rows, 10.0)
    m = 12  # the path moves a pixel at most ~10 frame pixels in 3 frames
    inner = support[:, m:-m, m:-m]
    for r, (t, nf, nb) in enumerate(rows):
        assert (inner[r] == nf + nb).all(), (r, np.unique(inner[r]))
        assert (support[r] <= nf + nb).all()


def test_constant_clip_comes_back_and_the_backward_side_mirrors_the_forward_side():
    rng = np.random.default_rng(3)
    F, H, W = 4, 9, 13
    fw = rng.normal(0, 1.5, (F - 1, 5, 7, 2)).astype(np.float32)
    bw = (-fw + rng.normal(0, 0.2, fw.shape)).astype(np.float32)
    flat = np.full((F, H, W, 3), 77, np.uint8)
    out, _ = DO.denoise_merge(flat, fw, bw, inpaint_rows(F, 2), 20.0)
    assert np.array_equal(out, flat)
    # the backward side is the forward side of the reversed clip: the same support, and with one side only (so that the
    # sums run in the same order) the same bytes
    frames = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    rows = inpaint_rows(F, 2)
    rev = np.stack([F - 1 - rows[::-1, 0], rows[::-1, 2], rows[::-1, 1]], 1)
    rframes, rfw, rbw = frames[::-1].copy(), bw[::-1].copy(), fw[::-1].copy()
    _, sup = DO.denoise_merge(frames, fw, bw, rows, 20.0)
    _, rsup = DO.denoise_merge(rframes, rfw, rbw, rev, 20.0)
    assert np.array_equal(rsup[::-1], sup) and sup.any()
    one = rows.copy()
    one[:, 2] = 0
    rone = np.stack([F - 1 - one[::-1, 0], one[::-1, 2], one[::-1, 1]], 1)
    out, sup = DO.denoise_merge(frames, fw, bw, one, 20.0)
    rout, rsup = DO.denoise_merge(rframes, rfw, rbw, rone, 20.0)
    assert np.array_equal(rout[::-1], out) and np.array_equal(rsup[::-1], sup)


def test_immerkaer_estimate():
    rng = np.random.default_rng(4)
    flat = np.full((4, 96, 128, 3), 128, np.uint8)
    assert D.sigma_from_sums(DO.noise_sums(flat), 96, 128) == 0.0
    for sigma in (5.0, 20.0):
        noisy = np.clip(np.rint(128 + sigma * rng.standard_normal(flat.shape)), 0, 255).astype(np.uint8)
        est = D.sigma_from_sums(DO.noise_sums(noisy), 96, 128)
        assert abs(est - sigma) < 0.03 * sigma, (est, sigma)


def test_protocol_noise_is_reproducible_and_per_frame():
    from raft_b200.davis import noisy_frame
    clean = np.full((40, 60, 3), 128, np.uint8)
    a = noisy_frame(clean, "bike-trial", 3, 20)
    assert np.array_equal(a, noisy_frame(clean, "bike-trial", 3, 20))
    assert not np.array_equal(a, noisy_frame(clean, "bike-trial", 4, 20))
    assert not np.array_equal(a, noisy_frame(clean, "boxing", 3, 20))
    assert a.dtype == np.uint8 and abs(a.astype(np.float64).std() - 20) < 1.0
    # a frame's noise is a function of (sequence, frame) alone: drawn in any order, in any grouping, it is the same
    seq = [noisy_frame(clean, "bike-trial", i, 20) for i in (5, 2, 3)]
    assert np.array_equal(seq[2], a)


@pytest.mark.parametrize("bad", [0, -1.0, float("nan"), float("inf"), "x", True, None, "0"])
def test_sigma_refusals(bad):
    with pytest.raises(ValueError):
        D.check_sigma(bad)


def test_sigma_accepts_numbers_and_auto():
    assert D.check_sigma("auto") == "auto"
    assert D.check_sigma(20) == 20.0 and D.check_sigma("12.5") == 12.5 and D.check_sigma(np.float32(3)) == 3.0


@pytest.mark.parametrize("bad", [0, 17, 2.5, True, None, -3])
def test_window_refusals(bad):
    with pytest.raises(ValueError):
        D.check_window(bad)


def test_header_constants_match():
    import os
    import re
    text = open(os.path.join(os.path.dirname(__file__), "..", "include", "raft_b200.h")).read()
    consts = dict(re.findall(r"#define RB_DENOISE_(\w+) ([0-9.]+)f?", text))
    assert (int(consts["SEARCH"]), int(consts["PATCH"]), int(consts["MAX_WINDOW"]), float(consts["H"])) == \
        (D.SEARCH, D.PATCH, D.MAX_WINDOW, D.H)


def _usage_error(argv, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


@pytest.mark.parametrize("argv,words", [
    (["--denoise", "20"], "needs --path"),
    (["--path", "f/", "--denoise", "0"], "SIGMA must be"),
    (["--path", "f/", "--denoise", "abc"], "SIGMA must be"),
    (["--path", "f/", "--denoise", "nan"], "SIGMA must be"),
    (["--path", "f/", "--denoise", "20", "--denoise-window", "0"], "--denoise-window"),
    (["--path", "f/", "--denoise", "20", "--denoise-window", "17"], "--denoise-window"),
    (["--path", "f/", "--denoise", "20", "--inpaint", "m/"], "cannot be combined with --inpaint"),
    (["--path", "f/", "--denoise", "20", "--stabilize", "5"], "cannot be combined with --stabilize"),
    (["--path", "f/", "--denoise", "20", "--warm-start"], "cannot be combined with --warm-start"),
    (["--path", "f/", "--denoise", "20", "--interpolate", "0.5"], "cannot be combined with --interpolate"),
    (["--path", "f/", "--denoise", "auto", "--scene-cut", "2"], "--scene-cut"),
    (["--path", "f/", "--denoise", "20", "--keep-size", "--flow-size", "64", "64"], "--flow-size"),
    (["--path", "f/", "--denoise-window", "3"], "--denoise-window goes with --denoise"),
    (["-m", "val", "--dataset", "sintel", "--data", "d/", "--denoise", "20"], "needs --dataset davis"),
    (["-m", "val", "--dataset", "davis", "--data", "d/", "--denoise", "auto"], "not auto"),
    (["-m", "val", "--dataset", "davis", "--data", "d/", "--denoise", "20", "--warm-start"], "--warm-start"),
    (["-m", "val", "--dataset", "davis", "--data", "d/", "--denoise", "20", "--keyframe-step", "5"],
     "--keyframe-step"),
    (["-m", "val", "--dataset", "davis", "--denoise", "20"], "--data"),
])
def test_cli_refusals(argv, words, capsys):
    assert words in _usage_error(argv, capsys)


def test_c_entries_refuse_bad_arguments_before_any_cuda_call():
    from raft_b200 import capi
    lib, fake = capi.lib, 4096  # a non-null pointer the checks never dereference
    args = [fake, 3, 8, 8, fake, fake, 4, 4, 1.0, 0.01, 0.5, fake, 1, 20.0, fake + 1, fake, None]
    for i, v, code in ((0, None, -2), (4, None, -2), (11, None, -2), (14, None, -2), (1, 0, -1), (2, 0, -1), (12, 0, -1),
                       (8, 0.0, -2), (8, float("nan"), -2), (9, -1.0, -2), (10, float("inf"), -2), (13, 0.0, -2),
                       (13, -2.0, -2), (13, float("nan"), -2), (13, float("inf"), -2), (14, fake, -2)):
        a = list(args)
        a[i] = v
        assert lib.rb_denoise_merge(*a) == code, (i, v)
    assert lib.rb_noise_sums(None, 1, 8, 8, fake, None) == -2
    assert lib.rb_noise_sums(fake, 1, 8, 8, None, None) == -2
    assert lib.rb_noise_sums(fake, 0, 8, 8, fake, None) == -1
    assert lib.rb_noise_sums(fake, 1, 2, 8, fake, None) == -1
    assert lib.rb_noise_sums(fake, 70000, 8, 8, fake, None) == -1
