"""F15 on the CPU: the numpy oracle of the scene-cut scores (np.bincount histograms, then the score formula), the pure
rules of raft_b200.video -- which input frame stands in for a cut pair's frames (cut_copy, split_cut_items), which pairs
of a warm-started video run cold (cold_start), the cut pairs of a pass (pass_cuts) -- the CLI's --scene-cut refusals and
the argument checks of rb_scene_cut_scores."""
import ctypes
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
BINS = 512


# ---- oracle ------------------------------------------------------------------------------------------------------
def scene_hist(frames):
    """[N,H,W,3] uint8 -> [N,512] int32: bin (c0 >> 5) 64 + (c1 >> 5) 8 + (c2 >> 5) of every pixel, counted once."""
    q = frames.astype(np.int64) >> 5
    bins = (q[..., 0] * 64 + q[..., 1] * 8 + q[..., 2]).reshape(len(frames), -1)
    return np.stack([np.bincount(b, minlength=BINS) for b in bins]).astype(np.int32)


def scene_scores(hist, npix):
    """fl32((H W - sum_b min(hist[k][b], hist[k+1][b])) / (H W)), the quotient in fp64."""
    inter = np.minimum(hist[:-1].astype(np.int64), hist[1:].astype(np.int64)).sum(axis=1)
    return ((npix - inter).astype(np.float64) / float(npix)).astype(np.float32)


def oracle(frames):
    h = scene_hist(frames)
    return scene_scores(h, frames.shape[1] * frames.shape[2]), h


def oracle_cuts(scores, thr):
    return [k for k, s in enumerate(scores) if float(s) > thr]


def test_oracle_values():
    rng = np.random.default_rng(1)
    f = rng.integers(0, 256, (4, 9, 7, 3), dtype=np.uint8)
    s, h = oracle(f)
    assert h.dtype == np.int32 and h.shape == (4, BINS) and (h.sum(axis=1) == 63).all()
    assert s.dtype == np.float32 and s.shape == (3,) and ((0 <= s) & (s <= 1)).all()
    # identical frames score exactly 0, frames without a common bin exactly 1
    same = np.repeat(f[:1], 3, axis=0)
    assert (oracle(same)[0] == 0.0).all()
    dark, light = np.full((1, 5, 6, 3), 31, np.uint8), np.full((1, 5, 6, 3), 32, np.uint8)
    assert oracle(np.concatenate([dark, light, dark]))[0].tolist() == [1.0, 1.0]
    # one pixel of 30 moved to another bin: 1/30 rounded once
    g = np.concatenate([dark, dark])
    g[1, 2, 3, 1] = 200
    assert oracle(g)[0][0] == np.float32(1.0 / 30.0)
    # a channel permutation of both frames permutes the bins: the scores do not change
    for perm in ([2, 1, 0], [1, 2, 0]):
        assert np.array_equal(oracle(f[..., perm])[0], s)
    # the bin formula on the corners of the cube
    px = np.array([[[[0, 0, 0], [255, 255, 255], [32, 0, 0], [0, 32, 0], [0, 0, 32], [224, 31, 95]]]], np.uint8)
    assert np.nonzero(scene_hist(px)[0])[0].tolist() == sorted([0, 511, 64, 8, 1, 7 * 64 + 0 * 8 + 2])


# ---- pure rules --------------------------------------------------------------------------------------------------
def test_cut_copy_rule():
    from raft_b200.video import cut_copy
    assert cut_copy(3, 0.25) == 3 and cut_copy(3, 0.5) == 3  # t = 0.5 goes to the earlier frame
    assert cut_copy(3, float(np.nextafter(0.5, 1.0))) == 4 and cut_copy(3, 0.75) == 4
    assert cut_copy(0, 0.2) == 0 and cut_copy(0, 0.8) == 1  # a cut at k = 0
    assert cut_copy(11, 0.6) == 12  # a cut at the last pair copies the last frame


def test_split_cut_items():
    from raft_b200.video import split_cut_items
    items = [(1, 0, 0.4), (2, 0, 0.8), (3, 1, 0.2), (4, 1, 0.6), (6, 2, 0.4), (7, 2, 0.8), (8, 3, 0.2), (9, 3, 0.5)]
    kept, copies = split_cut_items(items, [0, 3])  # the first and the last pair
    assert kept == [(3, 1, 0.2), (4, 1, 0.6), (6, 2, 0.4), (7, 2, 0.8)]
    assert copies == [(1, 0), (2, 1), (8, 3), (9, 3)]
    assert split_cut_items(items, []) == (items, [])
    assert split_cut_items(items, [0, 1, 2, 3]) == ([], [(1, 0), (2, 1), (3, 1), (4, 2), (6, 2), (7, 3), (8, 3), (9, 3)])


def test_cold_start_rule():
    from raft_b200.video import cold_start
    cuts = [0, 4, 8, 9, 11]  # 8 and 9: frame 9 is a one-frame shot
    cold = [k for k in range(12) if cold_start(k, cuts)]
    assert cold == [0, 1, 4, 5, 8, 9, 10, 11]
    assert [k for k in range(6) if cold_start(k, [])] == [0]
    assert [k for k in range(6) if cold_start(k, [2, 3])] == [0, 2, 3, 4]


def _shots(cuts, n_frames):
    """The frames of each shot: a cut at k ends a shot at frame k."""
    shots, cur = [], [0]
    for i in range(1, n_frames):
        if i - 1 in cuts:
            shots.append(cur)
            cur = []
        cur.append(i)
    return shots + [cur]


def test_cold_start_restarts_each_shot():
    """Warm pairs are exactly the pairs after the first of each shot, so each shot's chain is the chain on it alone."""
    from raft_b200.video import cold_start
    rng = np.random.default_rng(2)
    for _ in range(50):
        n = int(rng.integers(2, 20))
        cuts = sorted(int(k) for k in rng.choice(n - 1, int(rng.integers(0, n)), replace=False))
        warm = {k for k in range(n - 1) if not cold_start(k, cuts)}
        want = {s[i] for s in _shots(cuts, n) for i in range(1, len(s) - 1)}
        assert warm == want, (n, cuts)


def test_pass_cuts_ignores_idle_rows():
    from raft_b200.video import pass_cuts
    assert pass_cuts([6, 7, 8], [0.1, 0.9, 0.5], 0.5) == [7]  # strictly above the threshold
    assert pass_cuts([9, None, None], [0.9, 1.0, 1.0], 0.5) == [9]
    assert pass_cuts([0, 1], [1.0, 1.0], 1.0) == []


def test_check_scene_cut():
    from raft_b200.video import check_scene_cut
    assert check_scene_cut(0) == 0.0 and check_scene_cut("0.25") == 0.25 and check_scene_cut(1) == 1.0
    for bad in (-0.01, 1.01, float("nan"), float("inf"), "x", None):
        with pytest.raises(ValueError, match="scene_cut"):
            check_scene_cut(bad)


@pytest.mark.parametrize("batch", [1, 3, 8])
def test_fps_items_mapped_to_copies(batch):
    """24 -> 60 over 13 frames with cuts at 0, 4, 8, 9 and 11: every output frame is written once; a frame of a cut pair
    copies the input frame nearer to its time s, every other fractional s stays an item."""
    from raft_b200.video import fps_schedule, split_cut_items
    cuts = [0, 4, 8, 9, 11]
    passes = fps_schedule(13, 24, 60, batch)
    seen = {}
    for p in passes:
        items, copies = split_cut_items(p.items, cuts)
        for n, k, t in items:
            assert k not in cuts
            seen[n] = ("item", k, t)
        for n, i in p.copies + copies:
            assert i in p.frames
            assert n not in seen
            seen[n] = ("copy", i)
    assert sorted(seen) == list(range(31))
    for n, what in seen.items():
        s = Fraction(n * 24, 60)
        k = s.numerator // s.denominator
        if s.denominator == 1:
            assert what == ("copy", k)
        elif k in cuts:
            assert what == ("copy", k if s - k <= Fraction(1, 2) else k + 1), n
        else:
            assert what == ("item", k, float(s - k))


# ---- CLI ---------------------------------------------------------------------------------------------------------
def _frames_dir(tmp_path):
    for k in range(2):
        (tmp_path / f"f{k}.png").write_bytes(b"")  # never decoded: every refusal comes first
    return str(tmp_path)


@pytest.mark.parametrize("argv,what", [
    (["--scene-cut", "0.5"], "--interpolate, --input-fps/--fps or --warm-start"),
    (["--scene-cut", "0.5", "--batch", "4"], "--interpolate, --input-fps/--fps or --warm-start"),
    (["--scene-cut", "0.5", "--warm-start", "--nopath"], "--path"),
    (["--scene-cut", "0.5", "--interpolate", "0.5", "--nopath"], "--path"),
    (["--scene-cut", "-0.1", "--warm-start"], "[0, 1]"), (["--scene-cut", "1.5", "--warm-start"], "[0, 1]"),
    (["--scene-cut", "nan", "--warm-start"], "[0, 1]"), (["--scene-cut", "inf", "--warm-start"], "[0, 1]"),
    (["--scene-cut", "abc", "--warm-start"], "--scene-cut"),
    (["--scene-cut", "0.5", "--warm-start", "-m", "val", "--data", "x", "--dataset", "sintel"], "-m val"),
    (["--scene-cut", "0.5", "--warm-start", "--batch", "2"], "--batch 1"),
    (["--scene-cut", "0.5", "--interpolate", "0.5", "--warm-start"], "--warm-start"),
    (["--scene-cut", "0.5", "--input-fps", "24", "--fps", "60", "--warm-start"], "--warm-start"),
    (["--scene-cut", "0.5", "--input-fps", "24", "--fps", "24"], "exceed")])
def test_cli_scene_cut_refusals(tmp_path, argv, what):
    path = [] if "--nopath" in argv else ["--path", _frames_dir(tmp_path)]
    r = subprocess.run([sys.executable, CLI] + path + [a for a in argv if a != "--nopath"], capture_output=True,
                       text=True, timeout=120)
    error = r.stderr.strip().splitlines()[-1]  # the usage lines above it list every flag
    assert r.returncode == 2 and what in error, r.stderr


def test_cli_scene_cut_refusals_import_no_torch(tmp_path):
    """Every --scene-cut refusal comes before torch (and so the GPU) is imported."""
    code = ("import sys; sys.path.insert(0, sys.argv[1]); import infer_raft\n"
            "try:\n    infer_raft.main(sys.argv[2:])\nexcept SystemExit as e:\n    print(e.code, 'torch' in sys.modules)")
    d = _frames_dir(tmp_path)
    for argv in (["--path", d, "--scene-cut", "0.5"], ["--path", d, "--scene-cut", "2", "--warm-start"],
                 ["--scene-cut", "0.5", "--interpolate", "0.5"],
                 ["--path", d, "--scene-cut", "0.5", "--warm-start", "--batch", "3"]):
        r = subprocess.run([sys.executable, "-c", code, os.path.dirname(CLI)] + argv, capture_output=True, text=True,
                           timeout=120)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)


# ---- argument checks of rb_scene_cut_scores (host pointers: a launch would fail, not return these codes) ----------
def test_scene_cut_scores_argument_checks():
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG = -1, -2
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def refused(rc, code, *words):
        assert rc == code, (rc, code)
        msg = lib.rb_last_error()
        assert all(w in msg for w in words), msg

    for f, h, s in ((None, p, p), (p, None, p), (p, p, None)):
        refused(lib.rb_scene_cut_scores(f, 3, 4, 4, h, s, None), BAD_ARG, b"rb_scene_cut_scores", b"null")
    for n in (1, 0, -2):
        refused(lib.rb_scene_cut_scores(p, n, 4, 4, p, p, None), BAD_SHAPE, b"rb_scene_cut_scores", b"two frames")
    for H, W in ((0, 4), (4, 0), (-1, 4), (4, -3)):
        refused(lib.rb_scene_cut_scores(p, 3, H, W, p, p, None), BAD_SHAPE, b"rb_scene_cut_scores", b"bad shape")
    refused(lib.rb_scene_cut_scores(p, 2, 32768, 65536, p, p, None), BAD_SHAPE, b"2^31")  # H*W == 2^31
    refused(lib.rb_scene_cut_scores(p, 2, 65536, 65536, p, p, None), BAD_SHAPE, b"2^31")
    refused(lib.rb_scene_cut_scores(p, 5000, 46340, 46340, p, p, None), BAD_SHAPE, b"one grid")
