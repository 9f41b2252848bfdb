"""F32 on the CPU: shutter_schedule()'s sample times, clamping, pass split and m = 1 anchor, the shutter and density
checks, the CLI's --shutter refusals, the C entries' table refusals, and the quality of the numpy oracle's exposure
against the true box average of a high-frame-rate known-path clip."""
import math
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import shutter_oracle as SO
from vfi_oracle import frame_stats, psnr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")


def _flat(passes):
    return [s for p in passes for s in p.samples]


def _expected(F, fin, fout, A, D, cuts=()):
    """The samples by the formula of include/raft_b200.h, written out independently of shutter_schedule."""
    fin, fout, A = Fraction(fin), Fraction(fout), Fraction(A)
    e = A / 360 * fin / fout
    m = max(1, math.ceil(D * e))
    last = F - 1
    out = []
    for n in range(int(last * fout / fin) + 1):
        s = n * fin / fout
        k = math.floor(s)
        home = k if s == k or k not in cuts else (k if s - k <= Fraction(1, 2) else k + 1)
        a = max([c + 1 for c in cuts if c < home], default=0)
        b = min([c for c in cuts if c >= home], default=last)
        for j in range(m):
            u = min(max(s - e / 2 + (j + Fraction(1, 2)) * e / m, a), b)
            out.append((n, int(u), None) if u == int(u) else (n, math.floor(u), float(u - math.floor(u))))
    return out, m


@pytest.mark.parametrize("F,fin,fout,A,D", [(21, 60, 24, 180, 16), (9, 24, 60, 360, 16), (9, 24, 60, 180, 4),
                                            (8, 30, 30, 315, 8), (10, "24000/1001", "60000/1001", 270, 10),
                                            (33, 240, 30, 360, 2), (12, 50, 25, 90, 3)])
def test_schedule_sample_times(F, fin, fout, A, D):
    from raft_b200.video import exposure, parse_rate, shutter_schedule
    want, m = _expected(F, parse_rate(fin), parse_rate(fout), A, D)
    assert exposure(fin, fout, A, D)[1] == m
    for batch in (1, 4, 8):
        assert _flat(shutter_schedule(F, fin, fout, A, D, batch)) == want


def test_schedule_60_to_24_at_180():
    """e = 1.25 input frames, m = 20 at density 16; frame 0's exposure starts at -0.625, so its first 10 samples hold
    frame 0, and the last output frame is floor(20 * 24 / 60) = 8 at s = 20."""
    from raft_b200.video import exposure, shutter_schedule
    assert exposure(60, 24, 180, 16) == (Fraction(5, 4), 20)
    flat = _flat(shutter_schedule(21, 60, 24, 180, 16, 8))
    rows = {}
    for n, i, t in flat:
        rows.setdefault(n, []).append((i, t))
    assert sorted(rows) == list(range(9)) and all(len(v) == 20 for v in rows.values())
    assert rows[0][:10] == [(0, None)] * 10 and rows[0][10] == (0, 0.03125)
    # s = 2.5: u_j = 1.875 + (j + 1/2) / 16
    assert rows[1] == [(math.floor(u), float(u - math.floor(u))) if u != int(u) else (int(u), None)
                       for u in (Fraction(15, 8) + Fraction(2 * j + 1, 32) for j in range(20))]
    assert rows[8][-10:] == [(20, None)] * 10


@pytest.mark.parametrize("batch", range(1, 10))
def test_rows_span_passes(batch):
    """Every batch runs the same samples in the same order; each pass runs item (k, t) when it holds pair k and frame i
    when it holds pair min(i, F - 2); opens / closes name the pass of each frame's first / last sample."""
    from raft_b200.video import interp_schedule, shutter_schedule
    F, T = 23, batch
    ref = _flat(shutter_schedule(F, 60, 24, 300, 12, 1))
    passes = shutter_schedule(F, 60, 24, 300, 12, batch)
    assert _flat(passes) == ref
    assert [(p.frames, p.pairs) for p in passes] == [(p.frames, p.pairs) for p in interp_schedule(F, batch)]
    for j, p in enumerate(passes):
        for n, i, t in p.samples:
            assert j == (i // T if t is not None else min(i, F - 2) // T)
        ns = [n for n, _, _ in p.samples]
        assert ns == sorted(ns)
        assert p.opens == sorted(n for n in set(ns) if _first_pass(passes, n) == j)
        assert p.closes == sorted(n for n in set(ns) if _last_pass(passes, n) == j)


def _first_pass(passes, n):
    return next(j for j, p in enumerate(passes) if any(s[0] == n for s in p.samples))


def _last_pass(passes, n):
    return max(j for j, p in enumerate(passes) if any(s[0] == n for s in p.samples))


def test_a_row_spans_passes():
    from raft_b200.video import shutter_schedule
    passes = shutter_schedule(17, 60, 24, 360, 16, 2)
    assert any(set(p.closes) - set(p.opens) for p in passes[1:])


def test_clamping_at_ends_and_cuts():
    from raft_b200.video import shutter_schedule
    F, cuts = 13, [4, 8]
    flat = _flat(shutter_schedule(F, 30, 30, 360, 8, 3, cuts=cuts))
    assert flat == _expected(F, 30, 30, 360, 8, cuts)[0]
    rows = {}
    for n, i, t in flat:
        rows.setdefault(n, []).append(i + (0 if t is None else t))
    assert rows[0][:4] == [0] * 4 and rows[12][-4:] == [12] * 4  # the clip's ends hold their end frames
    assert rows[4][-4:] == [4] * 4 and rows[5][:4] == [5] * 4  # no exposure crosses cut pair 4
    assert all(min(v) >= 5 for n, v in rows.items() if n >= 5 and n <= 8) and all(max(v) <= 4 for n, v in rows.items()
                                                                                   if n <= 4)
    # inside a cut pair the frame belongs to cut_copy's shot: 30 -> 60 puts output 9 at s = 4.5 (frame 4's shot)
    r2 = {}
    for n, i, t in _flat(shutter_schedule(F, 30, 60, 360, 8, 3, cuts=cuts)):
        r2.setdefault(n, []).append(i + (0 if t is None else t))
    assert max(r2[9]) <= 4 and min(r2[11]) >= 5


def test_m1_is_the_conversion_without_shutter():
    """D e <= 1 gives m = 1 and u_0 = s: the items and copies of fps_schedule()."""
    from raft_b200.video import fps_schedule, shutter_schedule
    for fin, fout, A, D in ((24, 60, 90, 2), ("24000/1001", "60000/1001", 360, 1), (25, 60, 180, 4)):
        for batch in (1, 3, 8):
            a = shutter_schedule(30, fin, fout, A, D, batch)
            b = fps_schedule(30, fin, fout, batch)
            for p, q in zip(a, b):
                assert sorted(p.samples) == sorted([(n, k, t) for n, k, t in q.items] + [(n, i, None) for n, i in q.copies])
                assert p.opens == p.closes == sorted(n for n, _, _ in p.samples)


def test_fps_schedule_still_refuses_down_conversion():
    from raft_b200.video import fps_schedule
    for fin, fout in ((60, 24), (30, 30)):
        with pytest.raises(ValueError, match="goes up"):
            fps_schedule(10, fin, fout, 4)


@pytest.mark.parametrize("bad", [0, -10, 360.5, 1e9, "x", None, float("nan"), float("inf"), True])
def test_check_shutter_refusals(bad):
    from raft_b200.video import check_shutter
    with pytest.raises(ValueError, match="shutter angle"):
        check_shutter(bad)


def test_check_shutter_and_density():
    from raft_b200.video import check_density, check_shutter
    assert check_shutter(360) == 360 and check_shutter(172.8) == Fraction(864, 5) and check_shutter("315") == 315
    assert check_density(16) == 16 and check_density(np.int64(3)) == 3 and check_density(2.0) == 2
    for bad in (0, -1, 1.5, "x", None, True, float("nan")):
        with pytest.raises(ValueError, match="density"):
            check_density(bad)


def _frames_dir(tmp_path):
    import cv2
    d = tmp_path / "frames"
    d.mkdir(exist_ok=True)
    for i in range(3):
        cv2.imwrite(str(d / f"{i:04d}.png"), np.full((16, 16, 3), 10 * i, np.uint8))
    return str(d)


@pytest.mark.parametrize("argv,what", [
    (["--input-fps", "60", "--fps", "24"], "must exceed"),  # without --shutter nothing changes
    (["--shutter", "180"], "--shutter"),
    (["--fps", "24", "--shutter", "180"], "--shutter"),
    (["--input-fps", "60", "--fps", "24", "--shutter", "0"], "(0, 360]"),
    (["--input-fps", "60", "--fps", "24", "--shutter", "400"], "(0, 360]"),
    (["--input-fps", "60", "--fps", "24", "--shutter", "180", "--shutter-density", "0"], ">= 1"),
    (["--input-fps", "60", "--fps", "24", "--shutter-density", "4"], "goes with --shutter"),
    (["--interpolate", "0.5", "--shutter", "180"], "--shutter"),
    (["--denoise", "10", "--shutter", "180"], "--shutter"),
    (["--input-fps", "60", "--fps", "24", "--shutter", "180", "--warm-start"], "--warm-start")])
def test_cli_shutter_refusals(tmp_path, argv, what):
    r = subprocess.run([sys.executable, CLI, "--path", _frames_dir(tmp_path)] + argv, capture_output=True, text=True,
                       timeout=120)
    error = r.stderr.strip().splitlines()[-1]
    assert r.returncode == 2 and what in error, r.stderr


# ---- the C entries' table checks (host pointers: a launch would fail, not return these codes) ----------------------
BAD_SHAPE, BAD_ARG = -1, -2


def _call(resized=False, entries=((0, 0, 0.5),), rows=((0, 1, 1, 0, 0, 3),), n_slots=1, B=2, n_acc=2, n_out=1, bgr=0,
          frames_u8=1, acc=True, out=True, H=8, W=8):
    import ctypes
    from raft_b200 import capi
    buf = (ctypes.c_float * 16)()
    e = (capi.ExposeEntry * max(1, len(entries)))(*[capi.ExposeEntry(*x) for x in entries])
    r = (capi.ExposeRow * max(1, len(rows)))(*[capi.ExposeRow(*x) for x in rows])
    a = buf if acc else None
    o = buf if out else None
    if resized:
        return capi.lib.rb_frame_expose_items_resized(buf, frames_u8, H, W, buf, buf, buf, buf, H, W, n_slots, e,
                                                      len(entries), r, len(rows), a, n_acc, o, n_out, bgr, B, None)
    return capi.lib.rb_frame_expose_items(buf, H, W, 0, 0, buf, buf, buf, buf, n_slots, e, len(entries), r, len(rows),
                                          a, n_acc, o, n_out, bgr, B, H, W, None)


@pytest.mark.parametrize("resized", [False, True])
@pytest.mark.parametrize("kw,code,word", [
    (dict(entries=[(0, 0, 0.5)] * 65, rows=[(0, 65, 65, 0, 0, 3)]), BAD_ARG, "entries"),
    (dict(entries=(), rows=()), BAD_ARG, "entries"),
    (dict(entries=[(1, 0, 0.5)]), BAD_ARG, "slot"),
    (dict(entries=[(-2, 0, 0.5)]), BAD_ARG, "slot"),
    (dict(entries=[(0, 2, 0.5)]), BAD_ARG, "sample"),
    (dict(entries=[(-1, 3, 0.0)]), BAD_ARG, "sample"),
    (dict(entries=[(0, -1, 0.5)]), BAD_ARG, "sample"),
    (dict(entries=[(0, 0, 1.5)]), BAD_ARG, "t must"),
    (dict(entries=[(0, 0, float("nan"))]), BAD_ARG, "t must"),
    (dict(rows=[(0, 1, 0, 0, 0, 3)]), BAD_ARG, "m ="),
    (dict(rows=[(0, 2, 1, 0, 0, 3)]), BAD_ARG, "outside"),
    (dict(rows=[(0, 0, 1, 0, 0, 3)]), BAD_ARG, "outside"),
    (dict(rows=[(0, 1, 1, 0, 0, 4)]), BAD_ARG, "flags"),
    (dict(rows=[(0, 1, 1, 2, 0, 2)]), BAD_ARG, "acc"),
    (dict(rows=[(0, 1, 1, 0, 1, 3)]), BAD_ARG, "out"),
    (dict(entries=[(0, 0, 0.5)] * 2, rows=[(0, 1, 2, 0, 0, 1), (1, 1, 2, 0, 0, 2)]), BAD_ARG, "share acc"),
    (dict(entries=[(0, 0, 0.5)] * 2, rows=[(0, 1, 1, 0, 0, 3), (1, 1, 1, 1, 0, 3)], n_out=2), BAD_ARG, "share out"),
    (dict(rows=[(0, 1, 1, 0, 0, 2)], acc=False), BAD_ARG, "null"),
    (dict(out=False), BAD_ARG, "null"),
    (dict(bgr=2), BAD_ARG, "bgr"),
    (dict(B=0), BAD_SHAPE, "B ="),
    (dict(H=0), BAD_SHAPE, "shape")])
def test_expose_refusals(resized, kw, code, word):
    from raft_b200 import capi
    assert _call(resized, **kw) == code
    assert word in capi.lib.rb_last_error().decode()


def test_expose_resized_refuses_frames_flag():
    from raft_b200 import capi
    assert _call(True, frames_u8=2) == BAD_ARG and "frames_u8" in capi.lib.rb_last_error().decode()


# ---- quality: the exposure of 7 samples at stride 8 against the true box average ------------------------------------
def test_blur_beats_sharp_against_true_average():
    """A clip panned 1.5 / 0.7 pixels per frame at 8x the input rate: every 8th frame is an input, and the exposure of
    shutter 315 degrees at density 8 puts its 7 samples on the true frames 8c - 3 .. 8c + 3.  With exact flows the
    oracle's exposure is far closer to np.rint of their mean than the sharp input frame is."""
    from raft_b200.video import exposure, shutter_schedule
    S, M, hw, F = 8, 7, (64, 96), 6
    hi = SO.pan_clip(S * (F - 1) + 1, hw)
    frames = hi[::S]
    fw, bw = SO.pan_flows(F - 1, hw, S)
    A = Fraction(360 * M, S)
    _, m = exposure(1, 1, A, S)
    assert m == M
    (ps,) = shutter_schedule(F, 1, 1, A, S, F - 1)
    prepared = (frames.astype(np.float32) / np.float32(255)).astype(np.float32)
    out = SO.motion_blur(prepared, fw, bw, ps.samples, m)
    blur, sharp = [], []
    for c in range(1, F - 1):  # windows inside the clip
        gt = np.rint(hi[S * c - 3:S * c + 4].astype(np.float64).mean(0)).astype(np.uint8)
        crop = (slice(16, -16), slice(16, -16))  # away from the clamped borders of the reversal
        blur.append(psnr(frame_stats(out[c][crop][None], gt[crop][None])[0, 0], gt[crop].size))
        sharp.append(psnr(frame_stats(frames[c][crop][None], gt[crop][None])[0, 0], gt[crop].size))
    print(f"PSNR vs the true 7-frame average: exposure {np.mean(blur):.2f} dB, sharp frame {np.mean(sharp):.2f} dB")
    assert min(blur) > max(sharp) + 6.0, (blur, sharp)
