"""F14 on the CPU: the output schedule of frame-rate conversion (raft_b200.video.fps_schedule), its rate parsing, the
item checks of RaftEngine.interpolate_sequence_at, the CLI's --input-fps / --fps refusals, and the argument checks of
rb_flow_reverse_items and rb_frame_synthesize_items."""
import ctypes
import os
import subprocess
import sys
from fractions import Fraction

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")

CONVERSIONS = [(24, 60), (25, 60), (24, 25), ("24000/1001", 60), (30, 60), ("24000/1001", "60000/1001")]


# ---- schedule ----------------------------------------------------------------------------------------------------
def _flat(passes):
    return (sorted(it for p in passes for it in p.items), sorted(c for p in passes for c in p.copies))


@pytest.mark.parametrize("fin,fout", CONVERSIONS)
@pytest.mark.parametrize("n_frames", [2, 3, 10, 49])
def test_fps_schedule(fin, fout, n_frames):
    from raft_b200.video import fps_schedule, interp_schedule
    ratio = Fraction(fin) / Fraction(fout)
    count = (n_frames - 1) * Fraction(fout) / Fraction(fin)
    count = count.numerator // count.denominator + 1
    flat = None
    for batch in (1, 3, 8):
        passes = fps_schedule(n_frames, fin, fout, batch)
        plain = interp_schedule(n_frames, batch)
        assert [(p.frames, p.pairs) for p in passes] == [(p.frames, p.pairs) for p in plain]
        ns = []
        for p in passes:
            assert p.items, "every pass interpolates: an up-conversion puts a frame strictly inside every pair"
            for n, k, t in p.items:
                s = n * ratio
                assert s.denominator != 1 and k == s.numerator // s.denominator and t == float(s - k)
                assert 0.0 < t < 1.0 and k in p.pairs  # the pass that holds pair k
                ns.append(n)
            for n, i in p.copies:
                assert n * ratio == i and i in p.frames  # copies fall exactly at the integer times
                ns.append(n)
        assert sorted(ns) == list(range(count))  # every output index once
        if flat is None:
            flat = _flat(passes)
        assert _flat(passes) == flat  # the same schedule for every batch


def test_fps_schedule_24_to_60_phases():
    from raft_b200.video import fps_schedule
    (p,) = fps_schedule(5, 24, 60, 8)
    assert p.copies == [(0, 0), (5, 2), (10, 4)]
    assert [(k, t) for _, k, t in p.items] == [(0, 0.4), (0, 0.8), (1, 0.2), (1, 0.6), (2, 0.4), (2, 0.8), (3, 0.2),
                                                (3, 0.6)]


def test_fps_schedule_rates_and_errors():
    from raft_b200.video import fps_schedule, parse_rate
    assert parse_rate("59.94") == parse_rate(59.94) == Fraction(2997, 50)
    assert parse_rate("60000/1001") == Fraction(60000, 1001) and parse_rate(60) == 60
    assert _flat(fps_schedule(20, "23.976", "59.94", 4)) == _flat(fps_schedule(20, Fraction(23976, 1000), 59.94, 4))
    for bad in ("0", "-24", "abc", "inf", "nan", "1/0", None, float("inf"), 0):
        with pytest.raises(ValueError, match="frame rate"):
            parse_rate(bad)
    for fin, fout in ((60, 60), (60, 24), ("60000/1001", "59.94")):
        with pytest.raises(ValueError, match="exceed"):
            fps_schedule(10, fin, fout, 8)
    for n, batch in ((1, 8), (10, 0)):
        with pytest.raises(ValueError):
            fps_schedule(n, 24, 60, batch)


def test_interpolate_sequence_at_item_checks():
    from raft_b200.engine import _items
    assert _items([(0, 0.5), (2, 1), (1, 0.0)], 3) == ([0, 2, 1], [0.5, 1.0, 0.0])
    for bad in ([], [(3, 0.5)], [(-1, 0.5)], [(0, 1.01)], [(0, -0.1)], [(0, float("nan"))], [(0.5, 0.5)], [(0,)],
                [("a", 0.5)], [(0, 0.5, 1)]):
        with pytest.raises(ValueError):
            _items(bad, 3)


# ---- CLI ---------------------------------------------------------------------------------------------------------
def _frames_dir(tmp_path):
    for k in range(2):
        (tmp_path / f"f{k}.png").write_bytes(b"")  # never decoded: every refusal comes first
    return str(tmp_path)


@pytest.mark.parametrize("argv,what", [
    (["--fps", "60"], "--input-fps"), (["--input-fps", "24"], "--fps"),
    (["--input-fps", "24", "--fps", "60", "--nopath"], "--path"),
    (["--input-fps", "abc", "--fps", "60"], "--input-fps"), (["--input-fps", "24", "--fps", "1/0"], "--fps"),
    (["--input-fps", "0", "--fps", "60"], "--input-fps"), (["--input-fps", "24", "--fps", "-60"], "--fps"),
    (["--input-fps", "inf", "--fps", "60"], "--input-fps"), (["--input-fps", "24", "--fps", "nan"], "--fps"),
    (["--input-fps", "60", "--fps", "60"], "exceed"), (["--input-fps", "60", "--fps", "24"], "exceed"),
    (["--input-fps", "24", "--fps", "60", "--interpolate", "0.5"], "--interpolate"),
    (["--input-fps", "24", "--fps", "60", "--warm-start"], "--warm-start"),
    (["--input-fps", "24", "--fps", "60", "--native-flow"], "--native-flow"),
    (["--input-fps", "24", "--fps", "60", "--flo", "x"], "--flo"),
    (["--input-fps", "24", "--fps", "60", "--npy", "x"], "--npy"),
    (["--input-fps", "24", "--fps", "60", "--bidirectional"], "--bidirectional")])
def test_cli_fps_refusals(tmp_path, argv, what):
    path = [] if "--nopath" in argv else ["--path", _frames_dir(tmp_path)]
    r = subprocess.run([sys.executable, CLI] + path + [a for a in argv if a != "--nopath"], capture_output=True,
                       text=True, timeout=120)
    error = r.stderr.strip().splitlines()[-1]  # the usage lines above it list every flag
    assert r.returncode == 2 and what in error, r.stderr


def test_cli_fps_refusals_import_no_torch(tmp_path):
    """Every refusal, an empty frame directory included, comes before torch (and so the GPU) is imported."""
    code = ("import sys; sys.path.insert(0, sys.argv[1]); import infer_raft\n"
            "try:\n    infer_raft.main(sys.argv[2:])\nexcept SystemExit as e:\n    print(e.code, 'torch' in sys.modules)")
    d = _frames_dir(tmp_path)
    for argv in (["--path", d, "--fps", "60"], ["--path", d, "--input-fps", "24", "--fps", "24"],
                 ["--path", d, "--input-fps", "x", "--fps", "60"], ["--input-fps", "24", "--fps", "60"],
                 ["--path", d, "--input-fps", "24", "--fps", "60", "--flo", "x"],
                 ["--path", str(tmp_path / "empty"), "--input-fps", "24", "--fps", "60"],
                 ["--path", d, "--input-fps", "24", "--fps", "60", "--batch", "0"]):
        r = subprocess.run([sys.executable, "-c", code, os.path.dirname(CLI)] + argv, capture_output=True, text=True,
                           timeout=120)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)


# ---- argument checks of the item entries (host pointers: a launch would fail, not return these codes) -------------
BAD_SHAPE, BAD_ARG, WORKSPACE = -1, -2, -5


def _refused(rc, code, *words):
    from raft_b200 import capi
    assert rc == code, (rc, code)
    msg = capi.lib.rb_last_error()
    assert all(w in msg for w in words), msg


def _f(*v):
    return (ctypes.c_float * max(1, len(v)))(*v)


def _i(*v):
    return (ctypes.c_int32 * max(1, len(v)))(*v)


def test_reverse_items_argument_checks():
    from raft_b200 import capi
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def rev(flow=p, B=2, smp=_i(0, 1), steps=_f(0.5, 1.0), n=2, ft=p, empty=p, multi=p, H=4, W=4, ws=p, nbytes=1 << 20):
        return capi.lib.rb_flow_reverse_items(flow, B, smp, steps, n, ft, empty, multi, H, W, ws, nbytes, None)

    for kw in ({"flow": None}, {"smp": None}, {"steps": None}, {"ft": None}, {"empty": None}, {"multi": None},
               {"ws": None}):
        _refused(rev(**kw), BAD_ARG, b"rb_flow_reverse_items", b"null")
    for n in (0, -1, 65):
        _refused(rev(smp=_i(*([0] * 65)), steps=_f(*([0.5] * 65)), n=n), BAD_ARG, b"items (1..64)")
    for B, H, W in ((0, 4, 4), (2, 0, 4), (2, 4, -1)):
        _refused(rev(B=B, H=H, W=W), BAD_SHAPE, b"bad shape")
    _refused(rev(n=1, H=65535, W=65537), BAD_SHAPE, b"2^32")  # n_items*H*W + 1 == 2^32
    _refused(rev(H=32768, W=65536), BAD_SHAPE, b"2^32")  # two items reach 2^32
    for smp in (_i(0, 2), _i(-1, 0)):
        _refused(rev(smp=smp), BAD_ARG, b"item_sample[", b"outside [0, 2)")
    for bad in (float("nan"), float("inf"), -float("inf")):
        _refused(rev(steps=_f(0.5, bad)), BAD_ARG, b"item_step[1]", b"finite")
    _refused(rev(nbytes=64), WORKSPACE, b"too small")
    # 64 items, samples repeated and unsorted, are accepted up to the workspace check
    _refused(rev(smp=_i(*[(7 * i) % 3 for i in range(64)]), B=3, steps=_f(*([0.25] * 64)), n=64, nbytes=64), WORKSPACE,
             b"too small")


def test_synthesize_items_argument_checks():
    from raft_b200 import capi
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def syn(f0s=p, f1s=p, Hp=8, Wp=8, top=0, left=0, f0=p, f1=p, e0=p, e1=p, smp=_i(0), ts=_f(0.5), n=1, out=p, u8=0,
            bgr=0, B=1, H=8, W=8):
        return capi.lib.rb_frame_synthesize_items(f0s, f1s, Hp, Wp, top, left, f0, f1, e0, e1, smp, ts, n, out, u8, bgr,
                                                  B, H, W, None)

    for kw in ({"f0s": None}, {"f1s": None}, {"f0": None}, {"f1": None}, {"e0": None}, {"e1": None}, {"smp": None},
               {"ts": None}, {"out": None}):
        _refused(syn(**kw), BAD_ARG, b"rb_frame_synthesize_items", b"null")
    for n in (0, -3, 65):
        _refused(syn(smp=_i(*([0] * 65)), ts=_f(*([0.5] * 65)), n=n), BAD_ARG, b"items (1..64)")
    for u8, bgr in ((2, 0), (-1, 0), (1, 2), (0, -1)):
        _refused(syn(u8=u8, bgr=bgr), BAD_ARG, b"0 or 1")
    for t in (-0.01, 1.01, float("nan"), float("inf")):
        _refused(syn(smp=_i(0, 0), ts=_f(0.5, t), n=2), BAD_ARG, b"item_t[1]", b"[0, 1]")
    for B, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, -2)):
        _refused(syn(B=B, H=H, W=W), BAD_SHAPE, b"bad shape")
    for smp in (_i(0, 3), _i(-1, 0)):
        _refused(syn(smp=smp, ts=_f(0.5, 0.5), n=2, B=3), BAD_ARG, b"item_sample[", b"outside [0, 3)")
    for Hp, Wp, top, left in ((7, 8, 0, 0), (8, 7, 0, 0), (9, 8, 2, 0), (8, 8, -1, 0), (8, 8, 0, -1)):
        _refused(syn(Hp=Hp, Wp=Wp, top=top, left=left), BAD_SHAPE, b"outside")
