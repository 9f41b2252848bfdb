"""F16 on the CPU: the centre-containment rule of the resized blend's masks, the oracle's reduction to the plain blend at
equal sizes, the uint8 round trip that makes t = 0 the input frame, the argument checks of
rb_frame_synthesize_pairs_resized / _items_resized, and the CLI's --native-frames / --flow-size refusals."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import interp_oracle
import native_oracle as N
from test_fps import BAD_ARG, BAD_SHAPE, _f, _i, _refused
from test_video_interp import quantise

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")


# ---- the nearest rule --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 7, 57, 432, 1024])
def test_nearest_identity_at_equal_sizes(n):
    assert np.array_equal(N.nearest_index(n, n), np.arange(n))


@pytest.mark.parametrize("src,dst", [(432, 1080), (1024, 1920), (544, 2160), (960, 3840), (37, 100), (53, 141),
                                     (100, 37), (1, 9), (9, 1), (1080, 432)])
def test_nearest_in_range_and_contains_centre(src, dst):
    from fractions import Fraction
    idx = N.nearest_index(src, dst)
    assert idx.dtype == np.int64 and idx.min() >= 0 and idx.max() <= src - 1
    assert np.all(np.diff(idx) >= 0)
    for d in range(dst):  # output centre (d + 1/2) dst^-1 of the extent lies in source cell [i, i + 1) src^-1
        c = Fraction(2 * d + 1, 2 * dst) * src
        assert idx[d] <= c < idx[d] + 1, (d, idx[d], c)


def test_nearest_uses_64_bit_products():
    for src, dst in ((2160, 3840), (40000, 60000), (65535, 2 ** 31 - 1)):
        d = np.array([0, dst // 3, dst - 1], dtype=np.int64)
        want = [((2 * int(x) + 1) * src) // (2 * dst) for x in d]
        got = ((2 * d + 1) * np.int64(src)) // (2 * np.int64(dst))
        assert got.tolist() == want
        assert N.nearest_index(src, min(dst, 4096))[-1] <= src - 1


def test_nearest_is_not_cv2_nearest():
    cv2 = pytest.importorskip("cv2")
    H, W, Hs, Ws = 432, 1024, 1080, 1920
    rows = np.repeat(np.arange(H, dtype=np.uint16)[:, None], W, 1)
    cols = np.repeat(np.arange(W, dtype=np.uint16)[None, :], H, 0)
    for interp in (cv2.INTER_NEAREST, cv2.INTER_NEAREST_EXACT):
        got_r = cv2.resize(rows, (Ws, Hs), interpolation=interp)[:, 0].astype(np.int64)
        got_c = cv2.resize(cols, (Ws, Hs), interpolation=interp)[0].astype(np.int64)
        assert not (np.array_equal(got_r, N.nearest_index(H, Hs)) and np.array_equal(got_c, N.nearest_index(W, Ws)))


# ---- the oracle --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("u8", [True, False])
def test_oracle_reduces_to_synthesize_at_equal_sizes(u8):
    rng = np.random.default_rng(3)
    B, H, W = 2, 23, 31
    frames = [rng.integers(0, 256, (B, H, W, 3)).astype(np.uint8) if u8 else
              rng.uniform(-0.1, 1.1, (B, H, W, 3)).astype(np.float32) for _ in range(2)]
    f0, f1 = (rng.normal(0, 4, (B, H, W, 2)).astype(np.float32) for _ in range(2))
    f0[0, 3, 4] = np.nan
    e0, e1 = ((rng.random((B, H, W)) < 0.3).astype(np.uint8) for _ in range(2))
    for t in (0.0, 0.3, 0.5, 1.0):
        got = N.synthesize_resized(*frames, f0, f1, e0, e1, t)
        want = interp_oracle.synthesize(*(N.prepare(f) for f in frames), f0, f1, e0, e1, t)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), t


def test_uint8_round_trip_is_identity():
    u = np.arange(256, dtype=np.uint8)
    assert np.array_equal(quantise(N.prepare(u[None, None, :, None].repeat(3, -1))[0, 0, :, 0]), u)


def test_oracle_t0_returns_frame0_bytes():
    rng = np.random.default_rng(4)
    frames = [rng.integers(0, 256, (1, 40, 60, 3)).astype(np.uint8) for _ in range(2)]
    f0 = np.zeros((1, 16, 24, 2), np.float32)  # a zero flow to frame 0: every pixel samples itself
    f1 = rng.normal(0, 3, (1, 16, 24, 2)).astype(np.float32)
    e0 = np.zeros((1, 16, 24), np.uint8)
    e1 = (rng.random((1, 16, 24)) < 0.5).astype(np.uint8)
    assert np.array_equal(quantise(N.synthesize_resized(*frames, f0, f1, e0, e1, 0.0)), frames[0])


# ---- argument checks of both entries (host pointers: a launch would fail, not return these codes) -----------------
def _entries():
    from raft_b200 import capi
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def pairs(f0s=p, f1s=p, fu8=0, Hs=8, Ws=8, f0=p, f1=p, e0=p, e1=p, H=4, W=4, smp=None, ts=_f(0.5), n=1, out=p,
              u8=0, bgr=0, B=1):
        return capi.lib.rb_frame_synthesize_pairs_resized(f0s, f1s, fu8, Hs, Ws, f0, f1, e0, e1, H, W, ts, n, out, u8,
                                                          bgr, B, None)

    def items(f0s=p, f1s=p, fu8=0, Hs=8, Ws=8, f0=p, f1=p, e0=p, e1=p, H=4, W=4, smp=_i(0), ts=_f(0.5), n=1, out=p,
              u8=0, bgr=0, B=1):
        return capi.lib.rb_frame_synthesize_items_resized(f0s, f1s, fu8, Hs, Ws, f0, f1, e0, e1, H, W, smp, ts, n, out,
                                                          u8, bgr, B, None)
    return {"pairs": pairs, "items": items}


@pytest.mark.parametrize("entry", ["pairs", "items"])
def test_resized_argument_checks(entry):
    syn = _entries()[entry]
    name = f"rb_frame_synthesize_{entry}_resized".encode()
    nulls = ["f0s", "f1s", "f0", "f1", "e0", "e1", "ts", "out"] + (["smp"] if entry == "items" else [])
    for k in nulls:
        _refused(syn(**{k: None}), BAD_ARG, name, b"null")
    many = {"smp": _i(*([0] * 65)), "ts": _f(*([0.5] * 65))}
    for n in (0, -1, 65):
        _refused(syn(**many, n=n), BAD_ARG, name, b"(1..64)")
    for fu8, u8, bgr in ((2, 0, 0), (-1, 0, 0), (0, 2, 0), (0, -1, 0), (0, 1, 2), (0, 0, -1)):
        _refused(syn(fu8=fu8, u8=u8, bgr=bgr), BAD_ARG, name, b"0 or 1")
    what = b"item_t[1]" if entry == "items" else b"ts[1]"
    for t in (-0.01, 1.01, float("nan"), float("inf"), -float("inf")):
        _refused(syn(smp=_i(0, 0), ts=_f(0.5, t), n=2), BAD_ARG, name, what, b"[0, 1]")
    for kw in ({"B": 0}, {"H": 0}, {"W": -1}, {"Hs": 0}, {"Ws": -2}):
        _refused(syn(**kw), BAD_SHAPE, name, b"bad shape")
    _refused(syn(Hs=65536, Ws=65536), BAD_SHAPE, name, b"32-bit")  # Hs*Ws = 2^32
    _refused(syn(Hs=3, Ws=2 ** 31 - 1), BAD_SHAPE, name, b"32-bit")
    if entry == "items":
        for smp in (_i(0, 3), _i(-1, 0)):
            _refused(syn(smp=smp, ts=_f(0.5, 0.5), n=2, B=3), BAD_ARG, name, b"item_sample[", b"outside [0, 3)")


# ---- CLI ---------------------------------------------------------------------------------------------------------
def _frames_dir(tmp_path):
    for k in range(2):
        (tmp_path / f"f{k}.png").write_bytes(b"")  # never decoded: every refusal comes first
    return str(tmp_path)


@pytest.mark.parametrize("argv,what", [
    (["--interpolate", "0.5", "--native-frames", "--keep-size"], "--keep-size"),
    (["-m", "val", "--data", "x", "--dataset", "vimeo", "--native-frames"], "-m val"),
    (["--native-frames"], "interpolation mode"),
    (["--path", "@", "--native-frames"], "interpolation mode"),
    (["--flow-size", "544", "960", "--keep-size"], "--keep-size"),
    (["-m", "val", "--data", "x", "--dataset", "sintel", "--flow-size", "544", "960"], "-m val"),
    (["--flow-size", "56", "960"], "at least 57"),
    (["--flow-size", "544", "40"], "at least 57"),
    (["--flow-size", "120", "960", "--upstream"], "at least 121"),
    (["--path", "@", "--input-fps", "24", "--fps", "60", "--flow-size", "100", "56"], "at least 57")])
def test_cli_native_refusals(tmp_path, argv, what):
    d = _frames_dir(tmp_path)
    argv = [d if a == "@" else a for a in argv]
    r = subprocess.run([sys.executable, CLI] + argv, capture_output=True, text=True, timeout=120)
    error = r.stderr.strip().splitlines()[-1]  # the usage lines above it list every flag
    assert r.returncode == 2 and what in error, r.stderr


def test_cli_native_refusals_import_no_torch(tmp_path):
    """The flag refusals come before torch (and so the GPU) is imported."""
    code = ("import sys; sys.path.insert(0, sys.argv[1]); import infer_raft\n"
            "try:\n    infer_raft.main(sys.argv[2:])\nexcept SystemExit as e:\n    print(e.code, 'torch' in sys.modules)")
    d = _frames_dir(tmp_path)
    for argv in (["--native-frames"], ["--interpolate", "0.5", "--native-frames", "--keep-size"],
                 ["--flow-size", "50", "960"], ["--path", d, "--native-frames"],
                 ["--path", d, "--input-fps", "24", "--fps", "60", "--flow-size", "544", "960", "--keep-size"]):
        r = subprocess.run([sys.executable, "-c", code, os.path.dirname(CLI)] + argv, capture_output=True, text=True,
                           timeout=120)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)
