"""F13 on the CPU: the pass schedule and output numbering of raft_b200.video.video_interpolate, the CLI's --path
--interpolate refusals, the argument checks of rb_flow_reverse_multi and rb_frame_synthesize_pairs, and the numpy
restatement of the blend's uint8 output (quantise / synthesize_u8, on top of tests/interp_oracle.py)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import interp_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")


def quantise(x, bgr=False):
    """rb_frame_synthesize_pairs' uint8 output: min(max(rint(fl32(255 x)), 0), 255), NaN -> 0, channels reversed with
    bgr."""
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.rint(np.float32(255) * np.asarray(x, np.float32))
    q = np.fmin(np.fmax(q, np.float32(0)), np.float32(255)).astype(np.uint8)  # fmax(NaN, 0) = 0
    return q[..., ::-1] if bgr else q


def synthesize_u8(frame0, frame1, flow_t0, flow_t1, empty0, empty1, t, bgr=False):
    return quantise(O.synthesize(frame0, frame1, flow_t0, flow_t1, empty0, empty1, t), bgr)


# ---- quantisation ------------------------------------------------------------------------------------------------
def test_quantise_equals_cli_expression():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.uniform(-0.5, 1.5, 100000), (np.arange(512) + 0.5) / 255, np.arange(256) / 255,
                        [0.0, -0.0, 1.0, 1e-30, -1e30, 1e30, np.finfo(np.float32).max]]).astype(np.float32)
    with np.errstate(over="ignore"):
        want = np.clip(np.rint(255.0 * x), 0, 255).astype(np.uint8)  # infer_raft.py --interpolate
    assert np.array_equal(quantise(x), want)


def test_quantise_special_values_and_swap():
    x = np.array([[np.nan, np.inf, -np.inf], [0.5 / 255, 1.5 / 255, 2.5 / 255]], np.float32)
    q = quantise(x)
    assert q[0].tolist() == [0, 255, 0]
    assert q[1].tolist() == [0, 2, 2]  # ties to even
    assert np.array_equal(quantise(x, bgr=True), q[..., ::-1])


def test_synthesize_u8_at_the_end_points_recovers_the_frames():
    rng = np.random.default_rng(1)
    B, H, W = 2, 9, 13
    u8 = [rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8) for _ in range(2)]
    i0, i1 = (a.astype(np.float32) / np.float32(255) for a in u8)
    f = np.zeros((B, H, W, 2), np.float32)
    e = np.zeros((B, H, W), np.uint8)
    assert np.array_equal(synthesize_u8(i0, i1, f, f, e, e, 0.0), u8[0])
    assert np.array_equal(synthesize_u8(i0, i1, f, f, e, e, 1.0, bgr=True), u8[1][..., ::-1])


# ---- schedule and numbering --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_frames", [2, 3, 8, 9, 10, 17])
@pytest.mark.parametrize("batch", [1, 3, 8])
def test_interp_schedule(n_frames, batch):
    from raft_b200.video import interp_schedule
    passes = interp_schedule(n_frames, batch)
    assert len(passes) == -(-(n_frames - 1) // batch)
    assert [k for p in passes for k in p.pairs if k is not None] == list(range(n_frames - 1))
    for j, p in enumerate(passes):
        assert not p.carry and len(p.frames) == batch + 1 and len(p.pairs) == batch
        assert p.frames == [min(i, n_frames - 1) for i in range(j * batch, j * batch + batch + 1)]
        for r, k in enumerate(p.pairs):  # row r blends frames r and r + 1 of the pass
            if k is not None:
                assert (p.frames[r], p.frames[r + 1]) == (k, k + 1)
            else:
                assert p.frames[r] == p.frames[r + 1] == n_frames - 1  # idle: the repeated last frame


def test_interp_schedule_tail_and_errors():
    from raft_b200.video import interp_schedule
    passes = interp_schedule(10, 4)  # 9 pairs: 4 + 4 + 1
    assert [p.frames for p in passes] == [[0, 1, 2, 3, 4], [4, 5, 6, 7, 8], [8, 9, 9, 9, 9]]
    assert passes[-1].pairs == [8, None, None, None]
    for bad in ((1, 4), (5, 0)):
        with pytest.raises(ValueError):
            interp_schedule(*bad)


@pytest.mark.parametrize("n_frames,m", [(2, 1), (5, 1), (5, 3), (9, 7)])
def test_frame_numbering(n_frames, m):
    from raft_b200.video import frame_number
    nums = [frame_number(k, m) for k in range(n_frames)]
    nums += [frame_number(k, m, j) for k in range(n_frames - 1) for j in range(m)]
    assert sorted(nums) == list(range((n_frames - 1) * (m + 1) + 1))  # every index once, none missing
    assert frame_number(n_frames - 1, m) == (n_frames - 1) * (m + 1)  # the last input frame closes the sequence
    assert frame_number(1, m) == m + 1 and frame_number(0, m, m - 1) == m


def test_check_times():
    from raft_b200.video import check_times
    assert check_times([0.25, 0.5]) == [0.25, 0.5]
    for bad in ([], [0.0], [1.0], [0.5, 0.5], [0.6, 0.3], [-0.1], [float("nan")]):
        with pytest.raises(ValueError, match="strictly increasing"):
            check_times(bad)


# ---- CLI ---------------------------------------------------------------------------------------------------------
def _frames_dir(tmp_path):
    for k in range(2):
        (tmp_path / f"f{k}.png").write_bytes(b"")  # never decoded: every refusal comes first
    return str(tmp_path)


@pytest.mark.parametrize("extra,what", [
    (["--warm-start"], "--warm-start"), (["--native-flow"], "--native-flow"), (["--flo", "x"], "--flo"),
    (["--npy", "x"], "--npy"), (["--bidirectional"], "--bidirectional")])
def test_cli_path_interpolate_refusals(tmp_path, extra, what):
    r = subprocess.run([sys.executable, CLI, "--path", _frames_dir(tmp_path), "--interpolate", "0.5"] + extra,
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and what in r.stderr, r.stderr


@pytest.mark.parametrize("ts", [["0"], ["1"], ["0.5", "0.5"], ["0.7", "0.2"], ["0.5", "1.0"]])
def test_cli_path_interpolate_times(tmp_path, ts):
    r = subprocess.run([sys.executable, CLI, "--path", _frames_dir(tmp_path), "--interpolate"] + ts,
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "strictly increasing" in r.stderr, r.stderr


def test_cli_path_interpolate_refusals_import_no_torch(tmp_path):
    """Every refusal, an empty frame directory included, comes before torch (and so the GPU) is imported."""
    code = ("import sys; sys.path.insert(0, sys.argv[1]); import infer_raft\n"
            "try:\n    infer_raft.main(sys.argv[2:])\nexcept SystemExit as e:\n    print(e.code, 'torch' in sys.modules)")
    for argv in (["--path", _frames_dir(tmp_path), "--interpolate", "0.5", "--flo", "x"],
                 ["--path", _frames_dir(tmp_path), "--interpolate", "0.5", "0.25"],
                 ["--path", str(tmp_path / "empty"), "--interpolate", "0.5"]):
        r = subprocess.run([sys.executable, "-c", code, os.path.dirname(CLI)] + argv, capture_output=True, text=True,
                           timeout=120)
        assert r.stdout.split() == ["2", "False"], (argv, r.stdout, r.stderr)


def test_cli_bidirectional_message_names_only_bidirectional(tmp_path):
    r = subprocess.run([sys.executable, CLI, "--path", str(tmp_path), "--bidirectional"], capture_output=True, text=True,
                       timeout=120)
    error = r.stderr.strip().splitlines()[-1]  # the usage lines above it list every flag
    assert r.returncode == 2 and "--bidirectional" in error and "--interpolate" not in error, r.stderr


# ---- argument checks of the new entries (host pointers: a launch would fail, not return these codes) --------------
def test_multi_entry_argument_checks():
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG, WORKSPACE = -1, -2, -5
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def refused(rc, code, *words):
        assert rc == code, (rc, code)
        msg = lib.rb_last_error()
        assert all(w in msg for w in words), msg

    def steps(*v):
        return (ctypes.c_float * max(1, len(v)))(*v)

    def rev(flow=p, ts=steps(0.5, 1.0), n=2, ft=p, empty=p, multi=p, B=1, H=4, W=4, ws=p, nbytes=1 << 20):
        return lib.rb_flow_reverse_multi(flow, ts, n, ft, empty, multi, B, H, W, ws, nbytes, None)

    for kw in ({"flow": None}, {"ts": None}, {"ft": None}, {"empty": None}, {"multi": None}, {"ws": None}):
        refused(rev(**kw), BAD_ARG, b"rb_flow_reverse_multi", b"null")
    for n in (0, -1, 65):
        refused(rev(ts=steps(*([0.5] * 65)), n=n), BAD_ARG, b"time steps")
    for bad in (float("nan"), float("inf"), -float("inf")):
        refused(rev(ts=steps(0.5, bad)), BAD_ARG, b"time_steps[1]")
    for B, H, W in ((0, 4, 4), (1, 0, 4), (1, 4, -1)):
        refused(rev(B=B, H=H, W=W), BAD_SHAPE, b"bad shape")
    refused(rev(B=1, H=65535, W=65537, n=1), BAD_SHAPE, b"2^32")  # n_steps*B*H*W + 1 == 2^32
    refused(rev(B=1, H=32768, W=65536, ts=steps(0.5, 0.5)), BAD_SHAPE, b"2^32")  # two steps reach 2^32
    refused(rev(nbytes=64), WORKSPACE, b"too small")
    out = ctypes.c_size_t()
    refused(lib.rb_flow_reverse_multi_workspace_bytes(2, 1, 4, 4, None), BAD_ARG, b"null")
    refused(lib.rb_flow_reverse_multi_workspace_bytes(0, 1, 4, 4, ctypes.byref(out)), BAD_ARG, b"time steps")
    refused(lib.rb_flow_reverse_multi_workspace_bytes(65, 1, 4, 4, ctypes.byref(out)), BAD_ARG, b"time steps")
    refused(lib.rb_flow_reverse_multi_workspace_bytes(2, 1, 0, 4, ctypes.byref(out)), BAD_SHAPE, b"bad shape")
    refused(lib.rb_flow_reverse_multi_workspace_bytes(2, 1, 32768, 65536, ctypes.byref(out)), BAD_SHAPE, b"2^32")

    def syn(f0s=p, f1s=p, Hp=8, Wp=8, top=0, left=0, f0=p, f1=p, e0=p, e1=p, ts=steps(0.5), n=1, out=p, u8=0, bgr=0, B=1,
            H=8, W=8):
        return lib.rb_frame_synthesize_pairs(f0s, f1s, Hp, Wp, top, left, f0, f1, e0, e1, ts, n, out, u8, bgr, B, H, W,
                                             None)

    for kw in ({"f0s": None}, {"f1s": None}, {"f0": None}, {"f1": None}, {"e0": None}, {"e1": None}, {"ts": None},
               {"out": None}):
        refused(syn(**kw), BAD_ARG, b"rb_frame_synthesize", b"null")
    for n in (0, -3, 65):
        refused(syn(ts=steps(*([0.5] * 65)), n=n), BAD_ARG, b"times")
    for u8, bgr in ((2, 0), (-1, 0), (1, 2), (0, -1)):
        refused(syn(u8=u8, bgr=bgr), BAD_ARG, b"0 or 1")
    for t in (-0.01, 1.01, float("nan"), float("inf")):
        refused(syn(ts=steps(0.5, t), n=2), BAD_ARG, b"[0, 1]")
    for B, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, -2)):
        refused(syn(B=B, H=H, W=W), BAD_SHAPE, b"bad shape")
    for Hp, Wp, top, left in ((7, 8, 0, 0), (8, 7, 0, 0), (9, 8, 2, 0), (8, 8, -1, 0), (8, 8, 0, -1)):
        refused(syn(Hp=Hp, Wp=Wp, top=top, left=left), BAD_SHAPE, b"outside")
