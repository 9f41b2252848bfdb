"""F11 on the CPU: the colour-coding oracle (tests/flowviz_oracle.py) against flow_utils.flow_to_color and the reference's
own outputs (tests/golden/flow_to_color.npz), the frame listing and pass schedule of raft_b200.video, and the CLI's
--path argument errors."""
import os
import subprocess
import sys

import numpy as np
import pytest

import flowviz_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "flow_to_color.npz")


def _golden_cases():
    z = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in z.files if "/" in k})
    for n in names:
        clip = float(z[n + "/clip"])
        yield n, z[n + "/flow"], None if clip < 0 else clip, z


def raft_like(rng, H, W):
    """Smooth motion of RAFT's magnitude plus noise and a few sharp edges."""
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    a = rng.uniform(-1, 1, 6)
    u = 12 * a[0] + 8 * np.sin(xx / W * 4 + a[1]) + 4 * np.cos(yy / H * 3 + a[2])
    v = 6 * a[3] + 6 * np.cos(xx / W * 2 + a[4]) * np.sin(yy / H * 5 + a[5])
    f = np.stack([u, v], -1) + rng.normal(0, 0.3, (H, W, 2))
    f[H // 3:H // 2, W // 4:W // 2] *= -1.5
    return f.astype(np.float32)


def _numpy_atan_is_rounded(flow, clip):
    """Pixels where numpy's float32 arctan2 equals the fp64 value rounded to fp32 (where the host function and the
    oracle compute the same direction)."""
    f = np.clip(flow, 0, np.float32(clip)) if clip is not None else flow
    u, v = f[..., 0], f[..., 1]
    den = (np.sqrt(np.square(u) + np.square(v)).max() + np.float32(1e-5)).astype(np.float32)
    u, v = u / den, v / den
    return np.arctan2(-v, -u) == flowviz_oracle.atan2_f32(-v, -u)[0]


def _check_against_host(flow, clip):
    import flow_utils
    same = _numpy_atan_is_rounded(flow, clip)
    for bgr in (False, True):
        got, amb = flowviz_oracle.flow_to_color(flow, clip, bgr)
        host = flow_utils.flow_to_color(flow, clip_flow=clip, convert_to_bgr=bgr)
        assert np.array_equal(got[same], host[same]), bgr
        assert np.abs(got.astype(int) - host.astype(int)).max() <= 1
        assert amb.mean() < 0.01


@pytest.mark.parametrize("case", ["smooth", "noise", "clip", "zero", "axes"])
def test_oracle_equals_host_function_on_golden_cases(case):
    for n, flow, clip, _ in _golden_cases():
        if n == case:
            _check_against_host(flow, clip)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_equals_host_function_on_raft_like_flows(seed):
    rng = np.random.default_rng(seed)
    _check_against_host(raft_like(rng, 96, 160), None)
    _check_against_host(raft_like(rng, 40, 56), 10.0)


def test_oracle_within_one_lsb_of_reference_outputs():
    for n, flow, clip, z in _golden_cases():
        if flow.dtype != np.float32:
            continue
        for bgr in (0, 1):
            got, _ = flowviz_oracle.flow_to_color(flow, clip, bool(bgr))
            ref = z[f"{n}/bgr{bgr}/out"]
            assert np.abs(got.astype(int) - ref.astype(int)).max() <= 1, (n, bgr)


def test_ambiguous_mask_marks_midpoints():
    # the fp32 midpoint between 1 and its successor, as a double, is ambiguous; pi / 4 is not
    r, amb = flowviz_oracle.atan2_f32(np.array([1.0, 1.0]), np.array([1.0, -1.0]))
    assert not amb.any()
    mid = 1.0 + 2.0 ** -24  # halfway between 1.0f and its successor
    y, x = np.array([np.sin(mid)]), np.array([np.cos(mid)])
    d = np.arctan2(y, x)
    assert abs(d[0] - mid) <= 2 * np.spacing(mid)
    assert flowviz_oracle.atan2_f32(y, x)[1].all()


# ---- raft_b200.video: frames and schedule ------------------------------------------------------------------------
def test_list_frames_sorted_png_jpg_only(tmp_path):
    from raft_b200.video import list_frames
    for n in ("b.png", "a.jpg", "c.png", "d.jpeg", "e.txt", "f.PNG"):
        (tmp_path / n).write_bytes(b"")
    got = [os.path.basename(p) for p in list_frames(str(tmp_path))]
    assert got == ["a.jpg", "b.png", "c.png"]
    assert list_frames(["x", "y"]) == ["x", "y"]


def test_list_frames_needs_two(tmp_path):
    from raft_b200.video import list_frames
    (tmp_path / "a.png").write_bytes(b"")
    with pytest.raises(ValueError, match="two frames"):
        list_frames(str(tmp_path))
    with pytest.raises(ValueError, match="two frames"):
        list_frames(["only.png"])
    with pytest.raises(FileNotFoundError):
        list_frames(str(tmp_path / "missing"))


@pytest.mark.parametrize("n_frames", [2, 3, 8, 9, 10, 17, 30])
@pytest.mark.parametrize("batch", [1, 3, 8])
def test_schedule_covers_every_pair_once(n_frames, batch):
    from raft_b200.video import schedule
    passes = schedule(n_frames, batch)
    pairs = [k for p in passes for k in p.pairs if k is not None]
    assert pairs == list(range(n_frames - 1))
    assert not passes[0].carry and all(p.carry for p in passes[1:])
    assert len(passes[0].frames) == batch + 1 and all(len(p.frames) == batch for p in passes[1:])
    # the frames a pass sees: fresh [f_0 .. f_T], carry (previous last) + new; pair k of row r is (frame k, frame k + 1)
    prev_last = None
    for p in passes:
        seen = p.frames if not p.carry else [prev_last] + p.frames
        for r, k in enumerate(p.pairs):
            if k is not None:
                assert (seen[r], seen[r + 1]) == (k, k + 1)
        assert all(0 <= i < n_frames for i in p.frames)
        prev_last = seen[-1]


def test_schedule_tail_padding_and_idle_rows():
    from raft_b200.video import schedule
    passes = schedule(10, 4)  # 9 pairs: 4 + 4 + 1
    assert [p.frames for p in passes] == [[0, 1, 2, 3, 4], [5, 6, 7, 8], [9, 9, 9, 9]]
    assert passes[-1].pairs == [8, None, None, None]
    one = schedule(2, 8)  # T = 8 on a single pair: the last frame repeated, seven idle rows
    assert one[0].frames == [0, 1] + [1] * 7 and one[0].pairs == [0] + [None] * 7
    assert [p.frames for p in schedule(4, 1)] == [[0, 1], [2], [3]]


def test_schedule_warm_forces_one_pair_per_pass():
    from raft_b200.video import schedule
    passes = schedule(6, 1, warm_start=True)
    assert [p.pairs for p in passes] == [[0], [1], [2], [3], [4]]
    with pytest.raises(ValueError, match="batch must be 1"):
        schedule(6, 8, warm_start=True)
    with pytest.raises(ValueError):
        schedule(1, 1)
    with pytest.raises(ValueError):
        schedule(5, 0)


# ---- CLI ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra,what", [(["--bidirectional"], "--bidirectional"), (["--interpolate", "0.5"], "--interpolate"),
                                        (["--warm-start", "--batch", "8"], "--batch 1")])
def test_cli_path_errors(tmp_path, extra, what):
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    r = subprocess.run([sys.executable, cli, "--path", str(tmp_path)] + extra, capture_output=True, text=True,
                       timeout=120)
    assert r.returncode == 2 and what in r.stderr, r.stderr


def test_cli_path_flag_parses():
    import infer_raft
    a = infer_raft.parser().parse_args(["--path", "frames", "--batch", "8", "--flo", "f", "--npy", "n"])
    assert (a.path, a.batch, a.flo, a.npy) == ("frames", 8, "f", "n")
    assert infer_raft.parser().parse_args([]).path is None
