"""F17 on the GPU: rb_track_points_backward against the fp32 restatement (tests/track_backward_oracle.py) and against
rb_track_points on the reversed clip, bit for bit; carried reverse calls; RAFT.track(backward=True); and video_track /
infer_raft.py --track-backward end to end on shifted crops of tests/data/frame_0016.png."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import track_backward_oracle as B
import track_oracle as O
from test_gpu_track import _case, _model, _run, _weights
from test_gpu_video import _decoded, _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_bw(cuda, fw, bw, qframe, qpos, scale, tracks=None, status=None, state=None, first_frame=0, n_steps=None):
    from networks.utils import track_points_backward
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)  # noqa: E731
    return track_points_backward(t(fw), t(bw), t(qframe), t(qpos), tracks=tracks, status=status, state=state,
                                 first_frame=first_frame, n_steps=n_steps, flow_scale=scale)


@pytest.mark.parametrize("T,H,W,N,scale", [(3, 37, 53, 1, 1.0), (4, 37, 53, 300, 1.0), (4, 37, 53, 300, 8.0),
                                           (3, 1, 31, 64, 1.0), (3, 29, 1, 64, 1.0), (2, 1, 1, 5, 1.0),
                                           (5, 61, 97, 70000, 1.0), (2, 40, 60, 129, 8.0)])
def test_kernel_equals_fp32_restatement_bit_for_bit(cuda, T, H, W, N, scale):
    rng = np.random.default_rng(T * 100000 + H * 1000 + W + N + 7)
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    if scale != 1.0:
        fw, bw = fw / np.float32(scale), bw / np.float32(scale)
    want_t, want_s, (want_p, want_st) = B.track_backward(fw, bw, qframe, qpos, flow_scale=scale)
    tracks, status, (pos, st) = _run_bw(cuda, fw, bw, qframe, qpos, scale)
    assert tracks.shape == (T + 1, N, 2) and status.shape == (T + 1, N) and status.dtype == torch.uint8
    assert O.same_bits(tracks.cpu().numpy(), want_t), "tracks differ"
    assert np.array_equal(status.cpu().numpy(), want_s), f"{(status.cpu().numpy() != want_s).sum()} statuses differ"
    assert O.same_bits(pos.cpu().numpy(), want_p) and np.array_equal(st.cpu().numpy(), want_st)
    # the forward kernel on the reversed clip, from frame T - q, rows reversed
    rfw, rbw = B.reversed_clip(fw, bw)
    rt, rs, _ = _run(cuda, rfw, rbw, (T - qframe).astype(np.int32), qpos, scale)
    rows = np.arange(T + 1)[:, None] <= qframe
    assert O.same_bits(rt.cpu().numpy()[::-1][rows], tracks.cpu().numpy()[rows])
    assert np.array_equal(rs.cpu().numpy()[::-1][rows], status.cpu().numpy()[rows])
    # after the forward launch, on its buffers: the forward rows stay, the rows before the query are filled
    ft, fs, _ = _run(cuda, fw, bw, qframe, qpos, scale)
    keep_t, keep_s = ft.cpu().numpy(), fs.cpu().numpy()
    ct, cs, _ = _run_bw(cuda, fw, bw, qframe, qpos, scale, tracks=ft, status=fs)
    assert ct.data_ptr() == ft.data_ptr() and cs.data_ptr() == fs.data_ptr()
    after = np.arange(T + 1)[:, None] >= qframe
    assert O.same_bits(ct.cpu().numpy()[after], keep_t[after]) and np.array_equal(cs.cpu().numpy()[after], keep_s[after])
    assert O.same_bits(ct.cpu().numpy()[~after], want_t[~after]) and not (cs.cpu().numpy() == O.BEFORE).any()
    if N >= 300 and H * W > 1000:
        assert all((want_s[rows] == k).any() for k in range(3))


@pytest.mark.parametrize("split", [1, 3, 5])
def test_carried_reverse_calls_equal_one_launch(cuda, split):
    rng = np.random.default_rng(91 + split)
    T, H, W, N = 6, 33, 47, 1000
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    whole_t, whole_s, _ = _run_bw(cuda, fw, bw, qframe, qpos, 1.0)
    # the later pass first, padded as a short last pass of video_track is (n_steps < T), then the earlier one
    pad = lambda f: np.concatenate([f[split:], f[-1:].repeat(2, 0)])  # noqa: E731
    b_t, b_s, state = _run_bw(cuda, pad(fw), pad(bw), qframe, qpos, 1.0, first_frame=split, n_steps=T - split)
    a_t, a_s, _ = _run_bw(cuda, fw[:split], bw[:split], qframe, qpos, 1.0, state=state)
    assert O.same_bits(torch.cat([a_t, b_t[1:]]).cpu().numpy(), whole_t.cpu().numpy())
    assert torch.equal(torch.cat([a_s, b_s[1:]]), whole_s)
    assert O.same_bits(a_t[-1].cpu().numpy(), b_t[0].cpu().numpy())  # the shared row


def test_sentinel_rows_after_the_query_are_kept(cuda):
    rng = np.random.default_rng(5)
    T, H, W, N = 5, 31, 43, 2000
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    tr = torch.full((T + 1, N, 2), -12345.5, device=cuda)
    ss = torch.full((T + 1, N), 77, dtype=torch.uint8, device=cuda)
    t, s, _ = _run_bw(cuda, fw, bw, qframe, qpos, 1.0, tracks=tr, status=ss)
    after = torch.from_numpy(np.arange(T + 1)[:, None] > qframe).to(cuda)
    assert (t[after] == -12345.5).all() and (s[after] == 77).all() and (s[~after] != 77).all()
    want_t, want_s, _ = B.track_backward(fw, bw, qframe, qpos, np.full((T + 1, N, 2), -12345.5, np.float32),
                                         np.full((T + 1, N), 77, np.uint8))
    assert O.same_bits(t.cpu().numpy(), want_t) and np.array_equal(s.cpu().numpy(), want_s)


@pytest.mark.parametrize("input_size", [None, (128, 160)])
@pytest.mark.parametrize("upstream", [False, True])
@pytest.mark.parametrize("small", [False, True])
def test_track_backward_equals_the_flows_chained(cuda, small, upstream, input_size):
    m = _model(small, upstream=upstream, input_size=input_size)
    frames = _frames(5, 125, 150, seed=4800 + 2 * small + upstream)
    H, W = frames.shape[1:3]
    rng = np.random.default_rng(19)
    q = np.stack([rng.integers(0, 5, 800), rng.uniform(0, W - 1, 800), rng.uniform(0, H - 1, 800)], -1)
    q[:100, 0] = 4  # a grid of keyframe queries on the last frame
    fwd_t, fwd_s = m.track(frames, q)
    tracks, status = m.track(frames, q, backward=True)
    after = np.arange(5)[:, None] >= q[:, 0]
    assert O.same_bits(tracks.cpu().numpy()[after], fwd_t.cpu().numpy()[after])
    assert np.array_equal(status.cpu().numpy()[after], fwd_s.cpu().numpy()[after])
    assert not (status == O.BEFORE).any()
    fw, bw, _, _ = m.forward_sequence_bidirectional(frames, check=False)
    eng = m.engine()
    src, net = (H, W), eng.input_size if eng.input_size is not None else (H, W)
    qpos = O.to_network(q[:, 1:], src, net) if net != src else q[:, 1:].astype(np.float32)
    want_t, want_s, _ = B.track_backward(fw.cpu().numpy(), bw.cpu().numpy(), q[:, 0], qpos, flow_scale=eng.flow_scale)
    if net != src:
        want_t = O.from_network(want_t, src, net)
    assert O.same_bits(tracks.cpu().numpy()[~after], want_t[~after])
    assert np.array_equal(status.cpu().numpy()[~after], want_s[~after])
    assert (status.cpu().numpy()[~after] != O.LEFT).any()  # some points stay in the frame going back


def _vis_expected(frames, tracks, status):
    """The --track-vis drawing of every frame from the merged arrays: each status-0 point as a dot in its colour."""
    import cv2
    from raft_b200.video import track_colors
    colors = track_colors(tracks.shape[1])
    out = {}
    for f, img in enumerate(frames):
        img = img.copy()
        seen = np.flatnonzero(status[f] == 0)
        for i, (x, y) in zip(seen, np.rint(tracks[f][seen]).astype(np.int64)):
            cv2.circle(img, (int(x), int(y)), 2, colors[i].tolist(), -1)
        out[f"frame_{f:06d}.png"] = img
    return out


def test_video_track_backward_end_to_end(cuda, frame_dir, tmp_path):
    import cv2
    from raft_b200.video import video_track
    m = _model()
    frames = _decoded(frame_dir)
    F, H, W = frames.shape[:3]
    rng = np.random.default_rng(13)
    queries = np.concatenate([np.stack([rng.integers(0, F, 300), rng.uniform(0, W - 1, 300),
                                        rng.uniform(0, H - 1, 300)], -1), [[F - 1, 40.0, 60.0], [5, 70.0, 30.0]]])
    want_t, want_s = (x.cpu().numpy() for x in m.track(frames, queries, backward=True))
    assert not (want_s == O.BEFORE).any()
    runs = {}
    for batch in (1, 3, 8):
        for workers in (0, 4):
            out, vis = tmp_path / f"b{batch}w{workers}", tmp_path / f"vis{batch}w{workers}"
            files = video_track(m, frame_dir, str(out), queries=queries, batch=batch, workers=workers,
                                vis=str(vis) if workers else None, backward=True)
            assert files == (str(out / "tracks.npy"), str(out / "status.npy"))
            assert O.same_bits(np.load(files[0]), want_t), (batch, workers)
            assert np.array_equal(np.load(files[1]), want_s), (batch, workers)
            runs[(batch, workers)] = _files(str(out))
            if workers:
                runs[(batch, "vis")] = _files(str(vis))
    assert all(runs[k] == runs[(1, 0)] for k in runs if k[1] != "vis")
    assert all(runs[k] == runs[(3, "vis")] for k in runs if k[1] == "vis")
    want_vis = _vis_expected(frames, want_t, want_s)
    assert sorted(runs[(3, "vis")]) == sorted(want_vis)
    for name, img in want_vis.items():
        assert np.array_equal(cv2.imread(str(tmp_path / "vis3w4" / name)), img), name
    # a grid on frame 0: nothing before it, so no reverse pass runs and the files are those of the forward run
    a = video_track(m, frame_dir, str(tmp_path / "g0"), grid=16, batch=3, backward=True)
    b = video_track(m, frame_dir, str(tmp_path / "g1"), grid=16, batch=3)
    assert _files(os.path.dirname(a[0])) == _files(os.path.dirname(b[0]))


def test_cli_track_backward(cuda, frame_dir, tmp_path):
    from raft_b200.video import video_track
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    argv = [sys.executable, cli, "--path", frame_dir, "--out", str(tmp_path / "o"), "--load", npz, "--iters", "4",
            "--track-grid", "20", "--track-frame", "6", "--track-backward", "--batch", "4", "--keep-size"]
    r = subprocess.run(argv, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    files = video_track(_model(), frame_dir, str(tmp_path / "ref"), grid=20, grid_frame=6, backward=True)
    assert _files(str(tmp_path / "o")) == _files(os.path.dirname(files[0]))
    assert not (np.load(files[1]) == O.BEFORE).any()
