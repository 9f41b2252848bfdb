"""F16 on the GPU: rb_track_points against the fp32 restatement (tests/track_oracle.py) bit for bit, carried state across
launches, RAFT.track against forward_sequence_bidirectional's flows and occlusion masks, and video_track / infer_raft.py
--track end to end on shifted crops of tests/data/frame_0016.png."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import track_oracle as O
from test_gpu_video import _decoded, _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_WEIGHTS = {}


def _weights(small):
    from raft_b200 import synth
    if small not in _WEIGHTS:
        _WEIGHTS[small] = synth.make_weights(small)
    return _WEIGHTS[small]


def _model(small=False, iters=4, **kw):
    from networks.RAFT import RAFT
    return RAFT(None, SimpleNamespace(small=small), iters=iters, device="cuda:0", **kw).load(_weights(small))


def _case(rng, T, H, W, N, nan=3):
    fw = (rng.uniform(-0.3, 0.3, (T, H, W, 2)) * np.array([W, H])).astype(np.float32)  # many targets leave the frame
    bw = (-fw + rng.normal(0, 0.6, fw.shape)).astype(np.float32)
    for f in (fw, bw):
        for _ in range(nan if H * W > 1 else 0):
            f[rng.integers(T), rng.integers(H), rng.integers(W), rng.integers(2)] = np.nan
    qframe = rng.integers(0, T + 1, N).astype(np.int32)
    qpos = np.stack([rng.uniform(0, W - 1, N), rng.uniform(0, H - 1, N)], -1).astype(np.float32)
    centre = rng.random(N) < 0.3  # some pixel centres, whose samples hit one tap
    qpos[centre] = np.floor(qpos[centre])
    return fw, bw, qframe, qpos


def _run(cuda, fw, bw, qframe, qpos, scale, state=None, first_frame=0, n_steps=None):
    from networks.utils import track_points
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)  # noqa: E731
    return track_points(t(fw), t(bw), t(qframe), t(qpos), state=state, first_frame=first_frame, n_steps=n_steps,
                        flow_scale=scale)


@pytest.mark.parametrize("T,H,W,N,scale", [(3, 37, 53, 1, 1.0), (4, 37, 53, 300, 1.0), (4, 37, 53, 300, 8.0),
                                           (3, 1, 31, 64, 1.0), (3, 29, 1, 64, 1.0), (2, 1, 1, 5, 1.0),
                                           (5, 61, 97, 70000, 1.0), (2, 40, 60, 129, 8.0)])
def test_kernel_equals_fp32_restatement_bit_for_bit(cuda, T, H, W, N, scale):
    rng = np.random.default_rng(T * 100000 + H * 1000 + W + N)
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    if scale != 1.0:
        fw, bw = fw / np.float32(scale), bw / np.float32(scale)
    want_t, want_s, _ = O.track(fw, bw, qframe, qpos, flow_scale=scale)
    tracks, status, (pos, st) = _run(cuda, fw, bw, qframe, qpos, scale)
    assert tracks.shape == (T + 1, N, 2) and status.shape == (T + 1, N) and status.dtype == torch.uint8
    assert O.same_bits(tracks.cpu().numpy(), want_t), "tracks differ"
    assert np.array_equal(status.cpu().numpy(), want_s), f"{(status.cpu().numpy() != want_s).sum()} statuses differ"
    assert O.same_bits(pos.cpu().numpy(), want_t[-1]) and np.array_equal(st.cpu().numpy(), want_s[-1])
    if N >= 300 and H * W > 1000:
        assert all((want_s == k).any() for k in range(4))


@pytest.mark.parametrize("split", [1, 3, 5])
def test_carried_state_equals_one_launch(cuda, split):
    rng = np.random.default_rng(77 + split)
    T, H, W, N = 6, 33, 47, 1000
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    whole_t, whole_s, _ = _run(cuda, fw, bw, qframe, qpos, 1.0)
    a_t, a_s, state = _run(cuda, fw[:split], bw[:split], qframe, qpos, 1.0)
    # the second launch sees a padded pass, as a short last pass of video_track does: n_steps < T
    pad = lambda f: np.concatenate([f[split:], f[-1:].repeat(2, 0)])  # noqa: E731
    b_t, b_s, _ = _run(cuda, pad(fw), pad(bw), qframe, qpos, 1.0, state=state, first_frame=split, n_steps=T - split)
    assert O.same_bits(torch.cat([a_t, b_t[1:]]).cpu().numpy(), whole_t.cpu().numpy())
    assert torch.equal(torch.cat([a_s, b_s[1:]]), whole_s)


def _check_track(m, frames, queries):
    """RAFT.track against the restatement applied to the flows forward_sequence_bidirectional returns."""
    tracks, status = m.track(frames, queries)
    fw, bw, _, _ = m.forward_sequence_bidirectional(frames, check=False)
    eng = m.engine()
    src = tuple(frames.shape[1:3])
    net = eng.input_size if eng.input_size is not None else src
    q = np.asarray(queries, dtype=np.float64)
    qpos = O.to_network(q[:, 1:], src, net) if net != src else q[:, 1:].astype(np.float32)
    want_t, want_s, _ = O.track(fw.cpu().numpy(), bw.cpu().numpy(), q[:, 0], qpos, flow_scale=eng.flow_scale)
    if net != src:
        want_t = O.from_network(want_t, src, net)
    assert tracks.shape == (len(frames), len(q), 2) and status.shape == (len(frames), len(q))
    assert O.same_bits(tracks.cpu().numpy(), want_t) and np.array_equal(status.cpu().numpy(), want_s)
    return tracks, status, fw, bw


@pytest.mark.parametrize("input_size", [None, (128, 160)])
@pytest.mark.parametrize("upstream", [False, True])
@pytest.mark.parametrize("small", [False, True])
def test_track_equals_the_flows_chained(cuda, small, upstream, input_size):
    m = _model(small, upstream=upstream, input_size=input_size)
    frames = _frames(5, 125, 150, seed=4600 + 2 * small + upstream)
    H, W = frames.shape[1:3]
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    grid = np.stack([np.zeros(H * W), xs.ravel(), ys.ravel()], -1)
    rng = np.random.default_rng(9)
    later = np.stack([rng.integers(0, 5, 500), rng.uniform(0, W - 1, 500), rng.uniform(0, H - 1, 500)], -1)
    tracks, status, fw, bw = _check_track(m, frames, np.concatenate([grid, later]))
    if input_size is None:  # a dense frame-0 grid: the first step is the occlusion check and grid + s flow_fw[0]
        occ = m.forward_sequence_bidirectional(frames)[2][0].reshape(-1)
        assert torch.equal(status[1, :H * W], occ)
        s = m.engine().flow_scale
        inside = (occ != 2).cpu()
        want = torch.from_numpy(grid[:, 1:].astype(np.float32)) + s * fw[0].reshape(-1, 2).cpu()
        got = tracks[1, :H * W].cpu()
        assert O.same_bits(got[inside].numpy(), want[inside].numpy())


def test_track_inputs_and_duplicates(cuda):
    m = _model()
    frames = _frames(4, 64, 96, seed=4700)
    q = np.array([[0, 10.5, 20.0], [1, 3.0, 7.25], [0, 10.5, 20.0], [1, 3.0, 7.25], [3, 95.0, 63.0]])
    t8, s8 = m.track(frames, q)
    assert torch.equal(s8[:, 0], s8[:, 2]) and O.same_bits(t8[:, 0].cpu().numpy(), t8[:, 2].cpu().numpy())
    assert torch.equal(s8[:, 1], s8[:, 3]) and O.same_bits(t8[:, 1].cpu().numpy(), t8[:, 3].cpu().numpy())
    tf, sf = m.track(torch.from_numpy(frames).cuda(), torch.from_numpy(q))  # CUDA frames, tensor queries
    assert torch.equal(sf, s8) and O.same_bits(tf.cpu().numpy(), t8.cpu().numpy())
    a, _ = m.track(frames, q)
    assert a.data_ptr() != t8.data_ptr()  # fresh tensors
    for bad in ([[4, 1.0, 1.0]], [[0, 96.0, 1.0]], [[0, np.nan, 1.0]], np.zeros((0, 3)), [[0, 1.0]]):
        with pytest.raises(ValueError):
            m.track(frames, bad)


def test_video_track_end_to_end(cuda, frame_dir, tmp_path):
    from raft_b200.video import track_grid, video_track
    m = _model()
    frames = _decoded(frame_dir)
    F, H, W = frames.shape[:3]
    rng = np.random.default_rng(12)
    queries = np.concatenate([np.stack([rng.integers(0, F, 300), rng.uniform(0, W - 1, 300),
                                        rng.uniform(0, H - 1, 300)], -1), [[0, 40.0, 60.0]] * 2])
    want_t, want_s = (x.cpu().numpy() for x in m.track(frames, queries))
    assert O.same_bits(want_t[:, -1], want_t[:, -2])
    runs = {}
    for batch, workers in ((1, 0), (3, 4), (8, 4), (8, 0)):
        out, vis = tmp_path / f"b{batch}w{workers}", tmp_path / f"vis{batch}w{workers}"
        files = video_track(m, frame_dir, str(out), queries=queries, batch=batch, workers=workers,
                            vis=str(vis) if batch != 1 else None)
        assert files == (str(out / "tracks.npy"), str(out / "status.npy"))
        runs[(batch, workers)] = _files(str(out))
        if batch != 1:
            runs[(batch, workers, "vis")] = _files(str(vis))
    assert all(runs[k] == runs[(1, 0)] for k in runs if len(k) == 2)
    assert all(runs[k] == runs[(3, 4, "vis")] for k in runs if len(k) == 3)
    assert sorted(runs[(3, 4, "vis")]) == [f"frame_{i:06d}.png" for i in range(F)]
    out = tmp_path / "b8w4"
    assert O.same_bits(np.load(out / "tracks.npy"), want_t) and np.array_equal(np.load(out / "status.npy"), want_s)
    # a grid on a later frame
    g = video_track(m, frame_dir, str(tmp_path / "grid"), grid=16, grid_frame=2, batch=3)
    want = m.track(frames, track_grid(H, W, 16, 2))
    assert O.same_bits(np.load(g[0]), want[0].cpu().numpy()) and np.array_equal(np.load(g[1]), want[1].cpu().numpy())


def test_cli_track(cuda, frame_dir, tmp_path):
    from raft_b200.video import video_track
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    (tmp_path / "q.txt").write_text("0 20 30\n2 100.5 60.25\n")
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    argv = [sys.executable, cli, "--path", frame_dir, "--out", str(tmp_path / "o"), "--load", npz, "--iters", "4",
            "--track", str(tmp_path / "q.txt"), "--batch", "4", "--keep-size"]
    r = subprocess.run(argv, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    st = np.load(tmp_path / "o" / "status.npy")
    assert f"2 points tracked through 10 frames: {int((st[-1] == 0).sum())} consistent" in r.stdout, r.stdout
    files = video_track(_model(), frame_dir, str(tmp_path / "ref"), queries=[[0, 20, 30], [2, 100.5, 60.25]])
    assert _files(str(tmp_path / "o")) == _files(os.path.dirname(files[0]))
