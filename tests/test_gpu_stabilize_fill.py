"""F26 on the GPU: the flow extension and rb_frames_warp_affine_fill against the numpy oracle bit for bit
(tests/stabfill_oracle.py), the in-frame pixels against rb_frames_warp_affine, the known texture path at a realistic
size, RAFT.stabilize(fill=True) against its public parts, video_stabilize(fill=True) against RAFT.stabilize and the CLI.
The end-to-end tests run seeded weights (plumbing, not quality)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import stabfill_oracle as SF
import stabilize_oracle as SO
from raft_b200 import stabilize as S
from raft_b200.inpaint import inpaint_rows
from test_gpu_stabilize import every_pixel  # noqa: F401  (the fixture)
from test_gpu_track import _model, _weights
from test_gpu_video import _decoded, _files, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _motions(rng, T):
    th, s = rng.normal(0, 0.02, T), 1 + rng.normal(0, 0.02, T)
    return np.stack([s * np.cos(th), s * np.sin(th), rng.normal(0, 4, T), rng.normal(0, 4, T)], 1)


@pytest.mark.parametrize("T,net,hw,margin,scale", [(1, (24, 40), (48, 80), (3, 5), 1.0),
                                                   (3, (23, 37), (41, 67), (4, 2), 1.0),
                                                   (2, (31, 45), (31, 45), (6, 7), 8.0),
                                                   (2, (20, 30), (50, 70), (0, 0), 1.0)])
def test_flow_extension_matches_oracle(cuda, T, net, hw, margin, scale):
    from networks.utils import extend_flows
    rng = np.random.default_rng(T * 100 + net[0])
    mot = _motions(rng, T)
    fw = np.stack([SO.similarity_flow(m, *net, *hw, flow_scale=scale) for m in mot])
    fw += rng.normal(0, 0.5, fw.shape).astype(np.float32)  # a residual to extend
    bw = (-fw + rng.normal(0, 0.3, fw.shape)).astype(np.float32)
    efw, ebw = extend_flows(_t(cuda, fw), _t(cuda, bw), mot, hw, margin, scale)
    wfw, wbw = SF.extend_flows(fw, bw, mot, hw, margin, scale)
    assert np.array_equal(efw.cpu().numpy(), wfw) and np.array_equal(ebw.cpu().numpy(), wbw)
    my, mx = margin
    assert np.array_equal(efw.cpu().numpy()[:, my:my + net[0], mx:mx + net[1]], fw)
    # a field's bits do not depend on the batch
    one, _ = extend_flows(_t(cuda, fw[-1:]), _t(cuda, bw[-1:]), mot[-1:], hw, margin, scale)
    assert torch.equal(one[0], efw[-1])


def _fill_case(rng, F, hw, net, margin):
    frames = rng.integers(0, 256, (F,) + hw + (3,)).astype(np.uint8)
    mot = _motions(rng, F - 1)
    fw = np.stack([SO.similarity_flow(m, *net, *hw) for m in mot]) + rng.normal(0, 0.3, (F - 1,) + net + (2,))
    bw = np.stack([SO.similarity_flow(SF.inverse(m), *net, *hw) for m in mot]) + rng.normal(0, 0.3, (F - 1,) + net + (2,))
    efw, ebw = SF.extend_flows(fw.astype(np.float32), bw.astype(np.float32), mot, hw, margin)
    return frames, efw, ebw


def _raw_fill(cuda, frames, efw, ebw, net, margin, A, rows, a2=0.5):
    """rb_frames_warp_affine_fill called directly, so the table may hold what the wrapper refuses."""
    from raft_b200 import capi
    F, Hs, Ws, _ = frames.shape
    n = len(rows)
    f, fw, bw = _t(cuda, frames), _t(cuda, efw), _t(cuda, ebw)
    a, r = _t(cuda, np.asarray(A, np.float64)), _t(cuda, np.asarray(rows, np.int32))
    colour = torch.empty(n, Hs, Ws, 3, dtype=torch.float32, device=cuda)
    status = torch.empty(n, Hs, Ws, dtype=torch.uint8, device=cuda)
    with torch.cuda.device(cuda):
        capi.check(capi.lib.rb_frames_warp_affine_fill(capi.ptr(f), F, Hs, Ws, capi.ptr(fw), capi.ptr(bw), *net, *margin,
                                                       1.0, 0.01, a2, capi.ptr(a), capi.ptr(r), n, capi.ptr(colour),
                                                       capi.ptr(status), capi.stream()))
    return colour.cpu().numpy(), status.cpu().numpy()


def test_warp_fill_matches_oracle(cuda):
    rng = np.random.default_rng(5)
    F, hw, net, margin = 7, (45, 67), (21, 33), (4, 6)
    frames, efw, ebw = _fill_case(rng, F, hw, net, margin)
    rows = [[t, 3, 3] for t in range(F)] + [[3, 9, -2], [1, -1, 8], [-1, 2, 2], [F, 1, 1], [4, 0, 0], [2, 1, 1]]
    A = np.empty((len(rows), 2, 3))
    for r in range(len(rows)):
        th = rng.normal(0, 0.05)
        A[r] = [[np.cos(th), -np.sin(th), rng.normal(0, 5)], [np.sin(th), np.cos(th), rng.normal(0, 5)]]
    A[-2, 0, 2] = np.nan  # a NaN matrix: every source reads the clamped pixel
    A[-1] = [[1.0, 0, -30.0], [0, 1, 25.0]]  # sources far beyond the canvas
    for a2 in (0.5, 1e30):  # the test as in the occlusion check, and one every step passes
        colour, status = _raw_fill(cuda, frames, efw, ebw, net, margin, A, rows, a2)
        wc, ws = SF.warp_fill(frames, efw, ebw, net, margin, A, rows, a2=a2)
        assert np.array_equal(status, ws) and np.array_equal(colour.view(np.uint32), wc.view(np.uint32))
        assert (status[-4:-2] == 3).all() and (colour[-4:-2] == 0).all()  # absent rows
        assert (status[-2] == 0).all() and (status[-1] > 0).any()
        assert {1, 2}.issubset(set(np.unique(status[:F]).tolist())), np.unique(status)


def test_rows_before_a_cut_ignore_the_frames_after_it(cuda):
    from networks.utils import warp_frames_fill
    rng = np.random.default_rng(6)
    F, hw, net, margin = 8, (40, 60), (20, 30), (5, 5)
    frames, efw, ebw = _fill_case(rng, F, hw, net, margin)
    rows = inpaint_rows(F, 4, [3])
    A = np.tile(np.array([[1.0, 0, -6.0], [0, 1, 4.0]]), (F, 1, 1))
    run = lambda fr: [x.cpu().numpy() for x in warp_frames_fill(_t(cuda, fr), _t(cuda, efw), _t(cuda, ebw), net, margin,
                                                                A, rows, alpha2=1e30)]
    c0, s0 = run(frames)
    other = frames.copy()
    other[4:] = rng.integers(0, 256, other[4:].shape)
    c1, s1 = run(other)
    assert np.array_equal(c0[:4], c1[:4]) and np.array_equal(s0[:4], s1[:4])
    assert not np.array_equal(c0[4:], c1[4:])


def test_in_frame_pixels_are_the_warp_bytes(cuda):
    from networks.utils import extend_flows, warp_frames
    rng = np.random.default_rng(7)
    F, hw, net = 5, (44, 64), (22, 32)
    frames, efw, ebw = _fill_case(rng, F, hw, net, (3, 3))
    A = np.tile(np.array([[1.0, 0, 2.5], [0, 1, -3.25]]), (F, 1, 1))
    A[2] = [[0.99, -0.01, 1.0], [0.01, 0.99, 2.0]]
    margin = S.fill_margin(A, hw, net)
    assert margin != (0, 0)
    fw = _t(cuda, efw[:, 3:-3, 3:-3])
    efw_, ebw_ = extend_flows(fw, fw.clone(), np.tile([1.0, 0, 0, 0], (F - 1, 1)), hw, margin)
    out, status = S.fill_warp(_t(cuda, frames), efw_, ebw_, net, margin, _t(cuda, A), inpaint_rows(F, 10), 1.0)
    want = warp_frames(_t(cuda, frames), A)
    st = status.cpu().numpy()
    assert (st == 0).mean() > 0.8 and (st > 0).any()
    assert np.array_equal(out.cpu().numpy()[st == 0], want.cpu().numpy()[st == 0])
    # a path that needs no border: warp_frames' output exactly, all status 0, margin 0
    A = np.tile(np.array([[0.95, 0, 1.5], [0, 0.95, 1.1]]), (F, 1, 1))
    assert S.fill_margin(A, hw, net) == (0, 0)
    e = torch.zeros(F - 1, *net, 2, dtype=torch.float32, device=cuda)
    out, status = S.fill_warp(_t(cuda, frames), e, e, net, (0, 0), _t(cuda, A), inpaint_rows(F, 10), 1.0)
    assert torch.equal(out, warp_frames(_t(cuda, frames), A)) and (status == 0).all()


def test_known_path_at_a_realistic_size(cuda):
    """The texture clip of tests/test_stabilize_fill.py at 216 x 384 frames on a 108 x 192 grid, through the public
    pieces.  Thresholds as set from the CPU run of the oracle at 48 x 80."""
    from networks.utils import extend_flows
    F, hw, net = 16, (216, 384), (108, 192)
    G, mot = SF.jittered_path(F, 0, jitter=(3.0, 0.0), rot=0, zoom=0)
    frames = SF.render(G, hw)
    fw = np.stack([SO.similarity_flow(m, *net, *hw) for m in mot])
    bw = np.stack([SO.similarity_flow(SF.inverse(m), *net, *hw) for m in mot])
    A, _, _ = S.camera_transforms(mot, hw, 3.0, max_zoom=1.0)
    margin = S.fill_margin(A, hw, net)
    efw, ebw = extend_flows(_t(cuda, fw), _t(cuda, bw), mot, hw, margin)
    out, status = S.fill_warp(_t(cuda, frames), efw, ebw, net, margin, _t(cuda, A), inpaint_rows(F, 10), 1.0)
    out, st = out.cpu().numpy()[..., 0].astype(np.float64), status.cpu().numpy()
    true = SF.true_view(G, A, hw)
    rep = SO.warp(frames, A)[..., 0].astype(np.float64)
    filled = st > 0
    assert filled.sum() > 2000 and (st == 3).sum() == 0
    err, rerr = np.abs(out - true)[filled].mean(), np.abs(rep - true)[filled].mean()
    assert err < 0.6 and err < 0.15 * rerr, (err, rerr)


@pytest.fixture
def lenient(monkeypatch):
    """Seeded weights fail the forward-backward test almost everywhere, so every border pixel would go to the spatial
    fill and a wrong frame or pair index would change nothing.  Here the fill's alpha2 is so large that every step
    passes -- the real kernels on the real flows."""
    import raft_b200.engine as E
    monkeypatch.setattr(E, "FB_ALPHA2", 1e30)


def _composed(m, frames, sigma, window, cuts=()):
    """RAFT.stabilize(fill=True) from the public pieces."""
    from networks.utils import extend_flows, global_motion
    fw, bw, occ, _ = m.forward_sequence_bidirectional(frames)
    hw = frames.shape[1:3]
    params, _, _ = global_motion(fw, occ, hw, flow_scale=m.engine().flow_scale)
    A, _, _ = S.camera_transforms(params.cpu().numpy(), hw, sigma, cuts, 1.0)
    margin = S.fill_margin(A, hw, fw.shape[1:3])
    efw, ebw = extend_flows(fw, bw, S.fill_motions(params.cpu().numpy(), cuts), hw, margin, m.engine().flow_scale)
    out, st = S.fill_warp(_t("cuda:0", frames), efw, ebw, tuple(fw.shape[1:3]), margin, A,
                          inpaint_rows(len(frames), window, cuts), m.engine().flow_scale)
    return out, A, st


@pytest.mark.parametrize("small,size", [(False, None), (True, None), (False, (64, 96))])
def test_stabilize_fill_equals_its_parts(cuda, frame_dir, every_pixel, lenient, small, size):  # noqa: F811
    m = _model(small=small, input_size=size)
    frames = _decoded(frame_dir)
    out, A, status = m.stabilize(frames, 3.0, fill=True, window=4)
    want, wA, wst = _composed(m, frames, 3.0, 4)
    assert np.array_equal(A.cpu().numpy(), wA) and torch.equal(status, wst) and torch.equal(out, want)
    assert {1, 2, 3}.issubset(set(torch.unique(status).cpu().tolist())), torch.unique(status)
    plain, pA = m.stabilize(frames, 3.0, max_zoom=1.0)
    assert torch.equal(pA, A) and torch.equal(plain[status == 0], out[status == 0])
    with pytest.raises(ValueError, match="window"):
        m.stabilize(frames, 3.0, window=3)
    with pytest.raises(ValueError, match="window"):
        m.stabilize(frames, 3.0, fill=True, window=0)


# (1, 0, 2) keeps at most 7 of the 10 frames on the GPU, so the sweep drops frames it no longer needs
@pytest.mark.parametrize("batch,workers,window", [(1, 0, 10), (8, 4, 10), (3, 4, 10), (4, 0, 2), (1, 0, 2)])
def test_video_stabilize_fill_equals_stabilize(cuda, frame_dir, tmp_path, every_pixel, lenient, batch, workers, window,
                                               capsys):  # noqa: F811
    import cv2
    from raft_b200.video import video_stabilize
    m = _model(input_size=(64, 96))
    frames = _decoded(frame_dir)
    want, A, status = m.stabilize(frames, 2.5, fill=True, window=window)
    paths, info = video_stabilize(m, frame_dir, tmp_path, 2.5, batch=batch, workers=workers, fill=True, window=window)
    for i, p in enumerate(paths):
        assert np.array_equal(cv2.imread(p), want[i].cpu().numpy()), i
    assert np.array_equal(np.load(tmp_path / "transforms.npy"), A.cpu().numpy())
    counts = [int((status == s).sum()) for s in (1, 2, 3)]
    assert info["counts"] == counts and min(counts) > 0
    assert info["margin"] == S.fill_margin(A.cpu().numpy(), frames.shape[1:3], (64, 96))
    assert (f"stabilize fill: pixels filled from both sides {counts[0]}, from one side {counts[1]}, spatially "
            f"{counts[2]}") in capsys.readouterr().out


def test_video_stabilize_fill_across_a_scene_cut(cuda, frame_dir, tmp_path, every_pixel, lenient):  # noqa: F811
    import cv2
    from raft_b200.video import list_frames, video_stabilize
    d = tmp_path / "clip"
    d.mkdir()
    paths = []
    for i, p in enumerate(list_frames(frame_dir)):
        img = cv2.imread(p)
        paths.append(str(d / f"f{i:03d}.png"))
        cv2.imwrite(paths[-1], img if i < 6 else img // 5)  # a cut at pair 5
    m = _model()
    frames = np.stack([cv2.imread(p) for p in paths])
    want, A, status = m.stabilize(frames, 2.0, cuts=[5], fill=True, window=5)
    runs = {}
    for batch, workers in ((1, 0), (4, 4)):
        out = tmp_path / f"b{batch}"
        _, info = video_stabilize(m, paths, out, 2.0, batch=batch, workers=workers, scene_cut=0.5, fill=True, window=5)
        assert info["cuts"] == [5]
        runs[batch] = _files(out)
        for i in range(len(frames)):
            assert np.array_equal(cv2.imread(str(out / f"frame_{i:06d}.png")), want[i].cpu().numpy()), i
    assert runs[1] == runs[4]


def test_cli_writes_full_frames(cuda, frame_dir, tmp_path):
    import cv2
    np.savez(tmp_path / "w.npz", **_weights(False))
    out = tmp_path / "stable"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", frame_dir,
                        "--out", str(out), "--stabilize", "10", "--stabilize-fill", "--load", str(tmp_path / "w.npz"),
                        "--flow-size", "64", "96", "--iters", "4", "--batch", "3"], capture_output=True, text=True,
                       cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "zoom per shot 1.0000" in r.stdout and "stabilize fill: pixels filled from both sides" in r.stdout
    frames = _decoded(frame_dir)
    files = sorted(f for f in os.listdir(out) if f.endswith(".png"))
    assert len(files) == len(frames)
    assert all(cv2.imread(str(out / f)).shape == frames.shape[1:] for f in files)
