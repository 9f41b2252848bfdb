"""F22 / F23 on the GPU: rb_global_motion against the fp64 oracle (tests/stabilize_oracle.py) and its invariants,
rb_frames_warp_affine against the oracle bit for bit, RAFT.stabilize against the composition of its parts,
video_stabilize / infer_raft.py --stabilize end to end with seeded weights (plumbing, not quality), and the host path fed
the analytic flows of a known jittered camera path."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import stabilize_oracle as O
from raft_b200.stabilize import MOTION_ROUNDS
from test_gpu_track import _model, _weights
from test_gpu_video import _decoded, _files, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _pairs(rng, B, net, src, scale):
    """B flows of random similarities with noise, an outlier block, occluded pixels and a NaN, and their masks."""
    Hn, Wn = net
    flows, occs, truth = [], [], []
    for _ in range(B):
        th, s = rng.normal(0, 0.01), 1 + rng.normal(0, 0.01)
        M = (s * math.cos(th), s * math.sin(th), rng.normal(0, 5), rng.normal(0, 5))
        f = O.similarity_flow(M, Hn, Wn, *src, flow_scale=scale)
        f += rng.normal(0, 0.2 / scale, f.shape).astype(np.float32)
        h, w = max(1, Hn // 3), max(1, Wn // 3)
        f[:h, :w] += np.float32(6.0 / scale)
        if Hn * Wn > 4:
            f[Hn - 1, Wn - 1, 0] = np.nan
        flows.append(f)
        occs.append((rng.random((Hn, Wn)) < 0.15).astype(np.uint8))
        truth.append(M)
    return np.stack(flows), np.stack(occs), truth


@pytest.mark.parametrize("net,src,scale", [((432, 1024), (1080, 1920), 1.0), ((96, 160), (96, 160), 1.0),
                                           ((37, 53), (101, 149), 1.0), ((55, 71), (440, 568), 8.0)])
def test_global_motion_matches_oracle(cuda, net, src, scale):
    from networks.utils import global_motion
    rng = np.random.default_rng(net[0] + src[1])
    flow, occ, truth = _pairs(rng, 3, net, src, scale)
    f, o = _t(cuda, flow), _t(cuda, occ)
    # the sums of each round against the oracle's on the same previous-round parameters: only the summation order differs
    prev = None
    for r in sorted({0, 1, 2, MOTION_ROUNDS}):
        if r > 0:
            prev = global_motion(f, o, src, flow_scale=scale, rounds=r - 1)[0].cpu().numpy()
        sums = global_motion(f, o, src, flow_scale=scale, rounds=r, return_sums=True)[3].cpu().numpy()
        for b in range(len(flow)):
            w_sums, w_abs = O.round_sums(flow[b], occ[b], src, scale, None if prev is None else prev[b])
            err = np.abs(sums[b] - w_sums)
            assert (err <= 1e-12 * w_abs).all(), (r, b, (err / w_abs).max())
    params, weight, reliable = global_motion(f, o, src, flow_scale=scale)
    w_params, w_weight, w_flags, _, _ = O.global_motion(flow, occ, src, flow_scale=scale)
    assert np.array_equal(reliable.cpu().numpy(), w_flags == 0) and reliable.all()
    assert np.array_equal(weight.cpu().numpy(), w_weight)  # a count over Hn Wn: exact
    p = params.cpu().numpy()
    assert (np.abs(p - w_params) <= 1e-9 * np.maximum(1.0, np.abs(w_params))).all(), np.abs(p - w_params).max()
    for b, M in enumerate(truth):
        assert O.corner_error(p[b], M, src) < 0.5  # the outlier block and the noise are rejected


def test_global_motion_is_deterministic_and_batch_independent(cuda):
    from networks.utils import global_motion
    rng = np.random.default_rng(7)
    flow, occ, _ = _pairs(rng, 8, (108, 256), (270, 640), 1.0)
    f, o = _t(cuda, flow), _t(cuda, occ)
    a = global_motion(f, o, (270, 640), return_sums=True)
    b = global_motion(f, o, (270, 640), return_sums=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for i in (0, 3, 7):
        one = global_motion(f[i:i + 1].clone(), o[i:i + 1].clone(), (270, 640), return_sums=True)
        assert all(torch.equal(x[i:i + 1], y) for x, y in zip(a, one)), i


def test_unreliable_pairs_get_the_identity(cuda):
    from networks.utils import global_motion
    rng = np.random.default_rng(8)
    flow, occ, _ = _pairs(rng, 3, (40, 60), (80, 120), 1.0)
    occ[0] = 1  # every pixel occluded
    occ[1] = 1
    occ[1, :2, :2] = 0  # 4 of 2400 pixels: below the floor
    occ[2] = 1
    occ[2, :, 5:10] = 0  # a band of columns: 200 of 2400 pixels, above the floor
    params, weight, reliable = global_motion(_t(cuda, flow), _t(cuda, occ), (80, 120))
    p = params.cpu().numpy()
    assert reliable.cpu().tolist() == [False, False, True]
    assert np.array_equal(p[:2], [[1, 0, 0, 0]] * 2)
    assert weight.cpu().tolist()[:2] == [0.0, 4 / 2400]
    w_params, _, w_flags, _, _ = O.global_motion(flow, occ, (80, 120))
    assert w_flags.tolist() == [1, 1, 0]
    with pytest.raises(ValueError, match="occ_fw"):
        global_motion(_t(cuda, flow), _t(cuda, occ[:2]), (80, 120))


@pytest.mark.parametrize("F,H,W,C", [(1, 64, 96, 3), (3, 37, 53, 1), (4, 101, 149, 3), (2, 1, 7, 3)])
def test_warp_matches_oracle_bit_for_bit(cuda, F, H, W, C):
    from networks.utils import warp_frames
    rng = np.random.default_rng(F * 100 + H)
    frames = rng.integers(0, 256, (F, H, W, C)).astype(np.uint8)
    A = np.empty((F, 2, 3))
    for f in range(F):
        th, s = rng.normal(0, 0.3), math.exp(rng.normal(0, 0.2))
        A[f] = [[s * math.cos(th), -s * math.sin(th), rng.normal(0, W / 4)],
                [s * math.sin(th), s * math.cos(th), rng.normal(0, H / 4)]]  # many positions leave the frame
    if F > 2:
        A[1] = [[1, 0, 0.5], [0, 1, -0.25]]
        A[2, 0, 2] = np.nan
    got = warp_frames(_t(cuda, frames), A).cpu().numpy()
    assert np.array_equal(got, O.warp(frames, A))
    ident = np.tile(np.array([[1.0, 0, 0], [0, 1, 0]]), (F, 1, 1))
    assert np.array_equal(warp_frames(_t(cuda, frames), ident).cpu().numpy(), frames)


@pytest.fixture
def every_pixel(monkeypatch):
    """The end-to-end tests run seeded weights, whose flows fail the forward-backward check on most pixels: every pair
    would fall below the reliability floor, every motion would be the identity and every warp a copy, so a wrong pair or
    frame index in the sweeps would change nothing.  Here the fit counts every pixel instead -- the real kernel on the
    real flows -- so each pair gets its own non-identity motion and such an error changes the output."""
    import networks.utils as U
    real = U.global_motion

    def fit(flow_fw, occ_fw, *args, **kw):
        return real(flow_fw, torch.zeros_like(occ_fw), *args, **kw)
    monkeypatch.setattr(U, "global_motion", fit)


def _assert_moves(A, frames=None, out=None):
    """The precondition of the end-to-end comparisons: the transforms are not the identity and differ from frame to
    frame inside the clip (a shot's first and last frames keep their own path: their correction is only the zoom), and
    the warp changed the frames."""
    A = np.asarray(A)
    assert np.abs(A - np.array([[1.0, 0, 0], [0, 1, 0]])).max() > 1e-3
    assert len({a.tobytes() for a in A[1:-1]}) == len(A) - 2
    if out is not None:
        assert any(not np.array_equal(o, f) for o, f in zip(out, frames))


def _composed(m, frames, sigma, cuts=(), max_zoom=None):
    """RAFT.stabilize from the public pieces."""
    from networks.utils import global_motion, warp_frames
    from raft_b200.stabilize import DEFAULT_MAX_ZOOM, camera_transforms
    fw, _, occ, _ = m.forward_sequence_bidirectional(frames)
    hw = frames.shape[1:3]
    params, _, _ = global_motion(fw, occ, hw, flow_scale=m.engine().flow_scale)
    A, _, _ = camera_transforms(params.cpu().numpy(), hw, sigma, cuts, max_zoom or DEFAULT_MAX_ZOOM)
    return warp_frames(_t("cuda:0", frames), A), A


@pytest.mark.parametrize("small,size", [(False, None), (True, None), (False, (64, 96))])
def test_stabilize_equals_its_parts(cuda, frame_dir, every_pixel, small, size):
    m = _model(small=small, input_size=size)
    frames = _decoded(frame_dir)
    out, A = m.stabilize(frames, 3.0)
    want, wA = _composed(m, frames, 3.0)
    assert out.shape == frames.shape and out.dtype == torch.uint8
    _assert_moves(wA, frames, want.cpu().numpy())
    assert torch.equal(out, want) and np.array_equal(A.cpu().numpy(), wA)
    for bad, words in (({"sigma": 0}, "sigma"), ({"sigma": 2, "cuts": [9]}, "cuts"),
                       ({"sigma": 2, "max_zoom": 0.5}, "max_zoom")):
        with pytest.raises(ValueError, match=words):
            m.stabilize(frames, **bad)
    with pytest.raises(ValueError, match="uint8"):
        m.stabilize(frames.astype(np.float32) / 255, 2.0)


@pytest.mark.parametrize("batch,workers", [(1, 0), (8, 4), (3, 4)])
def test_video_stabilize_equals_stabilize(cuda, frame_dir, tmp_path, every_pixel, batch, workers):
    import cv2
    from raft_b200.video import video_stabilize
    m = _model(input_size=(64, 96))
    frames = _decoded(frame_dir)
    want, A = m.stabilize(frames, 2.5)
    _assert_moves(A.cpu().numpy(), frames, want.cpu().numpy())
    paths, info = video_stabilize(m, frame_dir, tmp_path, 2.5, batch=batch, workers=workers)
    assert len(paths) == len(want) and info["cuts"] == [] and len(info["zooms"]) == 1 and info["unreliable"] == []
    for i, p in enumerate(paths):
        assert np.array_equal(cv2.imread(p), want[i].cpu().numpy()), i
    assert np.array_equal(np.load(tmp_path / "transforms.npy"), A.cpu().numpy())


def test_scene_cuts_split_the_path(cuda, frame_dir, tmp_path, every_pixel):
    import cv2
    from raft_b200.video import list_frames, video_stabilize
    src = list_frames(frame_dir)
    d = tmp_path / "clip"
    d.mkdir()
    paths = []
    for i, p in enumerate(src):
        img = cv2.imread(p)
        if i >= 6:
            img = img // 5  # a darkened segment: a cut at pair 5
        paths.append(str(d / f"f{i:03d}.png"))
        cv2.imwrite(paths[-1], img)
    m = _model()
    runs = {}
    for batch, workers in ((1, 0), (4, 4)):
        out = tmp_path / f"b{batch}"
        _, info = video_stabilize(m, paths, out, 2.0, batch=batch, workers=workers, scene_cut=0.5)
        assert info["cuts"] == [5] and len(info["zooms"]) == 2 and info["unreliable"] == []
        runs[batch] = _files(out)
    assert runs[1] == runs[4]
    A = np.load(tmp_path / "b1" / "transforms.npy")
    _assert_moves(A[:6])
    _assert_moves(A[6:])
    for lo, hi in ((0, 6), (6, 10)):  # each shot alone
        out = tmp_path / f"shot{lo}"
        video_stabilize(m, paths[lo:hi], out, 2.0, batch=3, workers=0)
        assert np.array_equal(np.load(out / "transforms.npy"), A[lo:hi])
        for i in range(hi - lo):
            assert runs[1][f"frame_{lo + i:06d}.png"] == _files(out)[f"frame_{i:06d}.png"]
    frames = np.stack([cv2.imread(p) for p in paths])
    _, gA = m.stabilize(frames, 2.0, cuts=[5])
    assert np.array_equal(gA.cpu().numpy(), A)


def test_cli_writes_stabilized_frames(cuda, frame_dir, tmp_path):
    import cv2
    np.savez(tmp_path / "w.npz", **_weights(False))
    out = tmp_path / "stable"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", frame_dir,
                        "--out", str(out), "--stabilize", "10", "--load", str(tmp_path / "w.npz"), "--flow-size",
                        "64", "96", "--iters", "4", "--batch", "3"], capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "zoom per shot" in r.stdout and "scene cuts: 0" in r.stdout and "unreliable pairs" in r.stdout
    frames = _decoded(frame_dir)
    files = sorted(f for f in os.listdir(out) if f.endswith(".png"))
    assert len(files) == len(frames)
    assert all(cv2.imread(str(out / f)).shape == frames.shape[1:] for f in files)
    assert np.load(out / "transforms.npy").shape == (len(frames), 2, 3)


def test_known_jittered_path_is_recovered(cuda):
    """A clip rendered from a large texture along a known path -- a pan with rotation and zoom jitter -- and global_motion
    fed the analytic flows of that path: the transforms equal those of the true motions within 1e-3 px at the corners,
    and the stabilized clip moves less from frame to frame than the input."""
    from networks.utils import global_motion, warp_frames
    from raft_b200.stabilize import camera_transforms
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(11)
    F, Hs, Ws, Hn, Wn = 24, 216, 384, 108, 192
    t = np.arange(F)
    th = 0.002 * t + rng.normal(0, 0.01, F)
    sc = 1 + rng.normal(0, 0.01, F)
    tx, ty = 1.5 * t + rng.normal(0, 4, F), rng.normal(0, 4, F)
    G = np.stack([np.array([[s * math.cos(a), -s * math.sin(a), x], [s * math.sin(a), s * math.cos(a), y],
                                       [0, 0, 1]]) for s, a, x, y in zip(sc, th, tx, ty)])  # frame -> texture, centred
    M = np.stack([np.linalg.inv(G[k + 1]) @ G[k] for k in range(F - 1)])  # frame k -> frame k + 1
    motions = np.stack([M[:, 0, 0], M[:, 1, 0], M[:, 0, 2], M[:, 1, 2]], 1)
    flows = np.stack([O.similarity_flow(m, Hn, Wn, Hs, Ws) for m in motions])
    params, _, reliable = global_motion(_t(cuda, flows), torch.zeros(F - 1, Hn, Wn, dtype=torch.uint8, device=cuda),
                                        (Hs, Ws))
    assert reliable.all()
    got, _, _ = camera_transforms(params.cpu().numpy(), (Hs, Ws), 4.0)
    want, _, _ = camera_transforms(motions, (Hs, Ws), 4.0)
    c = np.array([[0, 0, 1], [Ws - 1, 0, 1], [0, Hs - 1, 1], [Ws - 1, Hs - 1, 1]], np.float64)
    assert np.abs(np.einsum("fij,cj->fci", got - want, c)).max() < 1e-3
    # render: frame t is the texture at G_t p, a centred crop of a warp of the 4x texture
    tex = gaussian_filter(rng.random((4 * Hs, 4 * Ws)), 3)
    tex = np.clip((tex - tex.mean()) / tex.std() * 50 + 128, 0, 255).astype(np.uint8)
    big = _t(cuda, np.repeat(tex[None, ..., None], F, 0))
    T = np.eye(3)
    T[:2, 2] = (2 * Ws - 0.5, 2 * Hs - 0.5)  # the texture's centre; the output crop's centre below is the same point
    Ti = np.linalg.inv(T)
    clip = warp_frames(big, (T @ G @ Ti)[:, :2])
    y0, x0 = (4 * Hs - Hs) // 2, (4 * Ws - Ws) // 2
    clip = clip[:, y0:y0 + Hs, x0:x0 + Ws].contiguous()
    stable = warp_frames(clip, got).cpu().numpy().astype(np.float64)[:, 40:-40, 60:-60]
    shaky = clip.cpu().numpy().astype(np.float64)[:, 40:-40, 60:-60]
    assert np.abs(np.diff(stable, axis=0)).mean() < 0.7 * np.abs(np.diff(shaky, axis=0)).mean()
