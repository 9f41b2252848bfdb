"""F18-F20 on the GPU: rb_flow_accumulate / _backward, rb_labels_propagate and rb_label_metrics against their
restatements (tests/propagate_oracle.py, tests/davis_oracle.py) bit for bit, RAFT.propagate against the composition of
the public pieces, and video_propagate / infer_raft.py --propagate end to end on shifted crops of
tests/data/frame_0016.png."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import davis_oracle as D
import propagate_oracle as P
from test_gpu_track import _model
from test_gpu_video import _decoded, _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def test_pillow_reads_label_maps():
    from PIL import Image  # noqa: F401  (the label PNG functions need it)


def _case(rng, T, H, W, nan=3):
    fw = (rng.uniform(-0.2, 0.2, (T, H, W, 2)) * np.array([W, H])).astype(F32)  # some pulls leave the frame
    bw = (-fw + rng.normal(0, 0.6, fw.shape)).astype(F32)
    for f in (fw, bw):
        for _ in range(nan):
            f[rng.integers(T), rng.integers(H), rng.integers(W), rng.integers(2)] = np.nan
    return fw, bw


def _t(cuda, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("T,H,W,scale", [(3, 37, 53, 1.0), (4, 37, 53, 8.0), (3, 1, 31, 1.0), (3, 29, 1, 1.0),
                                         (2, 1, 1, 1.0), (5, 96, 160, 1.0), (2, 61, 97, 8.0)])
@pytest.mark.parametrize("start", ["first", "middle", "last"])
def test_accumulate_equals_fp32_restatement_bit_for_bit(cuda, T, H, W, scale, start):
    from networks.utils import accumulate_flow, accumulate_flow_backward
    rng = np.random.default_rng(T * 1000 + H * 10 + W)
    fw, bw = _case(rng, T, H, W, nan=3 if H * W > 1 else 0)
    fw, bw = fw / F32(scale), bw / F32(scale)
    K = {"first": 0, "middle": T // 2, "last": T}[start]
    acc, st = P.keyframe_rows(T + 1, H, W, K)
    want_a, want_s = P.accumulate(fw, bw, acc, st, start=K, flow_scale=scale)
    want_a, want_s = P.accumulate_backward(fw, bw, want_a, want_s, start=K, flow_scale=scale)
    a, s = _t(cuda, acc), _t(cuda, st)
    accumulate_flow(_t(cuda, fw), _t(cuda, bw), a, s, start=K, flow_scale=scale)
    only_fw = a.cpu().numpy()
    assert np.isnan(only_fw[:K]).all() and (s.cpu().numpy()[:K] == 77).all()  # the forward entry leaves them alone
    accumulate_flow_backward(_t(cuda, fw), _t(cuda, bw), a, s, start=K, flow_scale=scale)
    assert _same(a.cpu().numpy(), want_a), "acc differs"
    assert np.array_equal(s.cpu().numpy(), want_s), f"{(s.cpu().numpy() != want_s).sum()} statuses differ"
    if H * W > 1000:
        assert all((want_s == k).any() for k in range(3))


@pytest.mark.parametrize("scale", [1.0, 8.0])
def test_first_row_is_the_occlusion_check_and_the_scaled_flow(cuda, scale):
    from networks.utils import accumulate_flow, fb_consistency
    rng = np.random.default_rng(11)
    T, H, W = 3, 45, 67
    fw, bw = _case(rng, T, H, W)
    fw, bw = _t(cuda, fw / F32(scale)), _t(cuda, bw / F32(scale))
    _, occ_bw = fb_consistency(fw, bw, flow_scale=scale)
    for K in range(T):
        a = torch.zeros(T + 1, H, W, 2, device=cuda)
        s = torch.zeros(T + 1, H, W, dtype=torch.uint8, device=cuda)
        accumulate_flow(fw, bw, a, s, start=K, flow_scale=scale)
        assert torch.equal(s[K + 1], occ_bw[K])
        inside = occ_bw[K] != 2
        assert _same(a[K + 1][inside].cpu().numpy(), (F32(scale) * bw[K]).cpu().numpy()[inside.cpu().numpy()])


def test_backward_equals_forward_on_the_reversed_clip(cuda):
    from networks.utils import accumulate_flow, accumulate_flow_backward
    rng = np.random.default_rng(12)
    T, H, W = 5, 50, 70
    fw, bw = _case(rng, T, H, W)
    rfw, rbw = P.reversed_clip(fw, bw)
    for K in (1, 3, 5):
        a, s = (_t(cuda, x) for x in P.keyframe_rows(T + 1, H, W, K))
        accumulate_flow_backward(_t(cuda, fw), _t(cuda, bw), a, s, start=K)
        ra, rs = (_t(cuda, x) for x in P.keyframe_rows(T + 1, H, W, T - K))
        accumulate_flow(_t(cuda, rfw), _t(cuda, rbw), ra, rs, start=T - K)
        assert _same(a.cpu().numpy()[:K + 1], ra.cpu().numpy()[::-1][:K + 1])
        assert np.array_equal(s.cpu().numpy()[:K + 1], rs.cpu().numpy()[::-1][:K + 1])


@pytest.mark.parametrize("bounds", [(0, 2, 6), (0, 1, 4, 6), (0, 3, 5, 6)])
def test_chained_passes_equal_one_pass(cuda, bounds):
    """Passes of 1-3 launches with row 0 carried, the later ones padded as a short last pass of video_propagate is."""
    from networks.utils import accumulate_flow
    rng = np.random.default_rng(13)
    T, H, W = 6, 41, 59
    fw, bw = _case(rng, T, H, W)
    whole_a, whole_s = (_t(cuda, x) for x in P.keyframe_rows(T + 1, H, W, 0))
    accumulate_flow(_t(cuda, fw), _t(cuda, bw), whole_a, whole_s)
    carry = (whole_a[0], whole_s[0])
    n_max = max(b - a for a, b in zip(bounds, bounds[1:]))
    for a, b in zip(bounds, bounds[1:]):
        pad = lambda f: np.concatenate([f[a:b]] + [f[b - 1:b]] * (n_max - (b - a)))  # noqa: E731
        ca = torch.full((b - a + 1, H, W, 2), float("nan"), device=cuda)
        cs = torch.full((b - a + 1, H, W), 9, dtype=torch.uint8, device=cuda)
        ca[0], cs[0] = carry
        accumulate_flow(_t(cuda, pad(fw)), _t(cuda, pad(bw)), ca, cs, n_steps=b - a)
        assert _same(ca.cpu().numpy(), whole_a[a:b + 1].cpu().numpy()) and torch.equal(cs, whole_s[a:b + 1])
        carry = (ca[-1], cs[-1])


@pytest.mark.parametrize("net,src", [((96, 160), (180, 320)), ((37, 53), (100, 150)), ((40, 60), (40, 60)),
                                     ((1, 31), (3, 40)), ((48, 64), (30, 50))])
def test_labels_equal_fp32_restatement_bit_for_bit(cuda, net, src):
    from networks.utils import accumulate_flow, propagate_labels
    rng = np.random.default_rng(net[0] * 7 + src[1])
    T, (H, W) = 3, net
    fw, bw = _case(rng, T, H, W, nan=0)
    acc, st = P.keyframe_rows(T + 1, H, W, 0)
    a, s = _t(cuda, acc), _t(cuda, st)
    accumulate_flow(_t(cuda, fw), _t(cuda, bw), a, s)
    key = rng.integers(0, 9, src).astype(np.uint8)
    key[src[0] // 3:, : src[1] // 2] = 4  # a region, so votes between equal labels happen too
    labels, status = propagate_labels(a, s, _t(cuda, key))
    want_l, want_s = P.propagate(a.cpu().numpy(), s.cpu().numpy(), key)
    assert np.array_equal(labels.cpu().numpy(), want_l), f"{(labels.cpu().numpy() != want_l).sum()} labels differ"
    assert np.array_equal(status.cpu().numpy(), want_s)
    assert np.array_equal(labels[0].cpu().numpy(), key) and (status[0] == 0).all()


def _masks(rng, n, H, W, objs):
    pred = np.zeros((n, H, W), np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    for i in range(n):
        for o in range(1, objs + 1):
            cy, cx = rng.uniform(-0.1, 1.1) * H, rng.uniform(-0.1, 1.1) * W  # some touch or cross the border
            ry, rx = rng.uniform(0.05, 0.4) * H + 1, rng.uniform(0.05, 0.4) * W + 1
            pred[i][((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1] = o
    gt = pred.copy()
    for i in range(n):
        gt[i] = np.roll(pred[i], rng.integers(-4, 5, 2), (0, 1))
        noise = rng.random((H, W)) < 0.01
        gt[i][noise] = rng.integers(0, objs + 2, noise.sum())
    if objs > 1:
        pred[:, pred[0] == 2] = 0  # an object that vanishes from the prediction
        gt[-1][gt[-1] == 1] = 0  # and one missing from the last ground truth
    return pred, gt


@pytest.mark.parametrize("n,H,W,objs,r", [(3, 64, 96, 3, 1), (2, 480, 854, 5, 8), (2, 480, 854, 12, 18),
                                         (4, 37, 53, 2, 8), (2, 33, 31, 1, 32), (3, 1, 45, 2, 3), (2, 20, 1, 2, 2),
                                         (1, 200, 300, 10, 18)])
def test_label_counts_equal_the_evaluator(cuda, n, H, W, objs, r):
    from networks.utils import label_metrics
    rng = np.random.default_rng(n * 100 + H + W + objs + r)
    pred, gt = _masks(rng, n, H, W, objs)
    got = label_metrics(_t(cuda, pred), _t(cuda, gt), objs, r).cpu().numpy()
    want = D.counts(pred, gt, objs, r)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]


def test_label_counts_of_random_and_border_masks(cuda):
    from networks.utils import label_metrics
    rng = np.random.default_rng(21)
    pred = rng.integers(0, 4, (2, 41, 67)).astype(np.uint8)
    gt = rng.integers(0, 4, (2, 41, 67)).astype(np.uint8)
    gt[1] = 1  # a full-frame object: its boundary is the last row and column of _seg2bmap only
    got = label_metrics(_t(cuda, pred), _t(cuda, gt), 3, 4).cpu().numpy()
    assert np.array_equal(got, D.counts(pred, gt, 3, 4))
    same = label_metrics(_t(cuda, gt), _t(cuda, gt), 3).cpu().numpy()  # DAVIS's radius for 41x67: 1
    assert np.array_equal(same[..., 4], same[..., 2]) and np.array_equal(same[..., 0], same[..., 1])


def _composed(m, frames, key, K):
    """RAFT.propagate from the public pieces: the flows of forward_sequence_bidirectional, accumulate_flow and
    accumulate_flow_backward from a zero row at K, propagate_labels at the frames' size."""
    from networks.utils import accumulate_flow, accumulate_flow_backward, propagate_labels
    fw, bw, _, _ = m.forward_sequence_bidirectional(frames, check=False)
    F, (H, W) = len(frames), fw.shape[1:3]
    a = torch.zeros(F, H, W, 2, device=fw.device)
    s = torch.zeros(F, H, W, dtype=torch.uint8, device=fw.device)
    kw = dict(start=K, flow_scale=m.engine().flow_scale)
    accumulate_flow(fw, bw, a, s, **kw)
    accumulate_flow_backward(fw, bw, a, s, **kw)
    return propagate_labels(a, s, _t(fw.device, key))


@pytest.mark.parametrize("input_size", [None, (128, 160)])
@pytest.mark.parametrize("upstream", [False, True])
@pytest.mark.parametrize("small", [False, True])
def test_raft_propagate_equals_the_public_pieces(cuda, small, upstream, input_size):
    m = _model(small, upstream=upstream, input_size=input_size)
    frames = _frames(5, 125, 150, seed=5100 + 2 * small + upstream)
    key = np.zeros((125, 150), np.uint8)
    key[30:90, 40:110] = 1
    key[50:70, 60:140] = 2
    for K in (0, 2, 4):
        labels, status = m.propagate(frames, key, frame=K)
        assert labels.shape == status.shape == (5, 125, 150) and labels.dtype == status.dtype == torch.uint8
        want_l, want_s = _composed(m, frames, key, K)
        assert torch.equal(labels, want_l) and torch.equal(status, want_s)
        assert np.array_equal(labels[K].cpu().numpy(), key) and (status[K] == 0).all()
        assert set(np.unique(labels.cpu().numpy())) <= {0, 1, 2}


def test_raft_propagate_refusals(cuda):
    m = _model()
    frames = _frames(3, 60, 80)
    for key, frame, words in ((np.zeros((60, 81), np.uint8), 0, "uint8 map"), (np.zeros((60, 80)), 0, "uint8 map"),
                              (np.zeros((60, 80), np.uint8), 3, r"\[0, 3\)"),
                              (np.zeros((60, 80), np.uint8), -1, r"\[0, 3\)")):
        with pytest.raises(ValueError, match=words):
            m.propagate(frames, key, frame=frame)


def test_video_propagate_end_to_end(cuda, frame_dir, tmp_path):
    from raft_b200.synth import DAVIS_PALETTE
    from raft_b200.video import read_labels, video_propagate, write_labels
    m = _model()
    frames = _decoded(frame_dir)
    F, H, W = frames.shape[:3]
    key = np.zeros((H, W), np.uint8)
    key[20:90, 30:100] = 3
    key[40:60, 50:140] = 7
    write_labels(tmp_path / "key.png", key, DAVIS_PALETTE)
    for K in (0, 5, F - 1):
        want_l, want_s = (x.cpu().numpy() for x in m.propagate(frames, key, frame=K))
        runs = {}
        for batch, workers in ((1, 0), (3, 4), (8, 4), (8, 0)):
            out = tmp_path / f"k{K}b{batch}w{workers}"
            files, last = video_propagate(m, frame_dir, str(out), str(tmp_path / "key.png"), frame=K, batch=batch,
                                          workers=workers)
            assert files == [str(out / f"label_{i:06d}.png") for i in range(F)]
            assert np.array_equal(last, want_s[-1])
            runs[(batch, workers)] = _files(str(out))
        assert all(r == runs[(1, 0)] for r in runs.values())
        got = np.stack([read_labels(f)[0] for f in files])
        assert np.array_equal(got, want_l)
        assert np.array_equal(read_labels(files[0])[1][:len(DAVIS_PALETTE)], DAVIS_PALETTE)
    grey, _ = video_propagate(m, frame_dir, str(tmp_path / "grey"), key, frame=5, batch=3)  # an array key: grey PNGs
    assert read_labels(grey[0])[1] is None and np.array_equal(read_labels(grey[5])[0], key)


def test_cli_propagate(cuda, frame_dir, tmp_path):
    from raft_b200 import synth
    from raft_b200.video import read_labels, write_labels
    np.savez(tmp_path / "w.npz", **synth.make_weights(False))
    H, W = _decoded(frame_dir).shape[1:3]
    key = np.zeros((H, W), np.uint8)
    key[10:80, 20:120] = 1
    write_labels(tmp_path / "key.png", key, synth.DAVIS_PALETTE)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", frame_dir,
                        "--out", str(tmp_path / "o"), "--propagate", str(tmp_path / "key.png"), "--propagate-frame",
                        "2", "--load", str(tmp_path / "w.npz"), "--keep-size", "--batch", "3", "--iters", "4"],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert "propagated through 10 frames" in r.stdout, r.stdout
    assert np.array_equal(read_labels(tmp_path / "o" / "label_000002.png")[0], key)
