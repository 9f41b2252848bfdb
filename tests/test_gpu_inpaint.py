"""F24 / F25 on the GPU: rb_masked_fill, rb_inpaint_masks and rb_inpaint_propagate against the numpy restatements bit
for bit (tests/inpaint_oracle.py), exact recovery of a translating background behind a moving occluder, RAFT.inpaint
against its parts and the oracle, video_inpaint against RAFT.inpaint for several batch, window and worker counts, scene
cuts and the CLI.  The end-to-end tests run seeded weights: plumbing, not quality."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import inpaint_oracle as O
from raft_b200 import inpaint as I
from test_gpu_track import _model, _weights
from test_gpu_video import _decoded, frame_dir  # noqa: F401  (frame_dir: the module fixture)
from test_inpaint import HOLES, field_of, hole_of

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.mark.parametrize("C", [2, 3])
def test_masked_fill_matches_oracle(cuda, C):
    from networks.utils import masked_fill
    vals = np.stack([field_of("smooth" if i % 2 else "noise", C, seed=i) for i in range(len(HOLES))])
    holes = np.stack([hole_of(k, seed=i) for i, k in enumerate(HOLES)]).astype(np.uint8)
    got, empty = masked_fill(_t(cuda, vals), _t(cuda, holes))
    got = got.cpu().numpy()
    assert not empty.any()
    for i in range(len(HOLES)):
        want, flag = O.masked_fill(vals[i], holes[i])
        assert flag == 0 and np.array_equal(got[i], want), HOLES[i]
    # a field's bits depend neither on B nor on its place, and repeated runs agree
    perm = [3, 0, 4, 2, 1]
    again, _ = masked_fill(_t(cuda, vals[perm]), _t(cuda, holes[perm]))
    assert np.array_equal(again.cpu().numpy(), got[perm])
    one, _ = masked_fill(_t(cuda, vals[2:3]), _t(cuda, holes[2:3]).bool())
    assert np.array_equal(one.cpu().numpy()[0], got[2])
    # a fully masked field gives zeros and the flag; a constant field stays bit for bit
    v = np.stack([vals[0], np.full_like(vals[0], 0.37)])
    h = np.stack([np.ones_like(holes[0]), holes[0]])
    out, empty = masked_fill(_t(cuda, v), _t(cuda, h))
    assert empty.cpu().tolist() == [True, False]
    assert not out[0].any() and np.array_equal(out[1].cpu().numpy(), v[1])


@pytest.mark.parametrize("shape", [(3, 1, 1), (2, 1, 37), (2, 17, 5), (1, 433, 1025)])
def test_masked_fill_odd_shapes(cuda, shape):
    from networks.utils import masked_fill
    rng = np.random.default_rng(sum(shape))
    v = rng.normal(0, 3, shape + (2,)).astype(np.float32)
    h = (rng.random(shape) < 0.3).astype(np.uint8)
    got, empty = masked_fill(_t(cuda, v), _t(cuda, h))
    for b in range(shape[0]):
        want, flag = O.masked_fill(v[b], h[b])
        assert np.array_equal(got[b].cpu().numpy(), want) and bool(empty[b]) == bool(flag)


@pytest.mark.parametrize("src,net,dilate,labels", [((41, 57), (41, 57), 2, None), ((72, 130), (32, 48), 1, [2, 5]),
                                                   ((23, 31), (40, 64), 0, None), ((30, 44), (30, 20), 3, [7])])
def test_masks_match_oracle(cuda, src, net, dilate, labels):
    from networks.utils import inpaint_masks
    rng = np.random.default_rng(src[0] + net[1])
    masks = (rng.integers(0, 8, (3,) + src) * (rng.random((3,) + src) < 0.05)).astype(np.uint8)
    hole, hole_net = inpaint_masks(_t(cuda, masks), net, dilate, labels)
    w_hole, w_net = O.inpaint_masks(masks, I.selection_table(labels), dilate, *net)
    assert np.array_equal(hole.cpu().numpy(), w_hole) and np.array_equal(hole_net.cpu().numpy(), w_net)


def _random_clip(rng, F, src, net, occ=0.15):
    Hs, Ws = src
    Hn, Wn = net
    frames = rng.integers(0, 256, (F, Hs, Ws, 3), dtype=np.uint8)
    hole = np.zeros((F, Hs, Ws), np.uint8)
    for f in range(F):  # a blob per frame, and scattered holes
        y, x = rng.integers(0, Hs - 8), rng.integers(0, Ws - 8)
        hole[f, y:y + Hs // 3, x:x + Ws // 3] = 1
    hole |= (rng.random(hole.shape) < occ).astype(np.uint8)
    fw = (rng.normal(0, 1.2, (F - 1, Hn, Wn, 2)) + np.array([0.7, -0.4])).astype(np.float32)
    bw = (-fw + rng.normal(0, 0.08, fw.shape)).astype(np.float32)
    return frames, hole, fw, bw


@pytest.mark.parametrize("src,net,scale", [((40, 56), (40, 56), 1.0), ((75, 101), (32, 48), 1.0),
                                           ((30, 44), (48, 64), 8.0)])
def test_inpaint_propagate_matches_oracle(cuda, src, net, scale):
    from networks.utils import inpaint_propagate
    rng = np.random.default_rng(src[1] + net[0])
    F = 8
    frames, hole, fw, bw = _random_clip(rng, F, src, net)
    fw, bw = fw / np.float32(scale), bw / np.float32(scale)
    rows = np.concatenate([I.inpaint_rows(F, 3), I.inpaint_rows(F, 2, [3])[::-1], I.inpaint_rows(F, 10, [0, 5])])
    colour, status = inpaint_propagate(_t(cuda, frames), _t(cuda, hole), _t(cuda, fw), _t(cuda, bw), rows,
                                       flow_scale=scale)
    w_colour, w_status = O.inpaint_propagate(frames, hole, fw, bw, rows, scale)
    assert np.array_equal(status.cpu().numpy(), w_status)
    assert np.array_equal(colour.cpu().numpy(), w_colour)
    st = w_status[hole[rows[:, 0]] == 1]
    assert (st == 1).any() and (st == 2).any() and (st == 3).any()  # every outcome is exercised


def test_inpaint_propagate_refuses_bad_tables(cuda):
    from networks.utils import inpaint_propagate
    rng = np.random.default_rng(0)
    frames, hole, fw, bw = _random_clip(rng, 4, (16, 20), (16, 20))
    args = [_t(cuda, a) for a in (frames, hole, fw, bw)]
    for rows in ([[4, 0, 0]], [[1, 3, 0]], [[1, 0, 2]], [[0, -1, 0]], [[0.5, 0, 0]], [0, 0, 0]):
        with pytest.raises(ValueError):
            inpaint_propagate(*args, rows)


def _recovery_clip(F, H, W, d, seed=4):
    """A textured background translating by the integer d per frame behind a textured rectangle that drifts down and
    wobbles: frames, occluder masks, the true background of every frame."""
    rng = np.random.default_rng(seed)
    from scipy.ndimage import gaussian_filter
    big = (gaussian_filter(rng.random((H + F * abs(d[1]) + 2, W + F * abs(d[0]) + 2, 3)), (1.5, 1.5, 0)) * 255 * 4
           ).clip(0, 255).astype(np.uint8)
    ox, oy = F * max(d[0], 0) + 1, F * max(d[1], 0) + 1
    bg = np.stack([big[oy - t * d[1]:oy - t * d[1] + H, ox - t * d[0]:ox - t * d[0] + W] for t in range(F)])
    frames = bg.copy()
    masks = np.zeros((F, H, W), np.uint8)
    tex = rng.integers(0, 256, (H // 4, W // 5, 3), dtype=np.uint8)
    for t in range(F):
        y, x = H // 3 + (t % 3) - t * d[1] // 2, W // 3 - t * d[0] + 2 * t
        y, x = int(np.clip(y, 0, H - tex.shape[0])), int(np.clip(x, 0, W - tex.shape[1]))
        frames[t, y:y + tex.shape[0], x:x + tex.shape[1]] = tex
        masks[t, y:y + tex.shape[0], x:x + tex.shape[1]] = 1
    return frames, masks, bg


def test_exact_recovery_of_a_translating_background(cuda):
    from networks.utils import inpaint_masks
    from raft_b200.inpaint import complete_flows, fill_frames
    F, H, W, d = 12, 60, 90, (2, -1)
    frames, masks, bg = _recovery_clip(F, H, W, d)
    fw = np.broadcast_to(np.array(d, np.float32), (F - 1, H, W, 2)).copy()
    bw = -fw
    # inside the occluder the given flows are the occluder's: completion must restore the background's
    fw[:, 28:34, 32:46] = 7.5  # inside every frame's occluder
    bw[:, 28:34, 32:46] = -3.25
    hole, hole_net = inpaint_masks(_t(cuda, masks), (H, W), 0)
    cfw, cbw = complete_flows(_t(cuda, fw), _t(cuda, bw), hole_net)
    out, status = fill_frames(_t(cuda, frames), hole, cfw, cbw, I.inpaint_rows(F, F), 1.0)
    out, status = out.cpu().numpy(), status.cpu().numpy()
    assert np.array_equal(out[masks == 0], frames[masks == 0]) and (status[masks == 0] == 0).all()
    seen = (status == 1) | (status == 2)
    assert seen.sum() > 0.9 * masks.sum()
    assert np.array_equal(out[seen], bg[seen])  # byte for byte wherever some frame in the window sees the background
    for t in range(F):  # what no frame sees stays within the range of the frame's known values
        left = status[t] == 3
        if left.any():
            known = out[t][~left]
            assert (out[t][left] >= known.min(0)).all() and (out[t][left] <= known.max(0)).all()


@pytest.fixture
def lenient(monkeypatch):
    """The end-to-end tests run seeded weights, whose flows fail the forward-backward test almost everywhere: every hole
    pixel would go to the spatial fill, so a wrong frame, pair or row index in the temporal fill or the sweep would
    change nothing.  Here the test's constant alpha2 is so large that every step passes -- the real kernels on the real
    flows -- so the sides chain through the flows and find other frames."""
    import raft_b200.engine as E
    monkeypatch.setattr(E, "FB_ALPHA2", 1e30)
    return 1e30


def _ellipse_masks(F, H, W, label=1):
    yy, xx = np.mgrid[0:H, 0:W]
    m = np.zeros((F, H, W), np.uint8)
    for t in range(F):
        cy, cx = H / 2 + 3 * np.sin(t / 2), W / 3 + 4 * t
        m[t][((yy - cy) / (H / 6)) ** 2 + ((xx - cx) / (W / 8)) ** 2 < 1] = label
    m[:, :4, :6] = label + 1  # a second object in the corner
    return m


@pytest.mark.parametrize("small,size", [(False, (64, 96)), (True, None)])
def test_raft_inpaint_equals_its_parts_and_the_oracle(cuda, frame_dir, lenient, small, size):
    from networks.utils import inpaint_masks
    from raft_b200.inpaint import complete_flows, fill_frames
    m = _model(small=small, input_size=size)
    frames = _decoded(frame_dir)
    F, Hs, Ws = frames.shape[:3]
    masks = _ellipse_masks(F, Hs, Ws)
    out, status = m.inpaint(frames, masks, window=3, dilate=1, labels=[1, 2], cuts=[6])
    eng = m.engine()
    fw, bw, _, _ = eng.forward_sequence_bidirectional(_t(cuda, frames), check=False)
    fw, bw = fw.clone(), bw.clone()
    hole, hole_net = inpaint_masks(_t(cuda, masks), fw.shape[1:3], 1, [1, 2])
    cfw, cbw = complete_flows(fw, bw, hole_net)
    rows = I.inpaint_rows(F, 3, [6])
    w_out, w_status = fill_frames(_t(cuda, frames), hole, cfw, cbw, rows, eng.flow_scale)
    assert torch.equal(out, w_out) and torch.equal(status, w_status)
    o_out, o_status = O.inpaint(frames, masks, fw.cpu().numpy(), bw.cpu().numpy(), rows, I.selection_table([1, 2]), 1,
                                eng.flow_scale, a2=lenient)
    assert np.array_equal(status.cpu().numpy(), o_status) and np.array_equal(out.cpu().numpy(), o_out)
    assert (o_status == 1).any() and (o_status == 2).any()  # the chains reach other frames


def test_inpaint_refusals(cuda, frame_dir):
    m = _model(input_size=(64, 96))
    frames = _decoded(frame_dir)
    F, Hs, Ws = frames.shape[:3]
    good = np.zeros((F, Hs, Ws), np.uint8)
    for kw in (dict(masks=good[:-1]), dict(masks=good.astype(np.int32)), dict(window=0), dict(dilate=40),
               dict(labels=[]), dict(cuts=[F - 1])):
        args = dict(masks=good) | kw
        with pytest.raises(ValueError):
            m.inpaint(frames, **args)
    with pytest.raises(ValueError):
        m.inpaint(frames.astype(np.float32), good)


def _mask_dir(d, masks):
    from raft_b200.video import write_labels
    d.mkdir()
    for i, mk in enumerate(masks):
        write_labels(d / f"m_{i:05d}.png", mk, palette=np.array([[0, 0, 0], [200, 0, 0], [0, 200, 0]], np.uint8))
    return str(d)


@pytest.mark.parametrize("batch,window,workers", [(1, 1, 1), (3, 4, 4), (8, 12, 1), (3, 1, 4), (1, 4, 4), (8, 4, 4)])
def test_video_inpaint_equals_inpaint(cuda, frame_dir, tmp_path, lenient, batch, window, workers):
    import cv2
    from raft_b200.video import video_inpaint
    m = _model(input_size=(64, 96))
    frames = _decoded(frame_dir)
    masks = _ellipse_masks(*frames.shape[:3])
    want, status = m.inpaint(frames, masks, window=window, labels=[1])
    paths, info = video_inpaint(m, frame_dir, tmp_path / "out", _mask_dir(tmp_path / "masks", masks), window=window,
                                labels=[1], batch=batch, workers=workers)
    assert len(paths) == len(frames) and info["cuts"] == []
    st = status.cpu().numpy()
    assert info["counts"] == [int((st == k).sum()) for k in (1, 2, 3)] and info["counts"][1] > 0
    for i, p in enumerate(paths):
        assert np.array_equal(cv2.imread(p), want[i].cpu().numpy()), i


def test_scene_cut_keeps_each_shot_apart(cuda, frame_dir, tmp_path, lenient):
    import cv2
    from raft_b200.video import list_frames, video_inpaint
    d = tmp_path / "clip"
    d.mkdir()
    for i, p in enumerate(list_frames(frame_dir)):
        img = cv2.imread(p) // 4
        img[..., 2 if i < 5 else 0] += 180  # shot A reddish, shot B bluish: disjoint ranges in channels 0 and 2
        cv2.imwrite(str(d / f"f{i:03d}.png"), img)
    frames = _decoded(str(d))
    masks = _ellipse_masks(*frames.shape[:3])
    m = _model(input_size=(64, 96))
    paths, info = video_inpaint(m, str(d), tmp_path / "out", _mask_dir(tmp_path / "masks", masks), window=6,
                                batch=3, scene_cut=0.5)
    assert info["cuts"] == [4]
    want, _ = m.inpaint(frames, masks, window=6, cuts=[4])
    for i, p in enumerate(paths):
        out = cv2.imread(p)
        assert np.array_equal(out, want[i].cpu().numpy())
        shot = frames[:5] if i < 5 else frames[5:]
        lo, hi = shot.reshape(-1, 3).min(0), shot.reshape(-1, 3).max(0)
        assert (out.reshape(-1, 3) >= lo).all() and (out.reshape(-1, 3) <= hi).all(), i


def test_cli_removes_an_annotated_object(cuda, tmp_path):
    import cv2
    from raft_b200 import synth
    from raft_b200.video import list_frames, read_labels
    root = tmp_path / "davis"
    name = synth.write_davis_tree(str(root), [("clip", 7)], H=64, W=96, objects=2)[0]
    np.savez(tmp_path / "w.npz", **_weights(False))
    frames_dir = root / "JPEGImages" / "480p" / name
    ann = root / "Annotations" / "480p" / name
    out = tmp_path / "clean"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", str(frames_dir),
                        "--out", str(out), "--inpaint", str(ann), "--inpaint-labels", "1", "--load",
                        str(tmp_path / "w.npz"), "--flow-size", "64", "96", "--iters", "4", "--batch", "3"],
                       capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "filled from both sides" in r.stdout and "scene cuts: 0" in r.stdout
    frames = np.stack([cv2.imread(p) for p in list_frames(str(frames_dir))])
    masks = np.stack([read_labels(p)[0] for p in sorted(ann.glob("*.png"))])
    hole, _ = O.inpaint_masks(masks, I.selection_table([1]), I.DEFAULT_DILATE, 64, 96)
    files = sorted(out.glob("frame_*.png"))
    assert len(files) == len(frames) and hole.any()
    for i, f in enumerate(files):
        img = cv2.imread(str(f))
        assert np.array_equal(img[hole[i] == 0], frames[i][hole[i] == 0])
