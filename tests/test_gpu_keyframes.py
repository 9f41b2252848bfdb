"""F21 on the GPU: rb_labels_propagate_keys against tests/keyframes_oracle.py bit for bit, its one-sided rows against
rb_labels_propagate, RAFT.propagate with several keyframes and cuts against the composition of the public pieces, and
video_propagate / infer_raft.py / DAVIS with keyframes end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import davis_oracle as D
import keyframes_oracle as KO
from test_gpu_davis import davis_root  # noqa: F401  (the module fixture)
from test_gpu_propagate import _case, _t
from test_gpu_track import _model, _weights
from test_gpu_video import _decoded, _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _chains(cuda, rng, n, H, W):
    """Two accumulated chains with NaNs and every status, as device tensors and host copies."""
    from networks.utils import accumulate_flow
    out = []
    for _ in range(2):
        fw, bw = _case(rng, n, H, W, nan=3 if H * W > 1 else 0)
        a = torch.zeros(n + 1, H, W, 2, device=cuda)
        s = torch.zeros(n + 1, H, W, dtype=torch.uint8, device=cuda)
        accumulate_flow(_t(cuda, fw), _t(cuda, bw), a, s)
        a, s = a[1:].contiguous(), s[1:].contiguous()
        if H * W > 4:
            a[0, 0, 0, 0] = float("nan")
        out += [a, s]
    return out


@pytest.mark.parametrize("net,src", [((37, 53), (100, 150)), ((96, 160), (180, 320)), ((40, 60), (40, 60)),
                                     ((1, 31), (3, 40)), ((29, 1), (29, 1))])
def test_kernel_equals_fp32_restatement_bit_for_bit(cuda, net, src):
    from networks.utils import propagate_labels_keys
    rng = np.random.default_rng(net[0] * 13 + src[1])
    n, m = 8, 3
    aa, sa, ab, sb = _chains(cuda, rng, n, *net)
    keys = rng.integers(0, 6, (m,) + src).astype(np.uint8)
    keys[1, src[0] // 3:, : src[1] // 2] = 4
    rows = np.array([[0, 1, 2, 1], [1, 2, 1, 3], [2, -1, 0, 0], [-1, 0, 0, 0], [-1, -1, 0, 0], [0, 2, 5, 5],
                     [2, 0, 7, 1], [1, 1, 4, 2]], np.int32)
    labels, status = propagate_labels_keys(aa, sa, ab, sb, _t(cuda, keys), rows)
    want_l, want_s = KO.propagate_keys(aa.cpu().numpy(), sa.cpu().numpy(), ab.cpu().numpy(), sb.cpu().numpy(), keys,
                                       rows)
    assert np.array_equal(labels.cpu().numpy(), want_l), f"{(labels.cpu().numpy() != want_l).sum()} labels differ"
    assert np.array_equal(status.cpu().numpy(), want_s)
    assert (status[4] == 3).all() and (labels[4] == 0).all()
    if net[0] * net[1] > 1000:
        assert all((want_s[:2] == k).any() for k in range(3))


def test_one_sided_rows_equal_single_key_propagation(cuda):
    from networks.utils import propagate_labels, propagate_labels_keys
    rng = np.random.default_rng(31)
    aa, sa, ab, sb = _chains(cuda, rng, 4, 48, 64)
    keys = rng.integers(0, 5, (2, 90, 130)).astype(np.uint8)
    k = _t(cuda, keys)
    want = propagate_labels(aa, sa, k[1])
    got = propagate_labels_keys(aa, sa, ab, sb, k, [[1, -1, 0, 0]] * 4)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    want = propagate_labels(ab, sb, k[0])
    got = propagate_labels_keys(aa, sa, ab, sb, k, [[-1, 0, 0, 0]] * 4)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    zero = torch.zeros_like(aa)
    zs = torch.zeros_like(sa)
    got = propagate_labels_keys(zero, zs, ab, sb, k, [[0, -1, 0, 0], [1, -1, 0, 0], [0, -1, 0, 0], [1, -1, 0, 0]])
    assert all(torch.equal(got[0][i], k[i % 2]) for i in range(4)) and (got[1] == 0).all()  # keyframe rows


def test_table_refusals(cuda):
    from networks.utils import propagate_labels_keys
    a = torch.zeros(2, 5, 6, 2, device=cuda)
    s = torch.zeros(2, 5, 6, dtype=torch.uint8, device=cuda)
    k = torch.zeros(2, 5, 6, dtype=torch.uint8, device=cuda)
    for rows, words in (([[0, -1, 0, 0]], r"\[n,4\]"), ([[0, 2, 1, 1]] * 2, "slots"), ([[-2, 0, 1, 1]] * 2, "slots"),
                        ([[0, 1, 0, 1]] * 2, "weights"), ([[0, 1, 1, 1 << 24]] * 2, "weights"),
                        (np.zeros((2, 4), np.float32), "integer")):
        with pytest.raises(ValueError, match=words):
            propagate_labels_keys(a, s, a, s, k, rows)
    with pytest.raises(ValueError, match="keys"):
        propagate_labels_keys(a, s, a, s, k[0], [[0, -1, 0, 0]] * 2)


def _composed(m, frames, keys, K, cuts=()):
    """RAFT.propagate with several keys from the public pieces: the flows, per key a forward chain to the frame before
    the next key and a backward chain to the frame after the previous one (each in buffers of its own, on slices of the
    flows), keyframe_rows and propagate_labels_keys."""
    from networks.utils import accumulate_flow, accumulate_flow_backward, propagate_labels_keys
    from raft_b200.video import keyframe_rows
    fw, bw, _, _ = m.forward_sequence_bidirectional(frames, check=False)
    F, (H, W), dev = len(frames), fw.shape[1:3], fw.device
    kw = dict(flow_scale=m.engine().flow_scale)
    acc = [torch.full((F, H, W, 2), float("nan"), device=dev) for _ in range(2)]
    st = [torch.full((F, H, W), 9, dtype=torch.uint8, device=dev) for _ in range(2)]

    def zeros(n):
        return torch.zeros(n, H, W, 2, device=dev), torch.zeros(n, H, W, dtype=torch.uint8, device=dev)

    for i, k in enumerate(K):
        hi = K[i + 1] - 1 if i + 1 < len(K) else F - 1
        a, s = zeros(hi - k + 1)
        if hi > k:
            accumulate_flow(fw[k:hi], bw[k:hi], a, s, **kw)
        acc[0][k:hi + 1], st[0][k:hi + 1] = a, s
        lo = K[i - 1] + 1 if i > 0 else 0
        a, s = zeros(k - lo + 1)
        if k > lo:
            accumulate_flow_backward(fw[lo:k], bw[lo:k], a, s, start=k - lo, **kw)
        acc[1][lo:k], st[1][lo:k] = a[:k - lo], s[:k - lo]
    return propagate_labels_keys(acc[0], st[0], acc[1], st[1], _t(dev, keys), keyframe_rows(F, K, cuts))


def _keys(m, H, W, seed):
    rng = np.random.default_rng(seed)
    keys = np.zeros((m, H, W), np.uint8)
    for i in range(m):
        y, x = rng.integers(10, H // 2), rng.integers(10, W // 2)
        keys[i, y:y + H // 3, x:x + W // 3] = 1 + i % 2
        keys[i, y + 10:y + 30, x + 5:x + W // 2] = 3
    return keys


@pytest.mark.parametrize("input_size", [None, (128, 160)])
@pytest.mark.parametrize("upstream", [False, True])
@pytest.mark.parametrize("small", [False, True])
def test_raft_propagate_with_keyframes_equals_the_public_pieces(cuda, small, upstream, input_size):
    m = _model(small, upstream=upstream, input_size=input_size)
    frames = _frames(7, 125, 150, seed=5200 + 2 * small + upstream)
    keys = _keys(3, 125, 150, 7)
    one = m.propagate(frames, keys[0], frame=2)
    listed = m.propagate(frames, keys[:1], frame=[2])
    assert torch.equal(one[0], listed[0]) and torch.equal(one[1], listed[1])
    for K, cuts in (([0, 3, 6], None), ([1, 4], [2]), ([0, 2, 5], [0, 3, 5]), ([3], [1])):
        got = m.propagate(frames, keys[:len(K)], frame=K, cuts=cuts)
        want = _composed(m, frames, keys[:len(K)], K, cuts or ())
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (K, cuts)
        lab = got[0].cpu().numpy()
        assert all(np.array_equal(lab[k], keys[i]) for i, k in enumerate(K))
        assert set(np.unique(lab)) <= {0, 1, 2, 3}
        if K == [3]:  # the cut at pair 1 keeps frames 0 and 1 from the only key
            assert (got[1][:2] == 3).all() and (got[0][:2] == 0).all() and (got[1][2:] != 3).all()


def test_raft_propagate_refusals(cuda):
    m = _model()
    frames = _frames(4, 60, 80)
    k = np.zeros((2, 60, 80), np.uint8)
    for labels, frame, cuts, words in ((k, [0], None, "2 key label maps for 1"), (k, [2, 1], None, "strictly"),
                                       (k, [0, 4], None, r"\[0, 4\)"), (k[:, :, :79].copy(), [0, 2], None, "uint8 stack"),
                                       (k.astype(np.int32), [0, 2], None, "uint8 stack"),
                                       (k, [0, 2], [3], "cuts"), (k[0], 0, [-1], "cuts")):
        with pytest.raises(ValueError, match=words):
            m.propagate(frames, labels, frame=frame, cuts=cuts)


def _write_keys(tmp_path, keys, palette=True):
    from raft_b200.synth import DAVIS_PALETTE
    from raft_b200.video import write_labels
    names = []
    for i, k in enumerate(keys):
        names.append(str(tmp_path / f"key{i}.png"))
        write_labels(names[-1], k, DAVIS_PALETTE if palette else None)
    return names


def test_video_propagate_with_keyframes(cuda, frame_dir, tmp_path):
    from raft_b200.video import read_labels, video_propagate
    m = _model()
    frames = _decoded(frame_dir)
    F, H, W = frames.shape[:3]
    for K, batches in ((list(range(0, F, 3)), ((8, 0), (8, 2), (1, 0), (2, 2))), ([0, F - 1], ((2, 0), (2, 2), (8, 2),
                                                                                             (1, 2))),
                       ([5, 8], ((2, 2), (3, 0), (8, 0)))):  # a reverse sweep before the first key
        keys = _keys(len(K), H, W, len(K))
        names = _write_keys(tmp_path, keys)
        want_l, want_s = (x.cpu().numpy() for x in m.propagate(frames, keys, frame=K))
        runs = {}
        for batch, workers in batches:
            out = tmp_path / f"k{len(K)}b{batch}w{workers}"
            files, last = video_propagate(m, frame_dir, str(out), names, frame=K, batch=batch, workers=workers)
            assert np.array_equal(last, want_s[-1])
            runs[(batch, workers)] = _files(str(out))
            got = np.stack([read_labels(f)[0] for f in files])
            assert np.array_equal(got, want_l), (K, batch)
        assert all(r == runs[batches[0]] for r in runs.values())


def test_video_propagate_stops_at_scene_cuts(cuda, frame_dir, tmp_path):
    import cv2
    from networks.utils import scene_cut_scores
    from raft_b200.video import read_labels, video_propagate
    m = _model()
    frames = _decoded(frame_dir)
    F, H, W = frames.shape[:3]
    d = tmp_path / "cut"
    d.mkdir()
    dark = frames.copy()
    dark[6:] = dark[6:] // 4  # a darkened tail: one cut at pair 5
    for i, f in enumerate(dark):
        cv2.imwrite(str(d / f"f{i:03d}.png"), f)
    clip = _decoded(str(d))
    thr = 0.5
    scores = scene_cut_scores(torch.from_numpy(clip).to(cuda)).cpu().numpy()
    cuts = [k for k in range(F - 1) if scores[k] > thr]
    assert 5 in cuts, scores
    keys = _keys(2, H, W, 3)
    names = _write_keys(tmp_path, keys)
    for K in ([2], [0, 8], [7]):
        want_l, want_s = (x.cpu().numpy() for x in m.propagate(clip, keys[:len(K)], frame=K, cuts=cuts))
        for batch, workers in ((3, 2), (8, 0)):
            out = tmp_path / f"c{len(K)}{K[0]}b{batch}"
            files, last, found = video_propagate(m, str(d), str(out), names[:len(K)] if len(K) > 1 else names[0],
                                                 frame=K if len(K) > 1 else K[0], batch=batch, workers=workers,
                                                 scene_cut=thr)
            assert found == cuts
            got = np.stack([read_labels(f)[0] for f in files])
            assert np.array_equal(got, want_l) and np.array_equal(last, want_s[-1]), (K, batch)
        if K == [2]:
            assert (want_s[6:] == 3).all() and (want_l[6:] == 0).all()
        if K == [7]:
            assert (want_s[:6] == 3).all()


def test_cli_with_two_keys_equals_the_api(cuda, frame_dir, tmp_path):
    from raft_b200.video import read_labels
    np.savez(tmp_path / "w.npz", **_weights(False))
    frames = _decoded(frame_dir)
    F, H, W = frames.shape[:3]
    keys = _keys(2, H, W, 11)
    names = _write_keys(tmp_path, keys)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", frame_dir,
                        "--out", str(tmp_path / "o"), "--propagate", *names, "--propagate-frame", "1", "6",
                        "--load", str(tmp_path / "w.npz"), "--keep-size", "--batch", "3", "--iters", "4"],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert f"labels of frames 1, 6 propagated through {F} frames" in r.stdout, r.stdout
    want = _model(iters=4).propagate(frames, keys, frame=[1, 6])[0].cpu().numpy()
    got = np.stack([read_labels(tmp_path / "o" / f"label_{i:06d}.png")[0] for i in range(F)])
    assert np.array_equal(got, want)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", frame_dir,
                        "--out", str(tmp_path / "c"), "--propagate", *names, "--propagate-frame", "1", "6",
                        "--load", str(tmp_path / "w.npz"), "--keep-size", "--iters", "4", "--scene-cut", "1.0"],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert "scene cuts: 0" in r.stdout and "reached by no key (status 3)" in r.stdout, r.stdout


def test_davis_with_keyframes(cuda, davis_root, tmp_path):  # noqa: F811
    from raft_b200.davis import davis_sequences, keyframe_frames, propagate_clip, scored_frames
    from raft_b200.evaluate import _engine, evaluate, summary_lines
    from raft_b200.video import read_labels
    m = _model(iters=4)
    res = {b: evaluate(m, davis_root, "davis", batch=b, iters=4, masks_out=str(tmp_path / f"m{b}"), keyframe_step=3)
           for b in (1, 8)}
    assert json.dumps(res[1], sort_keys=True) == json.dumps(res[8], sort_keys=True)
    assert res[1]["keyframe_step"] == 3
    assert summary_lines(res[1])[0].startswith("Validation DAVIS-2017 (val, a keyframe every 3): J&F: ")
    pairs = []
    for s in davis_sequences(davis_root):
        gt = np.stack([read_labels(p)[0] for p in s.annotations])
        gt[gt == 255] = 0
        pred = np.stack([read_labels(os.path.join(tmp_path / "m1", s.name, os.path.basename(p)))[0]
                         for p in s.annotations])
        K = keyframe_frames(len(gt), 3)
        assert all(np.array_equal(pred[k], gt[k]) for k in K)
        keep = [0] + scored_frames(len(gt), K) + [len(gt) - 1]  # the oracle drops the first and the last frame
        pairs.append((gt[keep], pred[keep]))
    want = D.evaluate_sequences(pairs)
    r = res[1]["splits"]["val"]
    for k, v in want.items():
        assert r[k] == pytest.approx(v, rel=1e-12, abs=1e-12), k
    longest = max(len(s.frames) for s in davis_sequences(davis_root))
    today = evaluate(m, davis_root, "davis", batch=2, iters=4)
    step = evaluate(m, davis_root, "davis", batch=2, iters=4, keyframe_step=longest)
    assert step.pop("keyframe_step") == longest
    assert json.dumps(step, sort_keys=True) == json.dumps(today, sort_keys=True)
    # propagate_clip with keyframes: RAFT.propagate's bits for every batch
    eng = _engine(m, 4, "sintel")
    clip = _frames(9, 64, 96, seed=77)
    keys = _keys(3, 64, 96, 5)
    want = eng.propagate(torch.from_numpy(clip), keys, frame=[0, 4, 8])
    for b in (1, 3, 8):
        got = propagate_clip(eng, clip, keys, b, frame=[0, 4, 8])
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), b
