"""F34 / F35 on the GPU: rb_homography_motion's sums, homographies and flags against the fp64 numpy restatement
(tests/motionseg_oracle.py) on the same previous-round estimate, its bits across calls and batch positions,
rb_motion_evidence and rb_motion_segment bit for bit with the oracle, and RAFT.segment_motion against its parts.  The
end-to-end test runs seeded weights: plumbing, not quality."""
import numpy as np
import pytest
import torch

import motionseg_oracle as MO
from networks import utils as U
from raft_b200 import motionseg as M
from test_gpu_inpaint import lenient  # noqa: F401  (the fixture)
from test_gpu_track import _model
from test_gpu_video import _decoded, frame_dir  # noqa: F401  (frame_dir: the module fixture)
from test_motionseg import _rotation

pytestmark = pytest.mark.gpu

SIZES = [((1080, 1920), (432, 1024), 1.0), ((96, 160), (96, 160), 1.0), ((101, 149), (37, 53), 1.0),
         ((96, 160), (48, 80), 8.0)]


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _fields(rng, T, src, net, scale):
    """T forward and T backward seeded fields on the network grid: a turning camera (exact per field), an object of
    its own motion, noise, occluded pixels and a few non-finite flows."""
    Hs, Ws = src
    Hn, Wn = net
    sx, sy = Ws / Wn, Hs / Hn
    i, j = (a.astype(np.float64) for a in np.mgrid[0:Hn, 0:Wn])
    x, y = (j + 0.5) * sx - 0.5, (i + 0.5) * sy - 0.5
    out = []
    for k in range(2 * T):
        Hm = _rotation((1.5 + 0.5 * k) * (1 if k < T else -1), src, 0.9 * Ws)
        X, Y, z = (Hm[r, 0] * x + Hm[r, 1] * y + Hm[r, 2] for r in range(3))
        u, v = (X / z - x) / sx, (Y / z - y) / sy
        obj = (np.abs(j - Wn * 0.6) < Wn * 0.12) & (np.abs(i - Hn * 0.4) < Hn * 0.15)
        u = np.where(obj, u + 2.5, u) + rng.normal(0, 0.05, u.shape)
        out.append(np.stack([u, v + rng.normal(0, 0.05, v.shape)], -1) / scale)
    flow = np.stack(out).astype(np.float32)
    occ = (rng.random(flow.shape[:3]) < 0.1).astype(np.uint8)
    for _ in range(3):
        flow[rng.integers(2 * T), rng.integers(Hn), rng.integers(Wn), rng.integers(2)] = np.nan
    return flow, occ


@pytest.mark.parametrize("src,net,scale", SIZES)
def test_homography_matches_oracle(cuda, src, net, scale):
    rng = np.random.default_rng(net[0])
    flow, occ = _fields(rng, 2, src, net, scale)
    f, o = _t(cuda, flow), _t(cuda, occ)
    params, _, reliable = U.global_motion(f, o, src, flow_scale=scale)
    sim, sflags = params.cpu().numpy(), (~reliable).cpu().numpy().astype(np.uint8)
    for rounds in (1, 3, M.ROUNDS):
        H, flags, sums = U.homography_motion(f, o, src, params, reliable, flow_scale=scale, rounds=rounds,
                                             return_sums=True)
        H, flags, sums = H.cpu().numpy(), flags.cpu().numpy(), sums.cpu().numpy()
        oH, oflags, _, _, _ = MO.homography(flow, occ, src, scale, sim, sflags, rounds)
        assert np.array_equal(flags, oflags)
        np.testing.assert_allclose(H, oH, rtol=0, atol=1e-9)
        # the last round's sums on the estimate the GPU's own previous round left
        if rounds > 1:
            prev, _ = U.homography_motion(f, o, src, params, reliable, flow_scale=scale, rounds=rounds - 1)
            prev = prev.cpu().numpy()
        else:
            prev = np.stack([MO.similarity_h(sim[b], 0.5 * max(src)) if not sflags[b] else np.eye(3)
                             for b in range(len(flow))])
        for b in range(len(flow)):
            s, a = MO.round_sums(flow[b], occ[b], src, scale, prev[b])
            assert (np.abs(sums[b] - s) <= 1e-12 * a + 1e-300).all(), (rounds, b, np.abs(sums[b] - s).max())
    assert (flags == 0).all()


def test_homography_bits_across_calls_and_batch(cuda):
    rng = np.random.default_rng(5)
    src, net = (101, 149), (37, 53)
    flow, occ = _fields(rng, 2, src, net, 1.0)
    f, o = _t(cuda, flow), _t(cuda, occ)
    p, _, r = U.global_motion(f, o, src)
    H, flags = U.homography_motion(f, o, src, p, r)
    H2, flags2 = U.homography_motion(f, o, src, p, r)
    assert torch.equal(H, H2) and torch.equal(flags, flags2)
    for b in range(len(flow)):
        Hb, fb = U.homography_motion(f[b:b + 1], o[b:b + 1], src, p[b:b + 1], r[b:b + 1])
        assert torch.equal(Hb[0], H[b]) and torch.equal(fb[0], flags[b])
    # an unreliable similarity gives the identity and flag 2
    Hu, fu = U.homography_motion(f, o, src, p, torch.zeros_like(r))
    assert (fu == 2).all() and torch.equal(Hu, torch.eye(3, dtype=torch.float64, device=cuda).expand(4, 3, 3))


@pytest.mark.parametrize("src,net,scale", SIZES)
def test_evidence_and_segment_match_oracle(cuda, src, net, scale):
    rng = np.random.default_rng(net[1])
    T = 2 if net[0] > 200 else 4
    flow, occ = _fields(rng, T, src, net, scale)
    fw, bw = flow[:T], flow[T:]
    # a consistent-looking backward field: the forward one reversed plus noise, so chains take steps
    bw = (-fw + rng.normal(0, 0.05, fw.shape)).astype(np.float32)
    flow = np.concatenate([fw, bw])
    f, o = _t(cuda, flow), _t(cuda, occ)
    H, flags = M.fit_fields(f, o, src, scale)
    cut = np.zeros(T, np.uint8)
    cut[T - 1] = 1
    for cuts in (None, cut):
        ev = U.motion_evidence(f[:T], f[T:], o[:T], o[T:], H, flags, src, None if cuts is None else _t(cuda, cuts),
                               flow_scale=scale, tau=0.7)
        oev = MO.evidence(fw, bw, occ[:T], occ[T:], H.cpu().numpy(), flags.cpu().numpy(), src, scale, cuts, 0.7)
        assert np.array_equal(ev.cpu().numpy(), oev)
    for window in (0, 3):
        rows = M.segment_rows(T + 1, window)
        mask, status = U.motion_segment(ev, f[:T], f[T:], src, rows, flow_scale=scale, alpha2=5.0)
        om, os_ = MO.segment(oev, fw, bw, src, rows, scale, 0.01, 5.0)
        assert np.array_equal(mask.cpu().numpy(), om) and np.array_equal(status.cpu().numpy(), os_)
    assert 0 < om.mean() < 1


def test_segment_motion_equals_its_parts(cuda, frame_dir, lenient):
    m = _model(input_size=(64, 96))
    frames = _decoded(frame_dir)
    F = len(frames)
    hw = frames.shape[1:3]
    mask, status, Hpix = m.segment_motion(frames, window=2, tau=0.5, cuts=[3])
    eng = m.engine()
    fw, bw, ofw, obw = eng.forward_sequence_bidirectional(_t(cuda, frames), check=True)
    H, flags = M.fit_fields(torch.cat([fw, bw]), torch.cat([ofw, obw]), hw, eng.flow_scale)
    ev = U.motion_evidence(fw, bw, ofw, obw, H, flags, hw, M.cut_flags([3], range(F - 1), cuda), eng.flow_scale, 0.5)
    w_mask, w_status = M.segment_frames(ev, fw, bw, hw, M.segment_rows(F, 2, [3]), eng.flow_scale)
    assert torch.equal(mask, w_mask) and torch.equal(status, w_status)
    assert mask.shape == (F, *hw) and mask.dtype == torch.uint8 and int(mask.max()) <= 1
    np.testing.assert_array_equal(Hpix, M.to_pixels(H[:F - 1].cpu().numpy(), hw))
    oev = MO.evidence(fw.cpu().numpy(), bw.cpu().numpy(), ofw.cpu().numpy(), obw.cpu().numpy(), H.cpu().numpy(),
                      flags.cpu().numpy(), hw, eng.flow_scale, M.cut_flags([3], range(F - 1), "cpu").numpy(), 0.5)
    assert np.array_equal(ev.cpu().numpy(), oev)
    for kw in (dict(window=-1), dict(window=17), dict(tau=0), dict(cuts=[F - 1])):
        with pytest.raises(ValueError):
            m.segment_motion(frames, **kw)


@pytest.mark.parametrize("batch,workers", [(1, 1), (3, 4), (8, 1), (8, 4)])
def test_video_segment_motion_equals_in_memory(cuda, frame_dir, lenient, tmp_path, batch, workers):
    from raft_b200.video import read_labels, video_segment_motion
    m = _model(input_size=(64, 96))
    frames = _decoded(frame_dir)
    want, _, Hpix = m.segment_motion(frames, window=2)
    paths, info = video_segment_motion(m, frame_dir, tmp_path / "out", window=2, batch=batch, workers=workers)
    assert len(paths) == len(frames) and info["cuts"] == []
    assert info["moving"] == pytest.approx(float(want.double().mean()), rel=0, abs=1e-12)
    for i, p in enumerate(paths):
        lab, _ = read_labels(p)
        assert np.array_equal(lab, want[i].cpu().numpy()), i
    assert np.array_equal(np.load(tmp_path / "out" / "homographies.npy"), Hpix)


def test_video_segment_motion_scene_cut(cuda, lenient, tmp_path):
    import cv2
    from raft_b200.video import read_labels, video_segment_motion
    src = cv2.imread(str(__import__("pathlib").Path(__file__).parent / "data" / "frame_0016.png"))
    frames = np.stack([src[100 + k:224 + k, 200 + 3 * k:350 + 3 * k] for k in range(5)] +
                      [255 - src[40 + k:164 + k, 20 + 2 * k:170 + 2 * k] for k in range(4)])
    d = tmp_path / "frames"
    d.mkdir()
    for k, f in enumerate(frames):
        cv2.imwrite(str(d / f"frame_{k:04d}.png"), f)
    m = _model(input_size=(64, 96))
    for batch in (2, 8):
        paths, info = video_segment_motion(m, str(d), tmp_path / f"out{batch}", window=3, batch=batch, scene_cut=0.5)
        assert info["cuts"] == [4]
        want, _, _ = m.segment_motion(frames, window=3, cuts=[4])
        for i, p in enumerate(paths):
            assert np.array_equal(read_labels(p)[0], want[i].cpu().numpy()), (batch, i)


def test_flagged_fields_match_oracle(cuda):
    """A singular field (flag 1: the similarity kept) and an unreliable one (flag 2: no evidence) beside two fitted
    ones: H and flags against the oracle, the evidence bit for bit."""
    from test_motionseg import _degenerate
    rng = np.random.default_rng(11)
    src, net = (24, 106), (12, 53)
    flow, occ = _fields(rng, 2, src, net, 1.0)
    dflow, docc = _degenerate(*net)
    flow[0], occ[0] = dflow[0], docc[0]
    f, o = _t(cuda, flow), _t(cuda, occ)
    params, _, reliable = U.global_motion(f, o, src)
    reliable[3] = False
    H, flags = U.homography_motion(f, o, src, params, reliable)
    sim, sflags = params.cpu().numpy(), (~reliable).cpu().numpy().astype(np.uint8)
    oH, oflags, _, _, _ = MO.homography(flow, occ, src, 1.0, sim, sflags)
    assert flags.cpu().tolist() == oflags.tolist() == [M.SINGULAR, M.FIT, M.FIT, M.UNRELIABLE]
    np.testing.assert_allclose(H.cpu().numpy(), oH, rtol=0, atol=1e-9)
    assert np.array_equal(H[0].cpu().numpy(), MO.similarity_h(sim[0], 0.5 * max(src)))
    ev = U.motion_evidence(f[:2], f[2:], o[:2], o[2:], H, flags, src)
    oev = MO.evidence(flow[:2], flow[2:], occ[:2], occ[2:], H.cpu().numpy(), flags.cpu().numpy(), src)
    assert np.array_equal(ev.cpu().numpy(), oev)
    # fields: forward 0, 1, backward 0, 1; frame 2 has only pair 1's backward field, flagged 2: no evidence
    assert ev[2, ..., 1].max() == 0 and ev[1, ..., 1].max() == 2


def test_cli_masks_feed_inpaint(cuda, tmp_path, frame_dir):
    import os
    import subprocess
    import sys
    from raft_b200.video import read_labels
    from test_gpu_track import _weights
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cli = os.path.join(root, "raft-tf_b200", "infer_raft.py")
    np.savez(tmp_path / "w.npz", **_weights(False))
    common = ["--load", str(tmp_path / "w.npz"), "--flow-size", "64", "96", "--iters", "4", "--batch", "3"]
    masks = tmp_path / "masks"
    r = subprocess.run([sys.executable, cli, "--path", frame_dir, "--out", str(masks), "--segment-motion",
                        "--segment-window", "2"] + common, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "segment motion:" in r.stdout and "motion masks written" in r.stdout
    files = sorted(masks.glob("mask_*.png"))
    assert len(files) == 10 and all(read_labels(str(p))[0].shape == (124, 150) for p in files)
    assert np.load(masks / "homographies.npy").shape == (9, 3, 3)
    r = subprocess.run([sys.executable, cli, "--path", frame_dir, "--out", str(tmp_path / "filled"), "--inpaint",
                        str(masks)] + common, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert len(sorted((tmp_path / "filled").glob("frame_*.png"))) == 10


def test_val_davis_motion_equals_the_host_recount(cuda, tmp_path):
    import json
    import os
    import subprocess
    import sys
    import davis_oracle as DAO
    from raft_b200 import synth
    from raft_b200.davis import davis_sequences, segment_clip
    from raft_b200.evaluate import _engine, _imread
    from raft_b200.video import read_labels
    from test_gpu_track import _weights
    from test_motionseg import _write_2016_list
    root = tmp_path / "davis"
    names = synth.write_davis_tree(str(root), [("alpha", 5), ("beta", 4)], H=64, W=96)
    _write_2016_list(str(root), names)
    np.savez(tmp_path / "w.npz", **_weights(False))
    out = tmp_path / "val"
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "raft-tf_b200", "infer_raft.py")
    r = subprocess.run([sys.executable, cli, "-m", "val", "--dataset", "davis", "--data", str(root), "--segment-motion",
                        "--load", str(tmp_path / "w.npz"), "--iters", "4", "--batch", "2", "--out", str(out)],
                       capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "Validation DAVIS-2016 motion segmentation (val): J&F: " in r.stdout
    res = json.load(open(out / "val_davis_motion.json"))
    assert [s["name"] for s in res["sequences"]] == names and res["iters"] == 4 and res["n_objects"] == 2
    eng = _engine(_model(), 4, "sintel")
    pairs = []
    for seq in davis_sequences(str(root), "val", year="2016"):
        gt = np.stack([read_labels(p)[0] for p in seq.annotations])
        gt = ((gt != 0) & (gt != 255)).astype(np.uint8)
        pred = np.stack([read_labels(str(out / "davis_motion" / seq.name / os.path.basename(p)))[0]
                         for p in seq.annotations])
        frames = np.stack([_imread(p, False) for p in seq.frames])
        got, _ = segment_clip(eng, _t(cuda, frames), batch=1)  # batch 1 gives the CLI's batch-2 bits
        want, _, _ = eng.segment_motion(_t(cuda, frames))
        assert torch.equal(got, want) and np.array_equal(got.cpu().numpy(), pred)
        pairs.append((gt, pred))
    host = DAO.evaluate_sequences(pairs)
    for k in ("J&F-Mean", "J-Mean", "F-Mean", "J-Recall", "F-Recall", "J-Decay", "F-Decay"):
        assert res[k] == pytest.approx(host[k], rel=1e-12, abs=1e-12, nan_ok=True), k
