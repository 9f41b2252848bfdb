"""F29 - F31 on the GPU: rb_tcons_terms, rb_screened_poisson and rb_warp_error against the numpy restatements
(tests/tcons_oracle.py) -- the terms and the solve bit for bit, the per-pair sums within 1e-12 relative -- and
RAFT.consistent / RAFT.warp_error against their parts.  The end-to-end tests run seeded weights: plumbing, not
quality."""
import numpy as np
import pytest
import torch

import tcons_oracle as TO
from raft_b200 import temporal as T
from test_gpu_denoise import _clip
from test_gpu_inpaint import lenient  # noqa: F401  (lenient: the fixture)
from test_gpu_track import _model
from test_gpu_video import _decoded, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
F32 = np.float32


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.mark.parametrize("src,net,scale", [((40, 56), (40, 56), 1.0), ((75, 101), (32, 48), 1.0),
                                           ((31, 45), (48, 64), 8.0), ((9, 13), (3, 2), 1.0)])
def test_terms_and_solve_match_oracle(cuda, src, net, scale):
    from networks.utils import screened_poisson, tcons_terms
    rng = np.random.default_rng(src[1] + net[0])
    frames, fw, bw = _clip(rng, 3, src, net, scale)
    P = np.clip(frames.astype(np.int32) + rng.integers(-30, 31, frames.shape), 0, 255).astype(np.uint8)
    prev_out = np.clip(P[0].astype(np.int32) + rng.integers(-8, 9, P[0].shape), 0, 255).astype(np.uint8)
    # the originals of frame 1 are frame 0 moved slightly, so some pixels pass the colour check and some do not
    frames[1] = np.clip(frames[0].astype(np.int32) + rng.integers(-25, 26, frames[0].shape), 0, 255).astype(np.uint8)
    for lam in (1e-3, 0.1, 10.0):
        c, r, st = tcons_terms(_t(cuda, frames[1]), _t(cuda, frames[0]), _t(cuda, P[1]), _t(cuda, prev_out),
                               _t(cuda, fw[0]), _t(cuda, bw[0]), lam, flow_scale=scale)
        wc, wr, wst = TO.tcons_terms(frames[1], frames[0], P[1], prev_out, fw[0], bw[0], lam, scale)
        assert np.array_equal(st.cpu().numpy(), wst)
        assert np.array_equal(c.cpu().numpy().view(np.uint32), wc.view(np.uint32))
        assert np.array_equal(r.cpu().numpy(), wr)
        D = screened_poisson(c, r)
        assert np.array_equal(D.cpu().numpy(), TO.screened_poisson(wc, wr))
        assert torch.equal(D, screened_poisson(c, r))  # deterministic run to run
    if src[0] > 9:
        assert all((wst == k).any() for k in (0, 1, 2))
    c3, r3, st3 = tcons_terms(None, None, _t(cuda, P[1]), None, None, None, 0.1)
    assert (st3 == 3).all() and not r3.any() and (c3 == F32(T.EPS)).all()
    assert not screened_poisson(c3, r3).any()


@pytest.mark.parametrize("hw", [(1, 1), (1, 9), (7, 1), (37, 53), (130, 97)])
@pytest.mark.parametrize("kind", ["ones", "half", "blobs", "point"])
def test_solve_matches_oracle_bit_for_bit(cuda, hw, kind):
    from networks.utils import screened_poisson
    from test_temporal import _system
    rng = np.random.default_rng(hw[0] * 7 + hw[1])
    for lam in (1e-4, 1.0, 10.0):
        c, r = _system(rng, *hw, lam, kind)
        D = screened_poisson(_t(cuda, c), _t(cuda, r)).cpu().numpy()
        assert np.array_equal(D, TO.screened_poisson(c, r))
        assert np.abs(D - TO.screened_poisson_f64(c, r)).max() <= 0.25


@pytest.mark.parametrize("src,net,scale", [((40, 56), (40, 56), 1.0), ((75, 101), (32, 48), 1.0),
                                           ((31, 45), (48, 64), 8.0)])
def test_warp_error_sums_match_oracle(cuda, src, net, scale):
    from networks.utils import warp_error
    rng = np.random.default_rng(src[0] + 3)
    frames, fw, bw = _clip(rng, 5, src, net, scale)
    sums = warp_error(_t(cuda, frames), _t(cuda, fw), _t(cuda, bw), flow_scale=scale).cpu().numpy()
    want = TO.warp_error_sums(frames, fw, bw, scale)
    assert np.array_equal(sums[:, 1], want[:, 1]) and (want[:, 1] > 0).all()
    assert np.allclose(sums[:, 0], want[:, 0], rtol=1e-12, atol=0)
    again = warp_error(_t(cuda, frames), _t(cuda, fw), _t(cuda, bw), flow_scale=scale).cpu().numpy()
    assert np.array_equal(sums, again)


@pytest.mark.parametrize("small,size,upstream", [(False, (64, 96), False), (True, None, False),
                                                 (False, (128, 160), True)])
def test_raft_consistent_equals_its_parts(cuda, frame_dir, lenient, small, size, upstream):
    m = _model(small=small, input_size=size, upstream=upstream)
    frames = _decoded(frame_dir)
    rng = np.random.default_rng(11)
    gain = rng.uniform(0.85, 1.15, (len(frames), 1, 1, 1))
    P = np.clip(np.rint(frames * gain + rng.uniform(-12, 12, (len(frames), 1, 1, 3))), 0, 255).astype(np.uint8)
    out, status = m.consistent(frames, P, 0.1, cuts=[6])
    eng = m.engine()
    fw, bw, _, _ = eng.forward_sequence_bidirectional(_t(cuda, frames), check=False)
    fw, bw = fw.cpu().numpy(), bw.cpu().numpy()
    w_out, w_st = TO.consistent(frames, P, fw, bw, 0.1, cuts=(6,), s=eng.flow_scale, a2=lenient)
    assert np.array_equal(status.cpu().numpy(), w_st) and np.array_equal(out.cpu().numpy(), w_out)
    assert out.shape == frames.shape and (w_st[1:6] == 0).any()
    assert np.array_equal(w_out[0], P[0]) and np.array_equal(w_out[7], P[7])
    e, per = m.warp_error(frames, out.cpu().numpy(), cuts=[6])
    sums = TO.warp_error_sums(w_out, fw, bw, eng.flow_scale, a2=lenient)
    w_e, w_per, excluded = T.pair_errors(sums, [6])
    assert excluded == [6] and np.isnan(per[6])
    assert np.allclose(per[~np.isnan(per)], w_per[~np.isnan(w_per)], rtol=1e-12, atol=0)
    assert abs(e - w_e) <= 1e-12 * abs(w_e)
    eP, _ = m.warp_error(frames, P, cuts=[6])
    assert e < eP


def test_consistent_refusals(cuda, frame_dir):
    m = _model()
    frames = _decoded(frame_dir)
    with pytest.raises(ValueError):
        m.consistent(frames, frames[:-1], 0.1)
    with pytest.raises(ValueError):
        m.consistent(frames, frames, 0.0)
    with pytest.raises(ValueError):
        m.consistent(frames, frames, 0.1, cuts=[len(frames)])
    with pytest.raises(ValueError):
        m.warp_error(frames, frames.astype(np.float32))


def test_solve_within_a_quarter_grey_level_at_480x854(cuda):
    """The lowest modes of large zero-weight regions are screened by eps alone: the solve at a real frame size, with
    half the frame and four fifths of the columns without a temporal term, against fp64 (measured with the oracle:
    2.7e-4 grey levels at lambda 1e-4, 8.9e-3 at lambda 10)."""
    from networks.utils import screened_poisson
    rng = np.random.default_rng(1)
    H, W = 480, 854
    for lam in (1e-4, 10.0):
        w = (rng.random((H, W)) ** 2).astype(F32)
        w[:, W // 5:] = 0
        w[H // 2:, :] = 0
        diff = rng.integers(-255, 256, (H, W, 3)).astype(F32) + F32(60)
        lw = (F32(lam) * w).astype(F32)
        c, r = (lw + F32(T.EPS)).astype(F32), (lw[..., None] * diff).astype(F32)
        D = screened_poisson(_t(cuda, c), _t(cuda, r)).cpu().numpy()
        assert np.array_equal(D, TO.screened_poisson(c, r))
        assert np.abs(D - TO.screened_poisson_f64(c, r)).max() <= 0.25


def _processed_dir(d, frames, seed=11):
    """Per-frame 'processed' frames (a seeded gain and offset per frame) written as PNGs; returns (dir, frames)."""
    import cv2
    rng = np.random.default_rng(seed)
    gain = rng.uniform(0.85, 1.15, (len(frames), 1, 1, 1))
    P = np.clip(np.rint(frames * gain + rng.uniform(-12, 12, (len(frames), 1, 1, 3))), 0, 255).astype(np.uint8)
    d.mkdir()
    for i, img in enumerate(P):
        cv2.imwrite(str(d / f"p{i:03d}.png"), img)
    return str(d), P


def _cut_clip(frame_dir, d):
    import cv2
    from raft_b200.video import list_frames
    d.mkdir()
    for i, p in enumerate(list_frames(frame_dir)):
        img = cv2.imread(p) // 4
        img[..., 2 if i < 5 else 0] += 180  # shot A reddish, shot B bluish: a cut at pair 4
        cv2.imwrite(str(d / f"f{i:03d}.png"), img)
    return str(d)


@pytest.mark.parametrize("batch,workers,size,cut", [(3, 2, (64, 96), False), (1, 0, None, False),
                                                    (4, 4, (64, 96), True), (9, 1, None, True)])
def test_video_consistent_equals_consistent(cuda, frame_dir, tmp_path, lenient, batch, workers, size, cut):
    import cv2
    from raft_b200.video import video_consistent
    src = _cut_clip(frame_dir, tmp_path / "clip") if cut else frame_dir
    frames = _decoded(src)
    pdir, P = _processed_dir(tmp_path / "proc", frames)
    m = _model(input_size=size)
    paths, info = video_consistent(m, src, pdir, tmp_path / "out", 0.1, batch=batch, workers=workers,
                                   scene_cut=0.5 if cut else None)
    assert info["cuts"] == ([4] if cut else [])
    want, status = m.consistent(frames, P, 0.1, cuts=info["cuts"])
    assert len(paths) == len(frames)
    for i, p in enumerate(paths):
        assert np.array_equal(cv2.imread(p), want[i].cpu().numpy()), i
    assert info["status"] == np.bincount(status.cpu().numpy().ravel(), minlength=4).tolist()
    e, per = m.warp_error(frames, want.cpu().numpy(), cuts=info["cuts"])
    assert info["output"]["E_warp"] == e and np.array_equal(np.array(info["output"]["E_pair"]), per, equal_nan=True)
    eP, perP = m.warp_error(frames, P, cuts=info["cuts"])
    assert info["input"]["E_warp"] == eP
    eI, _ = m.warp_error(frames, frames, cuts=info["cuts"])
    assert info["original"]["E_warp"] == eI
    if cut:
        assert info["output"]["excluded"] == [4] and (status.cpu().numpy()[5] == 3).all()


@pytest.mark.parametrize("batch,workers", [(2, 0), (5, 3)])
def test_video_warp_error_equals_warp_error(cuda, frame_dir, tmp_path, batch, workers):
    from raft_b200.video import video_warp_error
    frames = _decoded(frame_dir)
    pdir, P = _processed_dir(tmp_path / "proc", frames)
    m = _model(input_size=(64, 96))
    info = video_warp_error(m, frame_dir, pdir, batch=batch, workers=workers)
    e, per = m.warp_error(frames, P)
    assert info["input"]["E_warp"] == e and np.array_equal(np.array(info["input"]["E_pair"]), per, equal_nan=True)


def test_video_refuses_misaligned_frames(cuda, frame_dir, tmp_path):
    import cv2
    from raft_b200.video import video_consistent, video_warp_error
    frames = _decoded(frame_dir)
    short = tmp_path / "short"
    short.mkdir()
    for i in range(len(frames) - 1):
        cv2.imwrite(str(short / f"s{i:03d}.png"), frames[i])
    small = tmp_path / "small"
    small.mkdir()
    for i in range(len(frames)):
        cv2.imwrite(str(small / f"s{i:03d}.png"), frames[i][:-2])
    m = _model()
    with pytest.raises(ValueError, match="aligned"):
        video_consistent(m, frame_dir, str(short), tmp_path / "o1", 0.1)
    with pytest.raises(ValueError, match="aligned"):
        video_warp_error(m, frame_dir, str(small))


def test_cli_end_to_end(cuda, tmp_path, frame_dir):
    import json
    import os
    import subprocess
    import sys
    import cv2
    from test_gpu_track import _weights
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    np.savez(tmp_path / "w.npz", **_weights(False))
    pdir, _ = _processed_dir(tmp_path / "proc", _decoded(frame_dir))
    base = [sys.executable, os.path.join(root, "raft-tf_b200", "infer_raft.py"), "--path", frame_dir, "--load",
            str(tmp_path / "w.npz"), "--flow-size", "64", "96", "--iters", "4", "--batch", "3"]
    out = tmp_path / "stable"
    r = subprocess.run(base + ["--consistent", pdir, "--consistent-strength", "0.1", "--out", str(out)],
                       capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "consistent: E_warp original" in r.stdout and "status: used" in r.stdout
    files = sorted(out.glob("frame_*.png"))
    assert len(files) == 10 and all(cv2.imread(str(f)).shape == (124, 150, 3) for f in files)
    r = subprocess.run(base + ["--warp-error", str(out), "--out", str(tmp_path / "score")], capture_output=True,
                       text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "warp error: E_warp" in r.stdout
    rec = json.load(open(tmp_path / "score" / "warp_error.json"))
    assert len(rec["input"]["E_pair"]) == 9 and rec["cuts"] == []
