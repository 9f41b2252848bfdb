"""F27 / F28 on the GPU: rb_denoise_merge and rb_noise_sums against the numpy restatements bit for bit
(tests/denoise_oracle.py), the support against rb_track_points, RAFT.denoise against its parts, video_denoise against
RAFT.denoise for several batch, window and worker counts and a scene cut, the CLI and the DAVIS denoising protocol on a
synthetic tree.  The end-to-end tests run seeded weights: plumbing, not quality."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import denoise_oracle as DO
from raft_b200 import denoise as D
from raft_b200.inpaint import inpaint_rows
from test_gpu_inpaint import _random_clip, lenient  # noqa: F401  (lenient: the fixture)
from test_gpu_track import _model, _weights
from test_gpu_video import _decoded, frame_dir  # noqa: F401  (frame_dir: the module fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _clip(rng, F, src, net, scale=1.0):
    """Random frames and flows whose steps are partly consistent, partly occluded and partly leave the grid."""
    frames, _, fw, bw = _random_clip(rng, F, src, net)
    Hn, Wn = net
    fw[:, : Hn // 4, :, 0] += np.float32(Wn)  # the top rows step off the grid
    bw[:, Hn // 2:, : Wn // 3] += np.float32(3.0)  # occluded: the backward flow disagrees
    return frames, fw / np.float32(scale), bw / np.float32(scale)


@pytest.mark.parametrize("src,net,scale", [((40, 56), (40, 56), 1.0), ((75, 101), (32, 48), 1.0),
                                           ((31, 45), (48, 64), 8.0), ((9, 13), (3, 2), 1.0)])
def test_merge_matches_oracle(cuda, src, net, scale):
    from networks.utils import denoise_merge
    rng = np.random.default_rng(src[1] + net[0])
    F = 8
    frames, fw, bw = _clip(rng, F, src, net, scale)
    rows = np.concatenate([inpaint_rows(F, 3), inpaint_rows(F, 2, [3])[::-1], inpaint_rows(F, 16, [0, 5]),
                           [[4, 0, 0], [0, 0, 0], [7, 0, 7]]])
    for sigma in (7.5, 30.0):
        out, support = denoise_merge(_t(cuda, frames), _t(cuda, fw), _t(cuda, bw), rows, sigma, flow_scale=scale)
        w_out, w_support = DO.denoise_merge(frames, fw, bw, rows, sigma, scale)
        assert np.array_equal(support.cpu().numpy(), w_support)
        assert np.array_equal(out.cpu().numpy(), w_out)
    if src[0] > 9:  # every outcome is exercised: no match, some, and chains cut short
        s, full = w_support[:F], (rows[:F, 1] + rows[:F, 2])[:, None, None]
        assert (s == 0).any() and (s > 0).any() and (s < full).any()


def test_merge_at_the_longest_window_and_bad_tables(cuda):
    """Rows at RB_DENOISE_MAX_WINDOW each way, and tables the kernel clamps: an absent t, steps past the clip or the
    window (the raw C entry; the Python wrapper refuses them)."""
    from raft_b200 import capi
    rng = np.random.default_rng(11)
    F, src, net = 20, (33, 47), (17, 24)
    frames, fw, bw = _clip(rng, F, src, net)
    fw[:] = 0
    bw[:] = 0  # every step consistent, so the chains run the whole window
    rows = np.array([[16, 3, 16], [3, 16, 3], [10, 40, 99], [19, 5, 20], [-1, 2, 2], [F, 0, 0], [5, -3, -1]], np.int32)
    f, a, b, tab = _t(cuda, frames), _t(cuda, fw), _t(cuda, bw), _t(cuda, rows)
    out = torch.empty(len(rows), *src, 3, dtype=torch.uint8, device=cuda)
    support = torch.empty(len(rows), *src, dtype=torch.uint8, device=cuda)
    capi.check(capi.lib.rb_denoise_merge(capi.ptr(f), F, *src, capi.ptr(a), capi.ptr(b), *net, 1.0, 0.01, 0.5,
                                         capi.ptr(tab), len(rows), 12.0, capi.ptr(out), capi.ptr(support),
                                         capi.stream()))
    w_out, w_support = DO.denoise_merge(frames, fw, bw, rows, 12.0)
    assert np.array_equal(support.cpu().numpy(), w_support) and np.array_equal(out.cpu().numpy(), w_out)
    assert (w_support[0] == 19).all() and (w_support[2] == 9 + 10).all() and (w_support[3] == 16).all()
    assert not w_out[4].any() and not w_out[5].any() and not w_support[4:6].any() and not w_support[6].any()
    from networks.utils import denoise_merge
    for bad in ([[F, 0, 0]], [[1, 0, 2]], [[3, F, 0]], [[0.5, 0, 0]], [0, 0, 0]):
        with pytest.raises(ValueError):
            denoise_merge(f, a, b, bad, 12.0)
    with pytest.raises(ValueError):
        denoise_merge(f, a, b, [[0, 0, 0]], 0.0)


def test_row_bits_do_not_depend_on_the_table(cuda):
    from networks.utils import denoise_merge
    rng = np.random.default_rng(5)
    F = 6
    frames, fw, bw = _clip(rng, F, (29, 38), (15, 19))
    args = [_t(cuda, a) for a in (frames, fw, bw)]
    rows = inpaint_rows(F, 2)
    out, sup = denoise_merge(*args, rows, 15.0)
    perm = [4, 1, 5, 0, 3, 2]
    out2, sup2 = denoise_merge(*args, rows[perm], 15.0)
    assert torch.equal(out2, out[perm]) and torch.equal(sup2, sup[perm])
    one, one_sup = denoise_merge(*args, rows[3:4], 15.0)
    assert torch.equal(one[0], out[3]) and torch.equal(one_sup[0], sup[3])


def test_constant_clip_comes_back(cuda):
    from networks.utils import denoise_merge
    rng = np.random.default_rng(6)
    F = 5
    _, fw, bw = _clip(rng, F, (37, 50), (20, 26))
    flat = np.full((F, 37, 50, 3), (12, 130, 250), np.uint8)
    out, sup = denoise_merge(_t(cuda, flat), _t(cuda, fw), _t(cuda, bw), inpaint_rows(F, 3), 25.0)
    assert np.array_equal(out.cpu().numpy(), flat) and sup.any()


def test_forward_support_is_the_tracked_prefix(cuda):
    """The forward support of a pixel equals the number of leading status-0 rows of rb_track_points for a query at its
    network position p0 (same step, same test)."""
    from inpaint_oracle import _remap
    from networks.utils import denoise_merge, track_points
    rng = np.random.default_rng(9)
    F, src, net = 7, (26, 34), (26, 34)
    frames, fw, bw = _clip(rng, F, src, net)
    rows = np.array([[0, F - 1, 0]], np.int32)
    _, sup = denoise_merge(_t(cuda, frames), _t(cuda, fw), _t(cuda, bw), rows, 10.0)
    ys, xs = (a.reshape(-1) for a in np.mgrid[0:src[0], 0:src[1]])
    q = np.stack([_remap(xs, 1.0, src[1]), _remap(ys, 1.0, src[0])], -1).astype(np.float32)
    _, status, _ = track_points(_t(cuda, fw), _t(cuda, bw), np.zeros(len(q), np.int32), q)
    st = status.cpu().numpy()[1:]  # [F-1, N]: the rows after the query frame
    lead = np.argmax(np.vstack([st != 0, np.ones((1, st.shape[1]), bool)]), axis=0)
    assert np.array_equal(sup.cpu().numpy()[0].reshape(-1), lead)
    assert (lead > 0).any() and (lead < F - 1).any()


@pytest.mark.parametrize("shape", [(1, 3, 3), (3, 41, 57), (2, 1080, 1920)])
def test_noise_sums_match_oracle(cuda, shape):
    from networks.utils import noise_sigma, noise_sums
    rng = np.random.default_rng(sum(shape))
    frames = rng.integers(0, 256, shape + (3,), dtype=np.uint8)
    got = noise_sums(_t(cuda, frames)).cpu().numpy()
    assert np.array_equal(got, DO.noise_sums(frames))
    assert noise_sigma(_t(cuda, frames)) == D.sigma_from_sums(got, shape[1], shape[2])
    flat = np.full(shape + (3,), 128, np.uint8)
    assert noise_sigma(_t(cuda, flat)) == 0.0


def _noisy(frames, sigma, seed=0):
    rng = np.random.default_rng(seed)
    return np.clip(np.rint(frames + sigma * rng.standard_normal(frames.shape)), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("small,size,upstream", [(False, (64, 96), False), (True, None, False),
                                                 (False, (128, 160), True)])
def test_raft_denoise_equals_its_parts(cuda, frame_dir, lenient, small, size, upstream):
    m = _model(small=small, input_size=size, upstream=upstream)
    frames = _noisy(_decoded(frame_dir), 20)
    F = len(frames)
    out, support = m.denoise(frames, 20, window=2, cuts=[6])
    eng = m.engine()
    fw, bw, _, _ = eng.forward_sequence_bidirectional(_t(cuda, frames), check=False)
    rows = inpaint_rows(F, 2, [6])
    w_out, w_sup = D.merge_frames(_t(cuda, frames), fw, bw, rows, 20.0, eng.flow_scale)
    assert torch.equal(out, w_out) and torch.equal(support, w_sup)
    assert out.shape == frames.shape and support.float().mean() > 1.0
    o_out, o_sup = DO.denoise_merge(frames, fw.cpu().numpy(), bw.cpu().numpy(), rows, 20.0, eng.flow_scale, a2=lenient)
    assert np.array_equal(support.cpu().numpy(), o_sup) and np.array_equal(out.cpu().numpy(), o_out)
    # sigma="auto" is the estimate of the first frames; on noise-free flat frames it is 0 and the frames come back
    auto, _ = m.denoise(frames, "auto", window=2, cuts=[6])
    est = D.estimate_sigma(_t(cuda, frames))
    assert est > 0 and torch.equal(auto, D.merge_frames(_t(cuda, frames), fw, bw, rows, est, eng.flow_scale)[0])
    flat = np.full_like(frames, 90)
    same, sup0 = m.denoise(flat, "auto")
    assert np.array_equal(same.cpu().numpy(), flat) and not sup0.any()


def test_denoise_refusals(cuda, frame_dir):
    m = _model(input_size=(64, 96))
    frames = _decoded(frame_dir)
    for kw in (dict(sigma=0), dict(sigma="x"), dict(sigma=float("nan")), dict(sigma=20, window=0),
               dict(sigma=20, window=17), dict(sigma=20, cuts=[len(frames) - 1])):
        with pytest.raises(ValueError):
            m.denoise(frames, **kw)
    with pytest.raises(ValueError):
        m.denoise(frames.astype(np.float32), 20)


def _noisy_dir(d, frames):
    import cv2
    d.mkdir()
    for i, f in enumerate(frames):
        cv2.imwrite(str(d / f"f{i:03d}.png"), f)
    return str(d)


@pytest.mark.parametrize("batch,window,workers", [(1, 1, 1), (3, 3, 4), (8, 16, 1), (3, 2, 0), (8, 3, 4)])
def test_video_denoise_equals_denoise(cuda, frame_dir, tmp_path, lenient, batch, window, workers):
    import cv2
    from raft_b200.video import video_denoise
    m = _model(input_size=(64, 96))
    frames = _noisy(_decoded(frame_dir), 15, seed=batch)
    d = _noisy_dir(tmp_path / "noisy", frames)
    want, support = m.denoise(frames, 15, window=window)
    paths, info = video_denoise(m, d, tmp_path / "out", 15, window=window, batch=batch, workers=workers)
    assert len(paths) == len(frames) and info["cuts"] == [] and info["sigma"] == 15.0
    assert info["support"] == pytest.approx(float(support.double().mean()), rel=0, abs=1e-12) and info["support"] > 0
    for i, p in enumerate(paths):
        assert np.array_equal(cv2.imread(p), want[i].cpu().numpy()), i
    paths, info = video_denoise(m, d, tmp_path / "auto", "auto", window=window, batch=batch, workers=workers)
    want, _ = m.denoise(frames, "auto", window=window)
    assert info["sigma"] == D.estimate_sigma(_t(cuda, frames))
    for i, p in enumerate(paths):
        assert np.array_equal(cv2.imread(p), want[i].cpu().numpy()), i


def test_scene_cut_keeps_each_shot_apart(cuda, frame_dir, tmp_path, lenient):
    import cv2
    from raft_b200.video import list_frames, video_denoise
    d = tmp_path / "clip"
    d.mkdir()
    for i, p in enumerate(list_frames(frame_dir)):
        img = cv2.imread(p) // 4
        img[..., 2 if i < 5 else 0] += 180  # shot A reddish, shot B bluish: disjoint ranges in channels 0 and 2
        cv2.imwrite(str(d / f"f{i:03d}.png"), img)
    frames = _decoded(str(d))
    m = _model(input_size=(64, 96))
    paths, info = video_denoise(m, str(d), tmp_path / "out", 40, window=6, batch=3, scene_cut=0.5)
    assert info["cuts"] == [4]
    want, support = m.denoise(frames, 40, window=6, cuts=[4])
    rows = inpaint_rows(len(frames), 6, [4])
    assert (support.cpu().numpy() <= (rows[:, 1] + rows[:, 2])[:, None, None]).all()
    for i, p in enumerate(paths):
        out = cv2.imread(p)
        assert np.array_equal(out, want[i].cpu().numpy())
        shot = frames[:5] if i < 5 else frames[5:]
        lo, hi = shot.reshape(-1, 3).min(0), shot.reshape(-1, 3).max(0)
        assert (out.reshape(-1, 3) >= lo).all() and (out.reshape(-1, 3) <= hi).all(), i


def test_cli_writes_the_frames(cuda, tmp_path, frame_dir):
    import cv2
    np.savez(tmp_path / "w.npz", **_weights(False))
    d = _noisy_dir(tmp_path / "noisy", _noisy(_decoded(frame_dir), 25))
    out = tmp_path / "clean"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--path", d, "--out",
                        str(out), "--denoise", "25", "--denoise-window", "2", "--load", str(tmp_path / "w.npz"),
                        "--flow-size", "64", "96", "--iters", "4", "--batch", "3"],
                       capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "denoise: sigma 25" in r.stdout and "mean support" in r.stdout and "denoised frames written" in r.stdout
    files = sorted(out.glob("frame_*.png"))
    assert len(files) == 10 and all(cv2.imread(str(f)).shape == (124, 150, 3) for f in files)


def test_val_davis_denoise_equals_the_host_computation(cuda, tmp_path):
    from networks.utils import frame_metrics
    from raft_b200 import synth
    from raft_b200.davis import davis_frames, denoise_clip, noisy_frame, psnr_ssim
    from raft_b200.evaluate import _engine, _imread
    root = tmp_path / "davis"
    names = synth.write_davis_tree(str(root), [("alpha", 5), ("beta", 4)], H=64, W=96)
    os.replace(root / "ImageSets" / "2017" / "val.txt", root / "ImageSets" / "2017" / "test-dev.txt")
    np.savez(tmp_path / "w.npz", **_weights(False))
    out = tmp_path / "val"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "-m", "val", "--dataset",
                        "davis", "--data", str(root), "--denoise", "20", "--load", str(tmp_path / "w.npz"), "--iters",
                        "4", "--batch", "2", "--out", str(out)], capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert "Validation DAVIS-2017 denoising (test-dev, sigma 20): PSNR: " in r.stdout and "(noisy: PSNR: " in r.stdout
    res = json.load(open(out / "val_davis_denoise.json"))
    assert [s["name"] for s in res["sequences"]] == names and res["iters"] == 4
    m = _model()
    eng = _engine(m, 4, "sintel")
    psnr, ssim, npsnr = [], [], []
    for clip in davis_frames(str(root)):
        clean = np.stack([_imread(p, True) for p in clip.frames])
        noisy = np.stack([noisy_frame(c, clip.name, i, 20) for i, c in enumerate(clean)])
        clean, noisy = clean[..., ::-1].copy(), noisy[..., ::-1].copy()
        got, _ = denoise_clip(eng, _t(cuda, noisy), 20.0, None, 1)
        w, _ = D.merge_frames(_t(cuda, noisy), *eng.forward_sequence_bidirectional(_t(cuda, noisy), check=False)[:2],
                              inpaint_rows(len(noisy), D.DEFAULT_WINDOW), 20.0, eng.flow_scale)
        assert torch.equal(got, w)  # the per-pass flows give the one-pass bits
        H, W = clean.shape[1:3]
        host = got.cpu().numpy().astype(np.float64)
        sse = ((host - clean) ** 2).sum(axis=(1, 2, 3))
        stats = frame_metrics(got, _t(cuda, clean)).cpu().numpy()
        assert np.array_equal(stats[:, 0], sse)
        p, s = psnr_ssim(stats, H, W)
        assert np.allclose(p, 10 * np.log10(255.0 ** 2 * 3 * H * W / sse), rtol=0, atol=1e-12)
        psnr.append(p.mean())
        ssim.append(s.mean())
        npsnr.append(psnr_ssim(frame_metrics(_t(cuda, noisy), _t(cuda, clean)).cpu().numpy(), H, W)[0].mean())
    assert res["PSNR"] == pytest.approx(np.mean(psnr), rel=1e-12) and res["SSIM"] == pytest.approx(np.mean(ssim),
                                                                                                  rel=1e-12)
    assert res["noisy_PSNR"] == pytest.approx(np.mean(npsnr), rel=1e-12)
