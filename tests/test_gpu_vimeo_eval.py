"""F12 frame-interpolation validation on the GPU: rb_frame_metrics against the numpy / scipy restatement
(tests/vfi_oracle.py) -- SSE exactly, SSIM to 1e-10 -- on fp32 frames with planted rounding ties, out-of-range values and
NaNs and on uint8 frames; its batch invariance, determinism and graph capture; and raft_b200.evaluate's 'vimeo' dataset
end to end against RAFT.interpolate followed by the oracle (raft-things and raft-small, two frame sizes, batch and worker
counts, RGB frames upstream, the CLI)."""
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import vfi_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_WEIGHTS = {}


def _weights(small):
    from raft_b200 import synth
    if small not in _WEIGHTS:
        _WEIGHTS[small] = synth.make_weights(small)
    return _WEIGHTS[small]


def _halves():
    """fp32 x with fl32(255 x) = k + 0.5 exactly, k = 0..254: the rounding ties of the quantisation."""
    out = []
    for k in range(255):
        x = np.float32((k + 0.5) / 255)
        for c in (x, np.nextafter(x, np.float32(0)), np.nextafter(x, np.float32(1))):
            if np.float32(255) * c == np.float32(k + 0.5):
                out.append(c)
                break
    assert len(out) > 200
    return np.array(out, np.float32)


def _case(rng, B, H, W):
    """uint8 ground truth and an fp32 prediction near it with ties, negatives, values > 1 and NaNs planted."""
    gt = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    smooth = rng.random((B, 1, 1, 3)) * np.linspace(0, 1, W)[None, None, :, None]  # some structure across the frame
    gt = np.clip(0.5 * gt + 120 * smooth, 0, 255).astype(np.uint8)
    pred = (gt / np.float32(255) + rng.normal(0, 0.04, gt.shape)).astype(np.float32)
    flat = pred.reshape(-1)
    n = flat.size
    idx = rng.permutation(n)
    h = _halves()
    k = min(n // 4, 4 * h.size)
    m = n // 20
    flat[idx[:k]] = h[rng.integers(0, h.size, k)]
    flat[idx[k:k + m]] = -rng.random(m).astype(np.float32)
    flat[idx[k + m:k + 2 * m]] = (1 + rng.random(m)).astype(np.float32)
    flat[idx[k + 2 * m:k + 2 * m + 3]] = np.nan
    return pred, gt


def _gpu(pred, gt):
    from networks.utils import frame_metrics
    return frame_metrics(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()).cpu().numpy()


def _check(stats, pred, gt):
    want = vfi_oracle.frame_stats(pred, gt)
    assert stats.dtype == np.float64 and stats.shape == want.shape
    assert np.array_equal(stats[:, 0], want[:, 0]), (stats[:, 0], want[:, 0])
    assert np.abs(stats[:, 1] - want[:, 1]).max() <= 1e-10, (stats[:, 1], want[:, 1])


@pytest.mark.parametrize("B,H,W", [(1, 11, 11), (2, 11, 12), (3, 37, 53), (2, 65, 63), (2, 256, 448), (1, 436, 1024)])
def test_kernel_equals_oracle(cuda, B, H, W):
    rng = np.random.default_rng(B * 7919 + H * 31 + W)
    pred, gt = _case(rng, B, H, W)
    _check(_gpu(pred, gt), pred, gt)
    q = vfi_oracle.quantise(pred)
    stats = _gpu(q, gt)
    _check(stats, q, gt)
    assert np.array_equal(stats, _gpu(pred, gt))  # an fp32 frame scores as its quantised uint8 frame, bit for bit
    assert (stats[:, 1] < 1).all() and (stats[:, 0] > 0).all()


def test_identical_frames_score_ssim_one_and_zero_sse(cuda):
    rng = np.random.default_rng(3)
    _, gt = _case(rng, 2, 40, 50)
    stats = _gpu(gt, gt)
    assert stats[:, 0].tolist() == [0.0, 0.0] and np.abs(stats[:, 1] - 1).max() <= 1e-15


def test_batch_equals_single_calls_bit_for_bit_and_runs_repeat(cuda):
    rng = np.random.default_rng(9)
    B, H, W = 5, 67, 93
    pred, gt = _case(rng, B, H, W)
    batch = _gpu(pred, gt)
    assert np.array_equal(batch.view(np.int64), _gpu(pred, gt).view(np.int64))
    for b in range(B):
        one = _gpu(pred[b:b + 1], gt[b:b + 1])
        assert np.array_equal(one.view(np.int64), batch[b:b + 1].view(np.int64)), b
    perm = [3, 0, 4, 2, 1]
    moved = _gpu(np.ascontiguousarray(pred[perm]), np.ascontiguousarray(gt[perm]))
    assert np.array_equal(moved.view(np.int64), batch[perm].view(np.int64))


def test_graph_capture_equals_eager(cuda):
    from networks.utils import frame_metrics
    rng = np.random.default_rng(12)
    pred, gt = _case(rng, 3, 70, 90)
    p, g = torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda()
    eager = frame_metrics(p, g)  # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = frame_metrics(p, g)
    pred2, gt2 = _case(np.random.default_rng(13), 3, 70, 90)
    p.copy_(torch.from_numpy(pred2))
    g.copy_(torch.from_numpy(gt2))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured.view(torch.int64), frame_metrics(p, g).view(torch.int64))
    assert not torch.equal(captured, eager)


# ---- raft_b200.evaluate, dataset 'vimeo' ---------------------------------------------------------------------------
def _model(small=False, **kw):
    from networks.RAFT import RAFT
    return RAFT(None, SimpleNamespace(small=small), iters=4, **kw).load(_weights(small))


SIZES = [(64, 96), (72, 104), (64, 96), (72, 104), (64, 96)]  # interleaved: two graphs


@pytest.fixture(scope="module")
def vimeo_tree(tmp_path_factory):
    from raft_b200 import synth
    root = str(tmp_path_factory.mktemp("vimeo"))
    synth.write_vimeo_tree(root, SIZES)
    return root


def _oracle(model, root, rgb):
    """Per-triplet (psnr, ssim, mse) of model.interpolate(im1, im3, 0.5) scored by the oracle, in list order."""
    from raft_b200.evaluate import _decode_triplet, vimeo_triplets
    rows = []
    for t in vimeo_triplets(root):
        left, right, mid = _decode_triplet(t, rgb)
        pred = model.interpolate(left[None], right[None], 0.5).cpu().numpy()
        s = vfi_oracle.sse(pred[0], mid)
        rows.append((t.dir, vfi_oracle.psnr(s, mid.size), vfi_oracle.ssim(pred[0], mid), s / mid.size))
    return rows


def _same(res, oracle):
    assert [r["dir"] for r in res["triplets"]] == [o[0] for o in oracle] and res["n_triplets"] == len(oracle)
    for r, (_, p, s, mse) in zip(res["triplets"], oracle):
        assert r["psnr"] == p and r["mse"] == mse and abs(r["ssim"] - s) <= 1e-10, (r, p, s, mse)
    assert abs(res["psnr"] - np.mean([o[1] for o in oracle])) <= 1e-12 * res["psnr"]
    assert abs(res["ssim"] - np.mean([o[2] for o in oracle])) <= 1e-10


@pytest.mark.parametrize("small", [False, True])
def test_vimeo_end_to_end(cuda, vimeo_tree, small):
    from raft_b200.evaluate import evaluate
    model = _model(small)
    runs = [evaluate(model, vimeo_tree, "vimeo", batch=b, workers=w, iters=4) for b, w in ((1, 0), (3, 2), (3, 0), (1, 2))]
    assert runs[0] == runs[1] == runs[2] == runs[3]
    res = runs[0]
    assert res["dataset"] == "vimeo" and res["iters"] == 4 and res["pad_mode"] == "sintel" and list(res["splits"]) == ["vimeo"]
    r = res["splits"]["vimeo"]
    _same(r, _oracle(model, vimeo_tree, False))
    assert 10 < r["psnr"] < 60 and 0 < r["ssim"] < 1
    assert evaluate(model, vimeo_tree, "vimeo", dstypes=("final",), batch=2, iters=4) == res  # dstypes is ignored


def test_vimeo_upstream_decodes_rgb(cuda, tmp_path):
    from raft_b200 import synth
    from raft_b200.evaluate import evaluate
    root = str(tmp_path)
    synth.write_vimeo_tree(root, [(128, 160), (128, 160), (136, 168)], seed=4100)
    up = _model(upstream=True)
    r = evaluate(up, root, "vimeo", batch=2, workers=2, iters=4)["splits"]["vimeo"]
    rgb = _oracle(up, root, True)
    _same(r, rgb)
    bgr = _oracle(up, root, False)
    assert [o[1] for o in rgb] != [o[1] for o in bgr]


def test_cli_val_vimeo_writes_the_api_result(cuda, vimeo_tree, tmp_path):
    from raft_b200.evaluate import evaluate
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    out = tmp_path / "log"
    cli = [sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "-m", "val", "--dataset", "vimeo",
           "--data", vimeo_tree, "--out", str(out), "--load", npz, "--iters", "4", "--batch", "2"]
    r = subprocess.run(cli, cwd=tmp_path, env=dict(os.environ, PYTHONNOUSERSITE="1"), capture_output=True, text=True,
                       check=True)
    got = json.loads((out / "val_vimeo.json").read_text())
    want = json.loads(json.dumps(evaluate(_model(), vimeo_tree, "vimeo", iters=4)))
    assert got == want
    s = want["splits"]["vimeo"]
    assert "Validation Vimeo-90K: PSNR: %f, SSIM: %f" % (s["psnr"], s["ssim"]) in r.stdout.splitlines(), r.stdout
