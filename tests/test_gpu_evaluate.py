"""F9 validation on the GPU: rb_flow_metrics against the torch restatement of upstream's formulas (tests/eval_oracle.py),
its determinism, pad_mode='kitti', and raft_b200.evaluate end to end against the oracle applied to RAFT.forward of each
pair (Sintel both passes, raft-things and raft-small; KITTI at two frame sizes with sparse 16-bit ground truth; RGB frames
upstream; mixed precision; the CLI)."""
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from eval_oracle import aggregate_stats, pixel_terms, sample_stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_WEIGHTS = {}


def _weights(small):
    from raft_b200 import synth
    if small not in _WEIGHTS:
        _WEIGHTS[small] = synth.make_weights(small)
    return _WEIGHTS[small]


def _case(rng, B, H, W, scale):
    """Random flows and ground truth with the edge cases planted: gt = 0, EPE exactly 1, 3 and 5, EPE > 3 with |gt| = 0."""
    gt = rng.uniform(-40, 40, (B, H, W, 2)).astype(np.float32)
    flow = (gt + rng.normal(0, 3, gt.shape)).astype(np.float32)
    n = B * H * W
    flat_g, flat_f = gt.reshape(-1, 2), flow.reshape(-1, 2)
    idx = rng.permutation(n)
    planted = [((0, 0), (0, 0)), ((0, 0), (1, 0)), ((10, 0), (13, 0)), ((0, 0), (3, 4)), ((0, 0), (4, 3)),
               ((0, 0), (0, 7)), ((20, -5), (20, -2)), ((100, 0), (105, 0)), ((0, 80), (0, 84))]
    for (g, f), i in zip(planted, idx):
        flat_g[i], flat_f[i] = g, f
    flat_g[idx[len(planted):len(planted) + n // 10]] = 0  # 10 % zero ground truth
    return flow / np.float32(scale), gt  # x scale in the kernel is exact


def _metrics(flow, gt, valid=None, scale=1.0):
    from networks.utils import flow_metrics
    t = lambda a: None if a is None else torch.from_numpy(a).cuda()  # noqa: E731
    stats, epe = flow_metrics(t(flow), t(gt), t(valid), flow_scale=scale, return_epe=True)
    return stats.cpu(), epe.cpu()


def _check_against_oracle(stats, epe_gpu, flow, gt, valid, scale):
    e, _, _ = pixel_terms(flow, gt, scale)
    assert torch.equal(epe_gpu.view(torch.int32), e.view(torch.int32)), "per-pixel EPE differs"
    want = sample_stats(flow, gt, valid, scale)
    cols = [0, 2, 3, 4, 5]
    assert torch.equal(stats[:, cols], want[:, cols]), (stats, want)
    assert ((stats[:, 1] - want[:, 1]).abs() <= 1e-12 * want[:, 1].abs().clamp_min(1e-300)).all(), (stats[:, 1], want[:, 1])


@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (2, 5, 7), (3, 37, 53), (1, 64, 64), (2, 65, 63), (2, 436, 1024)])
@pytest.mark.parametrize("masked", [False, True])
def test_kernel_equals_oracle(cuda, B, H, W, masked):
    rng = np.random.default_rng(B * 7919 + H * 31 + W + masked)
    for scale in (1.0, 8.0):
        flow, gt = _case(rng, B, H, W, scale)
        valid = (rng.random((B, H, W)) < 0.6).astype(np.uint8) if masked else None
        stats, epe = _metrics(flow, gt, valid, scale)
        assert stats.dtype == torch.float64 and tuple(stats.shape) == (B, 6)
        _check_against_oracle(stats, epe, flow, gt, valid, scale)
        if H * W > 1000:
            assert (stats[:, 5] > 0).all() and (stats[:, 2] > 0).all()  # outliers and sub-pixel errors both occur


def test_planted_edge_cases_by_hand(cuda):
    gt = np.array([[[[0, 0], [0, 0], [10, 0], [0, 0], [0, 0], [100, 0], [0, 80]]]], np.float32)
    fl = np.array([[[[0, 0], [1, 0], [13, 0], [3, 4], [0, 7], [105, 0], [0, 84]]]], np.float32)
    stats, epe = _metrics(fl, gt)
    assert epe[0, 0].tolist() == [0, 1, 3, 5, 7, 5, 4]
    # EPE < 1: 0; < 3: 0, 1; < 5: 0, 1, 3, 4; outliers: 5 and 7 with |gt| = 0 (5 / 100 and 4 / 80 round to 0.05f: not above)
    assert stats[0].tolist() == [7, 25, 1, 2, 4, 2]


def test_nan_flow_propagates_into_the_sum(cuda):
    rng = np.random.default_rng(5)
    flow, gt = _case(rng, 2, 9, 11, 1.0)
    flow[1, 3, 4, 0] = np.nan
    stats, epe = _metrics(flow, gt)
    assert torch.isnan(epe[1, 3, 4]) and torch.isnan(stats[1, 1]) and not torch.isnan(stats[0, 1])
    want = sample_stats(flow, gt)
    assert torch.equal(stats[:, [0, 2, 3, 4, 5]], want[:, [0, 2, 3, 4, 5]])


def test_batch_equals_single_calls_bit_for_bit(cuda):
    rng = np.random.default_rng(9)
    B, H, W = 5, 301, 517
    flow, gt = _case(rng, B, H, W, 1.0)
    valid = (rng.random((B, H, W)) < 0.4).astype(np.uint8)
    for v in (None, valid):
        batch, epe = _metrics(flow, gt, v)
        again, epe2 = _metrics(flow, gt, v)
        assert torch.equal(batch.view(torch.int64), again.view(torch.int64)) and torch.equal(epe, epe2)
        for b in range(B):
            one, _ = _metrics(flow[b:b + 1], gt[b:b + 1], None if v is None else v[b:b + 1])
            assert torch.equal(one.view(torch.int64), batch[b:b + 1].view(torch.int64)), b


def _model(small=False, **kw):
    from networks.RAFT import RAFT
    return RAFT(None, SimpleNamespace(small=small), iters=4, **kw).load(_weights(small))


def test_pad_mode_kitti_equals_bottom_padding_on_the_host(cuda):
    from raft_b200 import synth
    H, W = 125, 203  # pads 3 rows and 5 columns
    l, r = synth.make_batch(2, H, W)
    ph, pw = (-H) % 8, (-W) % 8
    pad = ((0, 0), (0, ph), (pw // 2, pw - pw // 2), (0, 0))
    lp, rp = (np.pad(x, pad, mode="edge") for x in (l, r))
    ref = _model().forward(lp, rp)[:, :H, pw // 2:pw // 2 + W]
    kitti = _model(pad_mode="kitti").forward(l, r)
    sintel = _model().forward(l, r)
    assert torch.equal(kitti, ref)
    assert not torch.equal(kitti, sintel)


def _oracle_pairs(model, pairs, kitti, rgb, scale):
    """Per-pair oracle stats of model.forward on the decoded pairs, in order."""
    from raft_b200.evaluate import _decode
    rows = []
    for p in pairs:
        left, right, gt, valid = _decode(p, kitti, rgb)
        flow = model.forward(left[None], right[None]).cpu()
        rows.append(sample_stats(flow, gt[None], None if valid is None else valid[None], scale)[0])
    return torch.stack(rows).numpy()


def _same_stats(res, oracle, kitti):
    got = np.array([[r["n"], r["epe"] * r["n"]] for r in res["pairs"]])
    assert np.array_equal(got[:, 0], oracle[:, 0])
    for r, o in zip(res["pairs"], oracle):
        n = o[0]
        assert [round(r[k] * n) for k in ("1px", "3px", "5px")] == list(o[2:5]) and round(r["f1"] * n / 100) == o[5]
        assert abs(r["epe"] - o[1] / n) <= 1e-12 * abs(o[1] / n)
    want = aggregate_stats(oracle, kitti)
    assert all(abs(res[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])) for k in want), (res, want)


@pytest.fixture(scope="module")
def sintel_tree(tmp_path_factory):
    from raft_b200 import synth
    root = str(tmp_path_factory.mktemp("sintel"))
    assert synth.write_sintel_tree(root, 2, 4, 124, 200) == 6
    return root


@pytest.mark.parametrize("small", [False, True])
def test_sintel_end_to_end(cuda, sintel_tree, small):
    from raft_b200.evaluate import evaluate, sintel_pairs
    model = _model(small)
    runs = [evaluate(model, sintel_tree, "sintel", batch=b, workers=w, iters=4) for b, w in ((1, 0), (3, 4), (3, 0))]
    assert runs[0] == runs[1] == runs[2]
    res = runs[0]
    assert res["iters"] == 4 and res["pad_mode"] == "sintel" and list(res["splits"]) == ["clean", "final"]
    scale = 8.0 if small else 1.0  # raft-small's reference flow is in 1/8-resolution units
    for d in ("clean", "final"):
        pairs = sintel_pairs(sintel_tree, d)
        r = res["splits"][d]
        assert [p["image1"] for p in r["pairs"]] == [p.image1 for p in pairs] and r["pixels"] == 6 * 124 * 200
        _same_stats(r, _oracle_pairs(model, pairs, False, False, scale), False)
    assert res["splits"]["clean"]["epe"] != res["splits"]["final"]["epe"]


def _kitti_tree(root, rng):
    """Five pairs at two sizes (interleaved ids), sparse valid masks, 16-bit ground truth."""
    import cv2
    from raft_b200 import synth
    sizes = [(124, 200), (130, 211), (124, 200), (130, 211), (124, 200)]
    for i, (H, W) in enumerate(sizes):
        f1, f2, flow = synth.make_pair(H, W, 3000 + i, return_flow=True)
        for s, f in (("10", f1), ("11", f2)):
            d = os.path.join(root, "training", "image_2")
            os.makedirs(d, exist_ok=True)
            cv2.imwrite(os.path.join(d, f"{i:06d}_{s}.png"), np.round(255 * f).astype(np.uint8))
        raw = np.zeros((H, W, 3), np.uint16)
        raw[..., 2:0:-1] = np.clip(np.round(flow * 64 + 2 ** 15), 0, 65535).astype(np.uint16)
        raw[..., 0] = rng.random((H, W)) < 0.3
        d = os.path.join(root, "training", "flow_occ")
        os.makedirs(d, exist_ok=True)
        cv2.imwrite(os.path.join(d, f"{i:06d}_10.png"), raw)


def test_kitti_end_to_end(cuda, tmp_path):
    from raft_b200.evaluate import evaluate, kitti_pairs
    rng = np.random.default_rng(11)
    root = str(tmp_path)
    _kitti_tree(root, rng)
    model = _model()
    res = evaluate(model, root, "kitti", batch=2, workers=2, iters=4)
    assert res == evaluate(model, root, "kitti", batch=1, workers=0, iters=4)
    assert res["iters"] == 4 and res["pad_mode"] == "kitti" and list(res["splits"]) == ["kitti"]
    pairs = kitti_pairs(root)
    r = res["splits"]["kitti"]
    assert [p["image1"] for p in r["pairs"]] == [p.image1 for p in pairs]
    oracle = _oracle_pairs(_model(pad_mode="kitti"), pairs, True, False, 1.0)
    assert r["pixels"] == oracle[:, 0].sum() > 0
    _same_stats(r, oracle, True)
    assert abs(r["epe"] - np.mean(oracle[:, 1] / oracle[:, 0])) <= 1e-12 * r["epe"]


def test_upstream_feeds_rgb_and_mixed_precision_runs(cuda, sintel_tree):
    from raft_b200.evaluate import evaluate, sintel_pairs
    pairs = sintel_pairs(sintel_tree, "clean")
    up = _model(upstream=True)
    res = evaluate(up, sintel_tree, "sintel", dstypes=("clean",), batch=2, iters=4)["splits"]["clean"]
    rgb = _oracle_pairs(up, pairs, False, True, 1.0)
    _same_stats(res, rgb, False)
    bgr = _oracle_pairs(up, pairs, False, False, 1.0)
    assert not np.array_equal(rgb[:, 1], bgr[:, 1])
    mp = _model(mixed_precision=True)
    res = evaluate(mp, sintel_tree, "sintel", dstypes=("clean",), batch=3, iters=4)["splits"]["clean"]
    assert np.isfinite(res["epe"])
    _same_stats(res, _oracle_pairs(mp, pairs, False, False, 1.0), False)


def test_cli_val_writes_the_api_result(cuda, sintel_tree, tmp_path):
    from raft_b200.evaluate import evaluate
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    out = tmp_path / "log"
    cli = [sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "-m", "val", "--dataset", "sintel",
           "--data", sintel_tree, "--out", str(out), "--load", npz, "--iters", "4", "--batch", "2"]
    r = subprocess.run(cli, cwd=tmp_path, env=dict(os.environ, PYTHONNOUSERSITE="1"), capture_output=True, text=True,
                       check=True)
    got = json.loads((out / "val_sintel.json").read_text())
    want = json.loads(json.dumps(evaluate(_model(), sintel_tree, "sintel", iters=4)))
    assert got == want
    for d in ("clean", "final"):
        s = want["splits"][d]
        line = "Validation (%s) EPE: %f, 1px: %f, 3px: %f, 5px: %f" % (d, s["epe"], s["1px"], s["3px"], s["5px"])
        assert line in r.stdout.splitlines(), r.stdout
