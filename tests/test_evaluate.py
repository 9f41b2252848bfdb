"""F9 validation, host side (no GPU): Sintel / KITTI enumeration, read_kitti_flow, the oracle's aggregation on a
hand-computed case, the exact form of the F1 rule the kernel uses, the argument checks of rb_flow_metrics (before any CUDA
call) and the CLI's usage error."""
import ctypes
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from eval_oracle import aggregate_pixels, aggregate_stats, pixel_terms, sample_stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _touch(path, data=b""):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(data)


def _sintel_tree(root, scenes, dstypes=("clean", "final")):
    """scenes: {name: number of frames}; frames 1..n, ground truth for all but the last."""
    for scene, n in scenes.items():  # created in the given order: enumeration must sort
        for d in dstypes:
            for k in range(1, n + 1):
                _touch(os.path.join(root, "training", d, scene, f"frame_{k:04d}.png"))
        for k in range(1, n):
            _touch(os.path.join(root, "training", "flow", scene, f"frame_{k:04d}.flo"))


def test_sintel_pairs_within_scenes_in_sorted_order(tmp_path):
    from raft_b200.evaluate import sintel_pairs
    _sintel_tree(str(tmp_path), {"market_2": 3, "alley_1": 4})
    for d in ("clean", "final"):
        pairs = sintel_pairs(str(tmp_path), d)
        got = [(os.path.relpath(p.image1, tmp_path), os.path.relpath(p.image2, tmp_path), os.path.relpath(p.gt, tmp_path))
               for p in pairs]
        want = [(f"training/{d}/{s}/frame_{k:04d}.png", f"training/{d}/{s}/frame_{k + 1:04d}.png",
                 f"training/flow/{s}/frame_{k:04d}.flo") for s, n in (("alley_1", 4), ("market_2", 3)) for k in range(1, n)]
        assert got == want  # the last frame of each scene is unpaired; no pair crosses scenes
        assert sintel_pairs(str(tmp_path), d) == pairs


def test_sintel_missing_or_unmatched_files_are_named(tmp_path):
    from raft_b200.evaluate import sintel_pairs
    root = str(tmp_path)
    _sintel_tree(root, {"alley_1": 4, "bamboo_1": 3})
    flo = os.path.join(root, "training", "flow", "bamboo_1", "frame_0002.flo")
    os.remove(flo)
    with pytest.raises(FileNotFoundError, match="bamboo_1/frame_0002.flo"):
        sintel_pairs(root, "clean")
    _touch(flo)
    extra = os.path.join(root, "training", "flow", "alley_1", "frame_0009.flo")
    _touch(extra)
    with pytest.raises(FileNotFoundError, match="alley_1/frame_0009.flo"):
        sintel_pairs(root, "final")
    os.remove(extra)
    os.remove(os.path.join(root, "training", "clean", "alley_1", "frame_0002.png"))  # 0001 would pair with 0003
    with pytest.raises(FileNotFoundError, match="alley_1/frame_0003.png"):
        sintel_pairs(root, "clean")
    assert len(sintel_pairs(root, "final")) == 5
    with pytest.raises(FileNotFoundError, match="training/nope"):
        sintel_pairs(os.path.join(root, "training", "nope"), "clean")
    with pytest.raises(ValueError):
        sintel_pairs(root, "albedo")


def _kitti_tree(root, ids):
    for i in ids:
        for s in ("10", "11"):
            _touch(os.path.join(root, "training", "image_2", f"{i:06d}_{s}.png"))
        _touch(os.path.join(root, "training", "flow_occ", f"{i:06d}_10.png"))


def test_kitti_pairs_and_missing_files(tmp_path):
    from raft_b200.evaluate import kitti_pairs
    root = str(tmp_path)
    _kitti_tree(root, [3, 0, 1])
    pairs = kitti_pairs(root)
    assert [os.path.basename(p.image1) for p in pairs] == ["000000_10.png", "000001_10.png", "000003_10.png"]
    assert all(p.image2 == p.image1[:-6] + "11.png" and p.gt.endswith("flow_occ/" + os.path.basename(p.image1))
               for p in pairs)
    assert kitti_pairs(root) == pairs
    second = os.path.join(root, "training", "image_2", "000001_11.png")
    os.remove(second)
    with pytest.raises(FileNotFoundError, match="000001_11.png"):
        kitti_pairs(root)
    _touch(second)
    gt = os.path.join(root, "training", "flow_occ", "000003_10.png")
    os.remove(gt)
    with pytest.raises(FileNotFoundError, match="flow_occ/000003_10.png"):
        kitti_pairs(root)
    _touch(gt)
    _touch(os.path.join(root, "training", "flow_occ", "000007_10.png"))
    with pytest.raises(FileNotFoundError, match="000007_10.png"):
        kitti_pairs(root)


def test_read_kitti_flow_decodes_16bit_pngs(tmp_path):
    import cv2
    from flow_utils import read_kitti_flow
    rng = np.random.default_rng(0)
    H, W = 5, 7
    raw = rng.integers(0, 65536, (H, W, 3)).astype(np.uint16)
    raw[0, :3, 2] = (0, 32768, 65535)   # u at the ends of the range and zero
    raw[1, :3, 1] = (65535, 0, 32768)   # v
    raw[..., 0] = rng.integers(0, 2, (H, W))  # valid flag
    raw[2, 2, 0] = 0
    raw[3, 3, 0] = 65535  # any nonzero flag counts
    path = str(tmp_path / "000000_10.png")
    assert cv2.imwrite(path, raw)
    flow, valid = read_kitti_flow(path)
    assert flow.dtype == np.float32 and flow.shape == (H, W, 2) and valid.dtype == np.uint8 and valid.shape == (H, W)
    want = (raw[..., [2, 1]].astype(np.float64) - 2 ** 15) / 64.0
    assert np.array_equal(flow.astype(np.float64), want)  # exact in fp32
    assert flow[0, 0, 0] == -512.0 and flow[0, 1, 0] == 0.0 and flow[0, 2, 0] == 32767 / 64
    assert np.array_equal(valid, (raw[..., 0] > 0).astype(np.uint8)) and valid[2, 2] == 0 and valid[3, 3] == 1
    with pytest.raises(FileNotFoundError):
        read_kitti_flow(str(tmp_path / "missing.png"))
    assert cv2.imwrite(str(tmp_path / "u8.png"), np.zeros((2, 2, 3), np.uint8))
    with pytest.raises(ValueError, match="16-bit"):
        read_kitti_flow(str(tmp_path / "u8.png"))


def _hand_case():
    """Image A: EPE 1 and 2.  Image B: four pixels of EPE 4 with |gt| = 100 (4/100 < 0.05), 0 (outlier: e / 0 = inf),
    50 (0.08: outlier) and 80 (4/80 rounds to 0.05f: not above it)."""
    gtA = np.array([[[[0, 0], [10, 0]]]], np.float32)
    flA = gtA + np.array([[[[1, 0], [2, 0]]]], np.float32)
    gtB = np.array([[[[100, 0], [0, 0]], [[50, 0], [0, 80]]]], np.float32)
    flB = gtB + np.array([[[[4, 0], [0, 4]], [[-4, 0], [0, -4]]]], np.float32)
    return (flA, gtA), (flB, gtB)


def _close(got, want):
    return all(abs(got[k] - want[k]) <= 1e-15 * max(1.0, want[k]) for k in want)


def test_oracle_aggregation_by_hand():
    (flA, gtA), (flB, gtB) = _hand_case()
    sA, sB = sample_stats(flA, gtA), sample_stats(flB, gtB)
    assert sA[0].tolist() == [2, 3, 0, 2, 2, 0]
    assert sB[0].tolist() == [4, 16, 0, 0, 4, 2]
    eA, _, oA = pixel_terms(flA, gtA)
    eB, _, oB = pixel_terms(flB, gtB)
    stats = np.concatenate([sA.numpy(), sB.numpy()])
    sintel = {"epe": 19 / 6, "1px": 0.0, "3px": 2 / 6, "5px": 1.0, "f1": 100 * 2 / 6}
    kitti = dict(sintel, epe=(1.5 + 4.0) / 2)  # the mean of the per-image means, not the pooled 19 / 6
    for agg, want in ((aggregate_stats(stats, False), sintel), (aggregate_stats(stats, True), kitti),
                      (aggregate_pixels([eA, eB], [oA, oB], False), sintel),
                      (aggregate_pixels([eA, eB], [oA, oB], True), kitti)):
        assert agg.keys() == want.keys() and _close(agg, want), (agg, want)
    # the evaluator's own aggregation of the same stats
    from raft_b200.evaluate import Pair, aggregate
    pairs = [Pair("a1", "a2", "ag"), Pair("b1", "b2", "bg")]
    for kit, want in ((False, sintel), (True, kitti)):
        res = aggregate(pairs, stats, kit)
        assert _close(res, want) and res["pixels"] == 6 and res["n_pairs"] == 2
        assert [(r["image1"], r["n"], r["epe"], r["f1"]) for r in res["pairs"]] == [("a1", 2, 1.5, 0.0), ("b1", 4, 4.0, 50.0)]
    # a mask: only B's second row counts -> |gt| = 50 (an outlier) and |gt| = 80 (not one)
    s = sample_stats(flB, gtB, valid=np.array([[[0, 0], [1, 1]]], np.uint8))
    assert s[0].tolist() == [2, 8, 0, 0, 2, 1]


def test_f1_rule_without_division_equals_the_rounded_quotient():
    """The kernel decides fl32(e / m) > 0.05f as (double)e >= mid * (double)m with mid = 26843547 * 2^-29, the midpoint
    above 0.05f (csrc/metrics.cu).  Against torch's fp32 division, densely around the threshold and at the IEEE cases."""
    import torch
    mid = 26843547.0 / 536870912.0
    c = np.float32(0.05)
    assert mid == (float(c) + float(np.nextafter(c, np.float32(1)))) / 2
    rng = np.random.default_rng(3)
    e = np.concatenate([rng.uniform(3, 1e5, 400000), np.full(4, 4.0)]).astype(np.float32)
    m = (e / c).astype(np.float32)
    steps = rng.integers(-3, 4, e.size).astype(np.int32)
    m = (m.view(np.int32) + steps).view(np.float32)  # a few ulps either side of the threshold
    m = np.concatenate([m, np.float32([0, np.inf, 1e-45, np.nan, 80.0, 79.99999])])
    e = np.concatenate([e, np.float32([4, 4, 4, 4, 4, 4])])
    want = ((torch.from_numpy(e) / torch.from_numpy(m)) > 0.05).numpy()
    got = e.astype(np.float64) >= mid * m.astype(np.float64)
    assert np.array_equal(got, want) and want.any() and not want.all()


def test_flow_metrics_argument_checks_before_any_cuda_call():
    from raft_b200 import capi
    lib = capi.lib
    out = ctypes.c_size_t()
    assert lib.rb_flow_metrics_workspace_bytes(2, 436, 1024, ctypes.byref(out)) == 0
    assert out.value == 2 * 109 * 6 * 8  # 4096-pixel chunks, six fp64 partials each
    assert lib.rb_flow_metrics_workspace_bytes(1, 1, 1, ctypes.byref(out)) == 0 and out.value == 48
    assert lib.rb_flow_metrics_workspace_bytes(1, 4, 4, None) == -2
    for shape in ((0, 4, 4), (1, 0, 4), (1, 4, -1)):
        assert lib.rb_flow_metrics_workspace_bytes(*shape, ctypes.byref(out)) == -1
        assert b"rb_flow_metrics_workspace_bytes" in lib.rb_last_error()
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ok = dict(f=p, s=1.0, g=p, v=None, B=1, H=4, W=4, e=None, st=p, ws=p, wsb=48)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.rb_flow_metrics(a["f"], a["s"], a["g"], a["v"], a["B"], a["H"], a["W"], a["e"], a["st"], a["ws"],
                                   a["wsb"], None)

    cases = [(dict(f=None), -2), (dict(g=None), -2), (dict(st=None), -2), (dict(ws=None), -2),
             (dict(B=0), -1), (dict(H=0), -1), (dict(W=-2), -1), (dict(B=65536, wsb=1 << 30), -1),
             (dict(s=0.0), -2), (dict(s=-8.0), -2), (dict(s=float("nan")), -2), (dict(s=float("inf")), -2),
             (dict(wsb=47), -5), (dict(B=2, wsb=48), -5), (dict(H=4096, W=2, wsb=48), -5)]
    for kw, code in cases:
        assert call(**kw) == code, kw
        assert b"rb_flow_metrics" in lib.rb_last_error(), kw


def test_pad_mode_and_input_size_are_refused_without_a_gpu():
    from networks.RAFT import RAFT
    from raft_b200.engine import RaftEngine
    from raft_b200.evaluate import evaluate
    with pytest.raises(ValueError, match="pad_mode"):
        RAFT((64, 96, 3), SimpleNamespace(small=False), pad_mode="middlebury")
    with pytest.raises(ValueError, match="pad_mode"):
        RaftEngine({}, pad_mode="KITTI")
    m = RAFT(None, SimpleNamespace(small=False), input_size=(432, 1024))
    with pytest.raises(ValueError, match="own size"):
        evaluate(m, "/nonexistent", "sintel")
    with pytest.raises(ValueError, match="dataset"):
        evaluate(RAFT(None, SimpleNamespace(small=False)), "/nonexistent", "chairs")


def test_cli_val_needs_data_and_dataset(tmp_path):
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    for extra in ([], ["--data", str(tmp_path)], ["--dataset", "sintel"]):
        r = subprocess.run([sys.executable, cli, "-m", "val"] + extra, cwd=tmp_path, env=env, capture_output=True,
                           text=True)
        assert r.returncode == 2 and "-m val needs --data" in r.stderr, (extra, r.stderr)
    r = subprocess.run([sys.executable, cli, "-m", "flops"], cwd=tmp_path, env=env, capture_output=True, text=True)
    assert r.returncode == 0 and "has no implementation" in r.stdout
