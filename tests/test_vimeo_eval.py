"""F12 frame-interpolation validation, host side (no GPU): the SSIM restatement of tests/vfi_oracle.py against an
independent direct 2-D form, its invariants (reflect and constant padding agree on the crop, SSIM(x, x) = 1, the PSNR of
a constant offset), the quantisation, Vimeo-90K triplet enumeration, the vimeo aggregation and summary line, the argument
checks of rb_frame_metrics (before any CUDA call) and the CLI's refusals."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import vfi_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _direct_ssim_channel(x, y):
    """The 11x11 outer-product window applied at the interior pixels only, explicit sums, no scipy."""
    k = np.arange(-5, 6, dtype=np.float64)
    g = np.exp(-0.5 * k * k / 1.5 ** 2)
    g /= g.sum()
    w2 = np.outer(g, g)
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    H, W = x.shape
    S = []
    for i in range(5, H - 5):
        for j in range(5, W - 5):
            px, py = x[i - 5:i + 6, j - 5:j + 6], y[i - 5:i + 6, j - 5:j + 6]
            mx, my = (w2 * px).sum(), (w2 * py).sum()
            vx = (w2 * px * px).sum() - mx * mx
            vy = (w2 * py * py).sum() - my * my
            vxy = (w2 * px * py).sum() - mx * my
            C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
            S.append(((2 * mx * my + C1) * (2 * vxy + C2)) / ((mx * mx + my * my + C1) * (vx + vy + C2)))
    return float(np.mean(S))


def _frames(rng, H, W):
    gt = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    noise = rng.integers(-40, 41, (H, W, 3))
    pred = np.clip(gt.astype(np.int64) + noise, 0, 255).astype(np.uint8)
    return pred, gt


@pytest.mark.parametrize("H,W", [(11, 11), (11, 12), (19, 23), (32, 17)])
def test_oracle_ssim_equals_the_direct_window(H, W):
    rng = np.random.default_rng(H * 100 + W)
    pred, gt = _frames(rng, H, W)
    for c in range(3):
        got = vfi_oracle.ssim_channel(gt[..., c], pred[..., c])
        want = _direct_ssim_channel(gt[..., c], pred[..., c])
        assert abs(got - want) <= 1e-12, (c, got, want)
    want = np.mean([_direct_ssim_channel(gt[..., c], pred[..., c]) for c in range(3)])
    assert abs(vfi_oracle.ssim(pred, gt) - want) <= 1e-12


def test_padding_never_reaches_the_crop():
    rng = np.random.default_rng(2)
    pred, gt = _frames(rng, 23, 31)
    for c in range(3):
        a = vfi_oracle.ssim_channel(gt[..., c], pred[..., c], mode="reflect")
        b = vfi_oracle.ssim_channel(gt[..., c], pred[..., c], mode="constant")
        assert a == b, (a, b)


def test_ssim_of_a_frame_with_itself_is_one_and_psnr_of_an_offset():
    rng = np.random.default_rng(4)
    _, gt = _frames(rng, 40, 52)
    assert abs(vfi_oracle.ssim(gt, gt) - 1.0) <= 1e-15
    assert vfi_oracle.sse(gt, gt) == 0 and vfi_oracle.psnr(0, gt.size) == float("inf")
    base = rng.integers(20, 230, (40, 52, 3)).astype(np.uint8)
    for d in (1, 3, 7, 20):
        shifted = (base.astype(np.int64) + d).astype(np.uint8)  # no clipping
        s = vfi_oracle.sse(shifted, base)
        assert s == d * d * base.size
        assert abs(vfi_oracle.psnr(s, base.size) - 20 * np.log10(255 / d)) <= 1e-12
        assert vfi_oracle.ssim(shifted, base) < 1.0
    from raft_b200.evaluate import psnr
    assert psnr(np.array([0.0, 3 * 9.0 * 100]), np.array([300.0, 300.0])).tolist() == [float("inf"),
                                                                                        20 * np.log10(255 / 3)]


def test_quantisation_is_the_clis_expression():
    x = np.float32([0.0, 1.0, -0.3, 1.7, np.nan, np.inf, -np.inf, 0.5 / 255, 1.5 / 255, 2.5 / 255, 0.49999997])
    q = vfi_oracle.quantise(x)
    finite = np.isfinite(x)
    cli = np.clip(np.rint(255.0 * x[finite]), 0, 255).astype(np.uint8)  # infer_raft.py --interpolate
    assert np.array_equal(q[finite], cli)
    assert q[4] == 0 and q[5] == 255 and q[6] == 0
    # exact fp32 halves of 255 x round to even
    halves = np.float32([0.5, 1.5, 2.5, 127.5, 254.5]) / np.float32(255)
    prod = np.float32(255) * halves
    assert np.array_equal(vfi_oracle.quantise(halves), np.rint(prod).astype(np.uint8))


def _touch(path, data=b""):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(data)


def _vimeo_tree(root, entries, listing=None):
    for e in entries:
        for k in (1, 2, 3):
            _touch(os.path.join(root, "sequences", e, f"im{k}.png"))
    with open(os.path.join(root, "tri_testlist.txt"), "w") as f:
        f.write(listing if listing is not None else "\n".join(entries) + "\n")


def test_vimeo_triplets_in_list_order_and_missing_files_named(tmp_path):
    from raft_b200.evaluate import vimeo_triplets
    root = str(tmp_path)
    entries = ["00002/0001", "00001/0389", "00001/0007"]
    _vimeo_tree(root, entries, "  00002/0001\n\n00001/0389  \n\t00001/0007\n\n")
    trips = vimeo_triplets(root)
    assert [t.dir for t in trips] == entries  # list order, not sorted
    for t, e in zip(trips, entries):
        d = os.path.join(root, "sequences", e)
        assert (t.image1, t.gt, t.image2) == tuple(os.path.join(d, f"im{k}.png") for k in (1, 2, 3))
    for k in (1, 2, 3):
        p = os.path.join(root, "sequences", "00001", "0389", f"im{k}.png")
        os.remove(p)
        with pytest.raises(FileNotFoundError, match=f"00001/0389/im{k}.png"):
            vimeo_triplets(root)
        _touch(p)
    with open(os.path.join(root, "tri_testlist.txt"), "w") as f:
        f.write("\n  \n")
    with pytest.raises(FileNotFoundError, match="no triplets"):
        vimeo_triplets(root)
    os.remove(os.path.join(root, "tri_testlist.txt"))
    with pytest.raises(FileNotFoundError, match="tri_testlist.txt"):
        vimeo_triplets(root)


def test_vimeo_aggregate_and_summary_line():
    from raft_b200.evaluate import Triplet, aggregate_vimeo, summary_lines
    trips = [Triplet("a1", "a3", "a2", "00001/0001"), Triplet("b1", "b3", "b2", "00001/0002")]
    n = 3.0 * 64 * 96
    stats = np.array([[n, 4.0 * n, 0.9], [n, 25.0 * n, 0.7]])  # constant errors of 2 and 5
    r = aggregate_vimeo(trips, stats)
    p = [20 * np.log10(255 / 2), 20 * np.log10(255 / 5)]
    assert r["n_triplets"] == 2 and abs(r["psnr"] - np.mean(p)) <= 1e-12 and abs(r["ssim"] - 0.8) <= 1e-15
    assert [t["dir"] for t in r["triplets"]] == ["00001/0001", "00001/0002"]
    assert [t["mse"] for t in r["triplets"]] == [4.0, 25.0] and [t["ssim"] for t in r["triplets"]] == [0.9, 0.7]
    assert all(abs(t["psnr"] - q) <= 1e-12 for t, q in zip(r["triplets"], p))
    res = {"dataset": "vimeo", "iters": 20, "pad_mode": "sintel", "splits": {"vimeo": r}}
    assert summary_lines(res) == ["Validation Vimeo-90K: PSNR: %f, SSIM: %f" % (r["psnr"], r["ssim"])]
    assert summary_lines(res)[0].startswith("Validation Vimeo-90K: PSNR: ")
    # a perfect triplet: infinite PSNR, mse 0
    r = aggregate_vimeo(trips[:1], np.array([[n, 0.0, 1.0]]))
    assert r["psnr"] == float("inf") and r["triplets"][0]["mse"] == 0.0


def test_frame_metrics_argument_checks_before_any_cuda_call():
    from raft_b200 import capi
    lib = capi.lib
    out = ctypes.c_size_t()
    assert lib.rb_frame_metrics_workspace_bytes(2, 256, 448, ctypes.byref(out)) == 0
    assert out.value == 2 * (14 * 16) * 2 * 8  # 32 x 16 tiles, two fp64 partials each
    assert lib.rb_frame_metrics_workspace_bytes(1, 11, 11, ctypes.byref(out)) == 0 and out.value == 16
    assert lib.rb_frame_metrics_workspace_bytes(1, 11, 11, None) == -2
    for shape in ((0, 11, 11), (1, 0, 11), (1, 11, -1)):
        assert lib.rb_frame_metrics_workspace_bytes(*shape, ctypes.byref(out)) == -1
        assert b"rb_frame_metrics_workspace_bytes" in lib.rb_last_error()
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ok = dict(pr=p, u8=0, g=p, B=1, H=11, W=11, st=p, ws=p, wsb=16)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.rb_frame_metrics(a["pr"], a["u8"], a["g"], a["B"], a["H"], a["W"], a["st"], a["ws"], a["wsb"], None)

    cases = [(dict(pr=None), -2, b"null"), (dict(g=None), -2, b"null"), (dict(st=None), -2, b"null"),
             (dict(ws=None), -2, b"null"), (dict(u8=2), -2, b"pred_is_u8"), (dict(u8=-1), -2, b"pred_is_u8"),
             (dict(B=0), -1, b"bad shape"), (dict(H=0), -1, b"bad shape"), (dict(W=-2), -1, b"bad shape"),
             (dict(H=10), -1, b"11x11"), (dict(W=10), -1, b"11x11"), (dict(H=10, W=10), -1, b"11x11"),
             (dict(B=65536, wsb=1 << 30), -1, b"grid"),
             (dict(wsb=15), -5, b"workspace"), (dict(B=2, wsb=16), -5, b"workspace"),
             (dict(H=17, W=11, wsb=16), -5, b"workspace"), (dict(H=11, W=33, wsb=16), -5, b"workspace")]
    for kw, code, word in cases:
        assert call(**kw) == code, kw
        msg = lib.rb_last_error()
        assert b"rb_frame_metrics" in msg and word in msg, (kw, msg)


def test_frame_metrics_wrapper_refuses_bad_inputs_without_a_gpu():
    import torch
    from networks.utils import frame_metrics
    gt = torch.zeros(1, 16, 16, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="pred"):
        frame_metrics(torch.zeros(1, 16, 16, 3), gt)  # a host tensor
    with pytest.raises(ValueError, match="pred"):
        frame_metrics(np.zeros((1, 16, 16, 3), np.float32), gt)


def test_evaluate_refuses_warm_start_and_submit_for_vimeo():
    from types import SimpleNamespace
    from networks.RAFT import RAFT
    from raft_b200.evaluate import evaluate, submit
    m = RAFT(None, SimpleNamespace(small=False))
    with pytest.raises(ValueError, match="triplets are not chains"):
        evaluate(m, "/nonexistent", "vimeo", warm_start=True)
    with pytest.raises(ValueError, match="Vimeo-90K"):
        submit(m, "/nonexistent", "vimeo", "/nonexistent")


def test_cli_refuses_test_split_and_warm_start_for_vimeo(tmp_path):
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    for extra, words in ((["--split", "test"], "Vimeo-90K has no hidden-ground-truth split"),
                         (["--warm-start"], "Vimeo-90K's triplets are not chains")):
        r = subprocess.run([sys.executable, cli, "-m", "val", "--dataset", "vimeo", "--data", str(tmp_path)] + extra,
                           cwd=tmp_path, env=env, capture_output=True, text=True)
        assert r.returncode == 2 and words in r.stderr, (extra, r.stderr)
