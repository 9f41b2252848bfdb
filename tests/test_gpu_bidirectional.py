"""F5: bidirectional flow with the forward-backward occlusion check.

rb_flow_fb_check must equal the fp32 numpy restatement (tests/fb_oracle.py) bit for bit; forward_bidirectional must give
forward(L, R) and forward(R, L) bit for bit on every engine path, masks equal to the restatement applied to the returned
flows, fresh results when it alternates with forward on one engine, and share the feature encoder between directions."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from fb_oracle import fb_check

pytestmark = pytest.mark.gpu


def _flows(rng, B, H, W, nan=0):
    fw = rng.uniform(-0.3, 0.3, (B, H, W, 2)) * np.array([W, H])  # many targets leave the frame
    bw = -fw + rng.normal(0, 0.6, fw.shape)
    fw, bw = fw.astype(np.float32), bw.astype(np.float32)
    for f in (fw, bw):
        for _ in range(nan):
            f[rng.integers(B), rng.integers(H), rng.integers(W), rng.integers(2)] = np.nan
    return fw, bw


@pytest.mark.parametrize("B,H,W,scale,alphas", [(3, 37, 53, 1.0, (0.01, 0.5)), (3, 37, 53, 8.0, (0.01, 0.5)),
                                                (2, 61, 97, 1.0, (0.05, 0.1)), (2, 1, 31, 1.0, (0.01, 0.5)),
                                                (2, 29, 1, 1.0, (0.01, 0.5)), (1, 1, 1, 1.0, (0.01, 0.5))])
def test_kernel_equals_fp32_restatement_bit_for_bit(cuda, B, H, W, scale, alphas):
    from networks.utils import fb_consistency
    rng = np.random.default_rng(B * 1000 + H * 10 + W)
    fw, bw = _flows(rng, B, H, W, nan=3 if H * W > 1 else 0)
    if scale != 1.0:
        fw, bw = fw / np.float32(scale), bw / np.float32(scale)
    ref = fb_check(fw, bw, *alphas, flow_scale=scale)
    got = fb_consistency(torch.from_numpy(fw).to(cuda), torch.from_numpy(bw).to(cuda), *alphas, flow_scale=scale)
    for r, g in zip(ref, got):
        assert g.dtype == torch.uint8 and tuple(g.shape) == (B, H, W)
        g = g.cpu().numpy()
        assert np.array_equal(r, g), f"{(r != g).sum()} of {r.size} pixels differ"
    if H * W > 1000:
        assert all((ref[0] == k).any() for k in (0, 1, 2))


def _model(p, small, H, W, B, cuda, volume_free=None, graph=True, simt=False):
    from raft_b200 import capi
    from networks.RAFT import RAFT
    m = RAFT((H, W, 3), SimpleNamespace(small=small), iters=4, batch=B, device=cuda, volume_free=volume_free).load(p)
    eng = m.engine()
    eng.use_graph = graph
    if simt:
        eng.math_mode = capi.RB_MATH_SIMT
    return m


def _frames(B, H, W, u8):
    from raft_b200 import synth
    l, r = synth.make_batch(B, H, W)
    if u8:
        l, r = (np.round(l * 255).astype(np.uint8), np.round(r * 255).astype(np.uint8))
    return l, r


def _check_bidirectional(cuda, small, B, H, W, u8=False, volume_free=None, graph=True, simt=False):
    from raft_b200 import synth
    p = synth.make_weights(small)
    l, r = _frames(B, H, W, u8)
    mf = _model(p, small, H, W, B, cuda, volume_free, graph, simt)
    fw_ref, bw_ref = mf.forward(l, r), mf.forward(r, l)
    mb = _model(p, small, H, W, B, cuda, volume_free, graph, simt)
    fw, bw, ofw, obw = mb.forward_bidirectional(l, r)
    assert fw.shape == bw.shape == (B, H, W, 2) and ofw.shape == obw.shape == (B, H, W) and ofw.dtype == torch.uint8
    assert torch.equal(fw, fw_ref), (fw - fw_ref).abs().max().item()
    assert torch.equal(bw, bw_ref), (bw - bw_ref).abs().max().item()
    ref = fb_check(fw.cpu().numpy(), bw.cpu().numpy(), flow_scale=8.0 if small else 1.0)
    assert np.array_equal(ofw.cpu().numpy(), ref[0]) and np.array_equal(obw.cpu().numpy(), ref[1])
    # without the check: the same flows, no masks
    fw2, bw2, o1, o2 = mb.forward_bidirectional(l, r, check=False)
    assert o1 is None and o2 is None and torch.equal(fw2, fw) and torch.equal(bw2, bw)
    return fw, bw, ofw, obw


@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("B,H,W", [(1, 64, 96), (2, 64, 96), (1, 60, 100), (2, 60, 100)])
def test_flows_equal_forward_both_ways(cuda, small, B, H, W):
    _check_bidirectional(cuda, small, B, H, W)


@pytest.mark.parametrize("small", [False, True])
def test_uint8_frames(cuda, small):
    _check_bidirectional(cuda, small, 2, 60, 100, u8=True)


@pytest.mark.parametrize("small", [False, True])
def test_volume_free(cuda, small):
    _check_bidirectional(cuda, small, 2, 64, 96, volume_free=True)


def test_simt_back_end(cuda):
    _check_bidirectional(cuda, False, 1, 64, 96, graph=False, simt=True)


def test_eager_equals_graph(cuda):
    a = _check_bidirectional(cuda, False, 2, 60, 100, graph=False)
    b = _check_bidirectional(cuda, False, 2, 60, 100, graph=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_full_size(cuda):
    """436x1024 (padded to 440): the full-size pyramid at 2B pairs."""
    _check_bidirectional(cuda, False, 1, 436, 1024)


def test_alternating_modes_give_fresh_results(cuda):
    """forward and forward_bidirectional each keep their buffers and graph on one engine: results of an alternating
    sequence (different frames on every call) equal those of fresh models."""
    from raft_b200 import synth
    small, B, H, W = False, 1, 60, 100
    p = synth.make_weights(small)
    frames = [synth.make_batch(B, H, W, seed0=s) for s in (2000, 2100, 2200, 2300, 2400)]
    calls = [("f", frames[0]), ("b", frames[1]), ("f", frames[2]), ("b", frames[3]), ("n", frames[4]), ("b", frames[0])]

    def call(m, kind, lr):
        if kind == "f":
            return (m.forward(*lr),)
        return m.forward_bidirectional(*lr, check=kind == "b")

    one = _model(p, small, H, W, B, cuda)
    for kind, lr in calls:
        got = call(one, kind, lr)
        want = call(_model(p, small, H, W, B, cuda), kind, lr)
        for g, w in zip(got, want):
            assert (g is None and w is None) or torch.equal(g, w), kind


def test_feature_encoder_runs_once_per_pass(cuda):
    from raft_b200 import synth
    small, B, H, W = False, 2, 64, 96
    p = synth.make_weights(small)
    l, r = synth.make_batch(B, H, W)
    m = _model(p, small, H, W, B, cuda, graph=False)
    eng = m.engine()
    seen = []

    def counting(enc, name):
        def call(x, *a, **k):
            seen.append((name, x.shape[0]))
            return enc(x, *a, **k)
        return call

    eng.fnet, eng.cnet_bidir = counting(eng.fnet, "fnet"), counting(eng.cnet_bidir, "cnet")
    m.forward_bidirectional(l, r)
    assert seen == [("cnet", 2 * B), ("fnet", 2 * B)] or seen == [("fnet", 2 * B), ("cnet", 2 * B)], seen
    n_bidir = eng.launches_per_forward()
    m.forward(l, r)
    n_fwd = eng.launches_per_forward()
    assert n_bidir == n_fwd + 1, (n_bidir, n_fwd)  # + rb_flow_fb_check; the fmap copy is a memcpy, not a kernel


def test_cli_bidirectional(cuda, tmp_path, monkeypatch):
    import cv2
    import infer_raft
    from raft_b200 import synth
    l, r = synth.make_batch(1, 60, 100)
    for name, img in (("a.png", l[0]), ("b.png", r[0])):
        cv2.imwrite(str(tmp_path / name), (img * 255).astype(np.uint8))
    p = synth.make_weights(False)
    np.savez(tmp_path / "w.npz", **p)
    monkeypatch.chdir(tmp_path)
    base = ["--im1", "a.png", "--im2", "b.png", "--load", "w.npz", "--iters", "3", "--keep-size"]
    assert infer_raft.main(base + ["--npy", "plain.npy"]) == 0
    assert not os.path.exists("raft_occ_fw.png") and not os.path.exists("plain_bw.npy")
    assert infer_raft.main(base + ["--bidirectional", "--npy", "f.npy", "--flo", "f.flo"]) == 0
    for f in ("raft_flow_raft-things.png", "raft_flow_raft-things_bw.png", "raft_occ_fw.png", "raft_occ_bw.png",
              "f_bw.npy", "f.flo", "f_bw.flo"):
        assert os.path.exists(f), f
    fw, bw = np.load("f.npy"), np.load("f_bw.npy")
    assert np.array_equal(fw, np.load("plain.npy")) and fw.shape == bw.shape == (60, 100, 2)
    occ = cv2.imread("raft_occ_fw.png", cv2.IMREAD_UNCHANGED)
    ref = fb_check(fw[None], bw[None])[0][0]
    assert occ.shape == (60, 100) and np.array_equal(occ, np.array([0, 128, 255], np.uint8)[ref])
