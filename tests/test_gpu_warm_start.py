"""F10 warm start on the GPU: rb_flow_forward_interpolate against the fp64 oracle (tests/warm_oracle.py) bit for bit and
against upstream's scipy function where the nearest source is unique; forward(flow_init=..., return_low=True) against
the cold forward, the fp64 network oracle started from the same init, per-sample runs and the volume-free path; a warm
chain against one whose inits the oracle computes; submit() and evaluate(warm_start=True) against sequential loops of the
public API; and the CLI's --split test."""
import contextlib
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import warm_oracle
from oracle import raft_oracle as O
from test_warm_start import _upstream_nhwc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_WEIGHTS = {}


def _weights(small):
    from raft_b200 import synth
    if small not in _WEIGHTS:
        _WEIGHTS[small] = synth.make_weights(small)
    return _WEIGHTS[small]


def _bits(t):
    return np.ascontiguousarray(np.asarray(t.cpu() if isinstance(t, torch.Tensor) else t, np.float32)).view(np.int32)


def _fi(flow):
    from networks.utils import forward_interpolate
    return forward_interpolate(torch.from_numpy(np.ascontiguousarray(flow)).cuda()).cpu().numpy()


def _flows(rng, B, h, w):
    """Smooth motion plus noise; a global push moves a part of every sample's sources out of the grid."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    out = []
    for _ in range(B):
        a = rng.uniform(-3, 3, 4)
        u = a[0] + 0.2 * w * np.sin(xx / max(w, 1) * 3 + a[1]) / 4
        v = a[2] + 0.2 * h * np.cos(yy / max(h, 1) * 3 + a[3]) / 4
        out.append(np.stack([u, v], -1) + rng.normal(0, 0.7, (h, w, 2)))
    return np.stack(out).astype(np.float32)


# ---- the kernel -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(8, 8), (13, 37), (55, 128), (135, 240)])
@pytest.mark.parametrize("B", [1, 3])
def test_kernel_equals_oracle(cuda, B, h, w):
    rng = np.random.default_rng(B * 1000 + h * 7 + w)
    f = _flows(rng, B, h, w)
    f[0].reshape(-1, 2)[rng.choice(h * w, max(1, h * w // 50), replace=False), 0] = np.nan
    got = _fi(f)
    want, uniq = warm_oracle.forward_interpolate(f, return_unique=True)
    assert np.array_equal(_bits(got), _bits(want))
    if B == 1:  # upstream's scipy function wherever the nearest source is unique
        up = _upstream_nhwc(f[0])
        assert np.array_equal(got[0][uniq[0]], up[uniq[0]]) and uniq.mean() > 0.99
    for b in range(B):  # a batch gives the per-sample bits
        assert np.array_equal(_bits(_fi(f[b:b + 1])[0]), _bits(got[b]))


def test_kernel_degenerate_cases(cuda):
    h, w = 55, 128
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    none = np.full((h, w, 2), 500.0, np.float32)
    one = none.copy()
    one[40, 100] = (-77.25, -19.5)  # the only source, at (22.75, 20.5)
    cell = np.stack([10.0 + (xx * 0.37 % 1) - xx, 20.0 + (yy * 0.61 % 1) - yy], -1).astype(np.float32)  # all in cell (10, 20)
    cell[0, 0] = (500.0, 0.0)
    point = np.stack([10.25 - xx, 20.5 - yy], -1).astype(np.float32)  # every source lands at (10.25, 20.5): all tie
    f = np.stack([none, one, cell, point])
    got = _fi(f)
    assert not got[0].any()
    assert (got[1] == np.float32([-77.25, -19.5])).all()
    assert (got[3] == point[0, 0]).all()  # the lowest source index wins every tie
    assert np.array_equal(_bits(got), _bits(warm_oracle.forward_interpolate(f)))


def test_kernel_graph_replay_equals_eager(cuda):
    from networks.utils import forward_interpolate
    from raft_b200 import capi
    rng = np.random.default_rng(4)
    B, h, w = 2, 55, 128
    src = torch.from_numpy(_flows(rng, B, h, w)).cuda()
    out = torch.empty_like(src)
    n = capi.size_query(capi.lib.rb_flow_forward_interpolate_workspace_bytes, B, h, w)
    ws = torch.empty(n, dtype=torch.uint8, device=cuda)

    def call():
        capi.check(capi.lib.rb_flow_forward_interpolate(capi.ptr(src), capi.ptr(out), B, h, w, capi.ptr(ws), n,
                                                        capi.stream()))
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.Stream()):
        call()
    for seed in (5, 6):
        src.copy_(torch.from_numpy(_flows(np.random.default_rng(seed), B, h, w)))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), forward_interpolate(src).view(torch.int32))


# ---- the engine -------------------------------------------------------------------------------------------------------
def _model(small=False, iters=4, **kw):
    from networks.RAFT import RAFT
    return RAFT(None, SimpleNamespace(small=small), iters=iters, **kw).load(_weights(small))


def _frames(B, H, W, seed=1000):
    from raft_b200 import synth
    return synth.make_batch(B, H, W, seed)


def _init(rng, B, h, w, amp=1.5):
    return torch.from_numpy((amp * _flows(rng, B, h, w) / 3).astype(np.float32))


@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("kw", [{}, {"upstream": True}, {"volume_free": True}, {"mixed_precision": True}])
def test_zero_init_is_the_cold_forward(cuda, small, kw):
    l, r = _frames(2, 128, 160)
    m = _model(small, **kw)
    cold = m.forward(l, r)
    low_cold = m.engine().lowres_flow().clone()
    zeros = torch.zeros(2, 16, 20, 2)
    low, up = m.forward(l, r, flow_init=zeros, return_low=True)
    assert torch.equal(up, cold) and torch.equal(low, low_cold)
    low2, up2 = m.forward(l, r, return_low=True)  # no init: zeros
    assert torch.equal(up2, cold) and torch.equal(low2, low_cold)
    assert torch.equal(m.forward(l, r, flow_init=zeros.cuda()), cold)
    assert torch.equal(m.forward(l, r), cold)  # the cold graph is kept beside the warm one


def test_bad_flow_init_is_refused(cuda):
    l, r = _frames(1, 64, 96)
    m = _model()
    for bad in (torch.zeros(1, 8, 13, 2), torch.zeros(2, 8, 12, 2), torch.zeros(1, 8, 12, 3), torch.zeros(1, 8, 12, 2).double()):
        with pytest.raises(ValueError, match="flow_init"):
            m.forward(l, r, flow_init=bad)
    low, _ = m.forward(l, r, flow_init=np.zeros((1, 8, 12, 2), np.float32), return_low=True)
    assert low.shape == (1, 8, 12, 2)
    m = _model(input_size=(72, 100))  # the grid of input_size: 72 x 104 padded -> 9 x 13
    low, up = m.forward(*_frames(1, 64, 96), flow_init=torch.zeros(1, 9, 13, 2), return_low=True)
    assert low.shape == (1, 9, 13, 2) and up.shape == (1, 72, 100, 2)


def _oracle_warm(small, upstream, iters, l, r, init):
    """The fp64 network oracle (upstream semantics: tests/upstream_oracle.py) with coords1 = coords0 + init."""
    import upstream_oracle as U
    with (U.upstream_semantics() if upstream else contextlib.nullcontext()):
        o = O.RAFTOracle(_weights(small), small=small, iters=iters, dtype=torch.float64)
        st = o.prepare(torch.from_numpy(l), torch.from_numpy(r))
        st["coords1"] = st["coords0"] + init.double()
        _, mask, coords1 = o.iterate(st)
        low = coords1 - st["coords0"]
        return low, (O.upflow8(low) if small else O.upsample_flow(low, mask))


@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("upstream", [False, True])
def test_nonzero_init_matches_the_fp64_oracle(cuda, small, upstream):
    H, W = (128, 160) if upstream else (64, 96)
    l, r = _frames(1, H, W, 77)
    init = _init(np.random.default_rng(8), 1, H // 8, W // 8)
    m = _model(small, upstream=upstream)
    low, up = m.forward(l, r, flow_init=init, return_low=True)
    ref_low, ref_up = _oracle_warm(small, upstream, 4, l, r, init)
    assert (low.cpu().double() - ref_low).abs().max().item() < 1e-3
    assert (up.cpu().double() - ref_up).abs().max().item() < 1e-3
    assert not torch.equal(up, m.forward(l, r))  # the init matters


def test_nonzero_init_matches_the_oracle_at_20_iterations(cuda):
    l, r = _frames(1, 128, 256, 91)
    init = _init(np.random.default_rng(9), 1, 16, 32)
    _, up = _model(iters=20).forward(l, r, flow_init=init, return_low=True)
    _, ref = _oracle_warm(False, False, 20, l, r, init)
    assert (up.cpu().double() - ref).abs().max().item() < 1e-3


def test_mixed_batch_equals_per_sample_runs_and_volume_free_agrees(cuda):
    l, r = _frames(3, 128, 160, 55)
    init = _init(np.random.default_rng(10), 3, 16, 20)
    init[1] = 0
    m = _model()
    low, up = m.forward(l, r, flow_init=init, return_low=True)
    for b in range(3):
        lb, ub = m.forward(l[b:b + 1], r[b:b + 1], flow_init=init[b:b + 1], return_low=True)
        assert torch.equal(lb, low[b:b + 1]) and torch.equal(ub, up[b:b + 1])
    assert torch.equal(up[1:2], m.forward(l[1:2], r[1:2]))  # the zero row is the cold forward
    vf = _model(volume_free=True).forward(l, r, flow_init=init)
    assert (vf - up).abs().max().item() < 2e-4 * max(up.abs().max().item(), 1.0)


def test_four_frame_chain_equals_oracle_inits(cuda):
    from networks.utils import forward_interpolate
    from raft_b200 import synth
    frames = [synth.make_pair(124, 200, 300 + k)[0][None] for k in range(5)]
    m = _model(upstream=True)
    prev, gpu = None, []
    for k in range(4):
        low, up = m.forward(frames[k], frames[k + 1], flow_init=prev, return_low=True)
        gpu.append((low.cpu(), up.cpu()))
        prev = forward_interpolate(low)
    prev = None
    for k in range(4):
        low, up = m.forward(frames[k], frames[k + 1], flow_init=prev, return_low=True)
        assert torch.equal(low.cpu(), gpu[k][0]) and torch.equal(up.cpu(), gpu[k][1]), k
        prev = torch.from_numpy(warm_oracle.forward_interpolate(low.cpu().numpy()))


# ---- submit / evaluate ------------------------------------------------------------------------------------------------
SCENES = (("alley_1", 4, 124, 200), ("bamboo_2", 2, 124, 200), ("cave_4", 3, 130, 211), ("market_5", 5, 124, 200))


@pytest.fixture(scope="module")
def sintel_test_tree(tmp_path_factory):
    """Sintel's test layout: ragged scenes, one at another frame size."""
    import cv2
    from raft_b200 import synth
    root = str(tmp_path_factory.mktemp("sintel_test"))
    for i, (scene, n, H, W) in enumerate(SCENES):
        for d in ("clean", "final"):
            os.makedirs(os.path.join(root, "test", d, scene))
        for k in range(n):
            f = synth.make_pair(H, W, 500 + 10 * i + k // 2)[k % 2]
            for d in ("clean", "final"):
                img = f if d == "clean" else 0.8 * f + 0.1
                cv2.imwrite(os.path.join(root, "test", d, scene, f"frame_{k + 1:04d}.png"),
                            np.round(255 * img).astype(np.uint8))
    return root


def _files(out):
    res = {}
    for dp, _, fs in os.walk(out):
        for f in fs:
            p = os.path.join(dp, f)
            res[os.path.relpath(p, out)] = open(p, "rb").read()
    return res


def _loop(model, pairs, out, warm, write, scale=1.0):
    """The sequential reference: one RAFT.forward per pair, each scene's chain warm-started when warm."""
    from networks.utils import forward_interpolate
    from raft_b200.evaluate import _decode_frames, chains_of
    for chain in chains_of(pairs, warm):
        prev = None
        for i in chain:
            left, right = _decode_frames(pairs[i], False)
            if warm:
                low, flow = model.forward(left[None], right[None], flow_init=prev, return_low=True)
                prev = forward_interpolate(low)
            else:
                flow = model.forward(left[None], right[None])
            path = os.path.join(out, pairs[i].out)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            write(path, flow[0].cpu().numpy() * np.float32(scale))


@pytest.mark.parametrize("small", [False, True])
def test_submit_sintel_cold_and_warm(cuda, sintel_test_tree, tmp_path, small):
    from flow_utils import write_flo
    from raft_b200.evaluate import sintel_test_pairs, submit
    m = _model(small)
    scale = 8.0 if small else 1.0
    for warm in (False, True):
        runs = []
        for b, wk in ((1, 0), (3, 4), (3, 0)):
            out = str(tmp_path / f"w{warm}_b{b}_{wk}")
            files = submit(m, sintel_test_tree, "sintel", out, batch=b, workers=wk, iters=4, warm_start=warm)
            assert len(files) == 2 * sum(n - 1 for _, n, _, _ in SCENES)
            runs.append(_files(out))
        assert runs[0] == runs[1] == runs[2]
        ref = str(tmp_path / f"ref{warm}")
        for d in ("clean", "final"):
            _loop(m, sintel_test_pairs(sintel_test_tree, d), ref, warm, write_flo, scale)
        assert _files(ref) == runs[0]
        assert "clean/cave_4/frame0002.flo" in runs[0] and "final/market_5/frame0004.flo" in runs[0]
        if warm:
            assert runs[0] != cold
        cold = runs[0]


def test_submit_kitti(cuda, tmp_path):
    import cv2
    from flow_utils import write_kitti_flow
    from raft_b200 import synth
    from raft_b200.evaluate import kitti_test_pairs, submit
    root = str(tmp_path / "kitti")
    d = os.path.join(root, "testing", "image_2")
    os.makedirs(d)
    for i, (H, W) in enumerate([(124, 200), (130, 211), (124, 200)]):
        f1, f2 = synth.make_pair(H, W, 700 + i)
        for s, f in (("10", f1), ("11", f2)):
            cv2.imwrite(os.path.join(d, f"{i:06d}_{s}.png"), np.round(255 * f).astype(np.uint8))
    out = str(tmp_path / "out")
    files = submit(_model(), root, "kitti", out, batch=2, workers=2, iters=4)
    assert sorted(os.path.relpath(f, out) for f in files) == [f"{i:06d}_10.png" for i in range(3)]
    ref = str(tmp_path / "ref")
    _loop(_model(pad_mode="kitti"), kitti_test_pairs(root), ref, False, write_kitti_flow)
    assert _files(ref) == _files(out)


@pytest.fixture(scope="module")
def sintel_tree(tmp_path_factory):
    from raft_b200 import synth
    root = str(tmp_path_factory.mktemp("sintel"))
    assert synth.write_sintel_tree(root, 3, 4, 124, 200) == 9
    return root


def test_evaluate_warm_start(cuda, sintel_tree):
    from flow_utils import read_flo
    from networks.utils import flow_metrics, forward_interpolate
    from raft_b200.evaluate import aggregate, evaluate, sintel_pairs, _decode_frames
    m = _model()
    cold = evaluate(m, sintel_tree, "sintel", iters=4)
    assert evaluate(m, sintel_tree, "sintel", iters=4, warm_start=False) == cold
    runs = [evaluate(m, sintel_tree, "sintel", batch=b, workers=wk, iters=4, warm_start=True)
            for b, wk in ((1, 0), (2, 4), (3, 0))]
    assert runs[0] == runs[1] == runs[2]
    assert runs[0]["splits"]["clean"]["epe"] != cold["splits"]["clean"]["epe"]
    for d in ("clean", "final"):
        pairs = sintel_pairs(sintel_tree, d)
        stats, prev, scene = [], None, None
        for p in pairs:
            if os.path.dirname(p.image1) != scene:
                prev, scene = None, os.path.dirname(p.image1)
            left, right = _decode_frames(p, False)
            low, flow = m.forward(left[None], right[None], flow_init=prev, return_low=True)
            prev = forward_interpolate(low)
            stats.append(flow_metrics(flow, torch.from_numpy(read_flo(p.gt))[None].cuda())[0].cpu().numpy())
        assert runs[0]["splits"][d] == aggregate(pairs, np.stack(stats), False)


def test_cli_split_test_writes_the_api_files(cuda, sintel_test_tree, tmp_path):
    from raft_b200.evaluate import submit
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    out = tmp_path / "cli"
    cli = [sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "-m", "val", "--split", "test",
           "--dataset", "sintel", "--data", sintel_test_tree, "--out", str(out), "--load", npz, "--iters", "4",
           "--batch", "2", "--warm-start"]
    subprocess.run(cli, cwd=tmp_path, env=dict(os.environ, PYTHONNOUSERSITE="1"), capture_output=True, text=True,
                   check=True)
    api = str(tmp_path / "api")
    submit(_model(), sintel_test_tree, "sintel", api, iters=4, warm_start=True)
    assert _files(str(out)) == _files(api) and len(_files(api)) == 20
