"""F10 warm start, host side (no GPU): the fp64 forward_interpolate oracle against upstream's scipy griddata function,
the warm start on the CPU oracle of the network, the KITTI flow writer, the test-split enumeration, the lockstep chain
scheduler, the argument checks of the new C entry points (before any CUDA call) and the CLI's new flags."""
import ctypes
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import warm_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def upstream_forward_interpolate(flow):
    """upstream RAFT core/utils/utils.py forward_interpolate on a [2,h,w] float32 numpy flow (the .cpu().numpy() and
    torch.from_numpy(...).float() around it replaced by numpy)."""
    from scipy import interpolate
    dx, dy = flow[0], flow[1]
    ht, wd = dx.shape
    x0, y0 = np.meshgrid(np.arange(wd), np.arange(ht))
    x1 = x0 + dx
    y1 = y0 + dy
    x1 = x1.reshape(-1)
    y1 = y1.reshape(-1)
    dx = dx.reshape(-1)
    dy = dy.reshape(-1)
    valid = (x1 > 0) & (x1 < wd) & (y1 > 0) & (y1 < ht)
    x1 = x1[valid]
    y1 = y1[valid]
    dx = dx[valid]
    dy = dy[valid]
    flow_x = interpolate.griddata((x1, y1), dx, (x0, y0), method='nearest', fill_value=0)
    flow_y = interpolate.griddata((x1, y1), dy, (x0, y0), method='nearest', fill_value=0)
    flow = np.stack([flow_x, flow_y], axis=0)
    return flow.astype(np.float32)


def _upstream_nhwc(flow):
    with np.errstate(invalid="ignore"):
        return upstream_forward_interpolate(np.ascontiguousarray(flow.transpose(2, 0, 1))).transpose(1, 2, 0)


def _flow(rng, h, w, scale, nan=0):
    f = (rng.normal(0, scale, (h, w, 2))).astype(np.float32)
    if nan:
        f.reshape(-1, 2)[rng.choice(h * w, nan, replace=False), rng.integers(0, 2)] = np.nan
    return f


@pytest.mark.parametrize("h,w", [(1, 1), (5, 7), (8, 8), (13, 17), (24, 31), (55, 128)])
@pytest.mark.parametrize("scale,nan", [(2.0, 0), (40.0, 0), (3.0, 7)])
def test_oracle_equals_upstream_griddata(h, w, scale, nan):
    rng = np.random.default_rng(h * 1000 + w + int(scale) + nan)
    f = _flow(rng, h, w, scale, nan if h * w > nan else 0)
    with np.errstate(invalid="ignore"):
        n_valid = np.sum((np.arange(w)[None] + f[..., 0] > 0) & (np.arange(w)[None] + f[..., 0] < w)
                         & (np.arange(h)[:, None] + f[..., 1] > 0) & (np.arange(h)[:, None] + f[..., 1] < h))
    got, uniq = warm_oracle.forward_interpolate(f, return_unique=True)
    if n_valid == 0:  # upstream's griddata raises on an empty point set; the oracle returns zeros
        assert not got.any()
        return
    want = _upstream_nhwc(f)
    assert uniq.all()  # continuous random flows: no ties
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("h,w", [(6, 9), (16, 16), (21, 34)])
def test_oracle_equals_upstream_where_the_nearest_source_is_unique_on_ties(h, w):
    rng = np.random.default_rng(h + w)
    f = rng.integers(-2, 3, (h, w, 2)).astype(np.float32)  # integer targets: many equidistant sources
    f.reshape(-1, 2)[rng.choice(h * w, h * w // 4, replace=False)] += np.float32(0.5)
    got, uniq = warm_oracle.forward_interpolate(f, return_unique=True)
    want = _upstream_nhwc(f)
    assert 0 < uniq.sum() < h * w
    assert np.array_equal(got[uniq], want[uniq])
    assert set(map(tuple, got.reshape(-1, 2))) <= set(map(tuple, f.reshape(-1, 2)))  # every output is some source's flow


def test_oracle_tie_rule_and_no_valid_source():
    f = np.zeros((3, 4, 2), np.float32)
    f[..., 0] = 100.0  # every source leaves the frame
    assert not warm_oracle.forward_interpolate(f).any()
    f[1, 1] = (0.5, 0.0)   # lands at (1.5, 1): equidistant from grid x = 1 and x = 2
    f[1, 2] = (-0.5, 0.0)  # lands at (1.5, 1) as well: the lower index (1, 1) wins everywhere
    out = warm_oracle.forward_interpolate(f)
    assert (out == np.float32([0.5, 0.0])).all()
    f[0, 0] = (0.0, 0.0)  # x1 = 0 is not > 0: still invalid
    assert (warm_oracle.forward_interpolate(f) == out).all()
    b = warm_oracle.forward_interpolate(np.stack([f, np.full_like(f, 50.0)]))
    assert (b[0] == out).all() and not b[1].any()


def test_zero_init_on_the_cpu_oracle_is_the_cold_forward():
    from oracle.raft_oracle import RAFTOracle
    from raft_b200 import synth
    for small in (False, True):
        o = RAFTOracle(synth.make_weights(small), small=small, iters=2)
        l, r = (torch.from_numpy(x) for x in synth.make_batch(1, 64, 96))
        cold_up, cold_low = o.forward(l, r, return_lowres=True)
        st = o.prepare(l, r)
        st["coords1"] = st["coords0"] + torch.zeros_like(st["coords0"])
        _, _, coords1 = o.iterate(st)
        assert torch.equal(coords1 - st["coords0"], cold_low)
        st = o.prepare(l, r)
        st["coords1"] = st["coords0"] + torch.full_like(st["coords0"], 0.75)
        _, _, warm = o.iterate(st)
        assert not torch.equal(warm - st["coords0"], cold_low)


def upstream_write_flow_kitti(filename, uv):
    """upstream RAFT core/utils/frame_utils.py writeFlowKITTI."""
    import cv2
    uv = 64.0 * uv + 2**15
    valid = np.ones([uv.shape[0], uv.shape[1], 1])
    uv = np.concatenate([uv, valid], axis=-1).astype(np.uint16)
    cv2.imwrite(filename, uv[..., ::-1])


def test_write_kitti_flow_is_upstreams_bytes_and_round_trips(tmp_path):
    from flow_utils import read_kitti_flow, write_kitti_flow
    rng = np.random.default_rng(3)
    for H, W in ((5, 7), (37, 121)):
        flow = rng.uniform(-300, 300, (H, W, 2)).astype(np.float32)
        a, b = str(tmp_path / f"a{H}.png"), str(tmp_path / f"b{H}.png")
        write_kitti_flow(a, flow)
        upstream_write_flow_kitti(b, flow)
        assert open(a, "rb").read() == open(b, "rb").read()
        q = (np.round(flow * 64) / 64).astype(np.float32)  # on KITTI's 1/64 grid the round trip is exact
        write_kitti_flow(a, q)
        back, valid = read_kitti_flow(a)
        assert np.array_equal(back, q) and valid.all()
    with pytest.raises(ValueError):
        write_kitti_flow(str(tmp_path / "c.png"), np.zeros((4, 4, 3), np.float32))


def _touch(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "wb").close()


def test_sintel_test_pairs_layout_and_naming(tmp_path):
    from raft_b200.evaluate import chains_of, sintel_test_pairs
    root = str(tmp_path)
    for d in ("clean", "final"):
        for scene, n in (("market_1", 3), ("ambush_1", 4), ("cave_3", 2)):
            for k in range(1, n + 1):
                _touch(os.path.join(root, "test", d, scene, f"frame_{k:04d}.png"))
    for d in ("clean", "final"):
        pairs = sintel_test_pairs(root, d)
        got = [(os.path.relpath(p.image1, root), os.path.relpath(p.image2, root), p.out) for p in pairs]
        want = [(f"test/{d}/{s}/frame_{k:04d}.png", f"test/{d}/{s}/frame_{k + 1:04d}.png", f"{d}/{s}/frame{k:04d}.flo")
                for s, n in (("ambush_1", 4), ("cave_3", 2), ("market_1", 3)) for k in range(1, n)]
        assert got == want
        assert chains_of(pairs, True) == [[0, 1, 2], [3], [4, 5]]
        assert chains_of(pairs, False) == [[i] for i in range(6)]
    with pytest.raises(FileNotFoundError):
        sintel_test_pairs(str(tmp_path / "none"), "clean")
    with pytest.raises(ValueError):
        sintel_test_pairs(root, "albedo")


def test_kitti_test_pairs_layout_and_naming(tmp_path):
    from raft_b200.evaluate import kitti_test_pairs
    root = str(tmp_path)
    for i in (3, 0, 1):
        for s in ("10", "11"):
            _touch(os.path.join(root, "testing", "image_2", f"{i:06d}_{s}.png"))
    pairs = kitti_test_pairs(root)
    assert [(os.path.basename(p.image1), os.path.basename(p.image2), p.out) for p in pairs] == \
        [(f"{i:06d}_10.png", f"{i:06d}_11.png", f"{i:06d}_10.png") for i in (0, 1, 3)]
    os.remove(os.path.join(root, "testing", "image_2", "000001_11.png"))
    with pytest.raises(FileNotFoundError, match="000001_11.png"):
        kitti_test_pairs(root)


@pytest.mark.parametrize("lengths", [[5, 1, 3, 7, 2, 2, 4], [1], [3, 3, 3], [6, 0, 2, 1]])
def test_lockstep_schedule(lengths):
    from raft_b200.evaluate import warm_schedule
    inits = None
    for batch in range(1, len(lengths) + 3):
        steps = warm_schedule(lengths, batch)
        B = min(batch, len(lengths))
        assert all(len(row) == B for row in steps)
        ran = [e for row in steps for e in row if e is not None]
        assert sorted(ran) == [(c, k) for c, n in enumerate(lengths) for k in range(n)]  # every pair exactly once
        init = {}
        for t, row in enumerate(steps):
            for i, e in enumerate(row):
                if e is None:
                    continue
                c, k = e
                if k == 0:
                    init[e] = None  # a chain starts cold
                else:  # warm: from the same chain's previous pair, run in the same slot one step before
                    assert steps[t - 1][i] == (c, k - 1)
                    init[e] = (c, k - 1)
        inits = inits or init
        assert init == inits  # the pair -> init mapping does not depend on the batch size
    assert warm_schedule([], 4) == []


def test_new_entry_points_refuse_bad_arguments_before_any_cuda_call():
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG, WORKSPACE = -1, -2, -5
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def refused(rc, code, word):
        assert rc == code, (rc, code)
        assert word in lib.rb_last_error(), lib.rb_last_error()

    need = capi.size_query(lib.rb_flow_forward_interpolate_workspace_bytes, 2, 5, 7)
    assert need > 0 and capi.size_query(lib.rb_flow_forward_interpolate_workspace_bytes, 4, 5, 7) >= need
    fi = lib.rb_flow_forward_interpolate
    refused(fi(None, p, 2, 5, 7, p, need, None), BAD_ARG, b"rb_flow_forward_interpolate")
    refused(fi(p, None, 2, 5, 7, p, need, None), BAD_ARG, b"null")
    refused(fi(p, p, 2, 5, 7, None, need, None), BAD_ARG, b"null")
    for B, h, w in ((0, 5, 7), (2, 0, 7), (2, 5, -1), (1 << 16, 1 << 8, 1 << 7)):
        refused(fi(p, p, B, h, w, p, need, None), BAD_SHAPE, b"rb_flow_forward_interpolate")
    refused(fi(p, p, 2, 5, 7, p, need - 1, None), WORKSPACE, b"workspace")
    out = ctypes.c_size_t()
    refused(lib.rb_flow_forward_interpolate_workspace_bytes(1 << 16, 1 << 8, 1 << 7, ctypes.byref(out)), BAD_SHAPE, b"2^31")
    refused(lib.rb_flow_forward_interpolate_workspace_bytes(1, 2, 2, None), BAD_ARG, b"null")
    refused(lib.rb_coords_init(None, p, 1, 2, 2, None), BAD_ARG, b"rb_coords_init")
    refused(lib.rb_coords_init(p, None, 0, 2, 2, None), BAD_SHAPE, b"rb_coords_init")
    refused(lib.rb_coords_to_flow(p, None, 1, 2, 2, None), BAD_ARG, b"rb_coords_to_flow")
    refused(lib.rb_coords_to_flow(p, p, 1 << 16, 1 << 8, 1 << 7, None), BAD_SHAPE, b"rb_coords_to_flow")


def test_cli_split_and_warm_start_flags(tmp_path):
    import infer_raft
    a = infer_raft.parser().parse_args(["-m", "val", "--dataset", "sintel", "--data", "x"])
    assert a.split == "training" and a.warm_start is False
    a = infer_raft.parser().parse_args(["-m", "val", "--split", "test", "--warm-start", "--dataset", "sintel"])
    assert a.split == "test" and a.warm_start is True
    with pytest.raises(SystemExit):
        infer_raft.parser().parse_args(["--split", "validation"])
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    r = subprocess.run([sys.executable, cli, "-m", "val", "--dataset", "kitti", "--data", str(tmp_path), "--warm-start"],
                       cwd=tmp_path, env=dict(os.environ, PYTHONNOUSERSITE="1"), capture_output=True, text=True)
    assert r.returncode == 2 and "--warm-start" in r.stderr, r.stderr


def test_kitti_warm_start_is_refused_without_a_gpu():
    from networks.RAFT import RAFT
    from raft_b200.evaluate import evaluate, submit
    m = RAFT(None, SimpleNamespace(small=False))
    with pytest.raises(ValueError, match="warm_start"):
        evaluate(m, "/nonexistent", "kitti", warm_start=True)
    with pytest.raises(ValueError, match="warm_start"):
        submit(m, "/nonexistent", "kitti", "/nonexistent-out", warm_start=True)
