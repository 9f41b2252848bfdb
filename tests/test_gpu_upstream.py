"""RB_SEMANTICS_UPSTREAM on the GPU: the lookup entry points bit for bit against the fp32 restatement of the sampler
(tests/upstream_oracle.py) and against F.grid_sample on CUDA, the strided convs and encoders against PyTorch's padding, and
RAFT(..., upstream=True) end to end on weights that went through raft_b200.convert."""
import contextlib
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import upstream_oracle as U
from oracle import raft_oracle as O
from test_upstream_crosscheck import Upstream, UpstreamSmall

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def _upstream(on=True):
    from raft_b200 import capi
    capi.check(capi.lib.rb_set_semantics(capi.RB_SEMANTICS_UPSTREAM if on else capi.RB_SEMANTICS_REFERENCE))
    try:
        yield
    finally:
        capi.lib.rb_set_semantics(capi.RB_SEMANTICS_REFERENCE)


def _coords(B, h, w, seed):
    """Random coordinates and every border case: -1, 0, W-1, W, fractional negatives, +-1e4, NaN, and values just below
    integers (fl(c + d) rounding up across an integer: the `far` slack row of the materialised lookup)."""
    g = torch.Generator().manual_seed(seed)
    c = O.coords_grid(B, h, w) + (torch.rand(B, h, w, 2, generator=g) * 2 - 1) * 8.0
    below = lambda v: float(np.nextafter(np.float32(v), np.float32(0)))  # noqa: E731
    special = [(-1.0, -1.0), (0.0, 0.0), (w - 1.0, h - 1.0), (float(w), float(h)), (-0.75, -0.25), (-3.5, 2.0), (1e4, 3.0),
               (-1e4, -1e4), (float("nan"), 4.0), (5.0, float("nan")), (below(16.0), below(16.0)), (below(8.0), below(12.0)),
               (10.5, below(8.0)), (w + 3.25, h + 2.5), (-8.5, -6.0)]
    for k, (x, y) in enumerate(special):
        c[k % B, k // w, k % w] = torch.tensor([x, y])
    return c.contiguous()


def _pyramid_buffer(B, h, w, seed):
    """A random pyramid in the library's layout (levels concatenated, +64 floats of tail padding) and its host levels."""
    g = torch.Generator().manual_seed(seed)
    levels = [torch.randn(B * h * w, h >> l, w >> l, 1, generator=g) for l in range(4)]
    return torch.cat([p.reshape(-1) for p in levels] + [torch.zeros(64)]), levels


CASES = [(3, 16, 32, 4), (3, 17, 30, 3), (1, 55, 128, 4), (2, 18, 22, 4), (3, 21, 19, 3)]  # w_l % 4 != 0 -> plain loads


@pytest.mark.parametrize("B,h,w,r", CASES)
def test_materialised_lookup_is_the_fp32_restatement(cuda, B, h, w, r):
    from raft_b200 import capi
    lib = capi.lib
    buf, levels = _pyramid_buffer(B, h, w, 100 + h)
    coords = _coords(B, h, w, 7)
    ref = U.sample_corr_up(levels, coords, radius=r)
    K = (2 * r + 1) ** 2
    bd, cd = buf.to(cuda), coords.to(cuda)
    out = torch.empty(B, h, w, 4 * K, device=cuda)
    with _upstream():
        capi.check(lib.rb_corr_lookup(capi.ptr(bd), capi.ptr(cd), capi.ptr(out), B, h, w, r, capi.stream()))
    out = out.cpu()
    bad = ~((out == ref) | (torch.isnan(out) & torch.isnan(ref)))
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} taps differ, max {(out - ref).abs().max():.3e}"
    # the split form of the update block (rb_update_lookup) and the fused loop's lookup read the same kernel with SPLIT
    wsb = capi.size_query(lib.rb_update_workspace_bytes, int(r == 3), B, h, w)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
    with _upstream():
        capi.check(lib.rb_update_lookup(int(r == 3), capi.ptr(ws), capi.ptr(bd), capi.ptr(cd), B, h, w, capi.stream()))
    torch.cuda.synchronize()
    npix, pad = B * h * w, (4 * K + 63) // 64 * 64
    plane = (npix * pad * 2 + 1023) // 1024 * 1024
    hi = ws[:npix * pad * 2].view(torch.float16).view(npix, pad).float().cpu()
    lo = ws[plane:plane + npix * pad * 2].view(torch.float16).view(npix, pad).float().cpu()
    rec = (hi + lo / 2048.0)[:, :4 * K].reshape(B, h, w, 4 * K)
    err = (rec - ref).abs() / ref.abs().clamp_min(1e-2)
    assert err.max() < 2 ** -20, err.max()
    # the reference sampler did not leak: the same call without the selector is today's lookup
    ref_tf = O.sample_corr(levels, torch.nan_to_num(coords), radius=r)
    out_tf = torch.empty(B, h, w, 4 * K, device=cuda)
    capi.check(lib.rb_corr_lookup(capi.ptr(bd), capi.ptr(torch.nan_to_num(cd)), capi.ptr(out_tf), B, h, w, r, capi.stream()))
    assert torch.equal(out_tf.cpu(), ref_tf)


@pytest.mark.parametrize("B,h,w,r", [(3, 16, 32, 4), (1, 55, 128, 4), (3, 21, 19, 3)])
def test_lookup_matches_grid_sample_on_cuda(cuda, B, h, w, r):
    """The engine's own pyramid levels through F.grid_sample on CUDA (grid normalised in fp32 on the host, true division)."""
    from raft_b200 import capi
    buf, levels = _pyramid_buffer(B, h, w, 200 + w)
    coords = _coords(B, h, w, 9)
    K = (2 * r + 1) ** 2
    out = torch.empty(B, h, w, 4 * K, device=cuda)
    with _upstream():
        capi.check(capi.lib.rb_corr_lookup(capi.ptr(buf.to(cuda)), capi.ptr(coords.to(cuda)), capi.ptr(out), B, h, w, r,
                                           capi.stream()))
    d = torch.arange(-r, r + 1, dtype=torch.float32)
    c = coords.reshape(-1, 1, 1, 2)
    res, res_lit = [], []
    for l, vol in enumerate(levels):
        hl, wl = vol.shape[1:3]
        x, y = torch.broadcast_tensors(c[..., 0] / 2 ** l + d[:, None], c[..., 1] / 2 ** l + d[None, :])  # [N, i, j]: i walks x
        grid = torch.stack([2 * x / torch.tensor(wl - 1.0) - 1, 2 * y / torch.tensor(hl - 1.0) - 1], -1)
        vc = vol.permute(0, 3, 1, 2).to(cuda)
        res.append(F.grid_sample(vc, grid.to(cuda), mode="bilinear", padding_mode="zeros", align_corners=True).reshape(B, h, w, -1))
        xc, yc = x.to(cuda), y.to(cuda)  # upstream's literal expression, evaluated on CUDA
        gl = torch.stack([2 * xc / (wl - 1) - 1, 2 * yc / (hl - 1) - 1], -1)
        res_lit.append(F.grid_sample(vc, gl, mode="bilinear", padding_mode="zeros", align_corners=True).reshape(B, h, w, -1))
    gs, gl = torch.cat(res, -1), torch.cat(res_lit, -1)
    fin = torch.isfinite(coords).all(-1, keepdim=True).to(cuda)
    e = ((out - gs).abs() * fin).nan_to_num(0).max().item()
    e_lit = ((out - gl).abs() * fin).nan_to_num(0).max().item()
    scale = max(p.abs().max().item() for p in levels)
    print(f"\nmax |lookup - grid_sample| = {e:.3e} (literal 2x/(W-1)-1 on CUDA: {e_lit:.3e}), scale {scale:.2f}")
    # Measured on an H100 with torch 2.11: e is one ulp of the volume (PyTorch's compiled kernel rounds one step differently
    # from the stated sampler); the literal expression is further off because CUDA torch divides by a Python scalar as a
    # multiplication by its fp32 reciprocal, which moves ix by an ulp and the weights by ~1e-5 of the volume.
    assert e <= 1e-6 * scale and e_lit <= 1e-4 * scale


@pytest.mark.parametrize("B,h,w,C,r", [(3, 16, 32, 256, 4), (2, 17, 30, 128, 3), (1, 55, 128, 256, 4)])
def test_volume_free_lookup_matches_materialised_in_upstream_mode(cuda, B, h, w, C, r):
    from raft_b200 import capi
    from networks.model_utils import GetCorrPyramid
    lib = capi.lib
    g = torch.Generator().manual_seed(31)
    f1, f2 = (torch.randn(B, h, w, C, generator=g).to(cuda) for _ in range(2))
    coords = _coords(B, h, w, 11)
    coords = torch.nan_to_num(coords, nan=3.0).to(cuda)
    K = (2 * r + 1) ** 2
    with _upstream():
        pyr = GetCorrPyramid(f1, f2)
        ref = U.sample_corr_up([p.cpu() for p in pyr], coords.cpu(), radius=r)
        wsb = capi.size_query(lib.rb_corr_otf_workspace_bytes, B, h, w, C)
        ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
        out = torch.empty(B, h, w, 4 * K, device=cuda)
        capi.check(lib.rb_corr_otf_prepare(capi.ptr(f2), capi.ptr(ws), wsb, B, h, w, C, capi.stream()))
        capi.check(lib.rb_corr_otf_lookup(capi.ptr(f1), capi.ptr(f2), capi.ptr(ws), capi.ptr(coords), capi.ptr(out), B, h, w, C,
                                          r, capi.stream()))
    out = out.cpu()
    scale = ref.abs().max().item()
    assert (out - ref).abs().max().item() < 2e-4 * scale
    assert ((out == 0) == (ref == 0)).float().mean() > 0.999  # the same taps are zero padding


def _nchw(t):
    return t.permute(0, 3, 1, 2)


@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("k,cin,cout,H,W", [(3, 64, 96, 32, 48), (1, 64, 96, 32, 48), (7, 3, 64, 40, 56), (3, 24, 24, 30, 18)])
def test_conv2d_strided_pads_like_pytorch(cuda, mode, k, cin, cout, H, W):
    from raft_b200 import capi
    lib = capi.lib
    g = torch.Generator().manual_seed(41)
    x = torch.randn(2, H, W, cin, generator=g)
    Wt = torch.randn(k, k, cin, cout, generator=g) / (k * k * cin) ** 0.5
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(_nchw(x).double(), Wt.permute(3, 2, 0, 1).double(), b.double(), stride=2, padding=k // 2).permute(0, 2, 3, 1)
    wsb = capi.size_query(lib.rb_conv2d_workspace_bytes, 2, H, W, cin, cout, k, k)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
    xd = x.to(cuda)
    y = torch.empty(2, (H + 1) // 2, (W + 1) // 2, cout, device=cuda)
    Wc, bc = np.ascontiguousarray(Wt.numpy()), np.ascontiguousarray(b.numpy())
    capi.check(lib.rb_set_math_mode(capi.RB_MATH_TC if mode == "tc" else capi.RB_MATH_SIMT))
    try:
        with _upstream():
            capi.check(lib.rb_conv2d_strided(capi.ptr(xd), Wc.ctypes.data, bc.ctypes.data, capi.ptr(y), 2, H, W, cin, cout, k, k,
                                             2, 0, capi.ptr(ws), wsb, capi.stream()))
    finally:
        lib.rb_set_math_mode(capi.RB_MATH_TC)
    err = (y.cpu().double() - ref).abs().max().item()
    assert err < 2e-5 * max(ref.abs().max().item(), 1.0), err


@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("mode", ["tc", "simt"])
def test_encoders_pad_like_pytorch(cuda, small, mode):
    from raft_b200 import capi, synth
    from raft_b200.encoders import CudaEncoder
    p = synth.make_weights(small)
    H, W = 96, 128  # even at every strided conv
    x = torch.rand(2, H, W, 3, generator=torch.Generator().manual_seed(5))
    pt = {k: torch.from_numpy(v).double() for k, v in p.items()}
    fdim = 128 if small else 256
    enc = (O.small_encoder if small else O.basic_encoder)
    with U.upstream_semantics():
        ref = enc(2 * x.double() - 1, pt, "fnet", "instance")
    capi.check(capi.lib.rb_set_math_mode(capi.RB_MATH_TC if mode == "tc" else capi.RB_MATH_SIMT))
    try:
        with torch.cuda.device(cuda), _upstream():
            e = CudaEncoder(p, "fnet", small, "instance", fdim, cuda)
            out = torch.empty(2, H // 8, W // 8, fdim, device=cuda)
            e(x.to(cuda), out=out)
            torch.cuda.synchronize()
    finally:
        capi.lib.rb_set_math_mode(capi.RB_MATH_TC)
    err = (out.cpu().double() - ref).abs().max().item()
    print(f"\nencoder small={small} {mode}: max err {err:.2e}, scale {ref.abs().max().item():.2f}")
    assert err < 1e-3 * max(ref.abs().max().item(), 1.0)


# ---- end to end on converted checkpoints -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    """small -> (npz path, fp64 host params): torch.nn modules with the published architecture -> torch.save -> convert."""
    from raft_b200 import convert
    from raft_b200.weights import load_npz
    out = {}
    for small in (False, True):
        torch.manual_seed(99 + small)
        m = (UpstreamSmall() if small else Upstream()).eval()
        d = tmp_path_factory.mktemp("up")
        pth, npz = str(d / "m.pth"), str(d / "m.npz")
        torch.save({"module." + k: v for k, v in m.state_dict().items()}, pth)
        assert convert.main([pth, npz]) == 0
        out[small] = (npz, load_npz(npz))
    return out


def _frames(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, H, W, 3, generator=g)
    return x, torch.roll(x, shifts=(2, 3), dims=(1, 2)) * 0.9 + 0.05 * torch.rand(B, H, W, 3, generator=g)


def _model(ckpt, small, **kw):
    from networks.RAFT import RAFT
    return RAFT((0, 0, 3), SimpleNamespace(small=small), upstream=True, **kw).load(ckpt[small][0])


@pytest.mark.parametrize("small,H,W,iters", [(False, 256, 320, 12), (True, 216, 288, 12)])
def test_end_to_end_matches_fp64_upstream(cuda, ckpt, small, H, W, iters):
    l, r = _frames(1, H, W, 3)
    flow = _model(ckpt, small, iters=iters).forward(l, r).cpu()
    ref = U.UpstreamOracle(ckpt[small][1], small=small, iters=iters, dtype=torch.float64).forward(l.double(), r.double())
    err = (flow.double() - ref).abs().max().item()
    print(f"\nupstream small={small} {H}x{W} iters {iters}: max|flow| {ref.abs().max().item():.3f}, max err {err:.2e}")
    assert err < 1e-3
    vf = _model(ckpt, small, iters=iters, volume_free=True).forward(l, r).cpu()
    assert (vf - flow).abs().max().item() < 2e-4 * max(flow.abs().max().item(), 1.0)


@pytest.mark.parametrize("small", [False, True])
def test_graph_batch_bidirectional_interpolate_are_consistent(cuda, ckpt, small):
    from networks.utils import reverse_flow, synthesize
    from raft_b200.engine import RaftEngine
    l, r = _frames(3, 136, 200, 4)
    m = _model(ckpt, small, iters=6)
    batched = m.forward(l, r).cpu()
    for i in range(3):
        assert torch.equal(m.forward(l[i:i + 1], r[i:i + 1]).cpu(), batched[i:i + 1])
    eager = RaftEngine(ckpt[small][1], small=small, iters=6, device=cuda, use_graph=False, upstream=True)
    assert torch.equal(eager.forward(l, r).cpu(), batched)
    fw, bw, occ_fw, _ = m.forward_bidirectional(l, r)
    assert torch.equal(fw.cpu(), batched) and torch.equal(bw.cpu(), m.forward(r, l).cpu())
    assert occ_fw.shape == (3, 136, 200)
    if small:  # flows are in pixels upstream: the time steps are t, not 8t
        t = 0.375
        got = m.interpolate(l, r, t).cpu()
        fw, bw, _, _ = m.forward_bidirectional(l, r, check=False)
        ft0, e0 = reverse_flow(fw, t)[:2]
        ft1, e1 = reverse_flow(bw, 1.0 - t)[:2]
        want = synthesize(l.to(cuda), r.to(cuda), ft0, ft1, e0, e1, t).cpu()
        assert torch.equal(got, want)


def test_upstream_and_reference_engines_alternate(cuda, ckpt):
    from raft_b200.engine import RaftEngine
    l, r = _frames(1, 128, 160, 6)
    p = ckpt[False][1]
    up = RaftEngine(p, iters=4, device=cuda, upstream=True)
    tf = RaftEngine(p, iters=4, device=cuda)
    a, b = up.forward(l, r).clone(), tf.forward(l, r).clone()
    assert not torch.equal(a, b)
    for _ in range(2):
        assert torch.equal(tf.forward(l, r), b) and torch.equal(up.forward(l, r), a)


def test_frames_of_120_pixels_are_refused(cuda, ckpt):
    m = _model(ckpt, False, iters=2)
    l, r = _frames(1, 120, 256, 1)
    with pytest.raises(ValueError, match="121"):
        m.forward(l, r)
    l, r = _frames(1, 121, 256, 1)
    assert m.forward(l, r).shape == (1, 121, 256, 2)


def test_cli_upstream_keep_size_writes_forward_on_rgb_frames(cuda, ckpt, tmp_path):
    import cv2
    npz = ckpt[False][0]
    data = os.path.join(ROOT, "tests", "data")
    im1, im2 = os.path.join(data, "frame_0016.png"), os.path.join(data, "frame_0017.png")
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "raft-tf_b200"))
    subprocess.run([sys.executable, os.path.join(ROOT, "raft-tf_b200", "infer_raft.py"), "--im1", im1, "--im2", im2, "--load", npz,
                    "--iters", "4", "--keep-size", "--upstream", "--npy", str(tmp_path / "f.npy")], cwd=tmp_path, env=env, check=True)
    rgb = [np.float32(cv2.cvtColor(cv2.imread(p), cv2.COLOR_BGR2RGB))[None] / 255.0 for p in (im1, im2)]
    flow = _model(ckpt, False, iters=4).forward(*rgb).cpu().numpy()[0]
    assert np.array_equal(np.load(tmp_path / "f.npy"), flow)
