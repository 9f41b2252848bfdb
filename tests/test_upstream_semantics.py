"""RB_SEMANTICS_UPSTREAM on the CPU: the upstream oracle (tests/upstream_oracle.py) against independent PyTorch forms of
princeton-vl RAFT -- the torch.nn modules and the grid_sample CorrBlock of test_upstream_crosscheck.py -- at the sizes the
crosscheck cannot cover (even extents at the stride-2 convs, taps on and beyond the border), and the C ABI's argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import upstream_oracle as U
from oracle import raft_oracle as O
from test_upstream_crosscheck import _nhwc, _upstream_corr_lookup, converted, converted_small  # noqa: F401  (fixtures)


def _close(a, b, tol):
    return (a - b).abs().max().item() <= tol * max(b.abs().max().item(), 1.0)


@pytest.mark.parametrize("name,norm", [("fnet", "instance"), ("cnet", "batch")])
def test_basic_encoder_matches_upstream_module_at_even_sizes(converted, name, norm):
    m, p = converted
    x = torch.rand(2, 3, 64, 96, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 2 - 1  # 64 -> 32 -> 16 -> 8
    with torch.no_grad():
        ref = _nhwc(getattr(m, name)(x))
    with U.upstream_semantics():
        out = O.basic_encoder(_nhwc(x), p, name, norm)
    assert out.shape == ref.shape == (2, 8, 12, 256)
    assert _close(out, ref, 1e-9)
    assert not _close(O.basic_encoder(_nhwc(x), p, name, norm), ref, 1e-3), "TF padding should differ at even sizes"


def test_small_encoders_match_upstream_modules_at_even_sizes(converted_small):
    m, p = converted_small
    x = torch.rand(1, 3, 80, 48, generator=torch.Generator().manual_seed(4), dtype=torch.float64) * 2 - 1
    for name, norm in (("fnet", "instance"), ("cnet", "none")):
        with torch.no_grad():
            ref = _nhwc(getattr(m, name)(x))
        with U.upstream_semantics():
            out = O.small_encoder(_nhwc(x), p, name, norm)
        assert out.shape == ref.shape and _close(out, ref, 1e-9), name


def _border_coords(B, H, W, seed):
    """Random coordinates plus every kind of border tap: -1, 0, W-1, W, fractional negatives, far outside."""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    c = torch.stack([xs, ys], 0)[None].repeat(B, 1, 1, 1) + (torch.rand(B, 2, H, W, generator=g, dtype=torch.float64) * 10 - 5)
    special = [(-1.0, -1.0), (0.0, 0.0), (W - 1.0, H - 1.0), (float(W), float(H)), (-0.75, -0.25), (-4.5, 3.0),
               (1e4, -1e4), (-1e4, 5.0), (W + 4.0, H + 4.25), (-5.0, -4.0)]
    for k, (x, y) in enumerate(special):
        c[0, :, k // W, k % W] = torch.tensor([x, y], dtype=torch.float64)
    return c


@pytest.mark.parametrize("radius", [4, 3])
@pytest.mark.parametrize("H,W", [(40, 72), (37, 53)])
def test_sample_corr_up_matches_grid_sample_on_all_taps(radius, H, W):
    g = torch.Generator().manual_seed(5)
    B, Cc = 1, 16
    f1 = torch.randn(B, Cc, H, W, generator=g, dtype=torch.float64)
    f2 = torch.randn(B, Cc, H, W, generator=g, dtype=torch.float64)
    coords = _border_coords(B, H, W, 6)
    ref = _upstream_corr_lookup(f1, f2, coords, radius)
    out = U.sample_corr_up(O.get_corr_pyramid(_nhwc(f1), _nhwc(f2)), _nhwc(coords), radius=radius)
    assert out.shape == ref.shape
    assert _close(out, ref, 1e-10)
    assert (out == 0).any(), "taps outside every level must be present"


def test_fp32_restatement_matches_grid_sample_fp32():
    """The bit-level fp32 restatement of the GPU sampler against F.grid_sample in fp32 on the CPU (whose unnormalisation uses a
    precomputed scale, so not bit for bit)."""
    g = torch.Generator().manual_seed(7)
    B, Cc, H, W, r = 1, 16, 24, 40, 4
    f1 = torch.randn(B, Cc, H, W, generator=g)
    f2 = torch.randn(B, Cc, H, W, generator=g)
    coords = _border_coords(B, H, W, 8).float()
    pyr = O.get_corr_pyramid(_nhwc(f1), _nhwc(f2))
    out = U.sample_corr_up(pyr, _nhwc(coords), radius=r)
    assert out.dtype == torch.float32
    ref = _upstream_corr_lookup(f1, f2, coords, r)
    assert (out - ref).abs().max().item() <= 1e-6 * max(p.abs().max().item() for p in pyr)


def test_fma32_is_a_single_rounding():
    rng = np.random.default_rng(9)
    a, b, c = (rng.standard_normal(200000).astype(np.float32) for _ in range(3))
    r = U._fma32(a, b, c)
    exact = a.astype(np.longdouble) * b.astype(np.longdouble) + c.astype(np.longdouble)
    err = np.abs(r.astype(np.longdouble) - exact)
    ulp = np.spacing(np.abs(r)).astype(np.longdouble)
    assert (err <= ulp / 2).all()


def _upstream_raft(m, corr_fn, img1, img2, iters, small):
    """princeton-vl RAFT.forward(test_mode=True)[1] assembled from the torch.nn modules and the grid_sample CorrBlock."""
    hid, ctx = (96, 64) if small else (128, 128)
    i1, i2 = 2 * img1 - 1, 2 * img2 - 1
    f1, f2 = m.fnet(i1), m.fnet(i2)
    net, inp = torch.split(m.cnet(i1), [hid, ctx], dim=1)
    net, inp = torch.tanh(net), torch.relu(inp)
    N, _, h, w = f1.shape
    ys, xs = torch.meshgrid(torch.arange(h, dtype=img1.dtype), torch.arange(w, dtype=img1.dtype), indexing="ij")
    coords0 = torch.stack([xs, ys], 0)[None].repeat(N, 1, 1, 1)
    coords1 = coords0.clone()
    mask = None
    for _ in range(iters):
        corr = corr_fn(f1, f2, coords1, 3 if small else 4).permute(0, 3, 1, 2)
        flow = coords1 - coords0
        if small:
            net, delta = m.update_block(net, inp, corr, flow)
        else:
            net, mask, delta = m.update_block(net, inp, corr, flow)
        coords1 = coords1 + delta
    flow = coords1 - coords0
    if small:
        return 8 * F.interpolate(flow, size=(8 * h, 8 * w), mode="bilinear", align_corners=True)
    mk = torch.softmax(mask.view(N, 1, 9, 8, 8, h, w), dim=2)
    up = F.unfold(8 * flow, [3, 3], padding=1).view(N, 2, 9, 1, 1, h, w)
    return torch.sum(mk * up, dim=2).permute(0, 1, 4, 2, 5, 3).reshape(N, 2, 8 * h, 8 * w)


@pytest.mark.parametrize("small", [False, True])
def test_upstream_oracle_forward_matches_assembled_upstream_raft(converted, converted_small, small):
    m, p = converted_small if small else converted
    g = torch.Generator().manual_seed(12)
    l, r = (torch.rand(1, 3, 128, 192, generator=g, dtype=torch.float64) for _ in range(2))
    with torch.no_grad():
        ref = _nhwc(_upstream_raft(m, _upstream_corr_lookup, l, r, 4, small))
    out = U.UpstreamOracle({k: v.numpy() for k, v in p.items()}, small=small, iters=4,
                           dtype=torch.float64).forward(_nhwc(l), _nhwc(r))
    assert out.shape == ref.shape == (1, 128, 192, 2)
    # raft-small: the oracle's align_corners resize forms its source coordinates in fp32 like TF's kernel (~1e-6 pixel)
    assert _close(out, ref, 1e-5 if small else 1e-9)


# ---- C ABI (through the .so, no GPU needed) -------------------------------------------------------------------------------
def test_set_semantics_argument_checks():
    from raft_b200 import capi
    lib = capi.lib
    assert lib.rb_get_semantics() == capi.RB_SEMANTICS_REFERENCE
    for bad in (-1, 2, 99):
        assert lib.rb_set_semantics(bad) == -2 and b"rb_set_semantics" in lib.rb_last_error()
        assert lib.rb_get_semantics() == capi.RB_SEMANTICS_REFERENCE
    try:
        assert lib.rb_set_semantics(capi.RB_SEMANTICS_UPSTREAM) == 0 and lib.rb_get_semantics() == capi.RB_SEMANTICS_UPSTREAM
    finally:
        assert lib.rb_set_semantics(capi.RB_SEMANTICS_REFERENCE) == 0


def test_upstream_lookups_refuse_grids_below_16_before_any_cuda_call():
    """Frames below 121 pixels give a 1/8-resolution grid below 16, whose level 3 is 1 wide: upstream divides by W_l - 1.
    Dummy (never dereferenced) pointers: the refusal must come before any CUDA call."""
    from raft_b200 import capi
    lib, p = capi.lib, C.c_void_p(16)
    calls = {
        "rb_corr_lookup": lambda h, w: lib.rb_corr_lookup(p, p, p, 1, h, w, 4, None),
        "rb_update_lookup": lambda h, w: lib.rb_update_lookup(0, p, p, p, 1, h, w, None),
        "rb_raft_iterate": lambda h, w: lib.rb_raft_iterate(1, p, p, p, p, None, 1, h, w, 2, None),
        "rb_corr_otf_lookup": lambda h, w: lib.rb_corr_otf_lookup(p, p, p, p, p, 1, h, w, 256, 4, None),
        "rb_update_lookup_otf": lambda h, w: lib.rb_update_lookup_otf(0, p, p, p, p, p, 1, h, w, 256, None),
    }
    assert lib.rb_set_semantics(capi.RB_SEMANTICS_UPSTREAM) == 0
    try:
        for name, fn in calls.items():
            for h, w in ((15, 64), (64, 15), (8, 8)):
                assert fn(h, w) == -1, name
                assert b"upstream" in lib.rb_last_error(), (name, lib.rb_last_error())
    finally:
        lib.rb_set_semantics(capi.RB_SEMANTICS_REFERENCE)


def test_engine_refuses_small_frames_in_upstream_mode():
    pytest.importorskip("torch")
    from raft_b200 import engine
    assert engine.MIN_FRAME_UPSTREAM == 121 and (engine.MIN_FRAME_UPSTREAM + 7) // 8 >> 3 == 2
    assert (120 + 7) // 8 >> 3 == 1
    with pytest.raises(ValueError, match="121"):
        engine.RaftEngine({}, upstream=True, input_size=(120, 512))
