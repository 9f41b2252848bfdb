"""Direct tests of the pipeline edges the engine calls around the update loop: frame preparation (u8 -> fp32, replicate
padding), convex / bilinear 8x upsampling with the crop folded in, coords_grid and the general bilinear sampler --
each against numpy or the oracle at the shapes and values where such kernels go wrong -- and the engine's minimum frame
size."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import raft_oracle as O

pytestmark = pytest.mark.gpu


def _capi():
    from raft_b200 import capi
    return capi


def _f32(*bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


# ---- rb_frames_prepare ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pads", [(0, 0, 0, 0), (3, 4, 1, 6), (7, 0, 0, 7)], ids=lambda p: "-".join(map(str, p)))
@pytest.mark.parametrize("u8", [True, False], ids=["u8", "f32"])
def test_frames_prepare_bit_exact(cuda, u8, pads):
    """== np.pad(mode="edge") of np.float32(x) / np.float32(255) (uint8) or of x itself (fp32, NaN payloads, infinities,
    -0 and subnormals kept), bit for bit; pads are (top, bottom, left, right)."""
    capi = _capi()
    B, H, W = 2, 37, 53
    pt, pb, pl, pr = pads
    rng = np.random.default_rng(sum(pads) + u8)
    if u8:
        src = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
        src.reshape(-1)[:256] = np.arange(256)  # every value, most of them on the top row, which the padding replicates
        ref = np.pad(src, ((0, 0), (pt, pb), (pl, pr), (0, 0)), mode="edge").astype(np.float32) / np.float32(255)
    else:
        src = rng.random((B, H, W, 3), dtype=np.float32)
        special = _f32(0x7FC00000, 0x7FC12345, 0xFFC00001, 0x7F800000, 0xFF800000, 0x80000000, 0x00000001, 0x807FFFFF)
        for i, v in enumerate(special):  # corners and edges (replicated into the padding) and the interior
            src[i % B, (0, H - 1, 5, 0)[i % 4], (0, W - 1, 0, 9)[(i // 2) % 4], i % 3] = v
        ref = np.pad(src, ((0, 0), (pt, pb), (pl, pr), (0, 0)), mode="edge")
    src_d = torch.from_numpy(src).to(cuda)
    dst = torch.full((B, H + pt + pb, W + pl + pr, 3), float("nan"), device=cuda)
    capi.check(capi.lib.rb_frames_prepare(capi.ptr(src_d), int(u8), capi.ptr(dst), B, H, W, pt, pb, pl, pr, capi.stream()))
    got = dst.cpu().numpy()
    bad = got.view(np.int32) != ref.view(np.int32)
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} values differ, first at {np.argwhere(bad)[0]}"


# ---- rb_upsample_convex_crop / rb_upflow8_crop --------------------------------------------------------------------------
def _crops(h, w):
    """(top, left, out_h, out_w): the full field, an odd-sized interior crop at (3, 5), a single row, the bottom-right
    corner."""
    H, W = 8 * h, 8 * w
    return [(0, 0, H, W), (3, 5, H - 5, W - 7), (H // 2, 3, 1, W - 3), (H - 3, W - 5, 3, 5)]


def _coords_and_flow(B, h, w, seed, scale=3.0):
    """coords1 = grid + flow in fp32, and the flow the kernels form from it (coords1 - grid, fp32)."""
    g = torch.Generator().manual_seed(seed)
    grid = O.coords_grid(B, h, w)
    coords1 = (grid + torch.randn(B, h, w, 2, generator=g) * scale).contiguous()
    return coords1, coords1 - grid


def _mask(kind, B, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "randn":
        return torch.randn(B, h, w, 576, generator=g)
    if kind == "randn50":  # softmax saturates: most weights underflow to 0
        return torch.randn(B, h, w, 576, generator=g) * 50
    if kind == "equal":  # uniform weights 1/9
        return torch.full((B, h, w, 576), 1.75)
    # one dominant logit per fine pixel: softmax is one-hot up to e^-40
    m = torch.randn(B, h, w, 9, 64, generator=g)
    k = torch.randint(0, 9, (B, h, w, 1, 64), generator=g)
    return m.scatter_add(3, k, torch.full(k.shape, 40.0)).reshape(B, h, w, 576)


@pytest.mark.parametrize("kind", ["randn", "randn50", "equal", "dominant"])
@pytest.mark.parametrize("h,w", [(7, 9), (8, 8)], ids=lambda v: str(v))
def test_upsample_convex_crop_matches_fp64(cuda, h, w, kind):
    """rb_upsample_convex_crop == O.upsample_flow (RAFT.py:119-134) in fp64, then cropped; relative to max|8 flow|."""
    capi = _capi()
    B = 2
    coords1, flow = _coords_and_flow(B, h, w, seed=h * 10 + w)
    mask = _mask(kind, B, h, w, seed=h + w)
    ref = O.upsample_flow(flow.double(), mask.double())
    scale = 8 * flow.abs().max().item()
    c1, m = coords1.to(cuda), mask.to(cuda)
    for top, left, oh, ow in _crops(h, w):
        out = torch.full((B, oh, ow, 2), float("nan"), device=cuda)
        capi.check(capi.lib.rb_upsample_convex_crop(capi.ptr(c1), capi.ptr(m), capi.ptr(out), B, h, w, top, left, oh, ow,
                                                    capi.stream()))
        got = out.cpu().double()
        assert torch.isfinite(got).all(), f"crop {(top, left, oh, ow)}: unwritten outputs"
        err = (got - ref[:, top:top + oh, left:left + ow]).abs().max().item()
        assert err <= 4e-6 * scale, f"crop {(top, left, oh, ow)}: max-abs error {err:.3e}, max|8 flow| {scale:.2f}"


@pytest.mark.parametrize("scale", [1.0, 8.0])
@pytest.mark.parametrize("h,w", [(1, 6), (5, 1), (1, 1), (4, 7)], ids=lambda v: str(v))
def test_upflow8_crop_matches_fp64(cuda, h, w, scale):
    """rb_upflow8_crop == scale * O.upflow8 (align_corners bilinear x8, utils.py:105-111), cropped and uncropped.  The
    sample positions are fp32 in both (the oracle states TF's fp32 arithmetic), the interpolation is fp64 here."""
    capi = _capi()
    B = 2
    coords1, flow = _coords_and_flow(B, h, w, seed=h * 10 + w)
    ref = O.upflow8(flow.double()) * scale
    bound = 1e-6 * scale * flow.abs().max().item()
    c1 = coords1.to(cuda)
    for top, left, oh, ow in _crops(h, w):
        out = torch.full((B, oh, ow, 2), float("nan"), device=cuda)
        capi.check(capi.lib.rb_upflow8_crop(capi.ptr(c1), capi.ptr(out), B, h, w, scale, top, left, oh, ow, capi.stream()))
        got = out.cpu().double()
        assert torch.isfinite(got).all(), f"crop {(top, left, oh, ow)}: unwritten outputs"
        err = (got - ref[:, top:top + oh, left:left + ow]).abs().max().item()
        assert err <= bound, f"crop {(top, left, oh, ow)}: max-abs error {err:.3e} > {bound:.3e}"


# ---- rb_coords_grid, rb_bilinear_sample ---------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(7, 13), (1, 9), (11, 1)], ids=lambda v: str(v))
def test_coords_grid_exact(cuda, h, w):
    capi = _capi()
    out = torch.full((3, h, w, 2), float("nan"), device=cuda)
    capi.check(capi.lib.rb_coords_grid(capi.ptr(out), 3, h, w, capi.stream()))
    assert torch.equal(out.cpu(), O.coords_grid(3, h, w))


def _edge_coords(n, S, H, W, seed):
    """Random coordinates around the image, the first ones on the edges of tf_grid_sample's case analysis: exactly -1,
    in (-1, 0) (truncation toward zero), exact integers, exactly W-1 / H-1, the next fp32 above, and far outside."""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(n, S, 2, generator=g) * torch.tensor([W + 6.0, H + 6.0]) - 3.0

    def specials(L):
        up = float(np.nextafter(np.float32(L - 1), np.float32(np.inf)))
        return [-1.0, -0.75, float(np.nextafter(np.float32(-1), np.float32(0))), 0.0, float(L - 1), up, L - 0.5, 1e4, -1e4,
                3e6, -5e6]

    pairs = [(x, y) for x in specials(W) for y in specials(H)]
    for i in range(n):
        k = min(S, len(pairs))
        start = (i * 37) % len(pairs)  # every image gets a different window of the cross product
        sel = (pairs[start:] + pairs[:start])[:k]
        c[i, :k] = torch.tensor(sel)
    return c.contiguous()


@pytest.mark.parametrize("n,H,W,S", [(2, 6, 11, 1), (2, 6, 11, 1000), (3, 1, 9, 1000), (3, 7, 1, 1000), (2, 1, 1, 1000),
                                     (1, 1, 1, 1)], ids=lambda v: str(v))
def test_bilinear_sample_bit_exact_at_edges(cuda, n, H, W, S):
    """rb_bilinear_sample == O.bilinear_sampler (tf_grid_sample, utils.py:39-103) bit for bit."""
    capi = _capi()
    g = torch.Generator().manual_seed(n * 100 + H * 10 + W)
    img = torch.randn(n, H, W, 1, generator=g)
    coords = _edge_coords(n, S, H, W, seed=S)
    ref = O.bilinear_sampler(img, coords.view(n, S, 1, 2)).reshape(n, S)
    img_d, coords_d = img.to(cuda), coords.to(cuda)  # held: a freed temporary's block could be handed to the next one
    out = torch.full((n, S), float("nan"), device=cuda)
    capi.check(capi.lib.rb_bilinear_sample(capi.ptr(img_d), capi.ptr(coords_d), capi.ptr(out), n, H, W, S, capi.stream()))
    got = out.cpu()
    bad = got.view(torch.int32) != ref.view(torch.int32)
    assert not bad.any(), f"{int(bad.sum())} samples differ, e.g. at coords {coords[bad][:4].tolist()}"


# ---- engine: minimum frame size, and the smallest legal frames against the oracle -----------------------------------
@pytest.mark.parametrize("volume_free", [False, True], ids=["volume", "volume_free"])
def test_engine_rejects_frames_below_minimum_on_the_host(cuda, volume_free):
    """56 px -> a 7-pixel grid: too small for the 4-level pyramid.  Refused on the host before any work is done (the
    volume-free path used to get through both encoders first): no raft_b200 kernel is launched, and no device memory is
    allocated -- no engine buffer, no upload of the (host) frames."""
    from raft_b200 import capi, synth
    from raft_b200.engine import RaftEngine
    eng = RaftEngine(synth.make_weights(False), iters=2, device=cuda, volume_free=volume_free)
    for H, W in ((56, 100), (100, 56)):
        frames = torch.zeros(1, H, W, 3)
        torch.cuda.synchronize()
        allocated = torch.cuda.memory_allocated(cuda)
        capi.lib.rb_launch_count_reset()
        with pytest.raises(ValueError, match="at least 57"):
            eng.forward(frames, frames)
        assert capi.lib.rb_launch_count() == 0
        assert torch.cuda.memory_allocated(cuda) == allocated and eng._shape is None


@pytest.mark.parametrize("volume_free", [False, True], ids=["volume", "volume_free"])
def test_smallest_frames_match_oracle(cuda, volume_free):
    """57 x 61 frames, the smallest legal size: padded (3, 4, 1, 2) to 64 x 64, so the convex upsampling crops with
    left != 0 inside the engine.  Against the oracle on the edge-padded frames, cropped back, at 1e-3."""
    from raft_b200 import synth
    from networks.RAFT import RAFT
    H, W, iters = 57, 61, 4
    p = synth.make_weights(False)
    l, r = synth.make_batch(1, H, W)
    m = RAFT((H, W, 3), SimpleNamespace(small=False), iters=iters, device=cuda, volume_free=volume_free).load(p)
    out = m.forward(l, r).cpu()
    assert m.engine().pad == (3, 4, 1, 2)
    pad = ((0, 0), (3, 4), (1, 2), (0, 0))
    lp, rp = np.pad(l, pad, mode="edge"), np.pad(r, pad, mode="edge")
    ref = O.RAFTOracle(p, small=False, iters=iters).forward(torch.from_numpy(lp), torch.from_numpy(rp))[:, 3:3 + H, 1:1 + W]
    assert out.shape == ref.shape == (1, H, W, 2)
    err = (out - ref).abs().max().item()
    assert err < 1e-3, f"max-abs {err:.3e}, |flow|max {ref.abs().max():.2f}"
