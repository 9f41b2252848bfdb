"""The recurrent update loop, step by step, against fp64.

Every call goes through the C ABI in the order RaftEngine._hot_path uses: rb_corr_build (or rb_corr_otf_prepare) ->
rb_update_set_state_cnet -> rb_coords_grid -> N x (rb_update_lookup[_otf] + rb_update_step).  The loop is
teacher-forced: the reference for step k starts from the state the GPU left after step k-1 (net read back through
rb_update_get_net, coords1 read back), so an error in one step cannot hide in, or be blamed on, the compounding of the
others.  What each step is compared with:
  - corr: O.sample_corr on the GPU's own fp32 pyramid at the GPU's fp32 coords1 (bit-identical to the kernel's lookup,
    test_gpu_kernels.test_lookup_bit_exact), or on the fp64 pyramid of the same feature maps for the volume-free lookup;
  - net, delta, mask: O.basic_update_block / O.small_update_block in fp64 on (net_{k-1}, relu(cnet[..., hidden:]),
    corr, coords1_{k-1} - grid), within the tolerances of test_gpu_kernels.test_update_block;
  - coords1_k: fl32(coords1_{k-1} + delta_k), bit for bit.
This checks what one isolated update-block call cannot: the state the GRU epilogues write for the NEXT iteration (H in
fp32, the hidden slice of hx/qx as hi/lo fp16, the flow slot), the hoisted GRU contribution of `inp` (W.pre), and the
reuse of one workspace for a second frame pair.
"""
import contextlib

import numpy as np
import pytest
import torch

from oracle import raft_oracle as O

pytestmark = pytest.mark.gpu

NET_TOL, DELTA_TOL, MASK_TOL = 5e-5, 5e-5, 1e-4  # test_gpu_kernels.test_update_block
OTF_TOL = 1e-4  # volume-free lookup: the reference's pyramid is fp64, the kernel's dot products fp32


def _dims(small):
    """hidden, context, radius, feature channels (networks/RAFT.py:37-40)."""
    return (96, 64, 3, 128) if small else (128, 128, 4, 256)


def _modes():
    from raft_b200 import capi
    return {"tc": capi.RB_MATH_TC, "simt": capi.RB_MATH_SIMT}


@contextlib.contextmanager
def _math(mode):
    from raft_b200 import capi
    capi.check(capi.lib.rb_set_math_mode(mode))
    try:
        yield
    finally:
        capi.lib.rb_set_math_mode(capi.RB_MATH_TC)


@pytest.fixture(scope="module")
def weights(cuda):
    """small -> (packed device blob, fp64 host weights) of synth.make_weights(small)."""
    from raft_b200 import synth
    from raft_b200.weights import pack_update_block
    out = {}
    for small in (False, True):
        p = synth.make_weights(small)
        out[small] = (pack_update_block(p, small, cuda), {k: torch.from_numpy(v).double() for k, v in p.items()})
    return out


def _pair(small, B, h, w, seed):
    """Feature maps with unit variance (like instance-normed fnet output) and a raw context-encoder output."""
    hid, ctx, _, C = _dims(small)
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, h, w, C, generator=g), torch.randn(B, h, w, C, generator=g),
            torch.randn(B, h, w, hid + ctx, generator=g))


class _Loop:
    """Device buffers of one (variant, B, h, w) problem and the C-ABI calls of RaftEngine._hot_path on them."""

    def __init__(self, cuda, small, blob, B, h, w, volume_free=False):
        from raft_b200 import capi
        self.capi, self.lib = capi, capi.lib
        self.cuda, self.s, self.blob, self.B, self.h, self.w, self.vf = cuda, int(small), blob, B, h, w, volume_free
        self.hid, self.ctx, self.r, self.C = _dims(small)
        q = capi.size_query
        self.ws = torch.zeros(q(self.lib.rb_update_workspace_bytes, self.s, B, h, w), dtype=torch.uint8, device=cuda)
        if volume_free:
            self.pyramid = None
            self.cws_bytes = q(self.lib.rb_corr_otf_workspace_bytes, B, h, w, self.C)
        else:
            self.pyramid = torch.empty(q(self.lib.rb_corr_pyramid_bytes, B, h, w) // 4, device=cuda)
            self.cws_bytes = q(self.lib.rb_corr_workspace_bytes, B, h, w, self.C)
        self.cws = torch.zeros(self.cws_bytes, dtype=torch.uint8, device=cuda)
        self.coords1 = torch.empty(B, h, w, 2, device=cuda)
        self.delta = torch.empty(B, h, w, 2, device=cuda)
        self.mask = None if small else torch.empty(B, h, w, 576, device=cuda)
        self.net = torch.empty(B, h, w, self.hid, device=cuda)

    def _args(self):
        return self.B, self.h, self.w

    def set_pair(self, fmap1, fmap2, cnet):
        """Correlation volume (or pooled fmap2), recurrent state and context, coords1 = coords0."""
        c, lib, P, st = self.capi, self.lib, self.capi.ptr, self.capi.stream()
        self.f1, self.f2, self.cnet = (t.to(self.cuda).contiguous() for t in (fmap1, fmap2, cnet))
        if self.vf:
            c.check(lib.rb_corr_otf_prepare(P(self.f2), P(self.cws), self.cws_bytes, *self._args(), self.C, st))
        else:
            c.check(lib.rb_corr_build(P(self.f1), P(self.f2), P(self.pyramid), *self._args(), self.C, P(self.cws),
                                      self.cws_bytes, st))
        c.check(lib.rb_update_set_state_cnet(self.s, P(self.blob), P(self.ws), P(self.cnet), *self._args(), st))
        c.check(lib.rb_coords_grid(P(self.coords1), *self._args(), st))

    def step(self, with_mask=True):
        """One iteration of the engine's loop (lookup + update), with delta_out and (raft-things) mask_out."""
        c, lib, P, st = self.capi, self.lib, self.capi.ptr, self.capi.stream()
        if self.vf:
            c.check(lib.rb_update_lookup_otf(self.s, P(self.ws), P(self.f1), P(self.f2), P(self.cws), P(self.coords1),
                                             *self._args(), self.C, st))
        else:
            c.check(lib.rb_update_lookup(self.s, P(self.ws), P(self.pyramid), P(self.coords1), *self._args(), st))
        mask = self.mask if with_mask else None
        c.check(lib.rb_update_step(self.s, P(self.blob), P(self.ws), P(self.coords1), P(self.delta), P(mask),
                                   *self._args(), st))

    def iterate(self, iters):
        c, P = self.capi, self.capi.ptr
        c.check(self.lib.rb_raft_iterate(self.s, P(self.blob), P(self.ws), P(self.pyramid), P(self.coords1), P(self.mask),
                                         *self._args(), iters, c.stream()))

    def get_net(self):
        c, P = self.capi, self.capi.ptr
        c.check(self.lib.rb_update_get_net(self.s, P(self.ws), P(self.net), *self._args(), c.stream()))
        return self.net.cpu()

    def host_pyramid(self):
        """The device pyramid as O.sample_corr takes it: levels [B*h*w, h_l, w_l, 1] fp32."""
        import ctypes as C
        flat, levels = self.pyramid.cpu(), []
        for l in range(4):
            off, hl, wl = C.c_size_t(), C.c_int(), C.c_int()
            self.capi.check(self.lib.rb_corr_level_offset(*self._args(), l, C.byref(off), C.byref(hl), C.byref(wl)))
            n = self.B * self.h * self.w
            levels.append(flat[off.value:off.value + n * hl.value * wl.value].view(n, hl.value, wl.value, 1))
        return levels


def _bits(t):
    return t.contiguous().view(torch.int32)


def _ulps(a, b):
    """Distance in units in the last place between two fp32 tensors (+0 and -0 coincide)."""
    def key(t):
        i = t.contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return (key(a) - key(b)).abs()


def _teacher_forced(cuda, weights, small, mode, B, h, w, steps, volume_free=False, seed=0):
    """Run the loop, compare every step with fp64; returns the per-step errors (asserts at the end, naming the step)."""
    blob, pt = weights[small]
    hid, _, r, _ = _dims(small)
    f1, f2, cnet = _pair(small, B, h, w, seed=1000 * B + 10 * h + w + seed)
    inp = torch.relu(cnet[..., hid:]).double()
    grid = O.coords_grid(B, h, w)
    update = O.small_update_block if small else O.basic_update_block
    tols = (OTF_TOL,) * 3 if volume_free else (NET_TOL, DELTA_TOL, MASK_TOL)
    with _math(mode):
        lp = _Loop(cuda, small, blob, B, h, w, volume_free)
        lp.set_pair(f1, f2, cnet)
        net = lp.get_net()
        # set_state_cnet: tanh of the hidden half; CUDA documents tanhf at 2 ulp of the correctly rounded result
        tanh_ref = torch.tanh(cnet[..., :hid].double()).float()
        set_state_ulps = int(_ulps(net, tanh_ref).max())
        pyr = O.get_corr_pyramid(f1.double(), f2.double()) if volume_free else lp.host_pyramid()
        coords = grid.clone()
        rows, failures, outside = [], [], 0.0
        for k in range(steps):
            lp.step()
            c1, d, n1 = lp.coords1.cpu(), lp.delta.cpu(), lp.get_net()
            m = None if small else lp.mask.cpu()
            corr = O.sample_corr(pyr, coords.double() if volume_free else coords, radius=r).double()
            rn, rm, rd = update(net.double(), inp, corr, coords.double() - grid.double(), pt)
            e_net = (n1.double() - rn).abs().max().item()
            e_delta = (d.double() - rd).abs().max().item()
            e_mask = 0.0 if small else (m.double() - rm).abs().max().item()
            rows.append((e_net, e_delta, e_mask))
            for name, e, tol in zip(("net", "delta", "mask"), rows[-1], tols):
                if not e < tol:
                    failures.append(f"step {k}: {name} max-abs error {e:.3e} >= {tol:.0e}")
            if not torch.equal(_bits(c1), _bits(coords + d)):
                failures.append(f"step {k}: coords1 != fl32(coords1_prev + delta) in {int((c1 != coords + d).sum())} values")
            outside = max((-c1[..., 0]).max().item(), (c1[..., 0] - (w - 1)).max().item(),
                          (-c1[..., 1]).max().item(), (c1[..., 1] - (h - 1)).max().item(), outside)
            coords, net = c1, n1
    worst = [max(r_[i] for r_ in rows) for i in range(3)]
    print(f"\n{'small' if small else 'things'} B={B} h={h} w={w} mode={mode} volume_free={volume_free}: "
          f"set_state tanh {set_state_ulps} ulp; coords1 leave the grid by at most {outside:.3f} px")
    for k, (en, ed, em) in enumerate(rows):
        print(f"  step {k}: net {en:.2e} ({en / tols[0]:.2f} of tol)  delta {ed:.2e} ({ed / tols[1]:.2f})"
              f"  mask {em:.2e} ({em / tols[2]:.2f})")
    print(f"  worst: net {worst[0]:.2e} delta {worst[1]:.2e} mask {worst[2]:.2e}")
    assert set_state_ulps <= 2, f"rb_update_set_state_cnet: net is {set_state_ulps} ulp from tanh(cnet[..., :{hid}])"
    assert not failures, "\n".join(failures)
    return rows, outside


GRIDS = [(1, 8, 8),    # smallest legal grid: level 3 is 1x1
         (2, 12, 20),
         (3, 9, 17)]   # npix % 128 != 0; levels 4x8, 2x4, 1x2 (W % 4 != 0: the lookup's plain-load path, not TMA)


@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
@pytest.mark.parametrize("B,h,w", GRIDS, ids=lambda v: str(v))
def test_teacher_forced_steps_match_fp64(cuda, weights, B, h, w, small, mode):
    _teacher_forced(cuda, weights, small, _modes()[mode], B, h, w, steps=6)


@pytest.mark.parametrize("mode", ["tc", "simt"])
def test_teacher_forced_steps_above_cta_cap_threshold(cuda, weights, mode):
    """B*h*w = 16896 > 16384: update_step (csrc/update.cu) drops the CTA caps of convf1 / convf2 on the tensor cores, and
    the CUDA-core flow_conv7 that convf1 runs on in the CUDA-core math mode switches from 16- to 32-pixel blocks.  Many
    images of a modest size keep the B*(hw)^2 volume and the fp64 reference small."""
    B, h, w = 8, 48, 44
    assert B * h * w > 16384
    _teacher_forced(cuda, weights, False, _modes()[mode], B, h, w, steps=2)


@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
@pytest.mark.parametrize("B,h,w", [(2, 12, 20), (3, 9, 17)], ids=lambda v: str(v))
def test_volume_free_teacher_forced_steps_match_fp64(cuda, weights, B, h, w, small):
    """rb_corr_otf_prepare + rb_update_lookup_otf inside the loop, against the fp64 pyramid of the same feature maps.
    Far outside the image the reference's clamped-x1 weights grow like |x| and amplify the fp32-vs-fp64 difference of
    the dot products (test_gpu_kernels.test_volume_free_lookup_matches_materialised_path); here the centroids stay
    within a pixel of the grid, which is asserted so that the bound keeps meaning what it says.  The loop with most
    centroids off the image is test_gpu_volume_free_exact.test_loop_off_the_image_bit_identical: bit-identical to the
    materialised loop on feature maps whose dot products are exact."""
    _, outside = _teacher_forced(cuda, weights, small, _modes()["tc"], B, h, w, steps=6, volume_free=True)
    assert outside < 1.0, f"coords1 left the grid by {outside:.2f} px: the fixed tolerance no longer bounds the lookup"


@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_raft_iterate_equals_stepwise_loop(cuda, weights, small, mode):
    """rb_raft_iterate(N) (lookup fused in, mask on the last iteration only) == N x (rb_update_lookup + rb_update_step),
    bit for bit: coords1, and the mask of the LAST iteration."""
    B, h, w, N = 3, 9, 17, 3
    blob, _ = weights[small]
    pair = _pair(small, B, h, w, seed=5)
    with _math(_modes()[mode]):
        loop = _Loop(cuda, small, blob, B, h, w)
        loop.set_pair(*pair)
        masks = []
        for _ in range(N):
            loop.step()
            if not small:
                masks.append(loop.mask.clone())
        fused = _Loop(cuda, small, blob, B, h, w)
        fused.set_pair(*pair)
        fused.iterate(N)
        torch.cuda.synchronize()
    assert torch.equal(_bits(fused.coords1), _bits(loop.coords1))
    assert torch.equal(fused.get_net(), loop.get_net())
    if not small:
        assert not torch.equal(masks[0], masks[-1]), "the mask must change over the iterations for this test to mean anything"
        assert torch.equal(_bits(fused.mask), _bits(masks[-1])), "rb_raft_iterate's mask is not the last iteration's"


@pytest.mark.parametrize("volume_free", [False, True], ids=["volume", "volume_free"])
@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_workspace_reuse_equals_fresh_workspace(cuda, weights, small, mode, volume_free):
    """The engine replays pair after pair on one workspace: pair A for N steps, then rb_update_set_state_cnet(pair B) +
    N steps on the same workspace must equal pair B on a fresh zero-filled workspace, bit for bit (a stale hoisted W.pre,
    flow slot or qx slice would differ)."""
    B, h, w, N = 2, 12, 20, 3
    blob, _ = weights[small]
    pa, pb = _pair(small, B, h, w, seed=11), _pair(small, B, h, w, seed=12)
    with _math(_modes()[mode]):
        fresh = _Loop(cuda, small, blob, B, h, w, volume_free)
        fresh.set_pair(*pb)
        for _ in range(N):
            fresh.step()
        reused = _Loop(cuda, small, blob, B, h, w, volume_free)  # both workspaces stay alive: distinct addresses
        reused.set_pair(*pa)
        for _ in range(N):
            reused.step()
        coords_a = reused.coords1.clone()
        reused.set_pair(*pb)
        for _ in range(N):
            reused.step()
        torch.cuda.synchronize()
    assert not torch.equal(coords_a, fresh.coords1), "pairs A and B must give different flows for this test to mean anything"
    assert torch.equal(_bits(reused.coords1), _bits(fresh.coords1))
    assert torch.equal(_bits(reused.delta), _bits(fresh.delta))
    assert torch.equal(_bits(reused.get_net()), _bits(fresh.get_net()))
    if not small:
        assert torch.equal(_bits(reused.mask), _bits(fresh.mask))
