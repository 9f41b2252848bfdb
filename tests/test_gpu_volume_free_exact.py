"""The volume-free correlation lookup (F2: rb_corr_otf_lookup, rb_update_lookup_otf) bit for bit at every coordinate,
however far outside the image.

With small-integer feature maps (entries in {-3..3}, C = 128 or 256) every quantity before the division by sqrt(C) is
exact in fp32: every pooled fmap2 entry is a multiple of 2^-6 of magnitude <= 3, every product and every partial sum
(|sum| <= 2304, 6 fractional bits) is exact in any summation order, the warp butterfly included.  So every entry the
volume-free kernel evaluates is fl(exact dot / fl(sqrt C)), which is also level l of the exact pyramid
fl(fmap1 . pool^l(fmap2) / fl(sqrt C)) built here on the host.  From there the tap arithmetic is the reference's op for op,
so the volume-free lookup must equal O.sample_corr (U.sample_corr_up under RB_SEMANTICS_UPSTREAM) and the materialised
lookup on those levels BIT FOR BIT -- no cancellation of the reference's clamped-x1 weights (which grow like |x| outside
the image) can hide behind a tolerance.  The coordinate contract is at rb_corr_lookup in include/raft_b200.h: bit-exact
with the reference's 64-bit truncation for finite |c| < 2^62; beyond that and for +-inf / NaN unspecified values, but the
same ones from both lookups and no memory outside the level read.

test_realistic_statistics_far_outside covers randn feature maps with an a-priori error bound instead.
"""
import contextlib

import numpy as np
import pytest
import torch

import upstream_oracle as U
from oracle import raft_oracle as O
from test_gpu_update_loop import _Loop, _bits, _dims

pytestmark = pytest.mark.gpu

INF, NAN = float("inf"), float("nan")
# beyond the int32 range of a truncated coordinate (x0 + 1 used to wrap there); only compared between the two lookups
# and, below 2^62, with the oracle's 64-bit truncation
HUGE = [2.0 ** 31, 3e9, -3e9, 1e18, 3.4e38, INF, -INF, NAN]
ORACLE_LIMIT = 2.0 ** 62


def _below(v):
    return float(np.nextafter(np.float32(v), np.float32(0)))


def _above(v):
    return float(np.nextafter(np.float32(v), np.float32(np.inf) if v > 0 else np.float32(-np.inf)))


def _axis_values(n):
    """Special values of one coordinate axis, in units of a level that is n pixels wide."""
    return ([-1.0, 0.0, n - 1.0, float(n), -0.75, -0.25, -3.5]                                    # borders
            + [1.5 * n, -1.5 * n, 4.0 * n, -4.0 * n, 1e4, -1e4, 1e6, -1e6, 2.0 ** 30]             # far outside
            + [_below(2 ** 24), _above(2 ** 24), -_below(2 ** 24), -_above(2 ** 24)]             # around 2^24
            + [_below(8.0), _below(16.0), _below(32.0)])                                         # rounding slack


def _specials(h, w, gen, huge=True):
    """(x, y) pairs of every class at every level l (planted as c = v * 2^l, exact): x special with y inside the level,
    x inside with y special, and both special; then the HUGE values unscaled in the same three patterns."""
    out = []
    for l in range(4):
        hl, wl = h >> l, w >> l
        xs, ys = _axis_values(wl), _axis_values(hl)
        for i, (vx, vy) in enumerate(zip(xs, ys)):
            mx, my = (torch.rand(2, generator=gen) * torch.tensor([wl - 1.0, hl - 1.0])).tolist()
            out += [(vx * 2 ** l, my * 2 ** l), (mx * 2 ** l, vy * 2 ** l), (vx * 2 ** l, ys[(i + 3) % len(ys)] * 2 ** l)]
    if huge:
        for i, v in enumerate(HUGE):
            mx, my = (torch.rand(2, generator=gen) * torch.tensor([w - 1.0, h - 1.0])).tolist()
            out += [(v, my), (mx, v), (v, HUGE[(i + 1) % len(HUGE)])]
    return torch.tensor(out, dtype=torch.float32)


def _coord_sets(B, h, w, seed, huge=True):
    """Coordinate tensors [B,h,w,2] that together hold every special pair; the other half of each set (at least) are
    random in-image centroids (grid +- 8)."""
    gen = torch.Generator().manual_seed(seed)
    sp = _specials(h, w, gen, huge)
    npix = B * h * w
    per = max(npix // 2, 1)
    sets = []
    for k in range(0, len(sp), per):
        c = (O.coords_grid(B, h, w) + (torch.rand(B, h, w, 2, generator=gen) * 2 - 1) * 8.0).reshape(npix, 2)
        chunk = sp[k:k + per]
        idx = torch.randperm(npix, generator=gen)[:len(chunk)]
        c[idx] = chunk
        sets.append(c.reshape(B, h, w, 2).contiguous())
    return sets


def _int_maps(B, h, w, C, seed, lo=-3, hi=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(lo, hi + 1, (B, h, w, C), generator=g).float(),
            torch.randint(lo, hi + 1, (B, h, w, C), generator=g).float())


def _exact_levels(f1, f2):
    """Levels [B*h*w, h_l, w_l, 1] of fl(fmap1 . pool^l(fmap2) / fl(sqrt C)), the dot products exact in fp64."""
    B, h, w, C = f1.shape
    a = f1.double().reshape(B, h * w, C)
    pooled, levels = f2.double(), []
    for l in range(4):
        if l:
            pooled = O.avg_pool_2x2_valid(pooled)
        hl, wl = pooled.shape[1:3]
        dot = torch.einsum("bnc,bmc->bnm", a, pooled.reshape(B, hl * wl, C))
        assert torch.equal(dot.float().double(), dot), "the dot products must be exact in fp32"
        levels.append((dot.float() / torch.sqrt(torch.tensor(float(C)))).reshape(B * h * w, hl, wl, 1))
    return levels


def _pyramid_buffer(levels):
    """The library's pyramid layout: levels concatenated, 64 floats of tail padding (rb_corr_level_offset)."""
    return torch.cat([p.reshape(-1) for p in levels] + [torch.zeros(64)])


def _check_layout(lib, capi, B, h, w, levels):
    import ctypes as C
    for l in range(4):
        off, hl, wl = C.c_size_t(), C.c_int(), C.c_int()
        capi.check(lib.rb_corr_level_offset(B, h, w, l, C.byref(off), C.byref(hl), C.byref(wl)))
        assert off.value == sum(p.numel() for p in levels[:l]) and (hl.value, wl.value) == tuple(levels[l].shape[1:3])


@pytest.fixture(autouse=True)
def _reference_tc(cuda):
    """Every test starts in RB_SEMANTICS_REFERENCE / RB_MATH_TC: both are per-thread library state, and an engine leaves
    its own settings behind (RaftEngine.run sets them and does not restore them)."""
    from raft_b200 import capi
    capi.check(capi.lib.rb_set_semantics(capi.RB_SEMANTICS_REFERENCE))
    capi.check(capi.lib.rb_set_math_mode(capi.RB_MATH_TC))


@contextlib.contextmanager
def _semantics(up):
    from raft_b200 import capi
    capi.check(capi.lib.rb_set_semantics(capi.RB_SEMANTICS_UPSTREAM if up else capi.RB_SEMANTICS_REFERENCE))
    try:
        yield
    finally:
        capi.lib.rb_set_semantics(capi.RB_SEMANTICS_REFERENCE)


def _same(a, b):
    """Elementwise: the same fp32 bits, or both NaN (the payload is not specified)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return (na & nb) | (~na & ~nb & (_bits(a) == _bits(b)))


def _mismatch(got, want, rows, coords, what):
    """None if got == want (bits, NaN as NaN) on the [B,h,w] rows, else what differs and at which coordinates."""
    ok = _same(got, want) | ~rows[..., None]
    if ok.all():
        return None
    bad_rows = ~ok.all(-1)
    first = (~ok).nonzero()[0].tolist()
    c = coords[bad_rows]
    return (f"{what}: {int((~ok).sum())} taps of {int(bad_rows.sum())} pixels differ, first at {first}: "
            f"{got[tuple(first)].item()!r} != {want[tuple(first)].item()!r}; those pixels' |c| span "
            f"[{c.abs().max(-1).values.min().item():.3g}, {c.abs().max(-1).values.max().item():.3g}]")


def _assert_same(got, want, rows, coords, what):
    msg = _mismatch(got, want, rows, coords, what)
    assert msg is None, msg


class _Otf:
    """Device buffers of one (B, h, w, C) problem: feature maps, the volume-free workspace, the exact pyramid."""

    def __init__(self, cuda, f1, f2, levels):
        from raft_b200 import capi
        self.capi, self.lib, self.cuda = capi, capi.lib, cuda
        self.B, self.h, self.w, self.C = f1.shape
        self.f1, self.f2 = f1.to(cuda).contiguous(), f2.to(cuda).contiguous()
        _check_layout(self.lib, capi, self.B, self.h, self.w, levels)
        self.pyr = _pyramid_buffer(levels).to(cuda)
        self.wsb = capi.size_query(self.lib.rb_corr_otf_workspace_bytes, self.B, self.h, self.w, self.C)
        self.ws = torch.zeros(self.wsb, dtype=torch.uint8, device=cuda)
        capi.check(self.lib.rb_corr_otf_prepare(capi.ptr(self.f2), capi.ptr(self.ws), self.wsb, self.B, self.h, self.w,
                                                self.C, capi.stream()))

    def lookup(self, coords, r):
        """(volume-free, materialised) fp32 lookups at coords."""
        c, P, K = self.capi, self.capi.ptr, (2 * r + 1) ** 2
        cd = coords.to(self.cuda)
        otf = torch.full((self.B, self.h, self.w, 4 * K), 7.0, device=self.cuda)
        mat = torch.full((self.B, self.h, self.w, 4 * K), 7.0, device=self.cuda)
        c.check(self.lib.rb_corr_otf_lookup(P(self.f1), P(self.f2), P(self.ws), P(cd), P(otf), self.B, self.h, self.w,
                                            self.C, r, c.stream()))
        c.check(self.lib.rb_corr_lookup(P(self.pyr), P(cd), P(mat), self.B, self.h, self.w, r, c.stream()))
        torch.cuda.synchronize()
        return otf.cpu(), mat.cpu()

    def split_lookup(self, coords, small):
        """(volume-free, materialised) hi / lo planes of rb_update_lookup[_otf] as int16 bits [npix, pad]."""
        c, P = self.capi, self.capi.ptr
        r = 3 if small else 4
        K, npix = (2 * r + 1) ** 2, self.B * self.h * self.w
        pad = (4 * K + 63) // 64 * 64
        plane = (npix * pad * 2 + 1023) // 1024 * 1024
        cd = coords.to(self.cuda)
        out = []
        for otf in (True, False):
            wsb = c.size_query(self.lib.rb_update_workspace_bytes, int(small), self.B, self.h, self.w)
            ws = torch.zeros(wsb, dtype=torch.uint8, device=self.cuda)
            if otf:
                c.check(self.lib.rb_update_lookup_otf(int(small), P(ws), P(self.f1), P(self.f2), P(self.ws), P(cd), self.B,
                                                      self.h, self.w, self.C, c.stream()))
            else:
                c.check(self.lib.rb_update_lookup(int(small), P(ws), P(self.pyr), P(cd), self.B, self.h, self.w, c.stream()))
            torch.cuda.synchronize()
            hi = ws[:npix * pad * 2].view(torch.int16).view(npix, pad).cpu()
            lo = ws[plane:plane + npix * pad * 2].view(torch.int16).view(npix, pad).cpu()
            out.append((hi, lo))
        return out, 4 * K


def k_seed(h, w):
    return 7 * h + w


def _oracle_rows(coords):
    """[B,h,w] rows the reference's 64-bit truncation defines: finite, |c| < 2^62."""
    return (torch.isfinite(coords) & (coords.abs() < ORACLE_LIMIT)).all(-1)


# (B, h, w, C, r): 9 x 17 has levels narrower than the 11 evaluated columns, W_l % 4 != 0 and B*h*w % 16 != 0; at 8 x 8
# level 3 is 1 x 1; 55 x 128 is the full-size grid
CASES = [(3, 16, 32, 256, 4), (2, 17, 30, 128, 3), (1, 55, 128, 256, 4), (3, 9, 17, 256, 4), (1, 8, 8, 128, 3),
         (2, 21, 19, 256, 4)]
CASES_UP = [c for c in CASES if min(c[1:3]) >= 16]  # the upstream lookups need every level to be at least 2 x 2


@pytest.mark.parametrize("B,h,w,C,r", CASES, ids=str)
def test_volume_free_lookup_bit_exact_everywhere(cuda, B, h, w, C, r):
    f1, f2 = _int_maps(B, h, w, C, seed=h * w + C)
    levels = _exact_levels(f1, f2)
    p = _Otf(cuda, f1, f2, levels)
    n_oracle = n_beyond = 0
    for k, coords in enumerate(_coord_sets(B, h, w, seed=100 + k_seed(h, w))):
        otf, mat = p.lookup(coords, r)
        rows = _oracle_rows(coords)
        ref = O.sample_corr(levels, torch.where(rows[..., None], coords, torch.zeros(())), radius=r)
        msgs = [_mismatch(otf, ref, rows, coords, f"set {k}: volume-free lookup vs O.sample_corr on the exact pyramid"),
                _mismatch(mat, ref, rows, coords, f"set {k}: materialised lookup vs O.sample_corr on the exact pyramid"),
                _mismatch(otf, mat, torch.ones_like(rows), coords, f"set {k}: volume-free vs materialised lookup (every coordinate)")]
        msgs = [m for m in msgs if m]
        assert not msgs, "\n".join(msgs)
        n_oracle += int(rows.sum())
        n_beyond += int((~rows).sum())
    assert n_beyond >= 12 and n_oracle > 0, (n_oracle, n_beyond)  # +-inf, NaN and 3.4e38 in three patterns each


@pytest.mark.parametrize("B,h,w,C,r", CASES_UP, ids=str)
def test_volume_free_lookup_bit_exact_upstream(cuda, B, h, w, C, r):
    """RB_SEMANTICS_UPSTREAM: every coordinate, non-finite ones included, is defined (ix = -100 beyond 2^24 / NaN), so the
    volume-free and the materialised lookup must equal the fp32 restatement of the sampler everywhere."""
    f1, f2 = _int_maps(B, h, w, C, seed=h * w + C + 1)
    levels = _exact_levels(f1, f2)
    p = _Otf(cuda, f1, f2, levels)
    for k, coords in enumerate(_coord_sets(B, h, w, seed=200 + k_seed(h, w))):
        with _semantics(True):
            otf, mat = p.lookup(coords, r)
        with np.errstate(all="ignore"):
            ref = U.sample_corr_up(levels, coords, radius=r)
        every = torch.ones(coords.shape[:3], dtype=torch.bool)
        msgs = [_mismatch(otf, ref, every, coords, f"set {k}: volume-free lookup vs U.sample_corr_up on the exact pyramid"),
                _mismatch(mat, ref, every, coords, f"set {k}: materialised lookup vs U.sample_corr_up on the exact pyramid")]
        msgs = [m for m in msgs if m]
        assert not msgs, "\n".join(msgs)
        assert not torch.isnan(otf).any()


@pytest.mark.parametrize("up", [False, True], ids=["reference", "upstream"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
@pytest.mark.parametrize("B,h,w", [(3, 9, 17), (2, 17, 30), (1, 16, 32)], ids=str)
def test_split_planes_bit_exact(cuda, B, h, w, small, up):
    """rb_update_lookup_otf == rb_update_lookup on the exact pyramid: the hi and lo fp16 planes bit for bit, the channel
    padding zero."""
    if up and min(h, w) < 16:
        pytest.skip("the upstream lookups refuse grids below 16 x 16")
    C = _dims(small)[3]
    f1, f2 = _int_maps(B, h, w, C, seed=3 * h + w + C)
    p = _Otf(cuda, f1, f2, _exact_levels(f1, f2))
    for k, coords in enumerate(_coord_sets(B, h, w, seed=300 + k_seed(h, w))):
        with _semantics(up):
            ((hi_o, lo_o), (hi_m, lo_m)), nch = p.split_lookup(coords, small)
        for name, a, b in (("hi", hi_o, hi_m), ("lo", lo_o, lo_m)):
            assert torch.equal(a[:, :nch], b[:, :nch]), f"set {k}: {name} plane: {int((a != b).sum())} channels differ"
            assert (a[:, nch:] == 0).all() and (b[:, nch:] == 0).all(), f"set {k}: {name} plane: channel padding written"
        assert (hi_o[:, :nch] != 0).any()


# ---- d. the update loop off the image ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def blobs(cuda):
    """small -> packed device blob of synth.make_weights(small)."""
    from raft_b200 import synth
    from raft_b200.weights import pack_update_block
    return {small: pack_update_block(synth.make_weights(small), small, cuda) for small in (False, True)}


def _flow_init(B, h, w, seed):
    """Most centroids outside the image: +-(0.5..3) w / h in each axis; the last sample at +-1e4 (its NaN, once the fp16
    planes saturate, stays in that sample: no conv crosses samples)."""
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(B, h, w, 2, generator=g) < 0.5, -1.0, 1.0)
    mag = (0.5 + 2.5 * torch.rand(B, h, w, 2, generator=g)) * torch.tensor([float(w), float(h)])
    fi = sign * mag
    fi[-1] = sign[-1] * 1e4
    return fi.contiguous()


@pytest.mark.parametrize("mode", ["tc", "simt", "tc_fp16"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
@pytest.mark.parametrize("B,h,w", [(2, 12, 20), (3, 9, 17)], ids=str)
def test_loop_off_the_image_bit_identical(cuda, blobs, B, h, w, small, mode):
    """6 x (rb_update_lookup + rb_update_step) on the exact pyramid == 6 x (rb_update_lookup_otf + rb_update_step) on the
    same integer feature maps: coords1, delta, net and mask bit for bit after every step.  The lookups do not depend on
    the math mode and each step is deterministic."""
    from raft_b200 import capi
    mode_id = {"tc": capi.RB_MATH_TC, "simt": capi.RB_MATH_SIMT, "tc_fp16": capi.RB_MATH_TC_FP16}[mode]
    hid, ctx, _, C = _dims(small)
    f1, f2 = _int_maps(B, h, w, C, seed=17 * h + w, lo=-1, hi=1)
    cnet = torch.randn(B, h, w, hid + ctx, generator=torch.Generator().manual_seed(h + w))
    buf = _pyramid_buffer(_exact_levels(f1, f2))
    fi = _flow_init(B, h, w, seed=B + h).to(cuda)
    grid = O.coords_grid(B, h, w)
    capi.check(capi.lib.rb_set_math_mode(mode_id))
    try:
        loops = []
        for vf in (False, True):
            lp = _Loop(cuda, small, blobs[small], B, h, w, volume_free=vf)
            lp.set_pair(f1, f2, cnet)
            if not vf:
                assert lp.pyramid.numel() == buf.numel()
                lp.pyramid.copy_(buf.to(cuda))
            capi.check(capi.lib.rb_coords_init(capi.ptr(lp.coords1), capi.ptr(fi), B, h, w, capi.stream()))
            loops.append(lp)
        c0 = loops[0].coords1.cpu()
        out = ((c0[..., 0] < 0) | (c0[..., 0] > w - 1) | (c0[..., 1] < 0) | (c0[..., 1] > h - 1)).float().mean().item()
        assert out >= 0.5, f"only {out:.0%} of the centroids start outside the image"
        for k in range(6):
            for lp in loops:
                lp.step()
            torch.cuda.synchronize()
            mat, vf = loops
            for name, a, b in (("coords1", mat.coords1, vf.coords1), ("delta", mat.delta, vf.delta),
                               ("net", mat.get_net(), vf.get_net())) + ((("mask", mat.mask, vf.mask),) if not small else ()):
                assert torch.equal(_bits(a.cpu()), _bits(b.cpu())), f"step {k}: {name} differs in {int((a != b).sum())} values"
        c = loops[0].coords1.cpu()[:-1]  # the samples that started within a few frame sizes
        fin = torch.isfinite(c).all(-1)
        still = (fin & ((c[..., 0] < 0) | (c[..., 0] > w - 1) | (c[..., 1] < 0) | (c[..., 1] > h - 1))).float().mean().item()
        print(f"\n{mode} small={small} {B}x{h}x{w}: {out:.0%} of the centroids start outside; after 6 steps "
              f"{fin.float().mean().item():.0%} of the first {B - 1} samples are finite, {still:.0%} outside")
    finally:
        capi.lib.rb_set_math_mode(capi.RB_MATH_TC)


# ---- e. realistic statistics far outside the image --------------------------------------------------------------------------
def _taps(coords, hl, wl, l, r):
    """The reference's tap of every (pixel, window column i, window row j) at level l, as the kernels compute it: corner
    indices (clamped trunc) and the four fp32 weights (utils.py:54-89, no FMA)."""
    d = torch.arange(-r, r + 1, dtype=torch.float32)
    c = coords.reshape(-1, 2) / 2 ** l
    x = (c[:, 0:1] + d[None])[:, :, None].expand(-1, -1, 2 * r + 1)  # [N, i, j]: i walks x
    y = (c[:, 1:2] + d[None])[:, None, :].expand(-1, 2 * r + 1, -1)
    x0, y0 = torch.trunc(x).long(), torch.trunc(y).long()
    x1, y1 = (x0 + 1).clamp(0, wl - 1), (y0 + 1).clamp(0, hl - 1)
    x0, y0 = x0.clamp(0, wl - 1), y0.clamp(0, hl - 1)
    qx, qy = x1.float() - x, y1.float() - y
    w_ = (qx * qy, qx * (1.0 - qy), (1.0 - qx) * qy, (1.0 - qx) * (1.0 - qy))
    return (x0, x1, y0, y1), [t.double() for t in w_]


def _bound_check(f1, f2, coords, r):
    """(the fp64 reference, the per-tap bound, the change an Ib <-> Ic swap makes).  ref: the fp32 weights times the
    fp64 entries fmap1 . pool^l(fmap2) / sqrt(C).  Bound per tap: sum_corners |w| (C 2^-24 A + 2^-23 |I|) with
    A = sum_c |f1_c| pool^l(|f2|)_c / sqrt(C) (dot product and pooling rounding in fp32, division), plus 4.01 * 2^-24
    sum_corners |w| (|I| + that error) for the rounding of the four products and three additions of the tap sum."""
    B, h, w, C = f1.shape
    a, aa = f1.double().reshape(B, h * w, C), f1.double().abs().reshape(B, h * w, C)
    p, pa = f2.double(), f2.double().abs()
    sq = C ** 0.5
    refs, bounds, swaps = [], [], []
    for l in range(4):
        if l:
            p, pa = O.avg_pool_2x2_valid(p), O.avg_pool_2x2_valid(pa)
        hl, wl = p.shape[1:3]
        I = (torch.einsum("bnc,bmc->bnm", a, p.reshape(B, -1, C)) / sq).reshape(B * h * w, hl * wl)
        A = (torch.einsum("bnc,bmc->bnm", aa, pa.reshape(B, -1, C)) / sq).reshape(B * h * w, hl * wl)
        (x0, x1, y0, y1), wts = _taps(coords, hl, wl, l, r)
        n = x0.shape[0]

        def g(t, xx, yy):
            return torch.gather(t, 1, (yy * wl + xx).reshape(n, -1)).reshape(xx.shape)
        Is = [g(I, x0, y0), g(I, x0, y1), g(I, x1, y0), g(I, x1, y1)]  # Ia, Ib, Ic, Id (utils.py:66-69)
        As = [g(A, x0, y0), g(A, x0, y1), g(A, x1, y0), g(A, x1, y1)]
        e = [C * 2.0 ** -24 * Ak + 2.0 ** -23 * Ik.abs() for Ik, Ak in zip(Is, As)]
        ref = sum(wk * Ik for wk, Ik in zip(wts, Is))
        bnd = sum(wk.abs() * ek for wk, ek in zip(wts, e)) + 4.01 * 2.0 ** -24 * sum(
            wk.abs() * (Ik.abs() + ek) for wk, Ik, ek in zip(wts, Is, e))
        refs.append(ref.reshape(B, h, w, -1))
        bounds.append(bnd.reshape(B, h, w, -1))
        swaps.append(((wts[1] - wts[2]) * (Is[2] - Is[1])).reshape(B, h, w, -1))  # Ib <-> Ic
    ref, bound, swap = torch.cat(refs, -1), torch.cat(bounds, -1), torch.cat(swaps, -1)
    return ref, bound, swap


@pytest.mark.parametrize("B,h,w,C,r", [(2, 17, 30, 128, 3), (1, 55, 128, 256, 4), (3, 9, 17, 256, 4)], ids=str)
def test_realistic_statistics_far_outside(cuda, B, h, w, C, r):
    """randn feature maps (the dot products round in fp32): rb_corr_otf_lookup against fp64 under the per-tap a-priori
    bound of _bound_check, at the far-outside coordinate set (where a fixed tolerance fails: the weights grow like |x|).
    The bound is tight enough to catch a corner texel swapped for its neighbour (Ib <-> Ic): shown on a perturbed copy of
    the result made on the host."""
    from raft_b200 import capi
    lib = capi.lib
    g = torch.Generator().manual_seed(h + C)
    f1, f2 = torch.randn(B, h, w, C, generator=g), torch.randn(B, h, w, C, generator=g)
    f1d, f2d = f1.to(cuda), f2.to(cuda)
    wsb = capi.size_query(lib.rb_corr_otf_workspace_bytes, B, h, w, C)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
    capi.check(lib.rb_corr_otf_prepare(capi.ptr(f2d), capi.ptr(ws), wsb, B, h, w, C, capi.stream()))
    K = (2 * r + 1) ** 2
    worst, caught, n = 0.0, 0, 0
    for k, coords in enumerate(_coord_sets(B, h, w, seed=500 + k_seed(h, w), huge=False)):
        out = torch.empty(B, h, w, 4 * K, device=cuda)
        capi.check(lib.rb_corr_otf_lookup(capi.ptr(f1d), capi.ptr(f2d), capi.ptr(ws), capi.ptr(coords.to(cuda)), capi.ptr(out),
                                          B, h, w, C, r, capi.stream()))
        out = out.cpu().double()
        ref, bound, swap = _bound_check(f1, f2, coords, r)
        ratio = ((out - ref).abs() / bound.clamp_min(1e-300)).max().item()
        assert ratio <= 1.0, f"set {k}: the volume-free lookup leaves the a-priori bound (x{ratio:.2f})"
        worst = max(worst, ratio)
        pert = out + swap  # host-side copy with Ib and Ic swapped in every tap
        caught += int(((pert - ref).abs() > bound).sum())
        n += int((swap != 0).sum())
    print(f"\n{B}x{h}x{w} C={C}: worst |err| / bound {worst:.3f}; the Ib <-> Ic swap leaves the bound in {caught} of the "
          f"{n} taps it changes")
    assert caught >= 0.9 * n, "the bound is too loose to see a swapped corner texel"


# ---- f. engine level ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("volume_free", [False, True], ids=["volume", "volume_free"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_engine_survives_huge_and_infinite_flow_init(cuda, small, volume_free):
    """forward, then forward(flow_init=...) with entries of 3e9 and +inf (the fp16-range check runs on the first call
    only), then forward again: the warm call returns and raises nothing, and the last call equals the first bit for bit
    (no sticky CUDA error, no corrupted state)."""
    from raft_b200 import synth
    from raft_b200.engine import RaftEngine
    p = synth.make_weights(small)
    l, r = (torch.from_numpy(t) for t in synth.make_batch(2, 64, 96))
    eng = RaftEngine(p, small=small, iters=4, device=cuda, volume_free=volume_free)
    first = eng.forward(l, r).clone()
    fi = torch.zeros(2, 8, 12, 2)
    fi[0, :4, :, 0] = 3e9
    fi[0, 4:, :, 1] = INF
    fi[1, :, :6] = torch.tensor([-3e9, INF])
    low, up = eng.forward(l, r, flow_init=fi, return_low=True)
    torch.cuda.synchronize()
    assert up.shape == first.shape and low.shape == (2, 8, 12, 2)
    last = eng.forward(l, r).clone()
    torch.cuda.synchronize()
    assert torch.equal(_bits(last), _bits(first))


def test_bilinear_sample_huge_coordinates(cuda):
    """rb_bilinear_sample (the general sampler) has the same x0 + 1: bit-exact with the 64-bit truncation up to 2^62, and
    in bounds beyond (the values there are unspecified)."""
    from networks.utils import bilinear_sampler
    g = torch.Generator().manual_seed(4)
    img = torch.randint(-3, 4, (2, 9, 11, 1), generator=g).float()
    vals = _axis_values(11) + HUGE
    coords = torch.tensor([[a, b] for a in vals for b in vals[::3]], dtype=torch.float32)
    coords = torch.cat([coords, torch.rand(len(coords), 2, generator=g) * 10]).reshape(2, -1, 1, 2)
    out = bilinear_sampler(img.to(cuda), coords.to(cuda)).cpu()
    rows = _oracle_rows(coords)
    ref = O.bilinear_sampler(img, torch.where(rows[..., None], coords, torch.zeros(())))
    _assert_same(out, ref, rows, coords, "rb_bilinear_sample vs the 64-bit truncation")
