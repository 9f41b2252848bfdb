"""Configuration coverage of the wgmma conv kernel (conv_tc_kernel<BLOCK_N>, csrc/conv_tc.cu).

The kernel picks its tile width (choose_block_n), pixel box (choose_geom) and persistent grid / ring depth (launch_cfg) from
the problem size; at the small shapes of test_gpu_kernels.py that is almost always a 32-wide tile and one tile per CTA.
Here the test hook rb_debug_conv_override forces every width, box, ring depth and CTA cap, and each forced run is held to
  * the fp64 oracle, at the tolerance of test_gpu_kernels.py;
  * the automatic run, BIT FOR BIT wherever DESIGN section 4 says the accumulation order cannot depend on the configuration;
  * rb_debug_conv_last, which must report the forced configuration.
The division by sqrt(C) of the correlation epilogue is tested on operands whose products and sums are exact, so that the
quotient must equal the fp32 IEEE quotient bit for bit.  The last tests run the heuristic's own choices at full size.

Configurations recorded by rb_debug_conv_last are printed at the end of the module (pytest -s)."""
import contextlib
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import raft_oracle as O

pytestmark = pytest.mark.gpu

RING = {16: 5, 32: 5, 64: 4, 96: 3, 128: 3}  # TcCfg<N>::kStages: shared-memory ring depth per tile width
SEEN = set()  # (block_n, bw_log2, stages, tiles per CTA) of every launch this module checked

# (block_n, bw_log2, max_ctas, stages), 0 = automatic.  A pairwise set: together every width, every pixel box, stages 2 / 3 /
# the width's maximum, CTA caps 1 / 2 / 5 / none.  With a 1x1 conv over 64 channels (one k-iteration) every ring is deeper
# than the k loop; 18 k-iterations (3x3, 128 channels) do not divide by 4 or 5, so the ring wraps in the middle of a tile.
CONFIGS = [(16, 3, 1, 2), (32, 4, 2, 3), (64, 5, 5, 4), (96, 6, 0, 3), (128, 7, 1, 2),
           (32, 7, 5, 5), (96, 3, 2, 2), (128, 4, 0, 3), (64, 6, 1, 3), (16, 5, 0, 5)]


def _cfg_id(c):
    return "n{}_bw{}_cta{}_st{}".format(*c)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if SEEN:
        print("\nconv_tc configurations checked (BLOCK_N, bw_log2, stages, tiles per CTA):")
        for t in sorted(SEEN):
            print("  ", t)


# ---- the configuration the kernel should pick: a replay of choose_geom / choose_block_n / launch_cfg -----------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _geom(h, w, bwl=0):
    """(bw_log2, tiles_x, tiles_y) of choose_geom."""
    if bwl:
        return bwl, -(-w // (1 << bwl)), -(-h // (128 >> bwl))
    best = None
    for b in range(7, 2, -1):
        if (1 << b) > w and b > 3:
            continue
        t = (b, -(-w // (1 << b)), -(-h // (128 >> b)))
        if best is None or t[1] * t[2] < best[1] * best[2]:
            best = t
    return best


def _auto_block_n(cout, m_tiles, ctas):
    if cout <= 16:
        return 16
    best, best_cost = 128, None
    for n in (128, 96, 64, 32):
        waves = -(-(m_tiles * -(-cout // n)) // ctas)
        cost = waves * max(n + n // 2, 64 + (3 * n) // 4)
        if best_cost is None or cost < best_cost:
            best, best_cost = n, cost
    return best


def _ring(block_n, stages):
    return RING[block_n] if stages <= 0 else min(max(stages, 2), RING[block_n])


def _expected(cfg, B, h, w, cout):
    """Configuration of a stand-alone conv with output [B, h, w, cout] under `cfg` (no internal CTA limit)."""
    bn_f, bwl_f, ctas, st = cfg
    bwl, tx, ty = _geom(h, w, bwl_f)
    m_tiles = B * tx * ty
    bn = _auto_block_n(cout, m_tiles, _sms())
    if bn_f and bn != 16:
        bn = bn_f
    total = m_tiles * -(-cout // bn)
    units = min(ctas, _sms()) if ctas else _sms()
    return dict(block_n=bn, bw_log2=bwl, grid=min(total, units), stages=_ring(bn, st), total_tiles=total)


# ---- C ABI helpers ---------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _forced(cfg):
    from raft_b200 import capi
    capi.check(capi.lib.rb_debug_conv_override(*cfg))
    try:
        yield
    finally:
        capi.lib.rb_debug_conv_override(0, 0, 0, 0)


def _last():
    """rb_debug_conv_last as a dict (+ 'fused': convs since the override that produced fused instance-norm statistics)."""
    from raft_b200 import capi
    v = [C.c_int() for _ in range(5)]
    fused = capi.lib.rb_debug_conv_last(*[C.byref(x) for x in v])
    assert fused >= 0, capi.lib.rb_last_error()
    rec = dict(zip(("block_n", "bw_log2", "grid", "stages", "total_tiles"), (x.value for x in v)))
    rec["fused"] = fused
    SEEN.add((rec["block_n"], rec["bw_log2"], rec["stages"], -(-rec["total_tiles"] // rec["grid"])))
    return rec


def _check_record(rec, want, what):
    got = {k: rec[k] for k in want}
    assert got == want, f"{what}: rb_debug_conv_last reports {got}, expected {want}"


def _first_diff(a, b):
    d = (a != b) & ~(torch.isnan(a) & torch.isnan(b))
    i = tuple(int(j) for j in d.nonzero()[0])
    return f"{int(d.sum())} of {d.numel()} elements differ; first at {i}: {a[i].item()!r} vs {b[i].item()!r}"


def _assert_same_bits(out, want, what, against="the automatic configuration"):
    assert torch.equal(out, want), f"{what}: not bit-identical to {against}: {_first_diff(out, want)}"


def _assert_finite(t, what):
    assert torch.isfinite(t).all(), f"{what}: {int((~torch.isfinite(t)).sum())} non-finite outputs (unwritten?)"


# ---- a. stand-alone conv -----------------------------------------------------------------------------------------------------
from test_gpu_kernels import CONV_CASES  # noqa: E402  (the filter shapes of the update block + awkward tile geometries)

STRIDE2_CASES = [(2, 36, 52, 64, 96, 3), (1, 37, 51, 64, 96, 3)]  # even and odd sizes of test_conv2d_stride2
_CONV_REF = {}


def _conv_problem(B, h, w, cin, cout, kh, kw, stride, seed):
    key = (B, h, w, cin, cout, kh, kw, stride, seed)
    if key not in _CONV_REF:
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(B, h, w, cin, generator=g)
        W = torch.randn(kh, kw, cin, cout, generator=g) * (2.0 / (kh * kw * cin)) ** 0.5
        b = torch.randn(cout, generator=g) * 0.1
        _CONV_REF[key] = (x, W, b, O.conv2d(x.double(), W.double(), b.double(), stride, torch.relu))
    return _CONV_REF[key]


def _run_conv(cuda, x, W, b, stride, cfg):
    from raft_b200 import capi
    lib = capi.lib
    B, h, w, cin = x.shape
    kh, kw, _, cout = W.shape
    y = torch.full((B, -(-h // stride), -(-w // stride), cout), float("nan"), device=cuda)
    wsb = capi.size_query(lib.rb_conv2d_workspace_bytes, B, h, w, cin, cout, kh, kw)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
    xd = x.to(cuda)
    Wn, bn = np.ascontiguousarray(W.numpy()), np.ascontiguousarray(b.numpy())
    with _forced(cfg):
        if stride == 1:
            capi.check(lib.rb_conv2d(capi.ptr(xd), Wn.ctypes.data, bn.ctypes.data, capi.ptr(y), B, h, w, cin, cout, kh, kw, 1,
                                     capi.ptr(ws), wsb, capi.stream()))
        else:
            capi.check(lib.rb_conv2d_strided(capi.ptr(xd), Wn.ctypes.data, bn.ctypes.data, capi.ptr(y), B, h, w, cin, cout, kh,
                                             kw, stride, 1, capi.ptr(ws), wsb, capi.stream()))
        torch.cuda.synchronize()
        rec = _last()
    return y.cpu(), rec


def _conv_sweep(cuda, B, h, w, cin, cout, kh, kw, stride, seed):
    x, W, b, ref = _conv_problem(B, h, w, cin, cout, kh, kw, stride, seed)
    oh, ow = ref.shape[1], ref.shape[2]
    tol = 2e-5 * max(ref.abs().max().item(), 1.0)
    auto, rec = _run_conv(cuda, x, W, b, stride, (0, 0, 0, 0))
    _check_record(rec, _expected((0, 0, 0, 0), B, oh, ow, cout), "automatic")
    for cfg in CONFIGS:
        y, rec = _run_conv(cuda, x, W, b, stride, cfg)
        what = f"forced {_cfg_id(cfg)}"
        _check_record(rec, _expected(cfg, B, oh, ow, cout), what)
        _assert_finite(y, what)
        err = (y.double() - ref).abs().max().item()
        assert err < tol, f"{what}: max abs err {err:.3e} vs fp64 (tolerance {tol:.3e})"
        _assert_same_bits(y, auto, what)


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_forced_configs(cuda, case):
    """Every filter shape of the update block under every width / box / CTA cap / ring depth: fp64 parity and the same bits
    as the automatic configuration."""
    B, h, w, cin, cout, kh, kw = case
    _conv_sweep(cuda, B, h, w, cin, cout, kh, kw, 1, sum(case))


@pytest.mark.parametrize("case", STRIDE2_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_stride2_forced_configs(cuda, case):
    """The encoders' strided TMA views (TF SAME pads 0|1 on even, 1|1 on odd sizes) under forced configurations."""
    B, h, w, cin, cout, k = case
    _conv_sweep(cuda, B, h, w, cin, cout, k, k, 2, sum(case))


# ---- b. update block ---------------------------------------------------------------------------------------------------------
# widths whose z|r tile straddles `hidden`: things (hidden 128) 96 -> channels 96..191; small (hidden 96) 64 -> 64..127 and
# 128 -> 0..127.  CTA caps 1 and 2 run the whole block -- the forked convf1 / convf2 included -- with many tiles per CTA.
UPDATE_CONFIGS = {
    False: [(96, 0, 1, 0), (96, 5, 2, 2), (128, 3, 0, 3), (64, 7, 1, 4), (32, 4, 5, 5)],
    True: [(64, 0, 1, 0), (128, 4, 2, 2), (64, 6, 0, 3), (96, 3, 1, 3), (32, 7, 5, 5)],
}
_UPDATE_REF = {}


def _update_problem(small):
    if small not in _UPDATE_REF:
        from raft_b200 import synth
        B, h, w = 2, 12, 20
        hid, ctx, r = (96, 64, 3) if small else (128, 128, 4)
        p = synth.make_weights(small)
        g = torch.Generator().manual_seed(21)
        net = torch.tanh(torch.randn(B, h, w, hid, generator=g))
        inp = torch.relu(torch.randn(B, h, w, ctx, generator=g))
        corr = torch.randn(B, h, w, 4 * (2 * r + 1) ** 2, generator=g) * 3
        flow = torch.randn(B, h, w, 2, generator=g) * 2
        pt = {k: torch.from_numpy(v).double() for k, v in p.items()}
        blk = O.small_update_block if small else O.basic_update_block
        _UPDATE_REF[small] = (p, (net, inp, corr, flow), blk(net.double(), inp.double(), corr.double(), flow.double(), pt))
    return _UPDATE_REF[small]


def _run_update(cuda, small, args, cfg):
    from networks import model_utils as MU
    fn = MU.SmallUpdateBlock if small else MU.BasicUpdateBlock
    with _forced(cfg):
        n2, m2, d2 = fn(*[a.to(cuda) for a in args], "update_block", 96 if small else 128)
        torch.cuda.synchronize()
        rec = _last()
    return n2.cpu(), (None if m2 is None else m2.cpu()), d2.cpu(), rec


@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_update_block_forced_configs(cuda, small):
    from networks import model_utils as MU
    p, args, (rn, rm, rd) = _update_problem(small)
    MU.set_variables(p)
    auto = _run_update(cuda, small, args, (0, 0, 0, 0))
    for cfg in UPDATE_CONFIGS[small]:
        n2, m2, d2, rec = _run_update(cuda, small, args, cfg)
        what = f"{'small' if small else 'things'} forced {_cfg_id(cfg)}"
        # the last conv of the block: the flow head's 2-channel conv (16 wide, keeps its width) or the mask conv
        assert rec["block_n"] in (cfg[0], 16) and rec["stages"] == _ring(rec["block_n"], cfg[3]), (what, rec)
        assert rec["bw_log2"] == cfg[1] or not cfg[1], (what, rec)
        assert not cfg[2] or rec["grid"] <= cfg[2], (what, rec)
        outs = [("net", n2, auto[0], rn, 5e-5), ("delta", d2, auto[2], rd, 5e-5)]
        if not small:
            outs.append(("mask", m2, auto[1], rm, 1e-4))
        for name, out, a, ref, tol in outs:
            _assert_finite(out, f"{what} {name}")
            err = (out.double() - ref).abs().max().item()
            assert err < tol, f"{what} {name}: max abs err {err:.3e} vs fp64"
            _assert_same_bits(out, a, f"{what} {name}")


# ---- c. encoders -------------------------------------------------------------------------------------------------------------
ENCODER_CASES = [  # those of test_gpu_kernels.test_encoder
    (False, "fnet", "instance", 256, 2, 64, 96), (False, "cnet", "batch", 256, 1, 72, 104),
    (True, "fnet", "instance", 128, 2, 64, 96), (True, "cnet", "none", 160, 1, 72, 104),
    (False, "cnet", "batch", 256, 2, 71, 99), (True, "fnet", "instance", 128, 1, 67, 85)]
# width / CTA cap / ring depth only: the instance-norm statistics keep their strips, so the bits cannot change
ENCODER_EXACT = [(96, 0, 1, 2), (128, 0, 2, 3), (32, 0, 5, 5), (16, 0, 1, 0), (64, 0, 0, 4)]
# forced pixel boxes: the statistics strips follow the box, so their sums round differently (instance norm: tolerance only)
ENCODER_GEOM = [(0, 3, 0, 0), (0, 5, 2, 0), (128, 7, 1, 2)]
_ENC_REF = {}


def _run_encoder(cuda, p, name, small, norm, out_dim, img, cfg):
    from raft_b200.encoders import CudaEncoder
    with _forced(cfg):  # the workspace layout (statistics strips per tile) is sized under the same override
        out = CudaEncoder(p, name, small, norm, out_dim, cuda)(img.to(cuda))
        torch.cuda.synchronize()
        rec = _last()
    return out.cpu(), rec


@pytest.mark.parametrize("small,name,norm,out_dim,B,H,W", ENCODER_CASES)
def test_encoder_forced_configs(cuda, small, name, norm, out_dim, B, H, W):
    """The encoders under forced configurations.  With CTA caps 1 / 2 the fused instance-norm statistics are written by CTAs
    that walk many tiles; rb_debug_conv_last's count proves they were fused (and not the stand-alone pass)."""
    from raft_b200 import synth
    key = (small, name, norm, out_dim, B, H, W)
    p = synth.make_weights(small)
    img = torch.rand(B, H, W, 3, generator=torch.Generator().manual_seed(31))
    if key not in _ENC_REF:
        pt = {k: torch.from_numpy(v).double() for k, v in p.items()}
        _ENC_REF[key] = (O.small_encoder if small else O.basic_encoder)(2.0 * img.double() - 1.0, pt, name, norm)
    ref = _ENC_REF[key]
    tol = 1e-4 * max(ref.abs().max().item(), 1.0)
    auto, arec = _run_encoder(cuda, p, name, small, norm, out_dim, img, (0, 0, 0, 0))
    if norm == "instance":
        assert arec["fused"] > 0, "no conv produced fused instance-norm statistics"
    else:
        assert arec["fused"] == 0
    for cfg in ENCODER_EXACT + ENCODER_GEOM:
        out, rec = _run_encoder(cuda, p, name, small, norm, out_dim, img, cfg)
        what = f"{name} {norm} small={small} forced {_cfg_id(cfg)}"
        oh, ow = -(-H // 8), -(-W // 8)
        _check_record(rec, _expected(cfg, B, oh, ow, out_dim), what + " (last conv: conv2, 1x1)")
        assert rec["fused"] == arec["fused"], f"{what}: {rec['fused']} convs with fused statistics, {arec['fused']} without override"
        _assert_finite(out, what)
        err = (out.double() - ref).abs().max().item()
        assert err < tol, f"{what}: max abs err {err:.3e} vs fp64 (tolerance {tol:.3e})"
        if cfg[1] == 0 or norm != "instance":
            _assert_same_bits(out, auto, what)


# ---- d. correlation build ----------------------------------------------------------------------------------------------------
CORR_CONFIGS = [(128, 3, 1, 2), (96, 5, 2, 3), (64, 7, 5, 4), (32, 4, 0, 5), (16, 6, 1, 3)]


def _corr_build(cuda, f1, f2, cfg=(0, 0, 0, 0)):
    """rb_corr_build -> the four levels as [B*h*w, h_l*w_l] fp32 (CPU) and the record of the last GEMM (level 3)."""
    from raft_b200 import capi
    lib = capi.lib
    B, h, w, Cc = f1.shape
    nbytes = capi.size_query(lib.rb_corr_pyramid_bytes, B, h, w)
    buf = torch.full((nbytes // 4,), float("nan"), device=cuda)
    wsb = capi.size_query(lib.rb_corr_workspace_bytes, B, h, w, Cc)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
    f1d, f2d = f1.contiguous().to(cuda), f2.contiguous().to(cuda)
    with _forced(cfg):
        capi.check(lib.rb_corr_build(capi.ptr(f1d), capi.ptr(f2d), capi.ptr(buf), B, h, w, Cc, capi.ptr(ws), wsb, capi.stream()))
        torch.cuda.synchronize()
        rec = _last()
    levels, off = [], 0
    for l in range(4):
        n = B * h * w * (h >> l) * (w >> l)
        levels.append(buf[off:off + n].view(B * h * w, (h >> l) * (w >> l)))
        off += n
    return levels, rec


@pytest.mark.parametrize("B,h,w,Cc", [(1, 40, 56, 128), (2, 36, 44, 256)])
def test_corr_build_forced_configs(cuda, B, h, w, Cc):
    """The correlation GEMMs (per-batch B operand) under forced configurations: fp64 parity and the automatic run's bits."""
    g = torch.Generator().manual_seed(11)
    f1 = torch.randn(B, h, w, Cc, generator=g)
    f2 = torch.randn(B, h, w, Cc, generator=g)
    ref = [r.reshape(B * h * w, -1) for r in O.get_corr_pyramid(f1.double(), f2.double())]
    tol = 2e-5 * ref[0].abs().max().item()
    auto, _ = _corr_build(cuda, f1, f2)
    for cfg in CORR_CONFIGS:
        levels, rec = _corr_build(cuda, f1, f2, cfg)
        what = f"corr B={B} {h}x{w} C={Cc} forced {_cfg_id(cfg)}"
        rows3 = (h >> 3) * (w >> 3)
        _check_record(rec, _expected(cfg, B, h, w, rows3), what + " (level 3)")
        for l in range(4):
            out = levels[l].cpu()
            _assert_finite(out, f"{what} level {l}")
            err = (out.double() - ref[l]).abs().max().item()
            assert err < tol, f"{what} level {l}: max abs err {err:.3e} vs fp64 (tolerance {tol:.3e})"
            _assert_same_bits(out, auto[l].cpu(), f"{what} level {l}")


def _fp32_quotient(v, Cc):
    """The reference's corr / tf.sqrt(float(C)) in fp32 (model_utils.py:213): IEEE-rounded quotient."""
    return v.float() / torch.sqrt(torch.tensor(float(Cc)))


@pytest.mark.parametrize("Cc", [128, 256])
def test_corr_sqrt_c_division_exact(cuda, Cc):
    """Level 0 = fl(v / fl(sqrt C)) BIT FOR BIT when the GEMM result v is exact.  fmap1 is one-hot and every fmap2 entry has at
    most 22 significant bits (hi + 2^-11 lo is then exact), so each level-0 entry is one fmap2 entry: a dense sweep of
    quotients over 17 binades.  C = 128: the call-free correctly rounded division (div_rn); C = 256: the power-of-two scaling."""
    B, h, w = 1, 32, 48
    N = h * w
    g = torch.Generator().manual_seed(5)
    f1 = torch.zeros(N, Cc)
    f1[torch.arange(N), torch.arange(N) % Cc] = 1.0
    mant = torch.randint(0, 1 << 21, (N, Cc), generator=g, dtype=torch.int64)
    mant[0, :4] = torch.tensor([0, (1 << 21) - 1, 1 << 10, (1 << 11) - 1])  # 1.0, all 22 bits set, fp16 hi tie, hi rounds up
    expo = torch.randint(-6, 11, (N, Cc), generator=g, dtype=torch.int64)
    sign = torch.where(torch.rand(N, Cc, generator=g) < 0.5, -1.0, 1.0).double()
    v = sign * torch.ldexp(1.0 + mant.double() / (1 << 21), expo.double())
    f2 = v.float()
    assert torch.equal(f2.double(), v), "fmap2 entries must be exact fp32"
    levels, _ = _corr_build(cuda, f1.view(B, h, w, Cc), f2.view(B, h, w, Cc))
    got = levels[0].cpu()
    want = _fp32_quotient(f2.t()[torch.arange(N) % Cc], Cc)  # [n, m] = fmap2[m, n % C] / sqrt(C)
    _assert_same_bits(got, want, f"level 0, C={Cc}", "the fp32 quotient")


@pytest.mark.parametrize("Cc", [128, 256])
def test_corr_pyramid_levels_exact_small_integers(cuda, Cc):
    """With small-integer feature maps every pooled operand and every partial sum is exact in fp32, so level l must equal
    fl(fmap1 . pool^l(fmap2) / fl(sqrt C)) bit for bit at every level."""
    B, h, w = 2, 20, 28
    g = torch.Generator().manual_seed(9)
    f1 = torch.randint(-3, 4, (B, h, w, Cc), generator=g).float()
    f2 = torch.randint(-3, 4, (B, h, w, Cc), generator=g).float()
    levels, _ = _corr_build(cuda, f1, f2)
    pooled = f2.double()
    for l in range(4):
        if l:
            pooled = O.avg_pool_2x2_valid(pooled)
        exact = torch.einsum("bnc,bmc->bnm", f1.double().reshape(B, h * w, Cc), pooled.reshape(B, -1, Cc)).reshape(B * h * w, -1)
        assert torch.equal(exact.float().double(), exact)
        _assert_same_bits(levels[l].cpu(), _fp32_quotient(exact, Cc), f"level {l}, C={Cc}", "fl(exact sum / fl(sqrt C))")


# ---- e. the heuristic's own choices at full size (55 x 128 feature grid) ------------------------------------------------------
@pytest.mark.parametrize("cout,block_n", [(192, 96), (256, 128)])
def test_fullsize_conv_natural_config(cuda, cout, block_n):
    """3x3 conv over 256 channels at B = 2 on the 55 x 128 grid: the cost model picks a 96 / 128-wide tile and CTAs that walk
    more than one tile -- compared with fp64."""
    B, h, w, cin = 2, 55, 128, 256
    x, W, b, ref = _conv_problem(B, h, w, cin, cout, 3, 3, 1, 7)
    y, rec = _run_conv(cuda, x, W, b, 1, (0, 0, 0, 0))
    _check_record(rec, _expected((0, 0, 0, 0), B, h, w, cout), "automatic")
    assert rec["block_n"] == block_n and rec["total_tiles"] > rec["grid"], rec
    _assert_finite(y, "full size")
    err = (y.double() - ref).abs().max().item()
    assert err < 2e-5 * max(ref.abs().max().item(), 1.0), f"max abs err {err:.3e}"


def test_fullsize_corr_build_natural_config(cuda):
    """rb_corr_build at B = 2, 55 x 128, C = 256: level 0 runs 128-wide tiles, dozens per CTA, over the per-batch B operand.
    About 512 sampled rows per batch against fp64: level 0 as the fp64 matmul, levels 1-3 as VALID 2x2 pools of that row."""
    B, h, w, Cc = 2, 55, 128, 256
    N = h * w
    g = torch.Generator().manual_seed(13)
    f1 = torch.randn(B, h, w, Cc, generator=g)
    f2 = torch.randn(B, h, w, Cc, generator=g)
    levels, rec = _corr_build(cuda, f1, f2)
    # the last GEMM is level 3 (6 x 16 = 96 rows); the replay of the heuristic, which every automatic launch in this module
    # is held to, puts level 0 (7040 rows) on 128-wide tiles with many tiles per CTA
    _check_record(rec, _expected((0, 0, 0, 0), B, h, w, (h >> 3) * (w >> 3)), "level 3")
    lv0 = _expected((0, 0, 0, 0), B, h, w, N)
    assert lv0["block_n"] == 128 and lv0["total_tiles"] >= 8 * lv0["grid"], lv0
    rows = torch.randperm(N, generator=g)[:512]
    scale, errs = 0.0, [0.0] * 4
    for bb in range(B):
        r0 = f1[bb].reshape(N, Cc)[rows].double() @ f2[bb].reshape(N, Cc).double().t() / math.sqrt(Cc)  # [512, N]
        ref = r0.reshape(-1, h, w, 1)
        scale = max(scale, r0.abs().max().item())
        for l in range(4):
            if l:
                ref = O.avg_pool_2x2_valid(ref)
            out = levels[l][bb * N + rows.to(levels[l].device)].cpu()
            _assert_finite(out, f"level {l}")
            errs[l] = max(errs[l], (out.double() - ref.reshape(len(rows), -1)).abs().max().item())
    for l in range(4):
        assert errs[l] < 2e-5 * scale, f"level {l}: max abs err {errs[l]:.3e} (scale {scale:.2f})"
