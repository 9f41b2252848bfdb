"""Every conv path held BIT FOR BIT to the exact value of its arithmetic (tests/exact_oracle.py).

On operands whose products and partial sums are exact in fp32 (certified per conv), RB_MATH_TC must return
hi*hi + 2^-11 (hi*lo + lo*hi), RB_MATH_TC_FP16 hi*hi and RB_MATH_SIMT the product of the joined operands, exactly, whatever
tile width, pixel box, ring depth, CTA cap, split-K half or CTA pair the launch uses.  A dropped tap, a misread lo plane or
padding offset, or a wrong epilogue operand then shows as a nonzero difference.  Every comparison is torch.equal after a
finiteness check (torch.equal does not tell -0 from +0).  Every stand-alone conv runs with relu = 0, so negative outputs are
compared too.
  A. stand-alone rb_conv2d / rb_conv2d_strided: the shapes of test_gpu_kernels / test_gpu_conv_coverage, both semantics,
     every back end on each family its model covers, and every forced configuration of both configuration sweeps;
  B. both encoders with norm "none" (stem, strided views, residual joins, 16-wide tiles, channel padding);
  C. the update block's flow and mask heads: with convz at zero weight and bias -1000 the gate z is +0 exactly
     (sigmoid_f = rcp.approx(1 + ex2.approx(+1442.7)) = rcp(+inf) = +0), so net passes the GRU unchanged and delta, coords1
     and mask are exact functions of it.
Configurations recorded by rb_debug_conv_last are printed at the end of the module (pytest -s)."""
import contextlib
import functools

import numpy as np
import pytest
import torch

import exact_oracle as E
from oracle import raft_oracle as O
from test_gpu_conv_coverage import (CONFIGS, ENCODER_CASES, ENCODER_EXACT, ENCODER_GEOM, SEEN, STRIDE2_CASES, _cfg_id,
                                    _check_record, _expected, _first_diff, _forced, _last)
from test_gpu_kernels import CONV_CASES
from test_gpu_mixed_precision import CONFIGS as MP_CONFIGS, _passes, _ring as _mp_ring

pytestmark = pytest.mark.gpu


def _capi():
    from raft_b200 import capi
    return capi


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if SEEN:
        print("\nconv_tc configurations checked (BLOCK_N, bw_log2, stages, tiles per CTA):")
        for t in sorted(SEEN):
            print("  ", t)


@pytest.fixture(autouse=True)
def _reset_thread_state():
    yield
    c = _capi()
    c.lib.rb_set_math_mode(c.RB_MATH_TC)
    c.lib.rb_set_semantics(c.RB_SEMANTICS_REFERENCE)
    c.lib.rb_debug_conv_override(0, 0, 0, 0)


@contextlib.contextmanager
def _mode(back_end, upstream=False):
    c = _capi()
    c.check(c.lib.rb_set_math_mode({E.TC: c.RB_MATH_TC, E.SIMT: c.RB_MATH_SIMT, E.FP16: c.RB_MATH_TC_FP16}[back_end]))
    c.check(c.lib.rb_set_semantics(c.RB_SEMANTICS_UPSTREAM if upstream else c.RB_SEMANTICS_REFERENCE))
    try:
        yield
    finally:
        c.lib.rb_set_math_mode(c.RB_MATH_TC)
        c.lib.rb_set_semantics(c.RB_SEMANTICS_REFERENCE)


def _assert_exact(out, want, what):
    out = out.cpu()
    assert torch.isfinite(out).all(), f"{what}: {int((~torch.isfinite(out)).sum())} non-finite outputs (unwritten?)"
    assert out.dtype == torch.float32 and out.shape == want.shape, (what, out.dtype, out.shape, want.shape)
    want = want.float()
    assert torch.equal(out, want), f"{what}: not the exact value: {_first_diff(out, want)}"


# ---- A. stand-alone convs --------------------------------------------------------------------------------------------------
# (B, h, w, cin, cout, kh, kw), stride, upstream semantics
STRIDE2_MORE = [(1, 40, 56, 3, 64, 7), (1, 39, 57, 3, 32, 7), (1, 9, 300, 16, 16, 3)]  # test_gpu_kernels.test_conv2d_stride2
S2 = [(B, h, w, ci, co, k, k) for (B, h, w, ci, co, k) in STRIDE2_CASES + STRIDE2_MORE]
CASES = [(c, 1, False) for c in CONV_CASES] + [(c, 2, False) for c in S2] + [(c, 2, True) for c in S2]
_MODEL = {}


CASE_IDS = ["{}-s{}-{}".format("x".join(map(str, c)), s, "upstream" if u else "reference") for c, s, u in CASES]


@functools.lru_cache(maxsize=None)
def _operands(case, stride, upstream, family):
    B, h, w, cin, cout, kh, kw = case
    return E.operands(family, (B, h, w, cin), (kh, kw, cin, cout), sum(case) + stride, stride, upstream)


def _problem(case, stride, upstream, family, back_end):
    """(x, W, b, exact model value without activation), cached per case / family / back end."""
    key = (case, stride, upstream, family, back_end)
    if key not in _MODEL:
        x, W, b = _operands(case, stride, upstream, family)
        _MODEL[key] = (x, W, b, E.certify(x, W, b, stride, back_end, upstream))
    return _MODEL[key]


def _run(cuda, x, W, b, stride, relu, cfg=(0, 0, 0, 0), record=True):
    c = _capi()
    lib = c.lib
    B, h, w, cin = x.shape
    kh, kw, _, cout = W.shape
    y = torch.full((B, -(-h // stride), -(-w // stride), cout), float("nan"), device=cuda)
    wsb = c.size_query(lib.rb_conv2d_workspace_bytes, B, h, w, cin, cout, kh, kw)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
    xd = x.contiguous().to(cuda)
    Wn, bn = np.ascontiguousarray(W.numpy()), np.ascontiguousarray(b.numpy())
    with _forced(cfg):
        c.check(lib.rb_conv2d_strided(c.ptr(xd), Wn.ctypes.data, bn.ctypes.data, c.ptr(y), B, h, w, cin, cout, kh, kw, stride,
                                      relu, c.ptr(ws), wsb, c.stream()))
        torch.cuda.synchronize()
        rec = _last() if record else None
    return y.cpu(), rec


@pytest.mark.parametrize("case,stride,upstream", CASES, ids=CASE_IDS)
def test_conv_exact(cuda, case, stride, upstream):
    """Every back end on every family its model covers, relu = 0; relu = 1 once (family X, RB_MATH_TC)."""
    B, h, w, cin, cout, kh, kw = case
    for back_end, families in E.FAMILIES.items():
        for family in families:
            x, W, b, want = _problem(case, stride, upstream, family, back_end)
            what = f"{back_end} family {family}"
            with _mode(back_end, upstream):
                y, rec = _run(cuda, x, W, b, stride, 0, record=back_end != E.SIMT)
                if back_end == E.FP16:
                    assert _passes() == 1, what
                elif back_end == E.TC:
                    assert _passes() == 3, what
                    _check_record(rec, _expected((0, 0, 0, 0), B, want.shape[1], want.shape[2], cout), what)
            assert (want < 0).any() and (want > 0).any(), what
            _assert_exact(y, want, what)
    x, W, b, want = _problem(case, stride, upstream, "X", E.TC)
    with _mode(E.TC, upstream):
        y, _ = _run(cuda, x, W, b, stride, 1)
    _assert_exact(y, torch.relu(want), "tc family X relu")


SWEEP_CASES = [(c, 1, False) for c in CONV_CASES] + [(c, 2, False) for c in S2[:2]]


@pytest.mark.parametrize("family", ["X", "XW"])
@pytest.mark.parametrize("case,stride,upstream", SWEEP_CASES, ids=[CASE_IDS[CASES.index(c)] for c in SWEEP_CASES])
def test_conv_exact_forced_configs(cuda, case, stride, upstream, family):
    """test_gpu_conv_coverage.CONFIGS under RB_MATH_TC and test_gpu_mixed_precision.CONFIGS under RB_MATH_TC_FP16: every
    tile width, pixel box, ring depth and CTA cap gives the exact value, and rb_debug_conv_last reports the forced
    configuration."""
    B = case[0]
    for back_end, configs in ((E.TC, CONFIGS), (E.FP16, MP_CONFIGS)):
        x, W, b, want = _problem(case, stride, upstream, family, back_end)
        oh, ow, cout = want.shape[1:]
        for cfg in configs:
            what = f"{back_end} family {family} forced {_cfg_id(cfg)}"
            with _mode(back_end, upstream):
                y, rec = _run(cuda, x, W, b, stride, 0, cfg)
                assert _passes() == (1 if back_end == E.FP16 else 3), what
            exp = _expected(cfg, B, oh, ow, cout)
            if back_end == E.FP16:
                exp["stages"] = _mp_ring(cfg[3])
            _check_record(rec, exp, what)
            _assert_exact(y, want, what)


@pytest.mark.parametrize("cout,block_n", [(192, 96), (256, 128)])
def test_fullsize_conv_exact_natural_config(cuda, cout, block_n):
    """3x3 over 256 channels at B = 2 on the 55 x 128 grid: the heuristic's 96 / 128-wide tiles, CTAs walking many tiles."""
    case = (2, 55, 128, 256, cout, 3, 3)
    x, W, b, want = _problem(case, 1, False, "X", E.TC)
    y, rec = _run(cuda, x, W, b, 1, 0)
    _check_record(rec, _expected((0, 0, 0, 0), 2, 55, 128, cout), "automatic")
    assert rec["block_n"] == block_n and rec["total_tiles"] > rec["grid"], rec
    _assert_exact(y, want, "full size")


# ---- B. encoders -----------------------------------------------------------------------------------------------------------
ENC_SHAPES = sorted({(small, B, H, W) for (small, _, _, _, B, H, W) in ENCODER_CASES})
_ENC = {}


def _out_dim(small):
    return 128 if small else 256


def _encoder_problem(small, B, H, W, back_end, upstream):
    from raft_b200 import synth
    key = (small, B, H, W, back_end, upstream)
    if key not in _ENC:
        p = E.chain_weights(synth.make_weights(small), "fnet", 100 + int(small))
        img = E.exact_images(B, H, W, B * H + W)
        _ENC[key] = (p, img, E.encoder_model(p, "fnet", small, img, back_end, upstream))
    return _ENC[key]


def _run_encoder(cuda, p, small, img, cfg=(0, 0, 0, 0)):
    from raft_b200.encoders import CudaEncoder
    with _forced(cfg):
        out = CudaEncoder(p, "fnet", small, "none", _out_dim(small), cuda)(img.to(cuda))
        torch.cuda.synchronize()
        rec = _last()
    return out.cpu(), rec


@pytest.mark.parametrize("upstream", [False, True], ids=["reference", "upstream"])
@pytest.mark.parametrize("small,B,H,W", ENC_SHAPES, ids=lambda v: str(v))
def test_encoder_exact(cuda, small, B, H, W, upstream):
    for back_end in (E.TC, E.SIMT, E.FP16):
        p, img, want = _encoder_problem(small, B, H, W, back_end, upstream)
        with _mode(back_end, upstream):
            out, _ = _run_encoder(cuda, p, small, img)
        _assert_exact(out, want, f"{'small' if small else 'basic'} encoder {back_end}")


@pytest.mark.parametrize("small,B,H,W", ENC_SHAPES, ids=lambda v: str(v))
def test_encoder_exact_forced_configs(cuda, small, B, H, W):
    """test_gpu_conv_coverage's ENCODER_EXACT + ENCODER_GEOM: with norm "none" the forced pixel boxes give exact bits too."""
    p, img, want = _encoder_problem(small, B, H, W, E.TC, False)
    for cfg in ENCODER_EXACT + ENCODER_GEOM:
        what = f"{'small' if small else 'basic'} encoder forced {_cfg_id(cfg)}"
        out, rec = _run_encoder(cuda, p, small, img, cfg)
        _check_record(rec, _expected(cfg, B, -(-H // 8), -(-W // 8), _out_dim(small)), what + " (last conv: conv2, 1x1)")
        assert rec["fused"] == 0, what
        _assert_exact(out, want, what)


def test_encoder_exact_fullsize(cuda):
    """The basic encoder at 440 x 1024 in its natural configuration."""
    p, img, want = _encoder_problem(False, 1, 440, 1024, E.TC, False)
    out, _ = _run_encoder(cuda, p, False, img)
    _assert_exact(out, want, "basic encoder 440x1024")


# ---- C. update-block heads -------------------------------------------------------------------------------------------------
def _head_problem(small, B, h, w, family, seed):
    """Weights with convz at zero / bias -1000 and exact flow / mask heads, and the state: net from the family (X: H + L/2048,
    I: small integers), inp, corr."""
    from raft_b200 import synth
    hid, ctx = (96, 64) if small else (128, 128)
    p = dict(synth.make_weights(small))
    for z in (["gru/convz"] if small else ["gru/convz1", "gru/convz2"]):
        k = f"update_block/{z}"
        p[k + "/W"] = np.zeros_like(p[k + "/W"])
        p[k + "/b"] = np.full_like(p[k + "/b"], -1000.0)
    p = E.chain_weights(p, "update_block/flow_head", seed)
    if not small:
        p = E.chain_weights(p, "update_block/mask", seed + 1)
    g = torch.Generator().manual_seed(seed)
    net = E._activations(family, (B, h, w, hid), g).float()
    inp = torch.relu(torch.randn(B, h, w, ctx, generator=g))
    corr = torch.randn(B, h, w, 4 * (2 * (3 if small else 4) + 1) ** 2, generator=g) * 3
    return p, net, inp, corr


def _head_model(p, net, small, back_end):
    pt = {k: torch.from_numpy(np.asarray(v)).double() for k, v in p.items() if k.startswith("update_block/")}
    with E.exact_convs(back_end):
        delta = O.flow_head(net.double(), pt, "update_block/flow_head")
        mask = None
        if not small:
            m = O._conv(net.double(), pt, "update_block/mask/0", 1, torch.relu)
            mask = 0.25 * O._conv(m, pt, "update_block/mask/2", 1)
    return delta, mask


class _Heads:
    """rb_update_set_state + rb_update_set_corr + rb_coords_grid, then rb_update_step or rb_raft_iterate."""

    def __init__(self, cuda, small, p, net, inp, corr):
        from raft_b200.weights import pack_update_block
        c = _capi()
        self.c, self.lib, self.s = c, c.lib, int(small)
        self.B, self.h, self.w = net.shape[:3]
        self.blob = pack_update_block(p, small, cuda)
        q = c.size_query
        self.ws = torch.zeros(q(self.lib.rb_update_workspace_bytes, self.s, *self._dims()), dtype=torch.uint8, device=cuda)
        self.pyramid = torch.zeros(q(self.lib.rb_corr_pyramid_bytes, *self._dims()) // 4, device=cuda)
        self.coords1 = torch.empty(self.B, self.h, self.w, 2, device=cuda)
        self.delta = torch.full((self.B, self.h, self.w, 2), float("nan"), device=cuda)
        self.mask = None if small else torch.full((self.B, self.h, self.w, 576), float("nan"), device=cuda)
        self.net_out = torch.empty_like(net, device=cuda)
        self.net, self.inp, self.corr = (t.contiguous().to(cuda) for t in (net, inp, corr))
        P, st = c.ptr, c.stream()
        c.check(self.lib.rb_update_set_state(self.s, P(self.blob), P(self.ws), P(self.net), P(self.inp), *self._dims(), st))
        c.check(self.lib.rb_update_set_corr(self.s, P(self.ws), P(self.corr), *self._dims(), st))
        c.check(self.lib.rb_coords_grid(P(self.coords1), *self._dims(), st))

    def _dims(self):
        return self.B, self.h, self.w

    def step(self, with_mask=True):
        P = self.c.ptr
        self.c.check(self.lib.rb_update_step(self.s, P(self.blob), P(self.ws), P(self.coords1), P(self.delta),
                                             P(self.mask if with_mask else None), *self._dims(), self.c.stream()))
        torch.cuda.synchronize()

    def iterate(self, n):
        P = self.c.ptr
        self.c.check(self.lib.rb_raft_iterate(self.s, P(self.blob), P(self.ws), P(self.pyramid), P(self.coords1), P(self.mask),
                                              *self._dims(), n, self.c.stream()))
        torch.cuda.synchronize()

    def get_net(self):
        P = self.c.ptr
        self.c.check(self.lib.rb_update_get_net(self.s, P(self.ws), P(self.net_out), *self._dims(), self.c.stream()))
        return self.net_out.cpu()


def _check_heads(cuda, small, B, h, w, family, back_end, cfg):
    p, net, inp, corr = _head_problem(small, B, h, w, family, 7 * B + h + w)
    delta, mask = _head_model(p, net, small, back_end)
    grid = O.coords_grid(B, h, w)
    what = f"{'small' if small else 'things'} {B}x{h}x{w} family {family} {back_end} forced {_cfg_id(cfg)}"
    with _mode(back_end), _forced(cfg):
        hd = _Heads(cuda, small, p, net, inp, corr)
        hd.step(with_mask=False)  # the flow head's split-K conv is the step's last conv
        rec = _last() if back_end != E.SIMT else None
        _assert_exact(hd.get_net(), net.double(), what + " net")
        _assert_exact(hd.delta, delta, what + " delta")
        _assert_exact(hd.coords1, grid + delta.float(), what + " coords1")
        if not small:
            hd.step()
            _assert_exact(hd.mask, mask, what + " mask")
        fused = _Heads(cuda, small, p, net, inp, corr)
        fused.iterate(3)
        c1 = grid
        for _ in range(3):
            c1 = c1 + delta.float()
        _assert_exact(fused.coords1, c1, what + " rb_raft_iterate coords1")
        _assert_exact(fused.get_net(), net.double(), what + " rb_raft_iterate net")
        if not small:
            _assert_exact(fused.mask, mask, what + " rb_raft_iterate mask")
    return rec


@pytest.mark.parametrize("back_end", [E.TC, E.SIMT, E.FP16])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
@pytest.mark.parametrize("B,h,w", [(2, 12, 20), (1, 55, 128)], ids=lambda v: str(v))
def test_update_heads_exact(cuda, B, h, w, small, back_end):
    """net unchanged, delta = flow_head(net), coords1 = fl32(coords1 + delta), mask = 0.25 mask_head(net); N = 3 fused
    iterations = the stepwise fp32 sums.  At B = 1 on 55 x 128 the flow head's conv2 has 55 pixel tiles, 2 * 55 <= 132 SMs:
    launch_cfg puts its split-K halves on CTA pairs (grid 110); under rb_debug_conv_override(0, 0, 1, 0) no pairs."""
    for family in ("X", "I"):
        rec = _check_heads(cuda, small, B, h, w, family, back_end, (0, 0, 0, 0))
        if rec is not None:
            assert rec["block_n"] == 16, rec
            if B == 1 and (h, w) == (55, 128):
                assert rec["total_tiles"] == 55 and rec["grid"] == 2 * rec["total_tiles"], f"expected CTA pairs: {rec}"
        rec = _check_heads(cuda, small, B, h, w, family, back_end, (0, 0, 1, 0))
        if rec is not None:
            assert rec["grid"] == 1, rec
