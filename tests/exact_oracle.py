"""Exact models of the conv back ends on operands whose products and partial sums are exact (TEST INFRASTRUCTURE ONLY).

Every back end of include/raft_b200.h specifies its arithmetic exactly:
  * split_f32 (csrc/common.cuh): clamp to +-65504, hi = fp16_rn(a), lo = fp16_rn((a - hi) * 2048);
  * RB_MATH_TC: sum hi_a hi_w + 2^-11 sum (hi_a lo_w + lo_a hi_w), lo * lo dropped  (O.EMULATE = "fp16x3");
  * RB_MATH_TC_FP16: sum hi_a hi_w  (O.EMULATE = "fp16");
  * RB_MATH_SIMT: fp32 FMAs of the joined operands hi + 2^-11 lo  (plain fp64 on them).
If every term of every accumulator is a multiple of one quantum q and, for every output, sum |terms| + |bias| < 2^24 q, then
every partial sum is exact in fp32 in any order -- any tile width, pixel box, ring depth, CTA cap, split-K half, and whatever
order the tensor cores add in -- so the kernel must return the model's value bit for bit.  ``certify`` checks that condition
for one conv and returns the model's value; ``exact_convs`` swaps it into oracle.raft_oracle so that the encoders and heads
run on it, every conv certifying itself.

Operand families (``operands``), seeded and deterministic:
  I   small integers on both sides: both lo planes are zero;
  X   activations H + L/2048, integer H in +-[8, 16) or 0, L in [-7, 7] (hi = H, lo = L; for H = 0 hi = L/2048, lo = 0),
      small-integer weights;
  W   the mirror of X: small-integer activations, weights H + L/2048;
  XW  both operands H + L/2048 with H in +-{2, 3}, L in [-1, 1], or exactly 0.  RB_MATH_SIMT keeps the lo * lo terms,
      whose fp32 sums are not exact: XW is for RB_MATH_TC and RB_MATH_TC_FP16 only.
Biases are multiples of the quantum; the weights are thinned until the bound leaves a factor 2 of headroom.
"""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O

TC, SIMT, FP16 = "tc", "simt", "fp16"
FAMILIES = {TC: ("I", "X", "W", "XW"), SIMT: ("I", "X", "W"), FP16: ("I", "X", "W", "XW")}
LO = 2.0 ** -11
LIMIT = 2.0 ** 24    # sum |terms| < LIMIT * q: every partial sum exact in fp32
STORED = 2.0 ** 15   # stored activations stay below this: split exactly, and far inside the fp16 range
_EMULATE = {TC: "fp16x3", FP16: "fp16", SIMT: None}


# ---- split_f32 -------------------------------------------------------------------------------------------------------------
def split(a):
    """split_f32 bit for bit: fp32 values -> (hi, lo) as fp16 numpy arrays."""
    a = np.clip(np.asarray(a, dtype=np.float32), np.float32(-65504.0), np.float32(65504.0))
    hi = a.astype(np.float16)
    lo = ((a - hi.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
    return hi, lo


def planes(t):
    """(hi, lo, joined) of an fp32 tensor as fp64 torch tensors; joined = hi + 2^-11 lo, what the CUDA cores multiply."""
    hi, lo = split(t.detach().cpu().float().numpy())
    hi, lo = torch.from_numpy(hi.astype(np.float64)), torch.from_numpy(lo.astype(np.float64))
    return hi, lo, hi + LO * lo


def quantum(t) -> float:
    """The largest power of two that divides every entry of t (inf if t is all zero)."""
    v = np.abs(np.asarray(t, dtype=np.float64)).ravel()
    v = v[v != 0]
    if v.size == 0:
        return math.inf
    m, e = np.frexp(v)
    n = (m * 2.0 ** 53).astype(np.int64)
    low = (n & -n).astype(np.float64)
    return math.ldexp(1.0, int((np.log2(low) + e - 53).min()))


# ---- the models ----------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def model(back_end):
    """O.EMULATE of the back end while the block runs (None for RB_MATH_SIMT: fp64 on the joined operands)."""
    saved = O.EMULATE
    O.EMULATE = _EMULATE[back_end]
    try:
        yield
    finally:
        O.EMULATE = saved


def _conv(x, W, stride, upstream):
    """conv of NHWC x with HWIO W, no bias, under O.EMULATE.  Reference semantics: TF 'SAME' (O.conv2d); upstream stride 2:
    PyTorch's symmetric k // 2 (tests/upstream_oracle.conv2d_up), which calls F.conv2d directly -- routed through the
    emulation here."""
    kh, kw = int(W.shape[0]), int(W.shape[1])
    if upstream and stride != 1:
        pad = (kw // 2, kw // 2, kh // 2, kh // 2)
    else:
        pt, pb = O._same_pad(x.shape[1], kh, stride)
        pl, pr = O._same_pad(x.shape[2], kw, stride)
        pad = (pl, pr, pt, pb)
    xn = F.pad(x.permute(0, 3, 1, 2), pad)
    Wn = W.permute(3, 2, 0, 1).contiguous()
    op = lambda u, v: F.conv2d(u, v, None, stride=stride)  # noqa: E731
    y = op(xn, Wn) if O.EMULATE is None else O._emulated_bilinear(op, xn, Wn)
    return y.permute(0, 2, 3, 1)


def _terms(x, W, back_end):
    """[(activation operand, weight operand, scale)]: the products each back end accumulates."""
    ha, la, ja = planes(x)
    hw, lw, jw = planes(W)
    if back_end == TC:
        return [(ha, hw, 1.0), (ha, lw, LO), (la, hw, LO)]
    if back_end == FP16:
        return [(ha, hw, 1.0)]
    return [(ja, jw, 1.0)]


def _bound(x, W, b, stride, back_end, upstream):
    """(max over outputs of sum |terms| + |b|, the quantum q that divides every term and the bias, the bias in fp64)."""
    terms = _terms(x, W, back_end)
    b64 = torch.zeros(W.shape[3], dtype=torch.float64) if b is None else b.float().double()
    q = min([quantum(a) * quantum(w) * s for a, w, s in terms] + [quantum(b64)])
    with model(SIMT):
        bound = sum(_conv(a.abs(), w.abs(), stride, upstream) * s for a, w, s in terms) + b64.abs()
    return bound.max().item(), q, b64


def headroom(x, W, b=None, stride=1, back_end=TC, upstream=False):
    """max over outputs of (sum |terms| + |b|) / (2^24 q): certify requires < 1."""
    worst, q, _ = _bound(x.float(), W.float(), b, stride, back_end, upstream)
    return worst / (LIMIT * q)


def certify(x, W, b=None, stride=1, back_end=TC, upstream=False):
    """The back end's value of conv(x, W) + b (fp64, no activation), asserting that it is the kernel's exact result: every
    term a multiple of one quantum q, the bias too, sum |terms| + |b| < 2^24 q at every output, the value fp32.  x NHWC and
    W HWIO fp32; RB_MATH_SIMT additionally needs operands that equal their joined split."""
    x, W = x.float(), W.float()
    if back_end == SIMT:
        for t, name in ((x, "activation"), (W, "weight")):
            assert torch.equal(planes(t)[2], t.double()), f"SIMT: {name} operand is not hi + 2^-11 lo"
    worst, q, b64 = _bound(x, W, b, stride, back_end, upstream)
    assert q < math.inf, "all-zero operands"
    assert worst < LIMIT * q, f"sum |terms| reaches {worst / q:.3e} quanta (limit 2^24)"
    with model(back_end):
        y = _conv(x.double(), W.double(), stride, upstream) + b64
    assert torch.equal(y.float().double(), y), "model value not fp32-representable"
    return y.contiguous()


# ---- operand families -------------------------------------------------------------------------------------------------------
def _ints(shape, g, m):
    """integers in [-m, m]"""
    return torch.randint(-m, m + 1, shape, generator=g).double()


def _hl(shape, g, hmin, hmax, lmax, p_zero_h, p_exact_zero=0.0):
    """H + L/2048: |H| in [hmin, hmax) with a random sign, or H = 0 with probability p_zero_h; L in [-lmax, lmax];
    exactly 0 with probability p_exact_zero."""
    H = torch.randint(hmin, hmax, shape, generator=g).double() * torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    H = torch.where(torch.rand(shape, generator=g) < p_zero_h, torch.zeros(()).double(), H)
    v = H + _ints(shape, g, lmax) * LO
    return torch.where(torch.rand(shape, generator=g) < p_exact_zero, torch.zeros(()).double(), v)


def _activations(family, shape, g):
    if family in ("I", "W"):
        return _ints(shape, g, 3)
    if family == "X":
        return _hl(shape, g, 8, 16, 7, 0.25)
    return _hl(shape, g, 2, 4, 1, 0.0, 0.2)


def _weights(family, shape, g):
    if family in ("I", "X"):
        return _ints(shape, g, 3)
    if family == "W":
        return _hl(shape, g, 8, 16, 7, 0.25)
    return _hl(shape, g, 2, 4, 1, 0.0)


def operands(family, x_shape, w_shape, seed, stride=1, upstream=False):
    """(x NHWC, W HWIO, b) fp32 of a family: the weights thinned (halving their density) until every output of every back
    end the family is meant for has sum |terms| + |b| below 2^23 q, half the certificate's limit."""
    g = torch.Generator().manual_seed(seed)
    x = _activations(family, tuple(x_shape), g).float()
    W0 = _weights(family, tuple(w_shape), g)
    keep = torch.rand(tuple(w_shape), generator=g)
    # bias: in [-4, 4], integers (I) or multiples of 2^-11
    b = (_ints((w_shape[3],), g, 4) if family == "I" else _ints((w_shape[3],), g, 1 << 13) * LO).float()
    ends = [e for e in (TC, SIMT, FP16) if family in FAMILIES[e]]
    density = 1.0
    while True:
        W = torch.where(keep < density, W0, torch.zeros(()).double()).float()
        worst = max(headroom(x, W, b, stride, e, upstream) for e in ends)
        if worst < 0.5:
            return x, W, b
        density /= 2.0 ** max(1, math.ceil(math.log2(worst / 0.5)))  # the bound scales about linearly with the density
        assert density > 1e-4, "cannot thin the weights enough"


# ---- conv chains: encoders and update-block heads ---------------------------------------------------------------------------
def chain_weights(p, prefix, seed, fan_in=4):
    """``p`` with every conv under ``prefix`` replaced by exact weights: per output channel `fan_in` taps of +-1 (the rest
    zero) and a bias in multiples of 2^-5 -- the quantum of the input images 2 * (k / 64) - 1 -- in [-1/4, 1/4].  Each conv
    then at most multiplies the magnitude of its input by fan_in while keeping its quantum."""
    g = torch.Generator().manual_seed(seed)
    out = dict(p)
    for k in sorted(p):
        if not (k.startswith(prefix + "/") and k.endswith("/W")):
            continue
        kh, kw, cin, cout = p[k].shape
        K = kh * kw * cin
        W = torch.zeros(K, cout, dtype=torch.float64)
        for co in range(cout):
            idx = torch.randperm(K, generator=g)[:fan_in]
            W[idx, co] = torch.where(torch.rand(len(idx), generator=g) < 0.5, -1.0, 1.0).double()
        out[k] = W.reshape(kh, kw, cin, cout).numpy().astype(np.float32)
        out[k[:-2] + "/b"] = (_ints((cout,), g, 8) / 32.0).numpy().astype(np.float32)
    return out


def exact_images(B, H, W, seed):
    """[B, H, W, 3] images with pixels k / 64: 2x - 1 is exact in fp32 and fp16."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 65, (B, H, W, 3), generator=g).float() / 64.0


@contextlib.contextmanager
def exact_convs(back_end, upstream=False, record=None):
    """O.conv2d -> the certified exact model while the block runs: every conv asserts its certificate and that its input
    (a stored activation) is below 2^15 and split exactly; ``record`` collects (max |input|, headroom, input entries with a
    nonzero lo plane) per conv."""
    saved = O.conv2d

    def conv2d(x, W, b, stride=1, activation=None):
        xf = x.float()
        assert torch.equal(xf.double(), x.double()), "activation not fp32"
        top = x.abs().max().item()
        assert top < STORED, f"stored activation {top} >= 2^15"
        assert torch.equal(planes(xf)[2], x.double()), "activation not split exactly"
        y = certify(xf, W.float(), None if b is None else b.float(), stride, back_end, upstream)
        if record is not None:
            record.append((top, headroom(xf, W.float(), None if b is None else b.float(), stride, back_end, upstream),
                           int((planes(xf)[1] != 0).sum())))
        return activation(y) if activation is not None else y

    O.conv2d = conv2d
    try:
        yield
    finally:
        O.conv2d = saved


def encoder_model(p, name, small, img, back_end, upstream=False, record=None):
    """The encoder with norm "none" under the exact model of the back end (fp64 tensor)."""
    enc = O.small_encoder if small else O.basic_encoder
    pt = {k: torch.from_numpy(np.asarray(v)).double() for k, v in p.items() if k.startswith(name + "/")}
    with exact_convs(back_end, upstream, record):
        return enc(2.0 * img.double() - 1.0, pt, name, "none")
