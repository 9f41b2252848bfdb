"""The GRU gate epilogues and the convex upsampling held BIT FOR BIT on exact pre-activations.

The gates sigmoid_f / tanh_f (csrc/common.cuh: ex2.approx + rcp.approx on the SFU) cannot be restated bit for bit on the CPU,
but they are deterministic functions of their fp32 input.  So they are measured in isolation and every other path and
composite is held to the measured bits:
  * exact pre-activations: each GRU conv reads only `inp`, through its centre tap with weight +-1, plus a dyadic bias (0 on
    half the channels); its weights on h, motion and flow are zero, and the motion encoder and flow head are zero, so the
    flow stays 0.  A pre-activation is then s * inp + b, exact in fp32 (tests/test_exact_gates_model.py certifies every
    conv with exact_oracle.certify).  On raft-things it reaches the epilogue through the hoisted fp32 addend
    (precompute_inp); raft-small, which does not hoist, through the bias.  Every value of the sweep S (every multiple of
    2^-6 in [-24, 24] and +-{16, 17, 30, 64, 88, 89, 100, 1000, 60000}) is a pre-activation of the gate measured;
  * tanh table: convz's bias +1000 makes z = sigmoid_f(1000) = 1, so h' = fma(1, q, 0 h) = tanh_f(a_q);
    sigmoid table: h = 0 and convq's bias +1000 (q = 1) make h' = sigmoid_f(a_z);
    r: z = 1, h = 1 and r*h channel c routed to convq output c, so h' = tanh_f(join(split(sigmoid_f(a_r))));
    raft-things runs the other GRU pass transparent (z = 0: bias -1000), so h2 = h1 exactly;
  * against fp64: |sigmoid_f - sigmoid| and |tanh_f - tanh| <= 3e-7 on S, the saturated values exact for |x| >= 100, and the
    r path within the composed bound; the same output for every occurrence of a value (the gate is a function of a);
  * the same bits on every path: forced tile widths (16: unpaired epilogue lanes), pixel boxes, ring depths and CTA caps,
    RB_MATH_TC_FP16 and RB_MATH_SIMT, B = 2 and each sample alone, rb_update_set_state and rb_update_set_state_cnet, at
    2 x 5 x 7 and 1 x 55 x 128 (many tiles per CTA), and rb_raft_iterate (3 iterations for tanh_f, whose h' does not depend
    on h; 1 otherwise) at 55 x 128, where the 4-level correlation pyramid exists;
  * the composite: a_z and a_q drawn independently from S, h from exact_oracle's X family plus large, tiny and subnormal
    magnitudes; h' must equal fma(z_tab[a_z], q_tab[a_q], fl32(fl32(1 - z) h)) -- the combine both epilogues spell out with
    __fmaf_rn / __fmul_rn -- evaluated in exact rational arithmetic and rounded to fp32 once.
Convex upsampling (upsample_convex_kernel): mask logits from {L, L - 200}, so expf gives exactly 1 or 0 and the weights are
fl32(1/m) for m maxima; dyadic coordinates make 8 (c - x) exact.  All 511 tie patterns at interior, edge and corner pixels;
m in {1, 2, 4, 8} equals the rational value, any m the kernel's pinned order ax = fma(fx, p, ax), k = 0..8.
Largest gate errors and the configurations rb_debug_conv_last recorded are printed at the end of the module (pytest -s)."""
import contextlib
from fractions import Fraction

import numpy as np
import pytest
import torch

import exact_oracle as E
from oracle import raft_oracle as O
from test_gpu_conv_coverage import CONFIGS, SEEN, _cfg_id, _first_diff, _forced, _last, _ring
from test_gpu_edges import _crops

pytestmark = pytest.mark.gpu

# ---- the sweep and the construction (no GPU; tests/test_exact_gates_model.py checks it) ---------------------------------------
BIG = (16.0, 17.0, 30.0, 64.0, 88.0, 89.0, 100.0, 1000.0, 60000.0)
S = np.unique(np.concatenate([np.arange(-24 * 64, 24 * 64 + 1) / 64.0, BIG, -np.array(BIG)]))
SAT = 1000.0        # bias that saturates a gate: sigmoid_f(+-1000) = 1 / 0, tanh_f(1000) = 1
R_CONST = 2.5       # bias of a gate that is not measured and not saturated (r in the z and q runs)
GATE_BOUND = 3e-7   # DESIGN section 4: |gate_f - gate| for the sigmoid and tanh of the GRU epilogues
SHAPES = [(2, 5, 7), (1, 55, 128)]
MODES = ("sig", "tanh", "r")
# (sign, bias) of routed output channel c: class c % 4
CLASSES = ((1.0, 0.0), (-1.0, 0.0), (1.0, 3.0 / 64), (-1.0, -0.75))


def variant(small):
    """hidden, context, GRU passes (z, r, q conv names), centre tap of each pass, the conv input's channel count."""
    if small:
        return dict(hid=96, ctx=64, passes=(("convz", "convr", "convq"),), centre=((1, 1),), cin=242, radius=3)
    return dict(hid=128, ctx=128, passes=(("convz1", "convr1", "convq1"), ("convz2", "convr2", "convq2")),
                centre=((0, 2), (2, 0)), cin=384, radius=4)


def routing(small, gate):
    """(inp channel, sign, bias) of the routed output channels c < min(hidden, context) of gate 0 = z, 1 = r, 2 = q: a
    different permutation per gate, so an addend, a bias or a z | r half read from the wrong channel changes the value."""
    v = variant(small)
    n = min(v["hid"], v["ctx"])
    c = np.arange(n)
    perm = (c, (c + 37) % n, (5 * c + 11) % n)[gate]
    sign = np.array([CLASSES[k % 4][0] for k in c])
    bias = np.array([CLASSES[k % 4][1] for k in c])
    return perm, sign, bias


def _fp16_exact(t):
    return (np.abs(t) <= 65504) & (t.astype(np.float16).astype(np.float64) == t)


def admissible(sign, bias):
    """Values v of S that s * t + b reaches with an inp value t >= 0 that is exact in fp16 (so in every back end)."""
    t = sign * (S - bias)
    return S[(t >= 0) & _fp16_exact(t)]


def assign(small, gate, npix):
    """[npix, n] pre-activations from S for the routed channels of one gate: per class, the values the earlier classes left
    uncovered first (those fewest classes reach first), then the class's admissible values cyclically."""
    perm, sign, bias = routing(small, gate)
    n = len(perm)
    a = np.zeros((npix, n))
    covered = np.zeros(0)
    reach = sum(np.isin(S, admissible(*cl)).astype(int) for cl in CLASSES)
    for k in range(4):
        chans = np.arange(k, n, 4)
        adm = admissible(*CLASSES[k])
        todo = np.setdiff1d(adm, covered)
        todo = todo[np.argsort(reach[np.searchsorted(S, todo)], kind="stable")]
        seq = np.concatenate([todo, adm])
        j = (np.arange(npix)[:, None] * len(chans) + np.arange(len(chans))[None, :]) % len(seq)
        a[:, chans] = seq[j]
        covered = np.union1d(covered, a[:, chans].ravel())
    return a


def unrouted_bias(small, seed):
    """Biases of the output channels no inp channel feeds (raft-small: hidden 96 > context 64): constant values from S."""
    v = variant(small)
    n = min(v["hid"], v["ctx"])
    g = np.random.default_rng(seed)
    return S[g.integers(0, len(S), v["hid"] - n)]


def _zero_update_block(p):
    return {k: (np.zeros_like(v) if k.startswith("update_block/") else v) for k, v in p.items()}


def _set_gate(p, small, pas, gate, inp_weights=None, bias=0.0, extra=None):
    """Conv `gate` of GRU pass `pas`: weight sign[c] from inp channel perm[c] at the centre tap (inp_weights =
    (perm, sign)), plus `extra` = [(input channel, output channel, weight)], and `bias` (scalar or per channel)."""
    v = variant(small)
    name = f"update_block/gru/{v['passes'][pas][gate]}"
    W = np.zeros_like(p[name + "/W"])
    ky, kx = v["centre"][pas]
    if inp_weights is not None:
        perm, sign = inp_weights
        W[ky, kx, v["hid"] + perm, np.arange(len(perm))] = sign
    for ci, co, wt in extra or ():
        W[ky, kx, ci, co] = wt
    p[name + "/W"] = W
    p[name + "/b"] = np.broadcast_to(np.asarray(bias, dtype=np.float32), p[name + "/b"].shape).astype(np.float32).copy()


def _transparent(p, small, pas):
    _set_gate(p, small, pas, 0, bias=-SAT)
    _set_gate(p, small, pas, 1)
    _set_gate(p, small, pas, 2)


def problem(small, mode, pas, B, h, w, seed=0):
    """(weights, net, inp, pre-activation of the measured gate [B, h, w, hidden] fp64, pre-activation of a second gate or
    None).  mode: "sig", "tanh", "r" (one gate from S) or "composite" (z and q independently from S, biases 0)."""
    from raft_b200 import synth
    v = variant(small)
    hid, ctx = v["hid"], v["ctx"]
    npix = B * h * w
    n = min(hid, ctx)
    p = _zero_update_block(synth.make_weights(small))
    for other in range(len(v["passes"])):
        if other != pas:
            _transparent(p, small, other)
    g = np.random.default_rng((seed, pas, len(mode)))
    inp = np.zeros((npix, ctx))
    net = np.zeros((npix, hid))
    a2 = None
    if mode == "composite":
        tab = np.unique(np.abs(S))
        inp[:] = tab[g.integers(0, len(tab), inp.shape)]
        extra_b = unrouted_bias(small, seed + 1), unrouted_bias(small, seed + 2)
        pre = []
        for gate, eb in ((0, extra_b[0]), (2, extra_b[1])):
            perm, sign, _ = routing(small, gate)
            _set_gate(p, small, pas, gate, (perm, sign), np.concatenate([np.zeros(n), eb]))
            pre.append(np.concatenate([sign * inp[:, perm], np.broadcast_to(eb, (npix, hid - n))], axis=1))
        _set_gate(p, small, pas, 1, bias=R_CONST)
        a, a2 = pre
        hx = E._activations("X", (npix, hid), torch.Generator().manual_seed(seed + 3)).numpy()
        special = np.array([6e4, -6e4, 1e4, -3.0e3, 2.0 ** -100, -(2.0 ** -120), 1e-40, -3e-42, 0.0, 1.0])
        idx = g.choice(npix * hid, 4 * len(special), replace=False)
        hx.ravel()[idx] = np.tile(special, 4)
        net[:] = hx.astype(np.float32)
    else:
        gate = {"sig": 0, "r": 1, "tanh": 2}[mode]
        perm, sign, bias = routing(small, gate)
        a_r = assign(small, gate, npix)
        inp[:, perm] = sign * (a_r - bias)
        eb = unrouted_bias(small, seed + 4)
        a = np.concatenate([a_r, np.broadcast_to(eb, (npix, hid - n))], axis=1)
        _set_gate(p, small, pas, gate, (perm, sign), np.concatenate([bias, eb]))
        if mode == "sig":
            _set_gate(p, small, pas, 1, bias=R_CONST)
            _set_gate(p, small, pas, 2, bias=SAT)
        elif mode == "tanh":
            _set_gate(p, small, pas, 0, bias=SAT)
            _set_gate(p, small, pas, 1, bias=R_CONST)
        else:
            _set_gate(p, small, pas, 0, bias=SAT)
            _set_gate(p, small, pas, 2, extra=[(c, c, 1.0) for c in range(hid)])  # QX channel c = r * h, channel c
            net[:] = 1.0
    assert (inp >= 0).all() and _fp16_exact(inp).all()
    shape = (B, h, w)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).reshape(*shape, -1)  # noqa: E731
    return p, t(net).float(), t(inp).float(), t(a), None if a2 is None else t(a2)


def cnet_of(net, inp):
    """A raw context map whose tanh / relu (RAFT.py:85-87, libm tanhf) give net in {0, 1} and inp >= 0 exactly."""
    assert ((net == 0) | (net == 1)).all()
    return torch.cat([net * 100.0, inp], dim=-1).contiguous()


# ---- exact arithmetic ----------------------------------------------------------------------------------------------------------
def round_f32(fr):
    """The fp32 value nearest to the rational fr, ties to even mantissa."""
    c = np.float32(float(fr))
    cands = (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf)))
    return min(cands, key=lambda x: (abs(Fraction(float(x)) - fr), int(np.float32(x).view(np.uint32)) & 1))


def combine_exact(z, q, h):
    """fma(z, q, fl32(fl32(1 - z) h)) elementwise (fp32 arrays), the fma in exact rational arithmetic, one rounding."""
    t = (np.float32(1.0) - z) * h  # both fp32 operations, round to nearest
    out = np.empty(z.shape, dtype=np.float32)
    for i, (zz, qq, tt) in enumerate(zip(z.ravel(), q.ravel(), t.ravel())):
        out.ravel()[i] = round_f32(Fraction(float(zz)) * Fraction(float(qq)) + Fraction(float(tt)))
    return out


def fma_f32(a, b, c):
    """fl32(a b + c) with one rounding, vectorised: the product is exact in fp64, TwoSum gives the exact sum as s + e, and a
    sum that lands exactly on an fp32 midpoint is resolved by the sign of e (test_exact_gates_model checks it against
    Fraction)."""
    a, b, c = (np.asarray(x, dtype=np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)
    n = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    mid = (d != 0) & (2 * np.abs(d) == np.abs(n.astype(np.float64) - r.astype(np.float64)))
    return np.where(mid & (e != 0) & (np.sign(e) == np.sign(d)), n, r)


# ---- convex upsampling: all 511 tie patterns -------------------------------------------------------------------------------
UP_L = (1e4, 0.0, -37.5, 3.25, -1e4 + 0.5, 517.0625)


def upsample_problem(B, h, w, seed):
    """(coords1, mask, m = number of maxima per (b, y, x, t), pattern) with mask logits L (taps in the pattern) or L - 200;
    every category of coarse pixel (corner, edge, interior) runs through all 511 patterns."""
    g = torch.Generator().manual_seed(seed)
    grid = O.coords_grid(B, h, w).double()
    flow = torch.randint(-512, 513, (B, h, w, 2), generator=g).double() / 16
    coords1 = (grid + flow).float()
    assert torch.equal(coords1.double() - grid, flow)
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    border = (yy == 0).int() + (yy == h - 1).int() + (xx == 0).int() + (xx == w - 1).int()
    cat = torch.where(border >= 2, 2, torch.where(border == 1, 1, 0)).expand(B, h, w)  # 0 interior, 1 edge, 2 corner
    pattern = torch.zeros(B, h, w, 64, dtype=torch.int64)
    for k, off in ((0, 0), (1, 170), (2, 341)):
        sel = cat == k
        cnt = int(sel.sum()) * 64
        pattern[sel] = ((torch.arange(cnt) + off) % 511 + 1).reshape(-1, 64)
    bits = (pattern[..., None] >> torch.arange(9)) & 1  # [B, h, w, 64, 9]
    L = torch.tensor(UP_L, dtype=torch.float64)[torch.randint(0, len(UP_L), (B, h, w, 64, 1), generator=g)]
    logits = torch.where(bits == 1, L, L - 200.0)
    mask = logits.permute(0, 1, 2, 4, 3).reshape(B, h, w, 576).float()  # channel k * 64 + t
    assert torch.equal(mask.double(), logits.permute(0, 1, 2, 4, 3).reshape(B, h, w, 576))
    return coords1, mask, bits.sum(-1), bits, flow


def upsample_model(flow, bits):
    """The kernel's arithmetic on these inputs: p_k = fl32(1/m) on the maxima (expf(0) = 1, expf(-200) = 0, IEEE quotient),
    fx = 8 (c - x) or 0 outside the image, ax = fma(fx, p_k, ax) for k = 0..8.  [B, 8h, 8w, 2] fp32."""
    B, h, w, _ = flow.shape
    m = bits.sum(-1).numpy()
    pval = (np.float32(1.0) / m.astype(np.float32)).astype(np.float32)
    padded = torch.zeros(B, h + 2, w + 2, 2, dtype=torch.float64)
    padded[:, 1:-1, 1:-1] = 8.0 * flow
    out = []
    for ch in range(2):
        ax = np.zeros((B, h, w, 64), dtype=np.float32)
        for k in range(9):
            fx = padded[:, k // 3:k // 3 + h, k % 3:k % 3 + w, ch].numpy().astype(np.float32)[..., None]
            p = np.where(bits[..., k].numpy() == 1, pval, np.float32(0.0))
            ax = fma_f32(np.broadcast_to(fx, ax.shape), p, ax)
        out.append(ax)
    y = torch.from_numpy(np.stack(out, -1))  # [B, h, w, 64, 2]
    return y.reshape(B, h, w, 8, 8, 2).permute(0, 1, 3, 2, 4, 5).reshape(B, 8 * h, 8 * w, 2)


def upsample_rational(flow, bits):
    """sum_k p_k fx_k in fp64 with p_k = 1/m: exact for m in {1, 2, 4, 8} (dyadic operands of a few bits)."""
    B, h, w, _ = flow.shape
    m = bits.sum(-1).double()
    padded = torch.zeros(B, h + 2, w + 2, 2, dtype=torch.float64)
    padded[:, 1:-1, 1:-1] = 8.0 * flow
    acc = torch.zeros(B, h, w, 64, 2, dtype=torch.float64)
    for k in range(9):
        acc += padded[:, k // 3:k // 3 + h, k % 3:k % 3 + w, None, :] * (bits[..., k:k + 1].double() / m[..., None])
    return acc.reshape(B, h, w, 8, 8, 2).permute(0, 1, 3, 2, 4, 5).reshape(B, 8 * h, 8 * w, 2)


def fine_m(bits):
    B, h, w = bits.shape[:3]
    return bits.sum(-1).reshape(B, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(B, 8 * h, 8 * w)


# ---- GPU runs --------------------------------------------------------------------------------------------------------------------
def _capi():
    from raft_b200 import capi
    return capi


REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(REPORT):
        print(f"\n{k}: {REPORT[k]}")
    if SEEN:
        print("\nconv_tc configurations recorded by rb_debug_conv_last (BLOCK_N, bw_log2, stages, tiles per CTA):")
        for t in sorted(SEEN):
            print("  ", t)


@pytest.fixture(autouse=True)
def _reset_thread_state():
    yield
    c = _capi()
    c.lib.rb_set_math_mode(c.RB_MATH_TC)
    c.lib.rb_debug_conv_override(0, 0, 0, 0)


@contextlib.contextmanager
def _math(back_end):
    c = _capi()
    c.check(c.lib.rb_set_math_mode({E.TC: c.RB_MATH_TC, E.SIMT: c.RB_MATH_SIMT, E.FP16: c.RB_MATH_TC_FP16}[back_end]))
    try:
        yield
    finally:
        c.lib.rb_set_math_mode(c.RB_MATH_TC)


def run_gru(cuda, small, blob, net, inp, iterate=0, cnet=False):
    """net after one rb_update_step (iterate = 0) or rb_raft_iterate(iterate), with zero correlation features."""
    c = _capi()
    lib, s, P, st = c.lib, int(small), c.ptr, c.stream()
    B, h, w = net.shape[:3]
    dims = (B, h, w)
    ws = torch.zeros(c.size_query(lib.rb_update_workspace_bytes, s, *dims), dtype=torch.uint8, device=cuda)
    coords1 = torch.empty(B, h, w, 2, device=cuda)
    netd, inpd = net.contiguous().to(cuda), inp.contiguous().to(cuda)
    if cnet:
        cn = cnet_of(net, inp).to(cuda)
        c.check(lib.rb_update_set_state_cnet(s, P(blob), P(ws), P(cn), *dims, st))
    else:
        c.check(lib.rb_update_set_state(s, P(blob), P(ws), P(netd), P(inpd), *dims, st))
    corr = torch.zeros(B, h, w, 4 * (2 * variant(small)["radius"] + 1) ** 2, device=cuda)
    c.check(lib.rb_update_set_corr(s, P(ws), P(corr), *dims, st))
    c.check(lib.rb_coords_grid(P(coords1), *dims, st))
    if iterate:
        pyramid = torch.zeros(c.size_query(lib.rb_corr_pyramid_bytes, *dims) // 4, device=cuda)
        mask = None if small else torch.zeros(B, h, w, 576, device=cuda)
        c.check(lib.rb_raft_iterate(s, P(blob), P(ws), P(pyramid), P(coords1), P(mask), *dims, iterate, st))
    else:
        delta = torch.zeros(B, h, w, 2, device=cuda)
        c.check(lib.rb_update_step(s, P(blob), P(ws), P(coords1), P(delta), P(None), *dims, st))
    out = torch.empty(B, h, w, variant(small)["hid"], device=cuda)
    c.check(lib.rb_update_get_net(s, P(ws), P(out), *dims, st))
    torch.cuda.synchronize()
    assert torch.equal(coords1.cpu(), O.coords_grid(B, h, w)), "the flow must stay 0"
    return out.cpu()


def _blob(cuda, p, small):
    from raft_b200.weights import pack_update_block
    return pack_update_block(p, small, cuda)


def _assert_same(out, want, what):
    assert torch.isfinite(out).all(), f"{what}: non-finite outputs"
    assert torch.equal(out, want), f"{what}: not bit-identical: {_first_diff(out, want)}"


def table_of(a, out, what):
    """{value: fp32 output} from pre-activations a and outputs; asserts one output per value (bit patterns)."""
    a = a.reshape(-1).numpy()
    o = out.reshape(-1).numpy().view(np.uint32)
    vals, first, inv = np.unique(a, return_index=True, return_inverse=True)
    bad = o != o[first][inv]
    assert not bad.any(), f"{what}: {int(bad.sum())} outputs differ from another output of the same pre-activation " \
                          f"(first: a = {a[bad][0]!r})"
    return dict(zip(vals.tolist(), out.reshape(-1).numpy()[first].tolist()))


GATE_TABLES = {"sig": {}, "tanh": {}}


def merge_table(kind, tab, what):
    ref = GATE_TABLES[kind]
    for k, v in tab.items():
        if k in ref:
            assert np.float32(ref[k]).view(np.uint32) == np.float32(v).view(np.uint32), \
                f"{what}: {kind}({k!r}) = {v!r} here, {ref[k]!r} in another run"
        else:
            ref[k] = v


def _max_err(a, out, f):
    err = np.abs(out.double().numpy() - f(a.numpy()))
    i = int(np.argmax(err))
    return float(err.ravel()[i]), float(a.numpy().ravel()[i])


def _sigmoid(x):
    return 0.5 * (1.0 + np.tanh(0.5 * x))  # no overflow at -60000


def check_gate_bound(kind, a, out, what):
    f = _sigmoid if kind == "sig" else np.tanh
    err, at = _max_err(a, out, f)
    key = f"largest |{kind}_f - {kind}| (fp64)"
    if err >= REPORT.get(key, (-1.0, 0))[0]:
        REPORT[key] = (err, f"at x = {at!r}")
    assert err <= GATE_BOUND, f"{what}: |{kind}_f(x) - {kind}(x)| = {err:.3e} at x = {at!r} exceeds {GATE_BOUND}"
    big = a.abs() >= 100
    o = out[big]
    if kind == "sig":
        assert torch.equal(o, (a[big] > 0).float()), f"{what}: sigmoid_f not exactly 0 / 1 at |x| >= 100"
    else:
        assert torch.equal(o, torch.sign(a[big]).float()), f"{what}: tanh_f not exactly +-1 at |x| >= 100"


def _sweep_covered(a, what):
    missing = np.setdiff1d(S, a.numpy().ravel())
    assert missing.size == 0, f"{what}: {missing.size} values of S are no pre-activation (e.g. {missing[:4]})"


def paths(small, B, h, w, mode):
    """(name, back end, forced configuration, iterate, cnet) of every path a table must be identical on."""
    out = [("natural", E.TC, (0, 0, 0, 0), 0, False)]
    out += [(f"forced {_cfg_id(c)}", E.TC, c, 0, False) for c in CONFIGS]
    out += [("RB_MATH_SIMT", E.SIMT, (0, 0, 0, 0), 0, False)]
    if h >= 8 and w >= 8:  # rb_raft_iterate's 4-level correlation pyramid
        out += [("rb_raft_iterate", E.TC, (0, 0, 0, 0), 3 if mode == "tanh" else 1, False)]
    out += [("rb_update_set_state_cnet", E.TC, (0, 0, 0, 0), 0, True)]
    if mode != "r":  # with r * h as a conv operand, the single-pass mode multiplies hi(r) alone: checked on its own below
        out += [("RB_MATH_TC_FP16", E.FP16, (0, 0, 0, 0), 0, False)]
    return out


def _run_path(cuda, small, blob, net, inp, back_end, cfg, iterate, cnet):
    with _math(back_end), _forced(cfg):
        out = run_gru(cuda, small, blob, net, inp, iterate, cnet)
        rec = _last() if back_end != E.SIMT else None
    if rec is not None and cfg != (0, 0, 0, 0):  # the last conv of a step: the flow head's 16-wide conv2 (or the mask head)
        assert rec["stages"] == _ring(rec["block_n"], cfg[3]), rec
        assert not cfg[2] or rec["grid"] <= cfg[2], rec
        assert not cfg[1] or rec["bw_log2"] == cfg[1], rec
    return out


@pytest.mark.parametrize("B,h,w", SHAPES, ids=lambda v: str(v))
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_gate_tables(cuda, small, B, h, w):
    """Per GRU pass: the sigmoid and tanh tables and the r path, on every path, against fp64 and the measured bits."""
    for pas in range(len(variant(small)["passes"])):
        for mode in MODES:
            what = f"{'small' if small else 'things'} {B}x{h}x{w} pass {pas + 1} {mode}"
            p, net, inp, a, _ = problem(small, mode, pas, B, h, w)
            _sweep_covered(a, what)
            blob = _blob(cuda, p, small)
            base = None
            for name, back_end, cfg, it, cn in paths(small, B, h, w, mode):
                out = _run_path(cuda, small, blob, net, inp, back_end, cfg, it, cn)
                if base is None:
                    base = out
                else:
                    _assert_same(out, base, f"{what} {name}")
            if B > 1:
                for b in range(B):
                    out = _run_path(cuda, small, blob, net[b:b + 1], inp[b:b + 1], E.TC, (0, 0, 0, 0), 0, False)
                    _assert_same(out, base[b:b + 1], f"{what} sample {b} alone")
            if mode == "r":
                check_r(cuda, small, blob, net, inp, a, base, what)
            else:
                merge_table(mode, table_of(a, base, what), what)
                check_gate_bound(mode, a, base, what)


def check_r(cuda, small, blob, net, inp, a, out, what):
    """h' = tanh_f(a_q), a_q = join(split(r)) with r = sigmoid_f(a_r) (hi(r) alone under RB_MATH_TC_FP16): one output per
    a_q, and |h' - tanh(sigmoid(a_r))| <= 3e-7 + |a_q - sigmoid(a_r)|."""
    if not GATE_TABLES["sig"]:
        pytest.fail("the sigmoid table is measured first (mode order)")
    r = np.vectorize(lambda x: GATE_TABLES["sig"][x])(a.numpy()).astype(np.float32)
    hi, _, joined = E.planes(torch.from_numpy(r))
    exact = torch.from_numpy(np.tanh(_sigmoid(a.numpy())))
    for back_end, aq, got in ((E.TC, joined, out), (E.FP16, hi, None)):
        if got is None:
            with _math(back_end):
                got = run_gru(cuda, small, blob, net, inp)
        table_of(aq, got, f"{what} {back_end}")
        err = (got.double() - exact).abs()
        bound = GATE_BOUND + (aq - torch.from_numpy(_sigmoid(a.numpy()))).abs()
        worst = int(torch.argmax(err - bound))
        assert (err <= bound).all(), f"{what} {back_end}: r path error {err.view(-1)[worst]:.3e} > bound " \
                                     f"{bound.view(-1)[worst]:.3e} at a_r = {a.view(-1)[worst].item()!r}"
        REPORT[f"r path, largest |h' - tanh(sigmoid(a_r))| ({back_end})"] = f"{err.max().item():.3e}"


def _tables(cuda):
    """Measure the sigmoid and tanh tables (raft-things, pass 1, 2 x 5 x 7) unless a table test already did."""
    for mode in ("sig", "tanh"):
        if len(GATE_TABLES[mode]) < len(S):
            p, net, inp, a, _ = problem(False, mode, 0, 2, 5, 7)
            out = run_gru(cuda, False, _blob(cuda, p, False), net, inp)
            merge_table(mode, table_of(a, out, f"{mode} table"), f"{mode} table")
            check_gate_bound(mode, a, out, f"{mode} table")
    return GATE_TABLES["sig"], GATE_TABLES["tanh"]


@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_gru_composite_exact(cuda, small):
    """h' = fma(z_tab[a_z], q_tab[a_q], fl32(fl32(1 - z) h)) bit for bit, every pass, and the same bits on every path."""
    z_tab, q_tab = _tables(cuda)
    B, h, w = 2, 5, 7
    for pas in range(len(variant(small)["passes"])):
        what = f"{'small' if small else 'things'} composite pass {pas + 1}"
        p, net, inp, az, aq = problem(small, "composite", pas, B, h, w, seed=5)
        z = np.vectorize(lambda x: z_tab[x])(az.numpy()).astype(np.float32)
        q = np.vectorize(lambda x: q_tab[x])(aq.numpy()).astype(np.float32)
        want = torch.from_numpy(combine_exact(z, q, net.numpy()))
        blob = _blob(cuda, p, small)
        for name, back_end, cfg, it, cn in paths(small, B, h, w, "composite"):
            if cn:  # net here is no tanh of a context map
                continue
            out = _run_path(cuda, small, blob, net, inp, back_end, cfg, min(it, 1), False)
            _assert_same(out, want, f"{what} {name}")
        # the operands separate the pinned order from its alternatives (tests/test_exact_gates_model.py, fp64 stand-ins)
        t = (np.float32(1.0) - z) * net.numpy()
        alt = ((z * q).astype(np.float32) + t).astype(np.float32)
        n_alt = int((alt.view(np.uint32) != want.numpy().view(np.uint32)).sum())
        REPORT[f"{what}: entries where fl32(fl32((1-z) h) + fl32(z q)) differs"] = n_alt
        assert n_alt > 0


# ---- convex upsampling -------------------------------------------------------------------------------------------------------
def _upsample(cuda, coords1, mask, crop=None):
    c = _capi()
    B, h, w = coords1.shape[:3]
    top, left, oh, ow = crop or (0, 0, 8 * h, 8 * w)
    out = torch.full((B, oh, ow, 2), float("nan"), device=cuda)
    c1, m = coords1.contiguous().to(cuda), mask.contiguous().to(cuda)
    c.check(c.lib.rb_upsample_convex_crop(c.ptr(c1), c.ptr(m), c.ptr(out), B, h, w, top, left, oh, ow, c.stream()))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("h,w", [(5, 7), (6, 9)], ids=lambda v: str(v))
def test_upsample_convex_exact(cuda, h, w):
    """Every tie pattern at interior, edge and corner pixels, B = 2: the rational value for m in {1, 2, 4, 8}, the pinned
    fma order for every m, batched == each sample alone, and every crop == the same window of the full field."""
    B = 2
    coords1, mask, _, bits, flow = upsample_problem(B, h, w, 10 * h + w)
    want = upsample_model(flow, bits)
    full = _upsample(cuda, coords1, mask)
    _assert_same(full, want, "pinned fma order")
    pow2 = torch.isin(fine_m(bits), torch.tensor([1, 2, 4, 8]))
    rat = upsample_rational(flow, bits)
    assert torch.equal(rat[pow2].float().double(), rat[pow2]), "rational value not fp32"
    _assert_same(full[pow2], rat[pow2].float(), "m in {1, 2, 4, 8}: the rational value")
    for b in range(B):
        _assert_same(_upsample(cuda, coords1[b:b + 1], mask[b:b + 1]), full[b:b + 1], f"sample {b} alone")
    for crop in _crops(h, w):
        top, left, oh, ow = crop
        _assert_same(_upsample(cuda, coords1, mask, crop), full[:, top:top + oh, left:left + ow], f"crop {crop}")
