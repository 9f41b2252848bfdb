"""The construction of tests/test_gpu_exact_gates.py, checked without a GPU.

  * every GRU conv of every run certifies (exact_oracle.certify, all three back ends) and gives the intended
    pre-activations; every value of the sweep S is a pre-activation of the gate each run measures, in every pass and variant;
  * the saturation identities the runs rely on hold in a model of sigmoid_f / tanh_f with an exact exp2 and reciprocal;
  * planted defects are caught: with fp64 sigmoid / tanh standing in for the measured tables, the composite operands
    separate the pinned combine fma(z, q, fl32((1 - z) h)) from fma(1 - z, h, fl32(z q)) and from fl32(fl32((1 - z) h) +
    fl32(z q)) on many entries, and an addend read from the neighbouring channel, or the z and r halves swapped, change the
    expected output;
  * the exact-rounding helpers: fma_f32 equals the rational fma rounded once, also where fp64 alone rounds twice, and the
    upsampling model equals the rational value where the weights are powers of two."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import exact_oracle as E
import test_gpu_exact_gates as G


def _pass_convs(p, small, pas):
    names = G.variant(small)["passes"][pas]
    return [(p[f"update_block/gru/{n}/W"], p[f"update_block/gru/{n}/b"]) for n in names]


def _conv_input(small, net, inp, first=None):
    """The GRU conv input [first | inp | motion 0 | flow 0] (first = h for HX; r * h for QX)."""
    v = G.variant(small)
    B, h, w = net.shape[:3]
    rest = torch.zeros(B, h, w, v["cin"] - v["hid"] - v["ctx"])
    return torch.cat([net if first is None else first, inp, rest], dim=-1)


def pass_model(p, small, pas, net, inp, sig, tanh, defect=None, back_end=E.TC):
    """h' of one GRU pass from the certified pre-activations and the given gate functions (fp32 -> fp32).  defect:
    "neighbour" (every addend read one channel up) or "swap" (z and r halves of the z | r conv exchanged)."""
    hid = G.variant(small)["hid"]
    (Wz, bz), (Wr, br), (Wq, bq) = _pass_convs(p, small, pas)
    for Wg in (Wz, Wr, Wq):
        assert not Wg[:, :, :hid].any(), "the construction reads no h (and no r * h) channel here"
    x = _conv_input(small, torch.zeros_like(net), inp)
    zr = E.certify(x, torch.from_numpy(np.concatenate([Wz, Wr], -1)), torch.from_numpy(np.concatenate([bz, br])), 1, back_end)
    aq = E.certify(x, torch.from_numpy(Wq), torch.from_numpy(bq), 1, back_end)
    if defect == "neighbour":
        zr, aq = torch.roll(zr, -1, -1), torch.roll(aq, -1, -1)
    if defect == "swap":
        zr = torch.cat([zr[..., hid:], zr[..., :hid]], -1)
    z = sig(zr[..., :hid].float().numpy())
    q = tanh(aq.float().numpy())
    return torch.from_numpy(G.fma_f32(z, q, (np.float32(1.0) - z) * net.numpy())), zr, aq


def _sig64(x):
    return G._sigmoid(np.asarray(x, np.float64)).astype(np.float32)


def _tanh64(x):
    return np.tanh(np.asarray(x, np.float64)).astype(np.float32)


@pytest.mark.parametrize("mode", ["sig", "tanh", "r", "composite"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_routed_weights_certify_and_cover(small, mode):
    v = G.variant(small)
    hid = v["hid"]
    for pas in range(len(v["passes"])):
        p, net, inp, a, a2 = G.problem(small, mode, pas, 2, 5, 7)
        assert (inp >= 0).all() and G._fp16_exact(inp.double().numpy()).all()
        for other in range(len(v["passes"])):
            (Wz, bz), (Wr, br), (Wq, bq) = _pass_convs(p, small, other)
            if other != pas:  # transparent: z = sigmoid_f(-1000) = +0
                assert not (Wz.any() or Wr.any() or Wq.any() or br.any() or bq.any()) and (bz == -G.SAT).all()
        for back_end in (E.TC, E.SIMT, E.FP16):
            (Wz, bz), (Wr, br), (Wq, bq) = _pass_convs(p, small, pas)
            x = _conv_input(small, torch.zeros_like(net), inp)
            assert not (Wz[:, :, :hid].any() or Wr[:, :, :hid].any()), "z and r read no h channel"
            az = E.certify(x, torch.from_numpy(Wz), torch.from_numpy(bz), 1, back_end)
            ar = E.certify(x, torch.from_numpy(Wr), torch.from_numpy(br), 1, back_end)
            if mode == "r":  # q reads r * h, channel c -> output c, nothing else
                ref = np.zeros_like(Wq)
                ky, kx = v["centre"][pas]
                ref[ky, kx, np.arange(hid), np.arange(hid)] = 1.0
                assert np.array_equal(Wq, ref) and not bq.any()
                aq = None
            else:
                aq = E.certify(x, torch.from_numpy(Wq), torch.from_numpy(bq), 1, back_end)
            want = {"sig": (a, G.R_CONST, G.SAT), "tanh": (G.SAT, G.R_CONST, a), "r": (G.SAT, a, None),
                    "composite": (a, G.R_CONST, a2)}[mode]
            for got, exp in zip((az, ar, aq), want):
                if got is None:
                    continue
                exp = torch.full_like(got, exp) if isinstance(exp, float) else exp
                assert torch.equal(got, exp), f"{mode} pass {pas + 1} {back_end}: pre-activation"
        if mode != "composite":
            missing = np.setdiff1d(G.S, a.numpy().ravel())
            assert missing.size == 0, f"{mode} pass {pas + 1}: {missing.size} values of S missing"
        else:
            assert (a.abs() > 0).float().mean() > 0.9 and (a2.abs() > 0).float().mean() > 0.9


def test_sweep_covers_the_large_shape():
    for small in (False, True):
        for mode in G.MODES:
            _, _, _, a, _ = G.problem(small, mode, 0, 1, 55, 128)
            assert np.setdiff1d(G.S, a.numpy().ravel()).size == 0, (small, mode)


# ---- saturation identities ----------------------------------------------------------------------------------------------------
def _sfu_model(x, scale):
    """1 + exp2(scale * x) in fp32 (exact exp2 of the fp32 product, flushed below the normal range), then 1 / that."""
    t = (np.float32(scale) * np.asarray(x, np.float32)).astype(np.float32)
    with np.errstate(divide="ignore", over="ignore"):
        e = np.exp2(t.astype(np.float64)).astype(np.float32)
        e = np.where(np.abs(e) < np.finfo(np.float32).tiny, np.float32(0.0), e)
        return (np.float32(1.0) / (np.float32(1.0) + e)).astype(np.float32)


def test_saturation_identities():
    sig = lambda x: _sfu_model(x, -1.4426950408889634)  # noqa: E731
    tanh = lambda x: G.fma_f32(-2.0, _sfu_model(x, 2.8853900817779268), 1.0)  # noqa: E731
    assert sig(G.SAT) == 1.0 and sig(-G.SAT) == 0.0 and not np.signbit(sig(-G.SAT)) and tanh(G.SAT) == 1.0
    assert sig(0.0) == 0.5 and tanh(0.0) == 0.0
    g = np.random.default_rng(3)
    q = _tanh64(g.choice(G.S, 4096))
    z = _sig64(g.choice(G.S, 4096))
    h = (g.standard_normal(4096) * np.exp2(g.integers(-30, 16, 4096))).astype(np.float32)
    one, zero = np.float32(1.0), np.float32(0.0)
    assert np.array_equal(G.fma_f32(one, q, (one - one) * h), q), "z = 1: h' = q"
    assert np.array_equal(G.fma_f32(zero, q, (one - zero) * h), h), "z = 0: h' = h (transparent pass)"
    assert np.array_equal(G.fma_f32(z, one, (one - z) * zero), z), "h = 0, q = 1: h' = z"


# ---- planted defects ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_composite_separates_the_combine_orders(small):
    for pas in range(len(G.variant(small)["passes"])):
        p, net, inp, az, aq = G.problem(small, "composite", pas, 2, 5, 7, seed=5)
        z, q, h = _sig64(az.numpy()), _tanh64(aq.numpy()), net.numpy()
        want = G.combine_exact(z, q, h)
        assert np.array_equal(G.fma_f32(z, q, (np.float32(1.0) - z) * h), want)
        alt1 = G.fma_f32(np.float32(1.0) - z, h, z * q)
        alt2 = ((np.float32(1.0) - z) * h + z * q).astype(np.float32)
        for name, alt in (("fma(1 - z, h, fl32(z q))", alt1), ("fl32(fl32((1 - z) h) + fl32(z q))", alt2)):
            n = int((alt.view(np.uint32) != want.view(np.uint32)).sum())
            assert n >= 0.01 * want.size, f"pass {pas + 1}: {name} differs on only {n} of {want.size} entries"
        model, _, _ = pass_model(p, small, pas, net, inp, _sig64, _tanh64)
        assert np.array_equal(model.numpy(), want)


@pytest.mark.parametrize("mode", ["sig", "tanh", "composite"])
@pytest.mark.parametrize("defect", ["neighbour", "swap"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_planted_defects_change_the_output(small, defect, mode):
    for pas in range(len(G.variant(small)["passes"])):
        p, net, inp, a, _ = G.problem(small, mode, pas, 2, 5, 7, seed=5 if mode == "composite" else 0)
        good, _, _ = pass_model(p, small, pas, net, inp, _sig64, _tanh64)
        if mode != "composite":
            assert torch.equal(good, torch.from_numpy((_sig64 if mode == "sig" else _tanh64)(a.numpy())))
        bad, _, _ = pass_model(p, small, pas, net, inp, _sig64, _tanh64, defect)
        n = int((bad != good).sum())
        assert n >= 0.5 * good.numel(), f"{defect} pass {pas + 1}: only {n} of {good.numel()} outputs change"


# ---- exact-rounding helpers -----------------------------------------------------------------------------------------------------
def test_fma_f32_is_the_rational_fma_rounded_once():
    u = 2.0 ** -23
    # p = 1 - 2^-46 onto c = 2^24 + 2 / -(2^24 + 2): the fp64 sum lands on an fp32 midpoint and rounds to the wrong side
    crafted = [(1 + u, 1 - u, 2.0 ** 24 + 2), (1 + u, 1 - u, -(2.0 ** 24 + 2)), (1 + u, 1 - u, 2.0 ** 24)]
    g = np.random.default_rng(1)
    n = 20000
    a = np.concatenate([[c[0] for c in crafted], g.standard_normal(n) * np.exp2(g.integers(-10, 10, n))]).astype(np.float32)
    b = np.concatenate([[c[1] for c in crafted], g.standard_normal(n)]).astype(np.float32)
    c = np.concatenate([[c[2] for c in crafted], g.standard_normal(n) * np.exp2(g.integers(-30, 30, n))]).astype(np.float32)
    c[-100:] = np.float32(1e-40) * np.arange(100, dtype=np.float32)  # subnormal results
    a[-100:] *= np.float32(2.0 ** -120)
    got = G.fma_f32(a, b, c)
    exact = np.array([G.round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)],
                     dtype=np.float32)
    assert np.array_equal(got.view(np.uint32), exact.view(np.uint32))
    naive = (a.astype(np.float64) * b + c).astype(np.float32)
    assert naive[0] != exact[0] and naive[1] != exact[1], "the crafted cases round twice in plain fp64"


def test_round_f32_ties_to_even():
    assert G.round_f32(Fraction(1) + Fraction(1, 2 ** 24)) == np.float32(1.0)
    assert G.round_f32(Fraction(1) + Fraction(3, 2 ** 24)) == np.float32(1.0 + 2.0 ** -22)
    assert G.round_f32(Fraction(1, 3)) == np.float32(1.0) / np.float32(3.0)


@pytest.mark.parametrize("h,w", [(5, 7), (6, 9)], ids=lambda v: str(v))
def test_upsample_construction(h, w):
    """Every category of coarse pixel sees all 511 tie patterns; the logits are fp32; the fma model equals the rational value
    where m is a power of two and not everywhere else (the order is seen)."""
    coords1, mask, m, bits, flow = G.upsample_problem(2, h, w, 10 * h + w)
    pattern = (bits * (1 << torch.arange(9))).sum(-1)
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    border = ((yy == 0).int() + (yy == h - 1).int() + (xx == 0).int() + (xx == w - 1).int()).expand(2, h, w)
    for name, sel in (("interior", border == 0), ("edge", border == 1), ("corner", border == 2)):
        assert set(pattern[sel].unique().tolist()) == set(range(1, 512)), name
    assert set(m.unique().tolist()) == set(range(1, 10))
    model = G.upsample_model(flow, bits)
    rat = G.upsample_rational(flow, bits)
    pow2 = torch.isin(G.fine_m(bits), torch.tensor([1, 2, 4, 8]))
    assert torch.equal(model[pow2].double(), rat[pow2])
    assert (model[~pow2].double() != rat[~pow2]).any()
