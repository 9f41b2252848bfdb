"""The exact conv models of tests/exact_oracle.py, checked without a GPU.

  * ``split`` is the library's own host split bit for bit: the hi / lo planes the weight packers write, on weights with
    round-to-nearest-even ties of hi, residuals that make lo round, lo in the fp16 subnormal range, +-65504 and the
    saturation above it, and -0;
  * every case test_gpu_exact_conv.py runs meets its certificate, and families X, W and XW really carry nonzero lo planes;
  * why the exact file exists: a planted defect (one tap's a_lo * w_hi dropped, or one input channel's lo plane read as zero)
    stays inside the 2e-5 * max|y| tolerance of the randn conv tests after ReLU, and differs from the exact model on family
    data with relu = 0."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_oracle as E
from oracle import raft_oracle as O
from raft_b200 import capi, synth
from test_gpu_exact_conv import CASE_IDS, CASES, ENC_SHAPES, SWEEP_CASES, _encoder_problem, _head_model, _head_problem, _operands
from test_gpu_kernels import CONV_CASES

lib = capi.lib


# ---- split == the host packers ----------------------------------------------------------------------------------------------
def _edge_values(n, seed):
    """n fp32 weights: the edge cases first, then randn over many binades (residuals of up to 13 bits: lo rounds)."""
    f = np.float32
    u = 2.0 ** -11
    edges = [0.0, -0.0, 1 + u, 1 + 3 * u, -(1 + u), 2 + 2 * u, 1 + u - 2 ** -23, 1 + u + 2 ** -23,  # hi ties / near-ties
             1 + 2 ** -12 + 2 ** -23, 3.14159265, -2.71828183,                                      # lo rounds
             2 ** -8 + 2 ** -31, 2 ** -8 + 3 * 2 ** -30, -(2 ** -10 + 2 ** -33), 2 ** -12 + 2 ** -35,  # lo subnormal
             3e-6, -5.96e-8, 2 ** -24, 2 ** -25,                                                    # hi subnormal / flush
             65504.0, -65504.0, 65505.0, 65519.0, 65520.0, -65520.0, 1e6, -3e38, 32768.5, 2048.5]    # range, saturation
    g = np.random.default_rng(seed)
    rest = (g.standard_normal(n - len(edges)) * np.exp2(g.integers(-20, 12, n - len(edges)))).astype(f)
    return np.concatenate([np.array(edges, dtype=f), rest])


def _packed_planes(blob, hi, lo, cout_pad, taps, cin_pad):
    n = cout_pad * taps * cin_pad
    h = np.frombuffer(blob, dtype=np.uint16, count=n, offset=hi).reshape(cout_pad, taps, cin_pad)
    l = np.frombuffer(blob, dtype=np.uint16, count=n, offset=lo).reshape(cout_pad, taps, cin_pad)
    return h, l


def _assert_split_matches(W, h, l):
    """W HWIO fp32 against packed planes [cout_pad][tap][cin_pad] as fp16 bit patterns."""
    kh, kw, cin, cout = W.shape
    hi, lo = E.split(W.reshape(kh * kw, cin, cout).transpose(2, 0, 1))
    assert np.array_equal(h[:cout, :, :cin], hi.view(np.uint16)), "hi plane"
    assert np.array_equal(l[:cout, :, :cin], lo.view(np.uint16)), "lo plane"


@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_split_equals_update_packer(small):
    s = int(small)
    p = synth.make_weights(small)
    n = lib.rb_update_num_convs(s)
    Ws, bs, keep, names = (C.c_void_p * n)(), (C.c_void_p * n)(), [], []
    for i in range(n):
        name = lib.rb_update_conv_name(s, i).decode()
        W = np.ascontiguousarray(p[name + "/W"], dtype=np.float32)
        if name.endswith("flow_head/conv1"):
            W = np.ascontiguousarray(_edge_values(W.size, 3).reshape(W.shape))
        b = np.ascontiguousarray(p[name + "/b"], dtype=np.float32)
        keep += [W, b]
        names.append(name)
        Ws[i], bs[i] = W.ctypes.data, b.ctypes.data
    blob = np.zeros(capi.size_query(lib.rb_update_weights_bytes, s), dtype=np.uint8)
    capi.check(lib.rb_update_weights_pack_host(s, Ws, bs, blob.ctypes.data, blob.size))
    hi, lo, bias = C.c_size_t(), C.c_size_t(), C.c_size_t()
    kh, kw, cin_pad, cout, cout_pad = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
    checked = 0
    for cid, name in ((8, "flow_head/conv1"), (9, "flow_head/conv2"), (1, "encoder/convc2")):
        if small and cid == 1:
            continue
        capi.check(lib.rb_update_packed_conv(s, cid, C.byref(hi), C.byref(lo), C.byref(bias), C.byref(kh), C.byref(kw),
                                             C.byref(cin_pad), C.byref(cout), C.byref(cout_pad)))
        W = keep[2 * names.index("update_block/" + name)]
        h, l = _packed_planes(blob, hi.value, lo.value, cout_pad.value, kh.value * kw.value, cin_pad.value)
        _assert_split_matches(W, h, l)
        checked += 1
    assert checked == (2 if small else 3)


@pytest.mark.parametrize("small", [False, True], ids=["basic", "small"])
def test_split_equals_encoder_packer(small):
    """Norm "none": the packed weights are the given ones, unscaled."""
    s, out_dim = int(small), (128 if small else 256)
    p = synth.make_weights(small)
    n = lib.rb_encoder_num_convs(s)
    Ws, bs, bns, keep = (C.c_void_p * n)(), (C.c_void_p * n)(), (C.c_void_p * n)(), []
    for i in range(n):
        cname = f"fnet/{lib.rb_encoder_conv_name(s, i).decode()}"
        W = np.ascontiguousarray(p[cname + "/W"], dtype=np.float32)
        if i in (1, n - 1):
            W = np.ascontiguousarray(_edge_values(W.size, 10 + i).reshape(W.shape))
        b = np.ascontiguousarray(p[cname + "/b"], dtype=np.float32)
        keep += [W, b]
        Ws[i], bs[i] = W.ctypes.data, b.ctypes.data
    blob = np.zeros(capi.size_query(lib.rb_encoder_weights_bytes, s, out_dim), dtype=np.uint8)
    capi.check(lib.rb_encoder_weights_pack_host(s, 0, out_dim, Ws, bs, bns, blob.ctypes.data, blob.size))
    for i in (1, n - 1):
        hi, lo, bias = C.c_size_t(), C.c_size_t(), C.c_size_t()
        kh, kw, cin_pad, cout_pad = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        capi.check(lib.rb_encoder_packed_conv(s, out_dim, i, C.byref(hi), C.byref(lo), C.byref(bias), C.byref(kh), C.byref(kw),
                                              C.byref(cin_pad), C.byref(cout_pad)))
        h, l = _packed_planes(blob, hi.value, lo.value, cout_pad.value, kh.value * kw.value, cin_pad.value)
        _assert_split_matches(keep[2 * i], h, l)


def test_split_edge_cases_are_present():
    """The edge weights above really hit the cases they are named for."""
    v = _edge_values(64, 3)
    hi, lo = E.split(v)
    hf, lf = hi.astype(np.float32), lo.astype(np.float32)
    resid = (v[:40].astype(np.float64) - hf[:40]) * 2048
    assert (np.abs(resid) == 1).any(), "no hi tie"
    assert ((lf[:40] != resid) & np.isfinite(resid)).any(), "no lo rounding"
    assert ((lf != 0) & (np.abs(lf) < 2.0 ** -14)).any(), "no subnormal lo"
    assert (hf == 65504).any() and (hf == -65504).any() and (v > 65520).any(), "no saturation"
    assert np.signbit(hi[1]) and hi[1] == 0, "-0"
    assert np.isfinite(hf).all() and np.isfinite(lf).all()


# ---- the GPU file's preconditions --------------------------------------------------------------------------------------------
def _lo_nonzero(t):
    return bool((E.planes(t)[1] != 0).any())


@pytest.mark.parametrize("case,stride,upstream", CASES, ids=CASE_IDS)
def test_conv_cases_certified(case, stride, upstream):
    """Every stand-alone case of test_gpu_exact_conv.py meets its certificate under each back end its family is meant for;
    X / W / XW carry the lo planes they are named for, I none; the outputs take both signs."""
    for family in ("I", "X", "W", "XW"):
        x, W, b = _operands(case, stride, upstream, family)
        assert _lo_nonzero(x) == (family in ("X", "XW")), (family, "activation lo plane")
        assert _lo_nonzero(W) == (family in ("W", "XW")), (family, "weight lo plane")
        for back_end in (E.TC, E.SIMT, E.FP16):
            if family in E.FAMILIES[back_end]:
                y = E.certify(x, W, b, stride, back_end, upstream)
                assert (y < 0).any() and (y > 0).any()
        if family == "XW":
            with pytest.raises(AssertionError):  # lo * lo: the CUDA-core sums are not exact on XW
                E.certify(x, W, b, stride, E.SIMT, upstream)
    assert SWEEP_CASES and all(c in CASES for c in SWEEP_CASES)


@pytest.mark.parametrize("upstream", [False, True], ids=["reference", "upstream"])
@pytest.mark.parametrize("small,B,H,W", ENC_SHAPES, ids=lambda v: str(v))
def test_encoder_chains_certified(small, B, H, W, upstream):
    """Every conv of the encoders test_gpu_exact_conv.py runs certifies, its input below 2^15; the stored activations carry
    lo planes; the single-pass model differs from the three-pass one (the mode is seen)."""
    rec = []
    p, img, _ = _encoder_problem(small, B, H, W, E.TC, upstream)
    y = E.encoder_model(p, "fnet", small, img, E.TC, upstream, rec)
    assert sum(r[2] for r in rec) > 0, "no stored activation with a nonzero lo plane"
    assert max(r[1] for r in rec) < 1 and max(r[0] for r in rec) < E.STORED
    assert not torch.equal(y, E.encoder_model(p, "fnet", small, img, E.FP16, upstream))
    assert torch.equal(y, E.encoder_model(p, "fnet", small, img, E.SIMT, upstream))


@pytest.mark.parametrize("family", ["X", "I"])
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
def test_update_heads_certified(small, family):
    p, net, _, _ = _head_problem(small, 2, 12, 20, family, 7 * 2 + 12 + 20)
    assert _lo_nonzero(net) == (family == "X")
    for back_end in (E.TC, E.SIMT, E.FP16):
        delta, mask = _head_model(p, net, small, back_end)
        assert delta.abs().max() > 0 and (small or mask.abs().max() > 0)


# ---- why: a planted defect inside the tolerance, outside the exact comparison ---------------------------------------------
def _tc_conv(x, W, b, defect=None):
    """RB_MATH_TC's conv in fp64 from the split planes, with an optional planted defect:
    ("tap", ky, kx, ci): that tap's a_lo * w_hi dropped; ("lo", ci): input channel ci's lo plane read as zero."""
    ha, la, _ = E.planes(x)
    hw, lw, _ = E.planes(W)
    hw_x = hw.clone()
    if defect and defect[0] == "lo":
        la = la.clone()
        la[..., defect[1]] = 0
    with E.model(E.SIMT):
        y = E._conv(ha, hw, 1, False) + E.LO * (E._conv(ha, lw, 1, False) + E._conv(la, hw_x, 1, False))
        if defect and defect[0] == "tap":
            one = torch.zeros_like(hw)
            one[defect[1], defect[2], defect[3]] = hw[defect[1], defect[2], defect[3]]
            y = y - E.LO * E._conv(la, one, 1, False)
    return y + b.double()


@pytest.mark.parametrize("defect", [("tap", 1, 1, 5), ("lo", 5)], ids=["tap_alo_whi", "channel_lo"])
def test_planted_defect_passes_tolerance_fails_exact(defect):
    case = CONV_CASES[2]  # 3x3, 256 -> 192
    B, h, w, cin, cout, kh, kw = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(B, h, w, cin, generator=g)
    W = torch.randn(kh, kw, cin, cout, generator=g) * (2.0 / (kh * kw * cin)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    ref = O.conv2d(x.double(), W.double(), b.double(), 1, torch.relu)
    bad = torch.relu(_tc_conv(x, W, b, defect).float().double())
    good = torch.relu(_tc_conv(x, W, b).float().double())
    tol = 2e-5 * max(ref.abs().max().item(), 1.0)
    assert not torch.equal(bad, good), "the defect must change the output"
    assert (bad - ref).abs().max().item() < tol, "the defect is visible to the tolerance test"
    x, W, b = _operands(case, 1, False, "X")
    want = E.certify(x, W, b, 1, E.TC)
    got = _tc_conv(x, W, b, defect)
    assert torch.equal(_tc_conv(x, W, b), want)
    assert not torch.equal(got.float(), want.float()), "the exact comparison misses the defect"
