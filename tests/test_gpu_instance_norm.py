"""Instance norm of the feature encoders (csrc/encoder.cu) on ill-conditioned channels and flat frames, against fp64.

Instance norm is the one data-dependent reduction of every forward pass.  With seeded weights on random frames every channel
has |mean| / std of a few units, where any way of forming the variance is accurate.  These tests reach the other regime.

1. Bias-shift invariance.  IN(x + c) = IN(x) exactly for a per-channel constant c.  For the convs that instance norm follows
   (15 in the basic fnet, 21 in the small one), c_ch = rho * sqrt(sigma_ch^2 + 1e-5) is added to the bias, sigma_ch^2 being
   the fp64 variance of that conv's output (the largest over the batch), recorded from one pass of the fp64 oracle.  Channel
   (b, ch) then has |mean| / std of about rho_b,ch = c_ch / sqrt(sigma_b,ch^2 + 1e-5) >= rho; rho_eff is the largest over the
   shifted layers.  The fp64 oracle is invariant, so one pass is the reference of both runs.  The shifted run is held to the
   unshifted run and to the oracle within
       max(floor, KAPPA * rho_eff * u) * max(scale, 1),   u = 2^-24, scale = max |oracle output|,
   floor = 1e-4 (test_gpu_kernels.test_encoder), or under RB_MATH_TC_FP16 the larger of that and
   test_gpu_mixed_precision's encoder bound, 3 x the distance of the fp16-operand oracle from fp64.
   KAPPA = 16.  An implementation that keeps the conv output in fp32 and its moments in fp64 loses, per element of a
   normalised layer output y and in units of rho * u: <= 1 storing x = conv + c (|x| ~ rho * std) in fp32, <= 1 rounding
   the mean to fp32 before the (exact, Sterbenz) subtraction, <= |y| in rstd, since the stored values' errors move the
   std by up to rho * u relative.  That is (2 + |y|) rho u per layer, about 6 rho u at |y| ~ 4.  The next conv carries
   the perturbation with gain ~1 (He weights), the next norm divides the gain out again, and the independent errors of
   successive layers add incoherently.  Emulated in fp64 with exactly these roundings, the encoder output stays within
   6.6 rho_eff u over every encoder, size and rho below; 16 leaves 2.4x for the GPU's own fp32 operations.
   Forming var = E[x^2] - mean^2 from fp32 sums instead loses ~rho^2 u of the variance: at rho = 3e3 all of it.
   Measured on an H100 80GB HBM3 at a 700 W power limit: the largest error is 0.56 of its tolerance.  With the conv
   epilogue's former fp32 strip sums, 162 cases failed: RB_MATH_TC at every rho >= 1e3 and at 1e2 at 64 x 96,
   RB_MATH_TC_FP16 at every rho >= 3e3 and in 6 of 8 cases at 1e3, and every layer with fused statistics shifted alone;
   RB_MATH_SIMT and the stand-alone layers passed.
   Covered: rho in {1e2, 1e3, 3e3, 1e4} with every layer shifted, and each layer alone at rho = 3e3 (the failure names
   the layer); basic and small fnet; RB_MATH_TC, RB_MATH_SIMT, RB_MATH_TC_FP16; reference and upstream semantics;
   B = 2 at 64 x 96 and B = 1 at 436 x 1024.
2. Flat frames against the fp64 oracle at the same floors: uniform grey, black and white, a letterboxed frame (top and bottom
   quarters black) and a 16 x 16 textured patch on grey.  Their channels have var below eps, where rstd ~ 1 / sqrt(eps).
3. Which statistics path ran: under RB_MATH_TC and RB_MATH_TC_FP16 every instance-normed conv with a multiple of 16 output
   channels writes its statistics in the conv epilogue (rb_debug_conv_last's count), under RB_MATH_SIMT none does.  The
   small fnet's 8- and 24-channel convs take the stand-alone pass in every mode, so they are the control inside a mode.
"""
import contextlib
import ctypes as C

import pytest
import torch

import mixed_oracle as M
import upstream_oracle as U
from oracle import raft_oracle as O

pytestmark = pytest.mark.gpu

UNIT = 2.0 ** -24
KAPPA = 16.0
FLOOR = 1e-4
EPS = 1e-5
ENCODERS = {"basic": (False, 256), "small": (True, 128)}
SIZES = [(2, 64, 96), (1, 436, 1024)]
RHOS = [1e2, 1e3, 3e3, 1e4]
FLAT = ["grey", "black", "white", "letterbox", "patch"]


def _capi():
    from raft_b200 import capi
    return capi


def _modes():
    c = _capi()
    return {"tc": c.RB_MATH_TC, "simt": c.RB_MATH_SIMT, "fp16": c.RB_MATH_TC_FP16}


@pytest.fixture(autouse=True)
def _reset_thread_state():
    """The math mode, semantics and conv override are per-thread library state."""
    yield
    c = _capi()
    c.lib.rb_set_math_mode(c.RB_MATH_TC)
    c.lib.rb_set_semantics(c.RB_SEMANTICS_REFERENCE)
    c.lib.rb_debug_conv_override(0, 0, 0, 0)


def _norm_layers(small, out_dim):
    """(conv scope, cout) of every conv that instance norm follows, in execution order (= the oracle's call order)."""
    c = _capi()
    lib, out = c.lib, []
    for i in range(lib.rb_encoder_num_convs(int(small))):
        if not lib.rb_encoder_norm_name(int(small), i).decode():
            continue
        k, s, ci, co = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        c.check(lib.rb_encoder_conv_shape(int(small), i, out_dim, C.byref(k), C.byref(s), C.byref(ci), C.byref(co)))
        out.append((lib.rb_encoder_conv_name(int(small), i).decode(), co.value))
    return out


def _frame(kind, B, H, W):
    g = torch.Generator().manual_seed(1000 * B + H + W)
    rnd = torch.rand(B, H, W, 3, generator=g)
    if kind == "rand":
        return rnd
    if kind in ("grey", "black", "white"):
        return torch.full((B, H, W, 3), {"grey": 0.5, "black": 0.0, "white": 1.0}[kind])
    if kind == "letterbox":
        rnd[:, :H // 4] = 0.0
        rnd[:, H - H // 4:] = 0.0
        return rnd
    assert kind == "patch"
    img = torch.full((B, H, W, 3), 0.5)
    y, x = H // 2 - 8, W // 2 - 8
    img[:, y:y + 16, x:x + 16] = rnd[:, y:y + 16, x:x + 16]
    return img


@contextlib.contextmanager
def _recording_variances():
    """Wraps O.instance_norm (looked up by O._norm at call time): the fp64 [B, C] variance of every input, in call order."""
    inner, seen = O.instance_norm, []

    def rec(x, eps=EPS):
        seen.append(x.var(dim=(1, 2), unbiased=False))
        return inner(x, eps)

    O.instance_norm = rec
    try:
        yield seen
    finally:
        O.instance_norm = inner


def _weights(small):
    from raft_b200 import synth
    return synth.make_weights(small)


_ORACLE, _EMU, _BASE = {}, {}, {}


def _semantics_ctx(upstream):
    return U.upstream_semantics() if upstream else contextlib.nullcontext()


def _oracle(enc, upstream, B, H, W, frame):
    """fp64 encoder output and the variance of every instance-normed conv output."""
    key = (enc, upstream, B, H, W, frame)
    if key not in _ORACLE:
        small, out_dim = ENCODERS[enc]
        pt = {k: torch.from_numpy(v).double() for k, v in _weights(small).items()}
        fn = O.small_encoder if small else O.basic_encoder
        with _semantics_ctx(upstream), _recording_variances() as var:
            out = fn(2.0 * _frame(frame, B, H, W).double() - 1.0, pt, "fnet", "instance")
        layers = _norm_layers(small, out_dim)
        assert [v.shape[1] for v in var] == [co for _, co in layers], "oracle norms do not follow the library's conv order"
        _ORACLE[key] = (out, var)
    return _ORACLE[key]


def _emulated_fp16_gap(enc, upstream, B, H, W, frame):
    """Max-abs distance of the fp16-operand oracle (tests/mixed_oracle.py) from fp64: the mixed-precision error scale."""
    key = (enc, upstream, B, H, W, frame)
    if key not in _EMU:
        small, _ = ENCODERS[enc]
        pt = {k: torch.from_numpy(v).double() for k, v in _weights(small).items()}
        fn = O.small_encoder if small else O.basic_encoder
        with _semantics_ctx(upstream), M.fp16_convs():
            emu = fn(2.0 * _frame(frame, B, H, W).double() - 1.0, pt, "fnet", "instance")
        _EMU[key] = (emu - _oracle(*key)[0]).abs().max().item()
    return _EMU[key]


def _gpu(cuda, params, enc, mode, upstream, img):
    """The CUDA fnet on `img` -> (output fp64 on the CPU, convs that fused their instance-norm statistics)."""
    from raft_b200.encoders import CudaEncoder
    c = _capi()
    small, out_dim = ENCODERS[enc]
    c.check(c.lib.rb_set_math_mode(_modes()[mode]))
    c.check(c.lib.rb_set_semantics(c.RB_SEMANTICS_UPSTREAM if upstream else c.RB_SEMANTICS_REFERENCE))
    c.check(c.lib.rb_debug_conv_override(0, 0, 0, 0))  # restarts the fused-statistics count
    try:
        out = CudaEncoder(params, "fnet", small, "instance", out_dim, cuda)(img.to(cuda))
        torch.cuda.synchronize()
        fused = c.lib.rb_debug_conv_last(None, None, None, None, None)
        if fused < 0:  # no tensor-core conv has run on this thread yet: none can have fused statistics
            assert mode == "simt" and b"no tensor-core conv" in c.lib.rb_last_error(), c.lib.rb_last_error()
            fused = 0
    finally:
        c.lib.rb_set_math_mode(c.RB_MATH_TC)
        c.lib.rb_set_semantics(c.RB_SEMANTICS_REFERENCE)
    out = out.cpu().double()
    assert torch.isfinite(out).all(), f"{int((~torch.isfinite(out)).sum())} non-finite outputs"
    return out, fused


def _base(cuda, enc, mode, upstream, B, H, W, frame):
    key = (enc, mode, upstream, B, H, W, frame)
    if key not in _BASE:
        _BASE[key] = _gpu(cuda, _weights(ENCODERS[enc][0]), enc, mode, upstream, _frame(frame, B, H, W))
    return _BASE[key]


def _floor(enc, mode, upstream, B, H, W, frame, scale):
    """Absolute tolerance of a run without ill-conditioned channels."""
    tol = FLOOR * max(scale, 1.0)
    if mode == "fp16":
        tol = max(tol, 3.0 * _emulated_fp16_gap(enc, upstream, B, H, W, frame))
    return tol


def _shifted_params(enc, var, rho, only=None):
    """Weights with c_ch = rho * sqrt(max_b sigma_b,ch^2 + eps) added to the bias of the instance-normed convs (all, or
    the one at index `only`), and rho_eff, the largest |c| / sqrt(sigma^2 + eps) of a shifted channel."""
    small, out_dim = ENCODERS[enc]
    params = dict(_weights(small))
    rho_eff = 0.0
    for j, ((conv, _), v) in enumerate(zip(_norm_layers(small, out_dim), var)):
        if only is not None and j != only:
            continue
        c = rho * torch.sqrt(v.max(dim=0).values + EPS)
        rho_eff = max(rho_eff, (c / torch.sqrt(v + EPS)).max().item())
        name = f"fnet/{conv}/b"
        params[name] = (torch.from_numpy(params[name]).double() + c).float().numpy()
    return params, rho_eff


def _check_shift(cuda, enc, mode, upstream, B, H, W, rho, only=None):
    ref, var = _oracle(enc, upstream, B, H, W, "rand")
    base, _ = _base(cuda, enc, mode, upstream, B, H, W, "rand")
    params, rho_eff = _shifted_params(enc, var, rho, only)
    out, _ = _gpu(cuda, params, enc, mode, upstream, _frame("rand", B, H, W))
    scale = ref.abs().max().item()
    floor = _floor(enc, mode, upstream, B, H, W, "rand", scale)
    tol = max(floor, KAPPA * rho_eff * UNIT * max(scale, 1.0))
    e_base = (base - ref).abs().max().item()
    e_ref = (out - ref).abs().max().item()
    e_pair = (out - base).abs().max().item()
    what = f"{enc} {mode} {'upstream' if upstream else 'reference'} B={B} {H}x{W} rho={rho:g} (rho_eff {rho_eff:.3g})"
    if only is not None:
        what += f" shifting {_norm_layers(*ENCODERS[enc])[only][0]} only"
    print(f"\n{what}: unshifted vs fp64 {e_base:.2e}, shifted vs fp64 {e_ref:.2e}, shifted vs unshifted {e_pair:.2e}, "
          f"tol {tol:.2e} (scale {scale:.2f})")
    assert e_base < floor, f"{what}: unshifted run {e_base:.3e} from fp64 (tolerance {floor:.3e})"
    assert e_ref < tol, f"{what}: shifted run {e_ref:.3e} from fp64 (tolerance {tol:.3e})"
    assert e_pair < tol, f"{what}: shifted run {e_pair:.3e} from the unshifted run (tolerance {tol:.3e})"


_MODE_IDS = ["tc", "simt", "fp16"]
_SEM = pytest.mark.parametrize("upstream", [False, True], ids=["reference", "upstream"])
_MODE = pytest.mark.parametrize("mode", _MODE_IDS)
_ENC = pytest.mark.parametrize("enc", list(ENCODERS))
_SIZE = pytest.mark.parametrize("B,H,W", SIZES, ids=lambda v: str(v))


@pytest.mark.parametrize("rho", RHOS, ids=lambda r: f"rho{r:g}")
@_SIZE
@_SEM
@_MODE
@_ENC
def test_bias_shift_invariance(cuda, enc, mode, upstream, B, H, W, rho):
    _check_shift(cuda, enc, mode, upstream, B, H, W, rho)


NORMED_CONVS = {"basic": 15, "small": 21}  # rb_encoder_norm_name != "" (checked by test_statistics_path)


@_SEM
@_MODE
@pytest.mark.parametrize("enc,layer", [(e, j) for e, n in NORMED_CONVS.items() for j in range(n)],
                         ids=lambda v: str(v))
def test_bias_shift_invariance_per_layer(cuda, enc, layer, mode, upstream):
    _check_shift(cuda, enc, mode, upstream, 2, 64, 96, 3e3, only=layer)


@_SIZE
@_SEM
@_MODE
@_ENC
@pytest.mark.parametrize("frame", FLAT)
def test_flat_frames(cuda, frame, enc, mode, upstream, B, H, W):
    ref, _ = _oracle(enc, upstream, B, H, W, frame)
    out, _ = _base(cuda, enc, mode, upstream, B, H, W, frame)
    scale = ref.abs().max().item()
    tol = _floor(enc, mode, upstream, B, H, W, frame, scale)
    err = (out - ref).abs().max().item()
    print(f"\n{frame} {enc} {mode} upstream={upstream} B={B} {H}x{W}: vs fp64 {err:.2e}, tol {tol:.2e} (scale {scale:.2f})")
    assert err < tol, f"max abs err {err:.3e} vs fp64 (tolerance {tol:.3e}, scale {scale:.2f})"


@_SIZE
@_MODE
@_ENC
def test_statistics_path(cuda, enc, mode, B, H, W):
    small, out_dim = ENCODERS[enc]
    layers = _norm_layers(small, out_dim)
    fusable = sum(1 for _, co in layers if co % 16 == 0)
    assert len(layers) == NORMED_CONVS[enc]
    assert fusable == (13 if small else 15)  # the small fnet's 8- and 24-channel convs take the stand-alone pass
    _, fused = _base(cuda, enc, mode, False, B, H, W, "rand")
    assert fused == (0 if mode == "simt" else fusable), f"{fused} convs fused their statistics"
