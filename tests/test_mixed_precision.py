"""Mixed precision (RB_MATH_TC_FP16), the parts that need no GPU: the C ABI's mode and test-hook checks, the emulating
oracle of tests/mixed_oracle.py, and the CLI flag."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def lib():
    from raft_b200 import capi
    yield capi.lib
    capi.lib.rb_set_math_mode(capi.RB_MATH_TC)
    capi.lib.rb_debug_conv_override(0, 0, 0, 0)


def test_math_mode_values(lib):
    from raft_b200 import capi
    assert capi.RB_MATH_TC_FP16 == 2
    assert lib.rb_set_math_mode(capi.RB_MATH_TC_FP16) == 0
    assert lib.rb_get_math_mode() == 2
    for bad in (-1, 3, 7):
        assert lib.rb_set_math_mode(bad) == -2
        assert b"unknown mode" in lib.rb_last_error()
    assert lib.rb_get_math_mode() == 2  # a refused value leaves the mode alone
    assert lib.rb_set_math_mode(capi.RB_MATH_TC) == 0 and lib.rb_get_math_mode() == 0


RING_TC = {16: 5, 32: 5, 64: 4, 96: 3, 128: 3}  # TcCfg<N>::kStages, split operands
RING_FP16 = 6                                    # TcCfg<N, true>::kStages: the single-pass stage is half as big (cap 6)


def test_conv_override_validates_stages_against_the_current_modes_ring(lib):
    """rb_debug_conv_override checks `stages` against the ring of the kernel the thread's math mode launches, before any
    CUDA call (this box has no GPU)."""
    from raft_b200 import capi
    for mode, ring in ((capi.RB_MATH_TC, RING_TC), (capi.RB_MATH_SIMT, RING_TC),
                       (capi.RB_MATH_TC_FP16, {n: RING_FP16 for n in RING_TC})):
        assert lib.rb_set_math_mode(mode) == 0
        for n in (0,) + tuple(RING_TC):
            top = max(ring[16], ring[32]) if n == 0 else ring[n]
            for st in range(2, top + 1):
                assert lib.rb_debug_conv_override(n, 0, 0, st) == 0, (mode, n, st)
            assert lib.rb_debug_conv_override(n, 0, 0, top + 1) == -2, (mode, n, top + 1)
            assert b"stages" in lib.rb_last_error()
            assert lib.rb_debug_conv_override(n, 0, 0, 1) == -2
        assert lib.rb_debug_conv_override(48, 0, 0, 0) == -2
        assert lib.rb_debug_conv_override(0, 0, 0, 0) == 0


def test_conv_last_passes_before_any_launch(lib):
    # a fresh thread has launched nothing: the query refuses instead of reporting a stale record
    import threading
    out = []
    t = threading.Thread(target=lambda: out.append(lib.rb_debug_conv_last_passes()))
    t.start()
    t.join()
    assert out == [-2]


def test_fp16_emulation_rounds_conv_operands_only():
    """mixed_oracle.fp16_convs(): conv2d == F.conv2d of the fp16-rounded input and weights (in fp64), the correlation
    matmul == the matmul of the unrounded feature maps, and everything is restored afterwards -- also on top of upstream
    semantics, whose stride-2 conv is a different function."""
    import mixed_oracle as M
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 5, 7, 6, generator=g, dtype=torch.float64)
    W = torch.randn(3, 3, 6, 4, generator=g, dtype=torch.float64)
    b = torch.randn(4, generator=g, dtype=torch.float64)
    f1 = torch.randn(1, 8, 8, 16, generator=g, dtype=torch.float64)
    f2 = torch.randn(1, 8, 8, 16, generator=g, dtype=torch.float64)

    def hand_conv(xx, WW):
        y = F.conv2d(F.pad(xx.permute(0, 3, 1, 2), (1, 1, 1, 1)), WW.permute(3, 2, 0, 1).contiguous(), None)
        return y.permute(0, 2, 3, 1) + b

    def r16(t):
        return t.half().double()

    exact_corr = torch.matmul(f1.reshape(1, 64, 16), f2.reshape(1, 64, 16).transpose(1, 2)) / 4.0
    with M.fp16_convs():
        y = O.conv2d(x, W, b)
        pyr = O.get_corr_pyramid(f1, f2)
    assert (y - hand_conv(r16(x), r16(W))).abs().max() < 1e-12
    assert (y - hand_conv(x, W)).abs().max() > 1e-4  # the rounding is real at these operands
    assert torch.equal(pyr[0].reshape(1, 64, 64), exact_corr)
    conv_tf = O.conv2d
    import upstream_oracle as U
    with U.upstream_semantics(), M.fp16_convs():
        y2 = O.conv2d(x, W, b, 2)
    with U.upstream_semantics():
        assert torch.equal(y2, O.conv2d(r16(x), r16(W), b, 2))
        assert not torch.equal(y2, O.conv2d(x, W, b, 2))
    assert O.conv2d is conv_tf and O.EMULATE is None
    assert (O.conv2d(x, W, b) - hand_conv(x, W)).abs().max() < 1e-12


def test_fold_batch_norm_equals_conv_then_norm():
    """mixed_oracle.fold_batch_norm: the folded cnet with norm 'none' equals conv + batch norm in fp64 (up to the fp32
    rounding of the folded weights, as packed)."""
    import mixed_oracle as M
    from raft_b200 import synth
    p = synth.make_weights(False)
    q = M.fold_batch_norm(p, False, "cnet")
    img = 2.0 * torch.rand(1, 32, 48, 3, generator=torch.Generator().manual_seed(5), dtype=torch.float64) - 1.0
    pt = {k: torch.from_numpy(np.asarray(v)).double() for k, v in p.items()}
    qt = {k: torch.from_numpy(np.asarray(v)).double() for k, v in q.items()}
    ref = O.basic_encoder(img, pt, "cnet", "batch")
    out = O.basic_encoder(img, qt, "cnet", "none")
    assert (out - ref).abs().max() < 1e-4 * max(ref.abs().max().item(), 1.0)
    assert not torch.equal(qt["cnet/conv1/W"], pt["cnet/conv1/W"])


def test_infer_raft_parses_mixed_precision():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "raft-tf_b200"))
    import infer_raft
    assert infer_raft.parser().parse_args(["--mixed_precision"]).mixed_precision is True
    assert infer_raft.parser().parse_args([]).mixed_precision is False


def test_engine_refuses_mixed_precision_on_the_cuda_cores():
    """RaftEngine(mixed_precision=True, math_mode=RB_MATH_SIMT) raises ValueError before it needs a device."""
    from raft_b200 import capi
    from raft_b200.engine import RaftEngine
    with pytest.raises(ValueError, match="mixed_precision"):
        RaftEngine({}, mixed_precision=True, math_mode=capi.RB_MATH_SIMT)
