"""The halo A operand of the wgmma conv (ConvParams::halo, csrc/conv_tc.cu): one (box rows + kh - 1)-row activation box
per channel chunk and kx feeds all kh vertical taps.  The MMA operands and their order are those of one box per tap, so
every output must be BIT-IDENTICAL to the same conv with the halo off (rb_debug_conv_halo(-1)):
  * every kh > 1 filter shape of the update block, stand-alone, under every forced width, box, ring depth and CTA cap, in
    both tensor-core math modes, on grids whose edge tiles reach past the image (TMA zero fill = SAME padding in the halo
    rows);
  * both update blocks (raft-things and raft-small), two steps of rb_update_step, every output and the whole workspace.
The launch log (rb_debug_conv_log) must show the halo where the geometry and shared-memory arithmetic below says it fits."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_conv_coverage import CONFIGS, _conv_problem, _first_diff, _forced

HALO_SLOTS, RING_BYTES = 2, 227 * 1024 - 1024 - 2 * 64 * 36 * 4 - 256 - 1024


# ---- replay of the host arithmetic (conv_tc.cu: choose_geom, halo_b_stages) ----------------------------------------------
def halo_b_stages(block_n, planes, rows):
    n = (RING_BYTES - HALO_SLOTS * planes * rows * 128) // (planes * block_n * 128)
    return 0 if n < 2 else min(n, 6)


def halo_geom(h, w, kh, bwl=0):
    """bw_log2 choose_geom gives a halo conv with a kh-tall filter (forced bwl: that one)."""
    if bwl:
        return bwl
    best = None
    for b in range(7, 2, -1):
        bw, bh = 1 << b, 128 >> b
        if bw > w and b > 3:
            continue
        cost = -(-w // bw) * -(-h // bh) * ((bh + kh - 1) * bw + kh * 128)
        if best is None or cost < best[0]:
            best = (cost, b)
    return best[1]


def halo_rows(h, w, kh, block_n, planes, bwl=0):
    """Rows of the halo box the conv uses, 0 if it keeps one A box per tap."""
    b = halo_geom(h, w, kh, bwl)
    box_h = (128 >> b) + kh - 1
    rows = box_h << b
    return rows if box_h <= 256 and halo_b_stages(block_n, planes, rows) >= 2 else 0


def test_halo_arithmetic():
    """The 55 x 128 grid of a 440 x 1024 pair: 8 x 16 boxes for 3x3 and 5x1 (56 tiles), their rings; the 1-row box's
    halo does not fit beside two N = 128 stages."""
    assert halo_geom(55, 128, 3) == 4 and halo_geom(55, 128, 5) == 4
    assert halo_rows(55, 128, 3, 96, 2) == 160 and halo_rows(55, 128, 5, 128, 2) == 192
    assert halo_b_stages(128, 2, 160) == 3 and halo_b_stages(96, 2, 192) == 4 and halo_b_stages(32, 2, 160) == 6
    assert halo_b_stages(128, 2, 4 * 64) == 2 and halo_b_stages(128, 2, 3 * 128) == 0
    assert halo_rows(55, 128, 3, 128, 2, bwl=7) == 0 and halo_rows(55, 128, 3, 16, 2, bwl=7) == 384
    # every slot and stage is a whole number of 1024-byte swizzle atoms, tap offsets ky * BW * 128 bytes too (BW >= 8)
    for b in range(3, 8):
        for kh in (3, 5):
            assert (((128 >> b) + kh - 1) << b) * 128 % 1024 == 0 and (1 << b) * 128 % 1024 == 0


def test_halo_hook_argument_checks():
    from raft_b200 import capi
    lib = capi.lib
    for bad in (-2, 2):
        assert lib.rb_debug_conv_halo(bad) == -2
        assert b"rb_debug_conv_halo" in lib.rb_last_error()
    assert lib.rb_debug_conv_halo(0) == 0
    capi.check(lib.rb_debug_conv_override(0, 0, 0, 0))
    rec = (C.c_int * 10)()
    assert lib.rb_debug_conv_log(0, rec) == -2 and lib.rb_debug_conv_log(-1, rec) == -2


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def _log():
    from raft_b200 import capi
    rec = (C.c_int * 10)()
    n = capi.lib.rb_debug_conv_log(0, rec)
    out = []
    for i in range(max(n, 0)):
        assert capi.lib.rb_debug_conv_log(i, rec) == n
        out.append(dict(zip(("block_n", "bw_log2", "grid", "stages", "total_tiles", "halo_rows", "kh", "kw", "chunks",
                             "passes"), tuple(rec))))
    return out


class _Halo:
    def __init__(self, mode, math=0):
        self.mode, self.math = mode, math

    def __enter__(self):
        from raft_b200 import capi
        capi.check(capi.lib.rb_debug_conv_halo(self.mode))
        capi.check(capi.lib.rb_set_math_mode(self.math))

    def __exit__(self, *a):
        from raft_b200 import capi
        capi.lib.rb_debug_conv_halo(0)
        capi.lib.rb_set_math_mode(0)


# (B, h, w, cin, cout, kh, kw): the kh > 1 convs of the update block, and grids whose last tiles reach past the image
HALO_CASES = [(1, 16, 32, 256, 192, 3, 3), (1, 16, 32, 128, 64, 3, 3), (1, 16, 32, 256, 126, 3, 3),
              (1, 16, 32, 384, 128, 5, 1), (2, 13, 27, 242, 192, 3, 3), (1, 55, 128, 256, 96, 3, 3),
              (1, 55, 128, 256, 128, 5, 1), (2, 11, 21, 128, 64, 5, 1), (1, 9, 13, 64, 256, 3, 3)]
MATH = {"tc": (0, 2), "fp16": (2, 1)}  # math mode, operand planes


def _conv(cuda, x, W, b, cfg, mode, math):
    from raft_b200 import capi
    lib = capi.lib
    B, h, w, cin = x.shape
    kh, kw, _, cout = W.shape
    y = torch.full((B, h, w, cout), float("nan"), device=cuda)
    wsb = capi.size_query(lib.rb_conv2d_workspace_bytes, B, h, w, cin, cout, kh, kw)
    ws = torch.zeros(wsb, dtype=torch.uint8, device=cuda)
    xd = x.to(cuda)
    Wn, bn = np.ascontiguousarray(W.numpy()), np.ascontiguousarray(b.numpy())
    with _Halo(mode, math), _forced(cfg):
        capi.check(lib.rb_conv2d(capi.ptr(xd), Wn.ctypes.data, bn.ctypes.data, capi.ptr(y), B, h, w, cin, cout, kh, kw, 1,
                                 capi.ptr(ws), wsb, capi.stream()))
        torch.cuda.synchronize()
        log = _log()
    return y.cpu(), log[-1]


@pytest.mark.gpu
@pytest.mark.parametrize("math", sorted(MATH))
@pytest.mark.parametrize("case", HALO_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_halo_same_bits(cuda, case, math):
    B, h, w, cin, cout, kh, kw = case
    mode, planes = MATH[math]
    x, W, b, _ = _conv_problem(B, h, w, cin, cout, kh, kw, 1, 7)
    used = 0
    for cfg in [(0, 0, 0, 0)] + CONFIGS + [(0, 0, 0, 2), (0, 0, 1, 2), (0, 5, 3, 2), (0, 6, 0, 2)]:
        what = f"{case} {math} forced {cfg}"
        off, rec_off = _conv(cuda, x, W, b, cfg, -1, mode)
        on, rec_on = _conv(cuda, x, W, b, cfg, 1, mode)
        assert rec_off["halo_rows"] == 0, what
        want = halo_rows(h, w, kh, rec_on["block_n"], planes, cfg[1])
        assert rec_on["halo_rows"] == want and rec_on["bw_log2"] == halo_geom(h, w, kh, cfg[1]), (what, rec_on, want)
        if want and cfg[3]:
            assert rec_on["stages"] == min(cfg[3], halo_b_stages(rec_on["block_n"], planes, want)), (what, rec_on)
        used += want > 0
        assert torch.isfinite(off).all(), what
        assert torch.equal(on, off), f"{what}: halo differs from one box per tap: {_first_diff(on, off)}"
    assert used > 0, case


def _update_run(cuda, small, B, h, w, mode, cfg, math=0, steps=2):
    from raft_b200 import capi, synth
    from raft_b200.weights import pack_update_block
    lib, s = capi.lib, int(small)
    g = torch.Generator().manual_seed(11 + s)
    hid = 96 if small else 128
    ctx = 64 if small else 128
    pyr = (torch.randn(capi.size_query(lib.rb_corr_pyramid_bytes, B, h, w) // 4, generator=g)).to(cuda)
    grid = torch.stack(torch.meshgrid(torch.arange(w), torch.arange(h), indexing="xy"), -1).float()[None].repeat(B, 1, 1, 1)
    c1 = (grid + torch.rand(B, h, w, 2, generator=g) * 8 - 4).to(cuda).contiguous()
    ws = torch.zeros(capi.size_query(lib.rb_update_workspace_bytes, s, B, h, w), dtype=torch.uint8, device=cuda)
    blob = pack_update_block(synth.make_weights(small), small, cuda)
    net = torch.tanh(torch.randn(B, h, w, hid, generator=g)).to(cuda)
    inp = torch.relu(torch.randn(B, h, w, ctx, generator=g)).to(cuda)
    delta = torch.full((B, h, w, 2), float("nan"), device=cuda)
    mask = None if small else torch.full((B, h, w, 576), float("nan"), device=cuda)
    P, st = capi.ptr, capi.stream()
    with _Halo(mode, math), _forced(cfg):
        capi.check(lib.rb_update_set_state(s, P(blob), P(ws), P(net), P(inp), B, h, w, st))
        for i in range(steps):
            capi.check(lib.rb_update_lookup(s, P(ws), P(pyr), P(c1), B, h, w, st))
            capi.check(lib.rb_update_step(s, P(blob), P(ws), P(c1), P(delta), P(mask) if i == steps - 1 else None,
                                          B, h, w, st))
        torch.cuda.synchronize()
        log = _log()
    outs = [c1.cpu(), delta.cpu(), ws.cpu()] + ([] if small else [mask.cpu()])
    return outs, log


@pytest.mark.gpu
@pytest.mark.parametrize("math", sorted(MATH))
@pytest.mark.parametrize("small", [False, True], ids=["things", "small"])
@pytest.mark.parametrize("B,h,w", [(1, 55, 128), (2, 12, 20)], ids=lambda v: str(v))
def test_update_block_halo_same_bits(cuda, B, h, w, small, math):
    mode, _ = MATH[math]
    cfgs = [(0, 0, 0, 0), (0, 0, 0, 2), (0, 0, 3, 0)] + (CONFIGS if (B, h) == (2, 12) else [(96, 4, 0, 2), (128, 6, 5, 0)])
    for cfg in cfgs:
        what = f"{'small' if small else 'things'} B={B} {h}x{w} {math} forced {cfg}"
        off, log_off = _update_run(cuda, small, B, h, w, -1, cfg, mode)
        on, log_on = _update_run(cuda, small, B, h, w, 0, cfg, mode)
        assert all(r["halo_rows"] == 0 for r in log_off), what
        assert len(log_on) == len(log_off), what
        if cfg == (0, 0, 0, 0) and (B, h, w) == (1, 55, 128):
            # per step: convf1 convf2 [convc1 convc2] motion zr q [zr2 q2] fh1 fh2 (+ mask head on the last step)
            halo = [r["halo_rows"] > 0 for r in log_on]
            assert sum(halo) == (2 * 6 if not small else 2 * 5), (what, log_on)
            assert all(r["halo_rows"] == 0 for r in log_on if r["kh"] == 1 or r["block_n"] == 16), (what, log_on)
        for a, b, nm in zip(on, off, ["coords1", "delta", "workspace", "mask"]):
            assert torch.equal(a, b), f"{what}: {nm} differs with the halo: {_first_diff(a.float(), b.float())}"
