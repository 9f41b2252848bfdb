"""The conv launch log (rb_debug_conv_log) refuses launches it has not logged, and tools/conv_traffic.py's operand-byte and
FLOP arithmetic matches the shapes of the update block at 55 x 128 (the convc2 example of DESIGN section 8)."""
import ctypes as C
import importlib.util
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tool():
    spec = importlib.util.spec_from_file_location("conv_traffic", os.path.join(ROOT, "tools", "conv_traffic.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_conv_log_argument_checks():
    from raft_b200 import capi
    lib = capi.lib
    capi.check(lib.rb_debug_conv_override(0, 0, 0, 0))  # empties the log
    rec = (C.c_int * 10)()
    for i in (-1, 0, 64):
        assert lib.rb_debug_conv_log(i, rec) == -2
        assert b"rb_debug_conv_log" in lib.rb_last_error()


def test_operand_bytes_of_convc2():
    """convc2 (3x3, 256 -> 192) on 96-wide tiles: 55 pixel tiles x 2 channel tiles, 4 chunks, split planes."""
    t = _tool()
    rec = (96, 7, 110, 3, 110, 0, 3, 3, 4, 3)
    w, a = t.conv_bytes(rec)
    assert w == 110 * 4 * 2 * 9 * 96 * 128 and a == 110 * 4 * 2 * 9 * 128 * 128
    assert round(w / 1e6, 1) == 97.3 and round(a / 1e6, 1) == 129.8
    assert t.conv_flops(rec) == 2 * 110 * 128 * 96 * 64 * 4 * 9 * 3
    # single pass: one plane, one wgmma per product
    assert t.conv_bytes(rec[:-1] + (1,)) == (w // 2, a // 2)
    # halo: one 10 x 16-row box per (chunk, kx) on 8 x 16 tiles instead of three 128-row boxes
    hw, ha = t.conv_bytes((96, 4, 112, 5, 112, 160, 3, 3, 4, 3))
    assert hw == 112 * 4 * 2 * 9 * 96 * 128 and ha == 112 * 4 * 2 * 3 * 160 * 128
