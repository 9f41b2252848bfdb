"""The C-ABI library loads on a CPU-only box and exports every symbol include/raft_b200.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from raft_b200 import capi
    names = _declared()
    assert len(names) >= 25
    lib = ctypes.CDLL(capi.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in raft_b200.h but not exported"
    assert set(names) == set(capi.SIGNATURES), set(names) ^ set(capi.SIGNATURES)


def test_host_only_queries():
    from raft_b200 import capi
    lib = capi.lib
    assert lib.rb_version() >= 100
    assert lib.rb_update_num_convs(0) == 15 and lib.rb_update_num_convs(1) == 9
    assert lib.rb_update_conv_name(0, 5) == b"update_block/gru/convz1"
    assert lib.rb_update_conv_name(1, 8) == b"update_block/flow_head/conv2"
    # pyramid size at things@440x1024 = 261.3 MB (SURVEY section 6)
    assert capi.size_query(lib.rb_corr_pyramid_bytes, 1, 55, 128) == 4 * 7040 * (55 * 128 + 27 * 64 + 13 * 32 + 6 * 16) + 256
    # error path: status code + message, no abort
    out = ctypes.c_size_t()
    assert lib.rb_corr_pyramid_bytes(1, 4, 4, ctypes.byref(out)) == -1
    assert b"too small" in lib.rb_last_error()
    assert lib.rb_set_math_mode(7) == -2
    # argument checks come before any CUDA call: unsupported stride / even kernel -> RB_ERR_UNSUPPORTED on a CPU-only box
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.rb_conv2d_strided(p, p, None, p, 1, 8, 8, 4, 4, 3, 3, 3, 0, p, 64, None) == -3
    assert b"stride" in lib.rb_last_error()
    assert lib.rb_conv2d_strided(p, p, None, p, 1, 8, 8, 4, 4, 2, 2, 1, 0, p, 64, None) == -3
    assert lib.rb_update_packed_conv(0, 12, None, None, None, None, None, None, None, None) == -2


def test_pipeline_argument_checks():
    """Bad arguments of the frame, upsampling, loop and volume-free entry points return RB_ERR_* with a message before any
    CUDA call (every pointer below is a host address: a launch would fail, not return these codes)."""
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG = -1, -2
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def refused(rc, code, *words):
        assert rc == code, (rc, code)
        msg = lib.rb_last_error()
        assert all(w in msg for w in words), msg

    # rb_frames_prepare(src, u8, dst, B, H, W, top, bottom, left, right)
    refused(lib.rb_frames_prepare(None, 1, p, 2, 37, 53, 0, 0, 0, 0, None), BAD_ARG, b"rb_frames_prepare", b"null")
    refused(lib.rb_frames_prepare(p, 0, None, 2, 37, 53, 0, 0, 0, 0, None), BAD_ARG, b"rb_frames_prepare", b"null")
    for pads in ((-1, 0, 0, 0), (0, -1, 0, 0), (0, 0, -1, 0), (0, 0, 0, -3)):
        refused(lib.rb_frames_prepare(p, 1, p, 2, 37, 53, *pads, None), BAD_SHAPE, b"rb_frames_prepare", b"pad")
    # crops of the 8h x 8w = 56 x 72 field: (top, left, out_h, out_w)
    for top, left, oh, ow in ((0, 0, 57, 72), (0, 0, 56, 73), (50, 0, 7, 8), (0, 70, 8, 3), (-1, 0, 8, 8), (0, -2, 8, 8),
                              (0, 0, 0, 8), (0, 0, 8, 0), (4, 4, -1, 8)):
        refused(lib.rb_upsample_convex_crop(p, p, p, 2, 7, 9, top, left, oh, ow, None), BAD_SHAPE,
                b"rb_upsample_convex_crop", b"outside")
        refused(lib.rb_upflow8_crop(p, p, 2, 7, 9, ctypes.c_float(1.0), top, left, oh, ow, None), BAD_SHAPE,
                b"rb_upflow8_crop", b"outside")
    # rb_raft_iterate(small, weights, workspace, pyramid, coords1, mask_out, B, h, w, iters)
    for small in (0, 1):
        refused(lib.rb_raft_iterate(small, p, p, p, p, p, 1, 8, 8, 0, None), BAD_ARG, b"rb_raft_iterate", b"iters")
    refused(lib.rb_raft_iterate(0, p, p, p, p, None, 1, 8, 8, 4, None), BAD_ARG, b"rb_raft_iterate", b"mask_out")
    # volume-free lookups: C must be 128 or 256, the grid at least 8 x 8
    for B, h, w, C in ((1, 8, 8, 64), (1, 7, 8, 256), (1, 8, 7, 128)):
        refused(lib.rb_corr_otf_lookup(p, p, p, p, p, B, h, w, C, 4, None), BAD_SHAPE, b"volume-free")
        for small in (0, 1):
            refused(lib.rb_update_lookup_otf(small, p, p, p, p, p, B, h, w, C, None), BAD_SHAPE, b"volume-free")
    refused(lib.rb_corr_otf_prepare(p, p, 1 << 20, 1, 7, 8, 256, None), BAD_SHAPE, b"rb_corr_otf_prepare")


def test_conv_override_argument_checks():
    """The tensor-core conv test hook refuses configurations the kernel cannot run, without touching CUDA."""
    from raft_b200 import capi
    lib = capi.lib
    bad = [(48, 0, 0, 0), (8, 0, 0, 0), (256, 0, 0, 0), (-32, 0, 0, 0),  # tile widths
           (0, 8, 0, 0), (0, 2, 0, 0), (0, -1, 0, 0),                    # pixel boxes
           (0, 0, -1, 0),                                                 # CTA cap
           (0, 0, 0, 1), (0, 0, 0, -2), (0, 0, 0, 6),                    # a 1-stage ring deadlocks; no width has 6 stages
           (96, 0, 0, 4), (128, 0, 0, 4), (64, 0, 0, 5), (16, 0, 0, 6)]  # ring depth beyond that width's smem ring
    try:
        for args in bad:
            assert lib.rb_debug_conv_override(*args) == -2, args
            assert b"rb_debug_conv_override" in lib.rb_last_error()
        good = [(0, 0, 0, 0), (16, 3, 1, 2), (32, 7, 5, 5), (64, 4, 2, 4), (96, 5, 0, 3), (128, 6, 1, 3), (0, 0, 0, 5)]
        for args in good:
            assert lib.rb_debug_conv_override(*args) == 0, args
    finally:
        assert lib.rb_debug_conv_override(0, 0, 0, 0) == 0

