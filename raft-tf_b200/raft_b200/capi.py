"""ctypes binding of include/raft_b200.h.  There is no fallback: if the CUDA library is missing the
import fails loudly (build it with ``python raft-tf_b200/build.py`` or ``__graft_entry__.build()``)."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RAFT_B200_LIB") or os.path.join(_HERE, "..", "lib", "libraft_b200.so")  # env override: A/B of builds

RB_MATH_TC, RB_MATH_SIMT, RB_MATH_TC_FP16 = 0, 1, 2
RB_SEMANTICS_REFERENCE, RB_SEMANTICS_UPSTREAM = 0, 1

if not os.path.exists(LIB_PATH):
    raise ImportError(f"raft_b200: {LIB_PATH} not found -- the CUDA extension is required (no CPU fallback); "
                      "run `python raft-tf_b200/build.py`")
lib = C.CDLL(LIB_PATH)

_vp, _i, _sz, _f, _d = C.c_void_p, C.c_int, C.c_size_t, C.c_float, C.c_double
_pi, _psz = C.POINTER(C.c_int), C.POINTER(C.c_size_t)

# name -> (restype, argtypes); mirrors include/raft_b200.h one to one
SIGNATURES = {
    "rb_version": (_i, []),
    "rb_last_error": (C.c_char_p, []),
    "rb_set_math_mode": (_i, [_i]),
    "rb_get_math_mode": (_i, []),
    "rb_set_semantics": (_i, [_i]),
    "rb_get_semantics": (_i, []),
    "rb_set_device": (_i, [_i]),
    "rb_launch_count": (C.c_longlong, []),
    "rb_launch_count_reset": (None, []),
    "rb_debug_set_buffer": (_i, [_vp]),
    "rb_debug_conv_override": (_i, [_i, _i, _i, _i]),
    "rb_debug_conv_last": (_i, [_pi, _pi, _pi, _pi, _pi]),
    "rb_debug_conv_last_passes": (_i, []),
    "rb_debug_conv_halo": (_i, [_i]),
    "rb_debug_conv_log": (_i, [_i, _pi]),
    "rb_coords_grid": (_i, [_vp, _i, _i, _i, _vp]),
    "rb_coords_init": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "rb_coords_to_flow": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "rb_corr_pyramid_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_corr_level_offset": (_i, [_i, _i, _i, _i, _psz, _pi, _pi]),
    "rb_corr_workspace_bytes": (_i, [_i, _i, _i, _i, _psz]),
    "rb_corr_build": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _sz, _vp]),
    "rb_corr_lookup": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rb_bilinear_sample": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rb_conv2d_workspace_bytes": (_i, [_i, _i, _i, _i, _i, _i, _i, _psz]),
    "rb_conv2d": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    "rb_conv2d_strided": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    "rb_update_num_convs": (_i, [_i]),
    "rb_update_conv_name": (C.c_char_p, [_i, _i]),
    "rb_update_conv_shape": (_i, [_i, _i, _pi, _pi, _pi, _pi]),
    "rb_update_weights_bytes": (_i, [_i, _psz]),
    "rb_update_weights_pack": (_i, [_i, C.POINTER(_vp), C.POINTER(_vp), _vp, _sz, _vp]),
    "rb_update_weights_pack_host": (_i, [_i, C.POINTER(_vp), C.POINTER(_vp), _vp, _sz]),
    "rb_update_packed_conv": (_i, [_i, _i, _psz, _psz, _psz, _pi, _pi, _pi, _pi, _pi]),
    "rb_update_workspace_bytes": (_i, [_i, _i, _i, _i, _psz]),
    "rb_update_set_state": (_i, [_i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "rb_update_set_state_cnet": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "rb_update_get_net": (_i, [_i, _vp, _vp, _i, _i, _i, _vp]),
    "rb_update_lookup": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "rb_update_set_corr": (_i, [_i, _vp, _vp, _i, _i, _i, _vp]),
    "rb_update_step": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "rb_raft_iterate": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rb_corr_otf_workspace_bytes": (_i, [_i, _i, _i, _i, _psz]),
    "rb_corr_otf_prepare": (_i, [_vp, _vp, _sz, _i, _i, _i, _i, _vp]),
    "rb_corr_otf_lookup": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "rb_update_lookup_otf": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rb_upsample_convex": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "rb_upflow8": (_i, [_vp, _vp, _i, _i, _i, _f, _vp]),
    "rb_upsample_convex_crop": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rb_upflow8_crop": (_i, [_vp, _vp, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "rb_flow_fb_check": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _f, _f, _vp]),
    "rb_track_points": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _f, _f, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "rb_track_points_backward": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _f, _f, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "rb_flow_accumulate": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _f, _f, _i, _vp, _vp, _vp]),
    "rb_flow_accumulate_backward": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _f, _f, _i, _vp, _vp, _vp]),
    "rb_labels_propagate": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp]),
    "rb_labels_propagate_keys": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "rb_global_motion_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_global_motion": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _f, _i, _d, _d, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "rb_frames_warp_affine": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "rb_masked_fill_workspace_bytes": (_i, [_i, _i, _i, _i, _psz]),
    "rb_masked_fill": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "rb_inpaint_masks": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rb_inpaint_propagate": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _f, _f, _f, _vp, _i, _vp, _vp, _vp]),
    "rb_flow_extend_residual": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp]),
    "rb_flow_extend_finish": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp]),
    "rb_frames_warp_affine_fill": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, _f, _f, _f, _vp, _vp, _i, _vp, _vp,
                                        _vp]),
    "rb_denoise_merge": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _i, _f, _f, _f, _vp, _i, _f, _vp, _vp, _vp]),
    "rb_noise_sums": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "rb_tcons_terms": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _f, _f, _f, _f, _vp, _vp, _vp, _vp]),
    "rb_screened_poisson_workspace_bytes": (_i, [_i, _i, _psz]),
    "rb_screened_poisson": (_i, [_vp, _vp, _i, _i, _vp, _vp, _sz, _vp]),
    "rb_homography_motion_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_homography_motion": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp, _i, _d, _vp, _vp, _vp, _vp, _sz, _vp]),
    "rb_motion_evidence": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _vp, _vp]),
    "rb_motion_segment": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _i, _f, _f, _f, _vp, _i, _vp, _vp, _vp]),
    "rb_warp_error_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_warp_error": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _i, _f, _f, _f, _vp, _vp, _sz, _vp]),
    "rb_flow_reverse_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_flow_reverse": (_i, [_vp, _vp, _vp, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _sz, _vp]),
    "rb_frame_synthesize": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _f, _vp, _i, _i, _i, _vp]),
    "rb_flow_reverse_multi_workspace_bytes": (_i, [_i, _i, _i, _i, _psz]),
    "rb_flow_reverse_multi": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _sz, _vp]),
    "rb_frame_synthesize_pairs": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i,
                                       _vp]),
    "rb_flow_reverse_items": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _vp, _sz, _vp]),
    "rb_frame_synthesize_items": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i,
                                       _i, _vp]),
    "rb_frame_synthesize_pairs_resized": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _i, _vp, _i, _i,
                                               _i, _vp]),
    "rb_frame_synthesize_items_resized": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _vp, _i,
                                               _i, _i, _vp]),
    "rb_frame_expose_items": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _i,
                                   _i, _i, _i, _vp]),
    "rb_frame_expose_items_resized": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i,
                                           _vp, _i, _i, _i, _vp]),
    "rb_flow_metrics_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_flow_metrics": (_i, [_vp, _f, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "rb_frame_metrics_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_frame_metrics": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "rb_label_metrics": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "rb_scene_cut_scores": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "rb_flow_forward_interpolate_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_flow_forward_interpolate": (_i, [_vp, _vp, _i, _i, _i, _vp, _sz, _vp]),
    "rb_flow_to_color_workspace_bytes": (_i, [_i, _i, _i, _psz]),
    "rb_flow_to_color": (_i, [_vp, _i, _i, _i, _i, _f, _i, _vp, _vp, _sz, _vp]),
    "rb_frames_prepare": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rb_frames_resize": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "rb_flow_resize": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "rb_encoder_num_convs": (_i, [_i]),
    "rb_encoder_conv_name": (C.c_char_p, [_i, _i]),
    "rb_encoder_norm_name": (C.c_char_p, [_i, _i]),
    "rb_encoder_conv_shape": (_i, [_i, _i, _i, _pi, _pi, _pi, _pi]),
    "rb_encoder_weights_bytes": (_i, [_i, _i, _psz]),
    "rb_encoder_weights_pack": (_i, [_i, _i, _i, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), _vp, _sz, _vp]),
    "rb_encoder_weights_pack_host": (_i, [_i, _i, _i, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), _vp, _sz]),
    "rb_encoder_packed_conv": (_i, [_i, _i, _i, _psz, _psz, _psz, _pi, _pi, _pi, _pi]),
    "rb_encoder_workspace_bytes": (_i, [_i, _i, _i, _i, _psz]),
    "rb_encoder_forward": (_i, [_i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _sz, _vp]),
}
# F32's table rows (include/raft_b200.h)
RB_EXPOSE_FRAME, RB_EXPOSE_OPEN, RB_EXPOSE_CLOSE = -1, 1, 2


class ExposeEntry(C.Structure):  # rb_expose_entry
    _fields_ = [("slot", C.c_int32), ("sample", C.c_int32), ("t", C.c_float)]


class ExposeRow(C.Structure):  # rb_expose_row
    _fields_ = [(f, C.c_int32) for f in ("first", "count", "m", "acc", "out", "flags")]


for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)  # AttributeError here = the library does not export a declared symbol
    _fn.restype = _res
    _fn.argtypes = _args


class RaftB200Error(RuntimeError):
    pass


def check(rc: int) -> None:
    if rc != 0:
        raise RaftB200Error(f"raft_b200 error {rc}: {lib.rb_last_error().decode()}")


def ptr(t):
    """Device pointer of a contiguous torch CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "raft_b200 takes contiguous CUDA tensors"
    return t.data_ptr()


import threading

_tls = threading.local()


def stream():
    """Current torch stream handle for the enqueueing calls.  Also keeps the library's own CUDA runtime (statically linked:
    its per-thread current device is independent of torch's) on torch's current device -- every call that launches work
    takes stream() as an argument, so this is the one place that needs to know."""
    import torch
    dev = torch.cuda.current_device()
    if getattr(_tls, "device", None) != dev:
        check(lib.rb_set_device(dev))
        _tls.device = dev
    return torch.cuda.current_stream().cuda_stream


def size_query(fn, *args) -> int:
    out = C.c_size_t(0)
    check(fn(*args, C.byref(out)))
    return out.value
