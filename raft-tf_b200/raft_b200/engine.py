"""Host-side orchestration of one RAFT forward pass on one GPU.

rb_encoder_forward x2 (fnet on both frames, cnet on a forked stream; csrc/encoder.cu) -> rb_corr_build ->
rb_update_set_state_cnet -> rb_raft_iterate (lookup + update block per iteration) -> rb_upsample_convex /
rb_upflow8, all replayed from ONE CUDA graph.  Mirrors RAFT.network_graph (networks/RAFT.py:78-109).
forward_bidirectional runs both directions of B frame pairs as 2B pairs through the same path (each frame encoded once)
and adds the forward-backward consistency check (rb_flow_fb_check, csrc/consistency.cu) to the same graph.
interpolate runs the same bidirectional pass (without the check) from its own graph, then per time t two flow reversals
and the frame blend (rb_flow_reverse, rb_frame_synthesize, csrc/interp.cu) eagerly on the same stream.
forward(flow_init=..., return_low=True) is upstream's warm start: the same graph with rb_coords_init in place of
rb_coords_grid and rb_coords_to_flow (flow_low) after the loop, captured as a mode of its own (FORWARD_WARM).
forward_sequence(frames) is video: T + 1 frames give the T flows f_k -> f_(k+1), fnet once per frame, fmap1 = fmaps[:T] and
fmap2 = fmaps[1:] as overlapping views (SEQUENCE); carry=True continues from the previous call's last frame, whose image
and feature map the graph copies to row 0 before it encodes only the T new frames.
forward_sequence_bidirectional(frames) runs both directions of the T pairs of T + 1 frames as 2T pairs in the palindrome
order (0->1), ..., (T-1->T), (T->T-1), ..., (1->0): fmaps = [f_0 .. f_T, f_(T-1) .. f_0], so fmap1 = fmaps[:2T] and
fmap2 = fmaps[1:] overlap as in SEQUENCE, fnet and cnet run once per frame and the mirrored rows are device copies
(SEQUENCE_BIDIRECTIONAL); interpolate_sequence adds the per-t work of interpolate to it, and interpolate_sequence_at the
work of per-pair times, each (pair, t) item reversed and blended on its own (rb_flow_reverse_items,
rb_frame_synthesize_items).
With input_size set, every mode first resizes the frames to that size like the reference's cv2.resize (rb_frames_resize,
csrc/resize.cu, in the graph in place of rb_frames_prepare), and its outputs come back at that size -- except the frames
of interpolate* with native=True, blended at the frames' own size from the reversed flows at the network size
(rb_frame_synthesize_pairs_resized / _items_resized).
"""
from __future__ import annotations

import os
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import capi
from .encoders import CudaEncoder
from .weights import pack_update_block

# what one pass computes: L->R only (forward), both directions (forward_bidirectional), both plus the occlusion check,
# both directions for interpolate (which also holds the buffers of the per-t calls), L->R warm-started from flow_init with
# the 1/8-resolution flow kept (forward(flow_init=..., return_low=True)), T consecutive pairs of T + 1 frames, always
# started from flow_init (forward_sequence), both directions of T consecutive pairs (forward_sequence_bidirectional and
# interpolate_sequence)
FORWARD, BIDIRECTIONAL, BIDIRECTIONAL_CHECK, INTERPOLATE, FORWARD_WARM, SEQUENCE, SEQUENCE_BIDIRECTIONAL = range(7)
SEQUENCES = (SEQUENCE, SEQUENCE_BIDIRECTIONAL)
# forward-backward consistency thresholds of UnFlow (Meister et al. 2018): |f+b|^2 > a1 (|f|^2 + |b|^2) + a2
FB_ALPHA1, FB_ALPHA2 = 0.01, 0.5
# smallest frame side: the 4-level correlation pyramid needs a 1/8-resolution grid of at least 8 (level 3 is grid >> 3),
# and ceil(H / 8) >= 8 means H >= 57
MIN_FRAME = 57
# upstream mode divides by W_l - 1 at every pyramid level: level 3 must be at least 2 wide, a grid of 16, H >= 121
MIN_FRAME_UPSTREAM = 121
# upstream InputPadder's modes (pad_mode)
PAD_MODES = ("sintel", "kitti")
# most bytes the flow-reversal workspace of one interpolation chunk may take: interpolate, interpolate_sequence and
# interpolate_sequence_at reverse the flows of as many times (items) at once as fit, at least one; the results do not
# depend on it
REVERSE_WS_BOUND = 1 << 30
RB_INTERP_MAX_STEPS = 64  # include/raft_b200.h: times (items) per reversal / blend call


def _kept(parked, key):
    """Whether a call keyed `key` = (B, H, W, u8, mode) keeps the parked buffers of `parked`.  The pair modes keep each
    other at one (B, H, W, u8), as before; the buffers of each sequence mode survive any call of another mode at the same
    frame size (a carry continues across them), and a sequence call keeps the pair modes' buffers at its frame size and
    dtype.  A sequence call of another T or dtype replaces the buffers of its own mode."""
    if parked[4] == key[4] and key[4] in SEQUENCES:
        return parked == key
    if parked[4] in SEQUENCES:
        return parked[1:3] == key[1:3]
    if key[4] in SEQUENCES:
        return parked[1:4] == key[1:4]
    return parked[:4] == key[:4]


class RaftEngine:
    # everything _ensure allocates for one (B, H, W, u8, mode); parked per mode so alternating modes re-captures nothing
    _STATE = ("_key", "src_hw", "pad", "h", "w", "Hp", "Wp", "pairs", "pyr_bytes", "pyramid", "cws_bytes", "corr_ws",
              "ws_bytes", "ws", "coords1", "mask", "flow_up", "occ", "rev_ws_bytes", "rev_ws", "rev_rows", "flow_t", "empty_t", "flow_bw", "flow_init", "flow_low", "fmaps", "fmap1", "fmap2", "cmap", "images", "staged", "raw",
              "seq_enc", "_shape", "_graph", "_graph_carry")

    def __init__(self, params: Dict[str, np.ndarray], small: bool = False, iters: int = 20,
                 device: Optional[torch.device] = None, use_graph: bool = True, math_mode: int = capi.RB_MATH_TC,
                 volume_free: Optional[bool] = None, input_size: Optional[Tuple[int, int]] = None,
                 upstream: bool = False, mixed_precision: bool = False, pad_mode: str = "sintel"):
        # pad_mode: how frames are replicate-padded to a multiple of 8, like upstream's InputPadder -- 'sintel' splits the
        # padding top / bottom and left / right, 'kitti' pads the bottom only (and splits left / right)
        if pad_mode not in PAD_MODES:
            raise ValueError(f"raft_b200: pad_mode must be one of {PAD_MODES} (got {pad_mode!r})")
        self.pad_mode = pad_mode
        # mixed_precision: upstream RAFT's --mixed_precision boundary -- every conv as one fp16 x fp16 wgmma per product with
        # fp32 accumulation, the correlation and all elementwise work as in RB_MATH_TC (RB_MATH_TC_FP16, include/raft_b200.h)
        if mixed_precision:
            if math_mode == capi.RB_MATH_SIMT:
                raise ValueError("raft_b200: mixed_precision runs the convs on the tensor cores; it cannot be combined with "
                                 "math_mode=RB_MATH_SIMT")
            math_mode = capi.RB_MATH_TC_FP16
        self.mixed_precision = math_mode == capi.RB_MATH_TC_FP16
        # upstream: the numerics of princeton-vl RAFT (PyTorch), for checkpoints converted from its .pth files
        # (raft_b200.convert): grid_sample lookup, PyTorch's stride-2 padding, raft-small's flow scaled by 8
        # (RB_SEMANTICS_UPSTREAM, include/raft_b200.h)
        self.upstream = bool(upstream)
        self.semantics = capi.RB_SEMANTICS_UPSTREAM if self.upstream else capi.RB_SEMANTICS_REFERENCE
        self.min_frame = MIN_FRAME_UPSTREAM if self.upstream else MIN_FRAME
        # raft-small's flow: in 1/8-resolution units in the reference (upflow8 does not scale it), in pixels upstream
        self.flow_scale = 8.0 if small and not self.upstream else 1.0
        if input_size is not None:
            input_size = (int(input_size[0]), int(input_size[1]))
            if min(input_size) < self.min_frame:
                raise ValueError(f"raft_b200: input_size {input_size[0]}x{input_size[1]} is too small: frames must be at "
                                 f"least {self.min_frame} pixels on each side")
        if not torch.cuda.is_available():
            raise RuntimeError("raft_b200 needs a CUDA device (no CPU fallback)")
        # network size (Ho, Wo): frames of any size are resized to it on the GPU like the reference's test dataflow
        # (cv2.resize, test_dataflow.py:85-87); None runs frames at their own size (padded to a multiple of 8)
        self.input_size = input_size
        self.device = torch.device(device if device is not None else "cuda:0")
        self.small, self.iters = bool(small), int(iters)
        self.hidden, self.ctx, self.radius, self.fdim = (96, 64, 3, 128) if small else (128, 128, 4, 256)
        self.use_graph = use_graph and not os.environ.get("RAFT_B200_NO_GRAPH")
        # F2 (opt-in): no materialised correlation volume -- every iteration evaluates the dot products its taps touch
        # straight from the feature maps (rb_update_lookup_otf).  Saves 4*N^2*1.33 bytes per pair (261 MB at 440x1024),
        # costs ~100 k extra FMA per pixel and iteration on the CUDA cores; same flow up to fp32 summation order.
        self.volume_free = bool(os.environ.get("RAFT_B200_VOLUME_FREE")) if volume_free is None else bool(volume_free)
        self.math_mode = math_mode
        cnorm = "none" if small else "batch"
        with torch.cuda.device(self.device):
            self.fnet = CudaEncoder(params, "fnet", small, "instance", self.fdim, self.device)
            self.cnet = CudaEncoder(params, "cnet", small, cnorm, self.hidden + self.ctx, self.device)
            self.blob = pack_update_block(params, small, self.device)
        # the bidirectional pass runs the context encoder on 2B frames, forward on B: a twin with its own workspace keeps
        # the workspace each mode's CUDA graph was captured with (the feature encoder sees 2B frames in both modes)
        self.cnet_bidir = self.cnet.with_own_workspace()
        self._shape = None  # (B, H, W, u8, mode) at the size the network runs (input_size when set)
        self._key = None    # (B, H, W, u8, mode) at the frames' own size
        self._graph = None
        self._graph_carry = None  # SEQUENCE: the graph of carry=True calls (self._graph runs the fresh ones)
        self._carry = False       # the SEQUENCE pass being run continues from the previous one
        self._seq_last = None     # (T, H, W, u8, SEQUENCE) of the last forward_sequence call: what carry=True continues
        self.seq_enc = None
        self._parked = {}  # _key -> buffers and graph of the other modes at the current frame size
        self._enc_stream = None   # forked stream of the context encoder (encode())
        self._capture_stream = None  # CUDA-graph capture stream on this engine's device (run())
        self._cnet_pending = False
        self._range_checked = False  # first forward of this weight set: fp16-range check of the split path's inputs
        # motion_blur / expose: two fp32 accumulators [2,H,W,3]; an output frame whose samples span calls carries its sum
        # in one of them, expose_slot the one the next call reads
        self.expose_acc, self.expose_slot = None, 0

    # ---- buffers -------------------------------------------------------------------------------
    def _ensure(self, B: int, H: int, W: int, u8: bool = False, mode: int = FORWARD):
        """Buffers for B frame pairs of H x W pixels.  H, W need not be multiples of 8: frames are replicate-padded
        to (Hp, Wp) by rb_frames_prepare (upstream InputPadder's split of pad_mode, SURVEY 8(d)) and the flow is cropped
        back by the upsampling kernel -- the reference itself cannot run such shapes (SURVEY fact 6).

        In the bidirectional modes the hot path runs 2B pairs, (L_i -> R_i) then (R_i -> L_i): fmaps holds 3B feature
        maps [fL | fR | fL], so fmap1 = fmaps[:2B] and fmap2 = fmaps[B:] are both contiguous views.

        With input_size the frames' H x W (any size >= 1) only sizes the staging buffer; everything else is allocated
        for input_size, and the parking key keeps the frames' own size, so a new source size never finds a graph
        captured for another one."""
        key = (B, H, W, u8, mode)
        if self._key == key:
            return
        src_hw = (H, W)
        if self.input_size is not None:
            if H < 1 or W < 1:
                raise ValueError(f"raft_b200: empty {H}x{W} frames")
            H, W = self.input_size
        if H < self.min_frame or W < self.min_frame:  # refused here, before the encoders run or any buffer is allocated
            raise ValueError(f"raft_b200: {H}x{W} frames are too small: frames must be at least {self.min_frame} pixels on "
                             f"each side (a 1/8-resolution grid of at least {(self.min_frame + 7) // 8}x"
                             f"{(self.min_frame + 7) // 8} for the 4-level correlation pyramid)")
        # alternating modes on one frame size keeps every mode's buffers and CUDA graph; a new frame size drops them
        if self._key is not None:
            self._parked[self._key] = {k: getattr(self, k) for k in self._STATE}
        self._parked = {k: v for k, v in self._parked.items() if _kept(k, key)}
        if key in self._parked:
            self.__dict__.update(self._parked.pop(key))
            return
        bidir = mode not in (FORWARD, FORWARD_WARM, SEQUENCE)
        seq = mode in SEQUENCES
        NB = 2 * B if bidir else B  # frame pairs through the hot path
        ph, pw = (-H) % 8, (-W) % 8
        top = 0 if self.pad_mode == "kitti" else ph // 2
        self.pad = (top, ph - top, pw // 2, pw - pw // 2)  # top, bottom, left, right
        Hp, Wp = H + ph, W + pw
        h, w, s = Hp // 8, Wp // 8, int(self.small)
        d = self.device
        lib = capi.lib
        self.h, self.w, self.Hp, self.Wp, self.pairs = h, w, Hp, Wp, NB
        if self.volume_free:
            self.pyr_bytes, self.pyramid = 0, None
            self.cws_bytes = capi.size_query(lib.rb_corr_otf_workspace_bytes, NB, h, w, self.fdim)  # pooled fmap2, levels 1..3
        else:
            self.pyr_bytes = capi.size_query(lib.rb_corr_pyramid_bytes, NB, h, w)
            self.pyramid = torch.empty(self.pyr_bytes // 4, dtype=torch.float32, device=d)
            self.cws_bytes = capi.size_query(lib.rb_corr_workspace_bytes, NB, h, w, self.fdim)
        self.corr_ws = torch.zeros(self.cws_bytes, dtype=torch.uint8, device=d)
        self.ws_bytes = capi.size_query(lib.rb_update_workspace_bytes, s, NB, h, w)
        self.ws = torch.zeros(self.ws_bytes, dtype=torch.uint8, device=d)  # zero fill = channel padding
        self.coords1 = torch.empty(NB, h, w, 2, dtype=torch.float32, device=d)
        self.mask = None if self.small else torch.empty(NB, h, w, 576, dtype=torch.float32, device=d)
        self.flow_up = torch.empty(NB, H, W, 2, dtype=torch.float32, device=d)  # bidirectional: [L->R | R->L]
        self.occ = (torch.empty(2 * B, H, W, dtype=torch.uint8, device=d)
                    if mode in (BIDIRECTIONAL_CHECK, SEQUENCE_BIDIRECTIONAL) else None)
        # SEQUENCE_BIDIRECTIONAL: the backward flows in pair order (the pass leaves them in rows 2T-1 .. T)
        self.flow_bw = torch.empty(B, H, W, 2, dtype=torch.float32, device=d) if mode == SEQUENCE_BIDIRECTIONAL else None
        # the per-t buffers of interpolate / interpolate_sequence, allocated by _synthesize for the chunk it runs
        self.rev_ws_bytes, self.rev_ws, self.rev_rows, self.flow_t, self.empty_t = 0, None, 0, None, None
        if mode in (FORWARD_WARM, SEQUENCE):  # the caller's initial flow (copied in before each replay), the final 1/8-res flow
            self.flow_init = torch.zeros(B, h, w, 2, dtype=torch.float32, device=d)
            self.flow_low = torch.empty(B, h, w, 2, dtype=torch.float32, device=d)
        else:
            self.flow_init, self.flow_low = None, None
        # SEQUENCE: B = T pairs of T + 1 frames; fmap1 = fmaps[:T] and fmap2 = fmaps[1:] overlap, no copy.
        # SEQUENCE_BIDIRECTIONAL: 2T pairs, fmaps = [f_0 .. f_T, f_(T-1) .. f_0] (2T + 1 rows), fmap1 = fmaps[:2T] and
        # fmap2 = fmaps[1:]; cmap = [c_0 .. c_T, c_(T-1) .. c_1]
        nframes = B + 1 if seq else 2 * B
        self.fmaps = torch.empty(NB + 1 if seq else NB + B, h, w, self.fdim, dtype=torch.float32, device=d)
        self.fmap1, self.fmap2 = self.fmaps[:NB], self.fmaps[1 if seq else B:]
        self.cmap = torch.empty(NB, h, w, self.hidden + self.ctx, dtype=torch.float32, device=d)
        self.images = torch.empty(nframes, Hp, Wp, 3, dtype=torch.float32, device=d)  # [left | right], [0,1], padded
        # staging buffer of the raw frames (uint8 or unpadded fp32, at the frames' own size); fp32 frames that need no
        # resize and no padding go straight into self.images -- except in SEQUENCE, whose carry graph reads the previous
        # call's last frame from self.images, so the new frames must not land there before the replay
        self.staged = bool(u8 or ph or pw or self.input_size is not None or mode == SEQUENCE)
        self.raw = torch.empty(nframes, *src_hw, 3, dtype=torch.uint8 if u8 else torch.float32, device=d) if self.staged else None
        # SEQUENCE: the feature encoder sees T + 1 frames in the fresh graph and T in the carry graph, the context encoder T;
        # encoders with workspaces of their own keep the pointers each graph was captured with (CudaEncoder reallocates its
        # workspace when its batch changes), whatever the other modes run in between
        # SEQUENCE_BIDIRECTIONAL: both encoders see the T + 1 frames (twins for the same reason)
        if mode == SEQUENCE:
            self.seq_enc = (self.fnet.with_own_workspace(), self.fnet.with_own_workspace(), self.cnet.with_own_workspace())
        elif mode == SEQUENCE_BIDIRECTIONAL:
            self.seq_enc = (self.fnet.with_own_workspace(), self.cnet.with_own_workspace())
        else:
            self.seq_enc = None
        self.src_hw = src_hw
        self._key = key
        self._shape = (B, H, W, u8, mode)
        self._graph = None
        self._graph_carry = None

    # ---- stages --------------------------------------------------------------------------------
    def encode(self, defer_join: bool = False):
        """RAFT.py:53-59,79-87 on self.images = [left | right]: 2x-1, fnet(left), fnet(right), cnet(left).

        The context encoder is independent of the feature encoder (RAFT.py:79-87) and both are chains of ~50 small
        kernels at 1/4 and 1/8 resolution: cnet runs on a forked stream beside fnet (a fork/join that is captured into
        the CUDA graph like the flow branch of the update block).  With defer_join the caller joins (`_join_cnet`)
        where cmap is first needed -- after the correlation volume, which only needs the feature maps.

        Bidirectional modes: cnet runs on all 2B frames (the R->L pairs need the context of R), and the last B feature
        maps are a device-to-device copy of the first B (a copy-engine transfer, no kernel)."""
        B, H, W, u8, mode = self._shape
        bidir = mode not in (FORWARD, FORWARD_WARM, SEQUENCE, SEQUENCE_BIDIRECTIONAL)
        cnet, cframes = (self.cnet_bidir, self.images) if bidir else (self.cnet, self.images[:B])
        fnet, fout = self.fnet, self.fmaps[:2 * B]  # [fL | fR]
        cout = self.cmap
        raw, images = self.raw, self.images
        capi.check(capi.lib.rb_set_math_mode(self.math_mode))  # per-thread library state: set before ANY kernel of ours
        capi.check(capi.lib.rb_set_semantics(self.semantics))
        if mode == SEQUENCE:  # B = T pairs; the T + 1 frames all staged in self.raw
            fnet_fresh, fnet_carry, cnet = self.seq_enc
            if self._carry:  # the previous call's last frame becomes frame 0; only the T new frames are encoded
                self.images[0].copy_(self.images[B])
                self.fmaps[0].copy_(self.fmaps[B])
                raw, images = self.raw[1:], self.images[1:]
                fnet, fout = fnet_carry, self.fmaps[1:]
            else:
                fnet, fout = fnet_fresh, self.fmaps
        elif mode == SEQUENCE_BIDIRECTIONAL:  # B = T: both encoders on the T + 1 frames, the mirrored rows copied below
            fnet, cnet = self.seq_enc
            fout, cframes, cout = self.fmaps[:B + 1], self.images, self.cmap[:B + 1]
        n = images.shape[0]
        if self.input_size is not None:  # F3: cv2 resize, u8 -> fp32 /255 and replicate padding in one pass (csrc/resize.cu)
            capi.check(capi.lib.rb_frames_resize(capi.ptr(raw), int(u8), capi.ptr(images), n, *self.src_hw,
                                                 H, W, *self.pad, capi.stream()))
        elif self.staged:  # F3: u8 -> fp32 /255 and replicate padding in one pass (csrc/frames.cu)
            capi.check(capi.lib.rb_frames_prepare(capi.ptr(raw), int(u8), capi.ptr(images), n, H, W,
                                                  *self.pad, capi.stream()))
        main = torch.cuda.current_stream(self.device)
        if self._enc_stream is None:
            self._enc_stream = torch.cuda.Stream(device=self.device)
        side = self._enc_stream
        side.wait_stream(main)  # fork: the frames are in place
        with torch.cuda.stream(side):
            cnet(cframes, out=cout)
            if mode == SEQUENCE_BIDIRECTIONAL:  # cmap row T + i = c_(T-1-i): T - 1 copies
                for i in range(B - 1):
                    self.cmap[B + 1 + i].copy_(self.cmap[B - 1 - i])
        fnet(images, out=fout)
        self._cnet_pending = True
        if bidir:
            self.fmaps[2 * B:].copy_(self.fmaps[:B])  # contiguous, same dtype: cudaMemcpyAsync on the current stream
        elif mode == SEQUENCE_BIDIRECTIONAL:  # fmaps row T + 1 + i = f_(T-1-i): T copies
            for i in range(B):
                self.fmaps[B + 1 + i].copy_(self.fmaps[B - 1 - i])
        if self._cnet_pending and not defer_join:
            self._join_cnet()

    def _join_cnet(self):
        if self._cnet_pending:
            torch.cuda.current_stream(self.device).wait_stream(self._enc_stream)
            self._cnet_pending = False

    def _hot_path(self):
        """corr build + iterations + upsampling (+ the consistency check): hand-written kernels only (graph-capturable)."""
        B0, H, W, _, mode = self._shape
        B = self.pairs
        h, w, s, lib, st = self.h, self.w, int(self.small), capi.lib, capi.stream()
        capi.check(lib.rb_set_math_mode(self.math_mode))
        capi.check(lib.rb_set_semantics(self.semantics))
        if self.volume_free:
            capi.check(lib.rb_corr_otf_prepare(capi.ptr(self.fmap2), capi.ptr(self.corr_ws), self.cws_bytes, B, h, w, self.fdim, st))
        else:
            capi.check(lib.rb_corr_build(capi.ptr(self.fmap1), capi.ptr(self.fmap2), capi.ptr(self.pyramid), B, h, w,
                                         self.fdim, capi.ptr(self.corr_ws), self.cws_bytes, st))
        self._join_cnet()  # cmap (context encoder, forked stream) is first needed here
        capi.check(lib.rb_update_set_state_cnet(s, capi.ptr(self.blob), capi.ptr(self.ws), capi.ptr(self.cmap), B, h, w, st))
        if self.flow_init is not None:  # coords1 = grid + flow_init (upstream RAFT.forward)
            capi.check(lib.rb_coords_init(capi.ptr(self.coords1), capi.ptr(self.flow_init), B, h, w, st))
        else:
            capi.check(lib.rb_coords_grid(capi.ptr(self.coords1), B, h, w, st))
        if self.volume_free:  # RAFT.py:91-102 with the lookup evaluated on the fly
            for it in range(self.iters):
                capi.check(lib.rb_update_lookup_otf(s, capi.ptr(self.ws), capi.ptr(self.fmap1), capi.ptr(self.fmap2),
                                                    capi.ptr(self.corr_ws), capi.ptr(self.coords1), B, h, w, self.fdim, st))
                mask = self.mask if (it == self.iters - 1 and not self.small) else None
                capi.check(lib.rb_update_step(s, capi.ptr(self.blob), capi.ptr(self.ws), capi.ptr(self.coords1), None,
                                              capi.ptr(mask), B, h, w, st))
        else:
            capi.check(lib.rb_raft_iterate(s, capi.ptr(self.blob), capi.ptr(self.ws), capi.ptr(self.pyramid),
                                           capi.ptr(self.coords1), capi.ptr(self.mask), B, h, w, self.iters, st))
        if self.flow_init is not None:
            capi.check(lib.rb_coords_to_flow(capi.ptr(self.coords1), capi.ptr(self.flow_low), B, h, w, st))
        top, left = self.pad[0], self.pad[2]  # crop the padding away while upsampling
        if self.small:
            capi.check(lib.rb_upflow8_crop(capi.ptr(self.coords1), capi.ptr(self.flow_up), B, h, w, 8.0 / self.flow_scale,
                                           top, left, H, W, st))
        else:
            capi.check(lib.rb_upsample_convex_crop(capi.ptr(self.coords1), capi.ptr(self.mask), capi.ptr(self.flow_up),
                                                   B, h, w, top, left, H, W, st))
        if mode == BIDIRECTIONAL_CHECK:  # flow_scale: raft-small's reference flow is in 1/8-resolution units
            capi.check(lib.rb_flow_fb_check(capi.ptr(self.flow_up[:B0]), capi.ptr(self.flow_up[B0:]), capi.ptr(self.occ[:B0]),
                                            capi.ptr(self.occ[B0:]), B0, H, W, self.flow_scale, FB_ALPHA1,
                                            FB_ALPHA2, st))
        elif mode == SEQUENCE_BIDIRECTIONAL:  # pair (k+1 -> k) is row 2T-1-k: T copies into pair order
            for k in range(B0):
                self.flow_bw[k].copy_(self.flow_up[2 * B0 - 1 - k])

    def _all(self):
        self.encode(defer_join=True)
        self._hot_path()

    def launches_per_forward(self) -> int:
        """Number of raft_b200 kernels one forward pass launches (counted by the library)."""
        capi.lib.rb_launch_count_reset()
        with torch.cuda.device(self.device):
            self._all()
            torch.cuda.synchronize()
        return int(capi.lib.rb_launch_count())

    def run(self):
        """encoders + hot path on self.images, replayed from one CUDA graph."""
        if not self.use_graph:
            self._all()
            return
        attr = "_graph_carry" if self._carry else "_graph"
        if getattr(self, attr) is None:
            self._all()  # warm-up: function attributes, tensor-map cache
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            # torch.cuda.graph's default capture stream is a process-wide singleton on whichever device used it first, and
            # entering it switches the current device to THAT device: an engine on another device of the same process
            # would record its kernels there (illegal address at replay).  Capture on a stream of this engine's device.
            if self._capture_stream is None:
                self._capture_stream = torch.cuda.Stream(device=self.device)
            with torch.cuda.graph(g, stream=self._capture_stream):
                self._all()
            setattr(self, attr, g)
            if self._carry:  # the warm-up ran this pass; a replay would carry from the frame it has just encoded
                return
        getattr(self, attr).replay()

    @torch.no_grad()
    def forward(self, left: torch.Tensor, right: torch.Tensor, flow_init: Optional[torch.Tensor] = None,
                return_low: bool = False):
        """left/right: [B,H,W,3] frames, BGR like the reference: fp32 in [0,1] (RAFT.inputs(), RAFT.py:45-51) or
        uint8 in [0,255] (what cv2.imdecode yields, test_dataflow.py:56-61; the /255 then happens on the GPU).  Host
        (ideally pinned) or CUDA tensors; any H, W >= 57 (MIN_FRAME; 121 with upstream=True, whose weights expect RGB
        frames; smaller frames raise ValueError), or any size
        with input_size set, which resizes them to input_size first.  Returns the [B,H,W,2] flow (at input_size when
        set) -- the engine-owned buffer itself, overwritten by the next call (networks.RAFT.RAFT.forward hands
        out a copy).

        Warm start (upstream RAFT's flow_init): flow_init is a [B,h,w,2] fp32 host or CUDA tensor on the padded grid
        h, w = Hp / 8, Wp / 8 (of input_size when set), and the loop starts from coords1 = grid + flow_init.  With
        return_low the call returns (flow_low, flow_up), flow_low = coords1 - grid [B,h,w,2] after the last iteration,
        in the order of upstream's test_mode tuple; forward_interpolate(flow_low) is the next frame's flow_init.  Either
        argument runs a graph of its own (FORWARD_WARM, a zero init when flow_init is None); without them the call is the
        plain forward above.  A wrong shape or dtype raises ValueError."""
        if flow_init is None and not return_low:
            self._run_frames(left, right, FORWARD)
            return self.flow_up
        if flow_init is not None and (not isinstance(flow_init, torch.Tensor) or flow_init.dtype != torch.float32):
            raise ValueError(f"raft_b200: flow_init must be a float32 torch tensor (got "
                             f"{getattr(flow_init, 'dtype', type(flow_init))})")
        self._run_frames(left, right, FORWARD_WARM, flow_init)
        return (self.flow_low, self.flow_up) if return_low else self.flow_up

    @torch.no_grad()
    def forward_sequence(self, frames: torch.Tensor, carry: bool = False, flow_init: Optional[torch.Tensor] = None,
                         return_low: bool = False):
        """Video: the flows between consecutive frames.  frames is [T+1,H,W,3] (dtypes, sizes, input_size and padding as
        for forward()); the call returns the [T,H,W,2] flows f_k -> f_(k+1), each bit-identical to forward(f_k, f_(k+1)).
        The feature encoder runs once per frame (fmap1 = fmaps[:T] and fmap2 = fmaps[1:] are overlapping views), the
        context encoder on the first T frames, the hot path on T pairs.

        carry=True continues the previous forward_sequence call: frames is [T,H,W,3], T new frames after that call's last
        frame, giving the T pairs (last, g_0), (g_0, g_1), ...; the graph copies the last frame's image and feature map to
        row 0 on the device and encodes only the new frames, so a stream of clips encodes every frame once, at any T.  It
        raises ValueError without a preceding sequence call, when T, the frame size or the dtype differ from it, or when a
        call at another frame size released the buffers in between (pair-mode calls at the same size do not).

        Every sequence pass starts from coords = grid + flow_init ([T,h,w,2] on the padded 1/8-resolution grid, row i for
        pair i; zeros when None, which is the cold start bit for bit), so cold and warm calls share the graphs.  With
        return_low the call returns (flow_low, flow_up) as forward() does.  The returned tensors are engine-owned buffers,
        overwritten by the next call; one buffer set serves the fresh and the carry graph."""
        if not (isinstance(frames, torch.Tensor) and frames.dim() == 4 and frames.shape[-1] == 3
                and frames.dtype in (torch.uint8, torch.float32)):
            raise ValueError(f"raft_b200: frames must be a [N,H,W,3] uint8 or float32 tensor (got "
                             f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
        T = frames.shape[0] if carry else frames.shape[0] - 1
        if T < 1:
            raise ValueError(f"raft_b200: forward_sequence needs {'one new frame' if carry else 'two frames'} at least "
                             f"(got {frames.shape[0]})")
        if flow_init is not None and (not isinstance(flow_init, torch.Tensor) or flow_init.dtype != torch.float32):
            raise ValueError(f"raft_b200: flow_init must be a float32 torch tensor (got "
                             f"{getattr(flow_init, 'dtype', type(flow_init))})")
        key = (T, frames.shape[1], frames.shape[2], frames.dtype == torch.uint8, SEQUENCE)
        if carry:
            last = self._seq_last
            if last is None:
                raise ValueError("raft_b200: carry=True continues a forward_sequence call; there is none before it")
            for i, what in ((0, "T"), (slice(1, 3), "frame size"), (3, "dtype (uint8)")):
                if last[i] != key[i]:
                    raise ValueError(f"raft_b200: carry=True with another {what} than the previous sequence call "
                                     f"({key[i]} after {last[i]})")
            if key != self._key and key not in self._parked:
                raise ValueError("raft_b200: carry=True after a call at another frame size released the sequence buffers")
        with torch.cuda.device(self.device):
            self._ensure(*key)
            if flow_init is None:
                self.flow_init.zero_()
            elif tuple(flow_init.shape) != tuple(self.flow_init.shape):
                raise ValueError(f"raft_b200: flow_init must be [T,h,w,2] = {list(self.flow_init.shape)} on the padded "
                                 f"1/8-resolution grid (got {list(flow_init.shape)})")
            else:
                self.flow_init.copy_(flow_init, non_blocking=True)
            (self.raw[1:] if carry else self.raw).copy_(frames, non_blocking=True)
            self._carry = bool(carry)
            try:
                self.run()
            finally:
                self._carry = False
            self._seq_last = key
            if not self._range_checked:
                self._check_range()
        return (self.flow_low, self.flow_up) if return_low else self.flow_up

    @torch.no_grad()
    def forward_bidirectional(self, left: torch.Tensor, right: torch.Tensor, check: bool = True):
        """Both directions of B frame pairs in one pass: fnet once on the 2B frames, cnet on all 2B, the hot path on 2B
        pairs (L_i -> R_i, then R_i -> L_i).  Frames as for forward(); per pair the flows are bit-identical to
        forward(L, R) and forward(R, L) (every kernel is batch-invariant, DESIGN §4).  Returns (flow_fw, flow_bw, occ_fw,
        occ_bw): [B,H,W,2] fp32 flows and [B,H,W] uint8 masks of rb_flow_fb_check (0 consistent, 1 occluded, 2 leaves
        the frame; None when check is False) -- views of engine-owned buffers, overwritten by the next call.
        Alternating with forward() at one frame size keeps the buffers and CUDA graph of each mode (the memory of
        both); a call at another frame size releases them."""
        mode = BIDIRECTIONAL_CHECK if check else BIDIRECTIONAL
        self._run_frames(left, right, mode)
        B = left.shape[0]
        occ = (self.occ[:B], self.occ[B:]) if check else (None, None)
        return (self.flow_up[:B], self.flow_up[B:]) + occ

    @torch.no_grad()
    def forward_sequence_bidirectional(self, frames: torch.Tensor, check: bool = True):
        """Both directions of the T pairs of [T+1,H,W,3] frames (dtypes, sizes, input_size and padding as for forward())
        in one pass.  Returns (flow_fw, flow_bw, occ_fw, occ_bw): [T,H,W,2] fp32 flows in pair order, flow_fw[k] = f_k ->
        f_(k+1) bit-identical to forward(f_k, f_(k+1)) and flow_bw[k] = f_(k+1) -> f_k bit-identical to
        forward(f_(k+1), f_k), and the [T,H,W] uint8 masks of forward_bidirectional(f_k, f_(k+1)) (None when check is
        False; the check runs eagerly after the replay).  The 2T pairs run as one batch in the palindrome order (0->1), ...,
        (T-1->T), (T->T-1), ..., (1->0), so each frame goes through fnet once and cnet once; the mirrored feature and context
        rows and the backward flows in pair order are device copies in the graph.  Views of engine-owned buffers,
        overwritten by the next call.  Alternating with the other modes at one frame size keeps every mode's buffers and
        graph, and a pending forward_sequence carry survives it."""
        self._run_sequence(frames)
        T, H, W = self._shape[:3]
        if not check:
            return self.flow_up[:T], self.flow_bw, None, None
        with torch.cuda.device(self.device):
            capi.check(capi.lib.rb_flow_fb_check(capi.ptr(self.flow_up[:T]), capi.ptr(self.flow_bw),
                                                 capi.ptr(self.occ[:T]), capi.ptr(self.occ[T:]), T, H, W, self.flow_scale,
                                                 FB_ALPHA1, FB_ALPHA2, capi.stream()))
        return self.flow_up[:T], self.flow_bw, self.occ[:T], self.occ[T:]

    @torch.no_grad()
    def track(self, frames: torch.Tensor, queries, backward: bool = False):
        """Point tracking: queries [N,3] rows (frame, x, y), x and y in the frames' own pixels, followed from their frame
        to the last of the [F,H,W,3] frames (dtypes, sizes and input_size as for forward()).  One
        forward_sequence_bidirectional(check=False) pass, then one rb_track_points launch on its flows (flow_scale as in
        the occlusion check).  With input_size the positions are mapped to the network grid and the tracks back
        (track_queries, tracks_to_frames).  Returns fresh (tracks [F,N,2] fp32, status [F,N] uint8) CUDA tensors in the
        frames' own pixels: status 0 consistent, 1 inconsistent (occluded; the track goes on), 2 left the frame (NaN from
        then on), 3 before the query frame (NaN).  Bad queries raise ValueError before the pass.

        backward=True also follows each point from its frame back to frame 0: after the forward launch, one
        rb_track_points_backward launch on the same flows and buffers fills the rows before each query frame (status 0,
        1 or 2; 3 no longer occurs).  The rows at and after it are the bits of backward=False."""
        F = _sequence_length(frames) + 1
        src_hw = tuple(frames.shape[1:3])
        net_hw = self.input_size if self.input_size is not None else src_hw
        qframe, qpos = track_queries(queries, F, src_hw, net_hw)
        from networks.utils import track_points, track_points_backward
        flow_fw, flow_bw, _, _ = self.forward_sequence_bidirectional(frames, check=False)
        with torch.cuda.device(self.device):
            tracks, status, _ = track_points(flow_fw, flow_bw, qframe, qpos, flow_scale=self.flow_scale,
                                             alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)
            if backward:
                track_points_backward(flow_fw, flow_bw, qframe, qpos, tracks, status, flow_scale=self.flow_scale,
                                      alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)
            return tracks_to_frames(tracks, src_hw, net_hw), status

    @torch.no_grad()
    def propagate(self, frames: torch.Tensor, labels, frame=0, cuts=None):
        """Keyframe label propagation: the [Hs,Ws] uint8 label map `labels` of frame `frame` carried to every one of the
        [F,Hs,Ws,3] frames (dtypes, sizes and input_size as for forward()).  One forward_sequence_bidirectional(check=False)
        pass; a zero row at `frame`, one rb_flow_accumulate and one rb_flow_accumulate_backward launch on its flows
        (flow_scale and the forward-backward test as in the occlusion check), and one rb_labels_propagate over all rows
        at the frames' own size.  Returns fresh (labels [F,Hs,Ws] uint8, status [F,Hs,Ws] uint8) CUDA tensors: status 0
        consistent at every step back to the keyframe, 1 occluded at some step, 2 entered through the frame edge at some
        step; labels[frame] equals the key bit for bit.  A key that is not [Hs,Ws] uint8 or a frame outside [0, F) raises
        ValueError before the pass.

        Several keyframes: labels [m,Hs,Ws] uint8 and frame a strictly increasing sequence of m frame indices; cuts an
        iterable of scene-cut pairs (pair k between frames k and k + 1).  Each frame votes between the keyframes on
        either side of it that no cut separates from it (raft_b200.video.keyframe_rows): after the same pass, a zero row
        at every key, rb_flow_accumulate from each key to the frame before the next one and rb_flow_accumulate_backward
        from each key to the frame after the previous one (slices of the same flows), then one rb_labels_propagate_keys
        launch.  Status 3 (label 0): no keyframe reaches the frame.  A one-element list without cuts gives the single-key
        bits.  A count mismatch, keys not strictly increasing or outside [0, F), a key of the wrong size or dtype, or a
        cut outside [0, F - 1) raises ValueError before the pass."""
        from networks.utils import accumulate_flow, accumulate_flow_backward, propagate_labels, propagate_labels_keys
        from .video import check_cuts, check_keyframes, keyframe_rows
        F = _sequence_length(frames) + 1
        Hs, Ws = frames.shape[1:3]
        key = torch.as_tensor(labels)
        several = cuts is not None or not isinstance(frame, (int, np.integer))
        if not several:
            if not (key.dim() == 2 and key.dtype == torch.uint8 and tuple(key.shape) == (Hs, Ws)):
                raise ValueError(f"raft_b200: the key labels must be an [Hs,Ws] = [{Hs},{Ws}] uint8 map (got "
                                 f"{list(key.shape)} {key.dtype})")
            if not (0 <= frame < F):
                raise ValueError(f"raft_b200: the key frame must be an integer in [0, {F}) (got {frame!r})")
        else:
            K = check_keyframes(frame, F, "raft_b200")
            cuts = check_cuts(() if cuts is None else cuts, F, "raft_b200")
            if key.dim() == 2 and isinstance(frame, (int, np.integer)):
                key = key[None]
            if not (key.dim() == 3 and key.dtype == torch.uint8 and tuple(key.shape[1:]) == (Hs, Ws)):
                raise ValueError(f"raft_b200: the key labels must be an [m,Hs,Ws] = [m,{Hs},{Ws}] uint8 stack (got "
                                 f"{list(key.shape)} {key.dtype})")
            if key.shape[0] != len(K):
                raise ValueError(f"raft_b200: {key.shape[0]} key label maps for {len(K)} key frames")
        frame = int(frame) if not several else None
        flow_fw, flow_bw, _, _ = self.forward_sequence_bidirectional(frames, check=False)
        T, H, W = flow_fw.shape[:3]
        kw = dict(flow_scale=self.flow_scale, alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)
        with torch.cuda.device(self.device):
            if not several:
                acc = torch.empty(F, H, W, 2, dtype=torch.float32, device=self.device)
                status = torch.empty(F, H, W, dtype=torch.uint8, device=self.device)
                acc[frame].zero_()
                status[frame].zero_()
                accumulate_flow(flow_fw, flow_bw, acc, status, start=frame, **kw)
                accumulate_flow_backward(flow_fw, flow_bw, acc, status, start=frame, **kw)
                return propagate_labels(acc, status, key.to(self.device))
            acc = torch.empty(2, F, H, W, 2, dtype=torch.float32, device=self.device)  # side A, side B
            status = torch.empty(2, F, H, W, dtype=torch.uint8, device=self.device)
            for i, k in enumerate(K):
                acc[:, k].zero_()
                status[:, k].zero_()
                hi = K[i + 1] - 1 if i + 1 < len(K) else F - 1  # side A of frames k .. hi
                if hi > k:
                    accumulate_flow(flow_fw[k:hi], flow_bw[k:hi], acc[0, k:hi + 1], status[0, k:hi + 1], **kw)
                lo = K[i - 1] + 1 if i > 0 else 0  # side B of frames lo .. k - 1
                if k > lo:
                    accumulate_flow_backward(flow_fw[lo:k], flow_bw[lo:k], acc[1, lo:k + 1], status[1, lo:k + 1],
                                             start=k - lo, **kw)
            return propagate_labels_keys(acc[0], status[0], acc[1], status[1], key.to(self.device),
                                         keyframe_rows(F, K, cuts))

    @torch.no_grad()
    def stabilize(self, frames: torch.Tensor, sigma, cuts=None, max_zoom=None, fill=False, window=None):
        """Video stabilization of [F,Hs,Ws,3] uint8 frames (sizes and input_size as for forward()): one
        forward_sequence_bidirectional pass with the occlusion check, one rb_global_motion launch (networks.utils.
        global_motion: each pair's camera motion, a similarity fitted robustly to its consistent pixels), the host path
        of raft_b200.stabilize (the camera path per shot, smoothed by a Gaussian of sigma frames, one zoom per shot capped
        at max_zoom, default DEFAULT_MAX_ZOOM) and one rb_frames_warp_affine launch on the frames at their own size.
        cuts: scene-cut pair indices (pair k between frames k and k + 1), where the path restarts.  Returns fresh
        (frames [F,Hs,Ws,3] uint8, transforms [F,2,3] fp64) CUDA tensors, each transform mapping an output pixel to its
        source position in the frame's own pixels.  Non-uint8 frames, a sigma that is not finite and > 0, a max_zoom
        below 1 or bad cuts raise ValueError before the pass.

        fill=True fills the borders the correction uncovers instead of zooming them away (max_zoom then defaults to
        1.0; a larger cap keeps camera_transforms' zoom logic): after the same pass, fit and transforms, the flows of that
        pass are extended by raft_b200.stabilize.fill_margin's canvas margin (networks.utils.extend_flows), and one
        rb_frames_warp_affine_fill launch over raft_b200.inpaint.inpaint_rows(F, window, cuts) (window default
        DEFAULT_WINDOW frames each way; no side crosses a cut) and the spatial fill follow (raft_b200.stabilize.
        fill_warp).  Returns fresh (frames, transforms, status [F,Hs,Ws] uint8): status 0 the source lies in the frame
        (rb_frames_warp_affine's byte), 1 filled from both sides, 2 from one, 3 spatially.  A bad window, or a window
        without fill, raises ValueError before the pass."""
        from networks.utils import extend_flows, global_motion, warp_frames
        from .inpaint import DEFAULT_WINDOW, check_window, inpaint_rows
        from .stabilize import (DEFAULT_MAX_ZOOM, camera_transforms, check_max_zoom, check_sigma, fill_margin,
                                fill_motions, fill_warp)
        from .video import check_cuts
        F = _sequence_length(frames) + 1
        if frames.dtype != torch.uint8:
            raise ValueError(f"raft_b200: stabilize writes bytes: the frames must be uint8 (got {frames.dtype})")
        sigma = check_sigma(sigma, "raft_b200")
        if max_zoom is None:
            max_zoom = 1.0 if fill else DEFAULT_MAX_ZOOM
        max_zoom = check_max_zoom(max_zoom, "raft_b200")
        cuts = check_cuts(() if cuts is None else cuts, F, "raft_b200")
        if window is not None and not fill:
            raise ValueError("raft_b200: stabilize's window is the reach of fill=True")
        if fill:
            window = check_window(DEFAULT_WINDOW if window is None else window, "raft_b200")
        hw = tuple(frames.shape[1:3])
        flow_fw, flow_bw, occ_fw, _ = self.forward_sequence_bidirectional(frames, check=True)
        with torch.cuda.device(self.device):
            params, _, _ = global_motion(flow_fw, occ_fw, hw, flow_scale=self.flow_scale)
            motions = params.cpu().numpy()
            A, _, _ = camera_transforms(motions, hw, sigma, cuts, max_zoom)
            if not fill:
                A = torch.from_numpy(A).to(self.device)
                return warp_frames(frames.to(self.device), A), A
            net_hw = tuple(flow_fw.shape[1:3])
            margin = fill_margin(A, hw, net_hw)
            ext_fw, ext_bw = extend_flows(flow_fw, flow_bw, fill_motions(motions, cuts), hw, margin, self.flow_scale)
            A = torch.from_numpy(A).to(self.device)
            out, status = fill_warp(frames.to(self.device), ext_fw, ext_bw, net_hw, margin, A,
                                    inpaint_rows(F, window, cuts), self.flow_scale)
            return out, A, status

    @torch.no_grad()
    def inpaint(self, frames: torch.Tensor, masks, window=None, dilate=None, labels=None, cuts=None):
        """Object removal from [F,Hs,Ws,3] uint8 frames (sizes and input_size as for forward()): masks [F,Hs,Ws] uint8
        label maps at the frames' size, a pixel removed where its value is non-zero (with labels: one of them), dilated
        by the (2 dilate + 1)^2 square (default raft_b200.inpaint.DEFAULT_DILATE).  One forward_sequence_bidirectional
        (check=False) pass; rb_inpaint_masks; the 2T flows completed inside the holes on the network grid as one
        rb_masked_fill batch; one rb_inpaint_propagate launch, each hole pixel followed through the completed flows up to
        `window` frames each way (default DEFAULT_WINDOW; never across a scene-cut pair of cuts) to the nearest frames
        that see behind it; one rb_masked_fill of what no frame sees, and the rounding.  Returns fresh (frames
        [F,Hs,Ws,3] uint8, status [F,Hs,Ws] uint8) CUDA tensors: status 0 not a hole (the bytes as they were), 1 filled
        from both sides, 2 from one, 3 spatially.  Non-uint8 frames, bad masks, window, dilate, labels or cuts raise
        ValueError before the pass."""
        from networks.utils import inpaint_masks
        from .inpaint import (DEFAULT_DILATE, DEFAULT_WINDOW, check_dilate, check_window, complete_flows, fill_frames,
                              inpaint_rows, selection_table)
        from .video import check_cuts
        F = _sequence_length(frames) + 1
        if frames.dtype != torch.uint8:
            raise ValueError(f"raft_b200: inpaint writes bytes: the frames must be uint8 (got {frames.dtype})")
        Hs, Ws = frames.shape[1:3]
        m = torch.as_tensor(masks)
        if not (m.dtype == torch.uint8 and tuple(m.shape) == (F, Hs, Ws)):
            raise ValueError(f"raft_b200: the masks must be [F,Hs,Ws] = [{F},{Hs},{Ws}] uint8 label maps (got "
                             f"{list(m.shape)} {m.dtype})")
        window = check_window(DEFAULT_WINDOW if window is None else window, "raft_b200")
        dilate = check_dilate(DEFAULT_DILATE if dilate is None else dilate, "raft_b200")
        selection_table(labels, "raft_b200")
        rows = inpaint_rows(F, window, check_cuts(() if cuts is None else cuts, F, "raft_b200"))
        flow_fw, flow_bw, _, _ = self.forward_sequence_bidirectional(frames, check=False)
        with torch.cuda.device(self.device):
            hole, hole_net = inpaint_masks(m.to(self.device), flow_fw.shape[1:3], dilate, labels)
            fw, bw = complete_flows(flow_fw, flow_bw, hole_net)
            return fill_frames(frames.to(self.device), hole, fw, bw, rows, self.flow_scale)

    @torch.no_grad()
    def denoise(self, frames: torch.Tensor, sigma, window=None, cuts=None):
        """Video denoising of [F,Hs,Ws,3] uint8 frames (sizes and input_size as for forward()): sigma the noise's
        standard deviation in grey levels, or "auto" (raft_b200.denoise.estimate_sigma on the first frames; an estimate
        of 0 returns the frames unchanged without a flow pass).  One forward_sequence_bidirectional(check=False) pass and
        one rb_denoise_merge launch over raft_b200.inpaint.inpaint_rows(F, window, cuts) (window default
        raft_b200.denoise.DEFAULT_WINDOW frames each way; no side crosses a cut): each pixel merged with its patch matches
        in frame t and in every frame the chained flows reach through the forward-backward test.  Returns fresh (frames
        [F,Hs,Ws,3] uint8, support [F,Hs,Ws] uint8: the matched frames per pixel) CUDA tensors at the frames' own size.
        Non-uint8 frames, a bad sigma, window or cuts raise ValueError before the pass."""
        from .denoise import DEFAULT_WINDOW, check_sigma, check_window, estimate_sigma, merge_frames
        from .inpaint import inpaint_rows
        from .video import check_cuts
        F = _sequence_length(frames) + 1
        if frames.dtype != torch.uint8:
            raise ValueError(f"raft_b200: denoise writes bytes: the frames must be uint8 (got {frames.dtype})")
        sigma = check_sigma(sigma, "raft_b200")
        window = check_window(DEFAULT_WINDOW if window is None else window, "raft_b200")
        rows = inpaint_rows(F, window, check_cuts(() if cuts is None else cuts, F, "raft_b200"))
        with torch.cuda.device(self.device):
            on_dev = frames.to(self.device)
            if sigma == "auto":
                sigma = estimate_sigma(on_dev)
            if sigma == 0:
                return merge_frames(on_dev, None, None, rows, 0, self.flow_scale)
        flow_fw, flow_bw, _, _ = self.forward_sequence_bidirectional(frames, check=False)
        with torch.cuda.device(self.device):
            return merge_frames(on_dev, flow_fw, flow_bw, rows, sigma, self.flow_scale)

    @torch.no_grad()
    def segment_motion(self, frames: torch.Tensor, window=None, tau=None, cuts=None):
        """Motion segmentation of [F,Hs,Ws,3] uint8 frames (F >= 2; sizes and input_size as for forward()): the pixels
        whose motion departs from the camera's.  One forward_sequence_bidirectional(check=True) pass; global_motion and
        one rb_homography_motion on the 2T fields (forward then backward) as one batch; one rb_motion_evidence launch
        (tau in network pixels, default raft_b200.motionseg.TAU; scene-cut pairs of cuts contribute nothing); one
        rb_motion_segment launch over raft_b200.motionseg.segment_rows(F, window, cuts) (window default DEFAULT_WINDOW
        frames each way; no chain crosses a cut).  Returns fresh (masks [F,Hs,Ws] uint8 in {0, 1}, status [F,Hs,Ws]
        uint8: 1 where no evidence reached the pixel, homographies [F-1,3,3] fp64 host array: the forward pairs' H in
        the frames' own pixels, h33 = 1).  Non-uint8 frames, a bad window, tau or cuts raise ValueError before the
        pass."""
        from networks.utils import motion_evidence
        from .motionseg import (DEFAULT_WINDOW, TAU, check_tau, check_window, cut_flags, fit_fields, segment_frames,
                                segment_rows, to_pixels)
        from .video import check_cuts
        F = _sequence_length(frames) + 1
        if frames.dtype != torch.uint8:
            raise ValueError(f"raft_b200: segment_motion reads bytes: the frames must be uint8 (got {frames.dtype})")
        window = check_window(DEFAULT_WINDOW if window is None else window, "raft_b200")
        tau = check_tau(TAU if tau is None else tau, "raft_b200")
        cuts = check_cuts(() if cuts is None else cuts, F, "raft_b200")
        rows = segment_rows(F, window, cuts)
        hw = tuple(frames.shape[1:3])
        flow_fw, flow_bw, occ_fw, occ_bw = self.forward_sequence_bidirectional(frames, check=True)
        T = F - 1
        with torch.cuda.device(self.device):
            H, flags = fit_fields(torch.cat([flow_fw, flow_bw]), torch.cat([occ_fw, occ_bw]), hw, self.flow_scale)
            ev = motion_evidence(flow_fw, flow_bw, occ_fw, occ_bw, H, flags, hw, cut_flags(cuts, range(T), self.device),
                                 self.flow_scale, tau)
            mask, status = segment_frames(ev, flow_fw, flow_bw, hw, rows, self.flow_scale)
            return mask, status, to_pixels(H[:T].cpu().numpy(), hw)

    def _consistent_args(self, frames, other, name, cuts, what):
        F = _sequence_length(frames) + 1
        if frames.dtype != torch.uint8:
            raise ValueError(f"raft_b200: {what} compares bytes: the frames must be uint8 (got {frames.dtype})")
        o = torch.as_tensor(other)
        if not (o.dtype == torch.uint8 and tuple(o.shape) == tuple(frames.shape)):
            raise ValueError(f"raft_b200: the {name} must be [F,Hs,Ws,3] = {list(frames.shape)} uint8 frames aligned "
                             f"with the frames (got {list(o.shape)} {o.dtype})")
        from .video import check_cuts
        return F, o, check_cuts(() if cuts is None else cuts, F, "raft_b200")

    @torch.no_grad()
    def consistent(self, frames: torch.Tensor, processed, strength, cuts=None):
        """Blind video temporal consistency (Bonneel et al., SIGGRAPH Asia 2015) of processed, [F,Hs,Ws,3] uint8 frames
        made from the [F,Hs,Ws,3] uint8 frames one at a time (sizes and input_size as for forward()).  One
        forward_sequence_bidirectional(check=False) pass on the originals, then the frames in order on the stream, with
        no host synchronisation per frame: frame 0 and the first frame after each scene-cut pair of cuts are P byte for
        byte; every other frame is raft_b200.temporal.consistent_frame (rb_tcons_terms, rb_screened_poisson, the
        rounding) against the previous output.  strength (lambda > 0) trades the pull toward the previous output
        against P's gradients.  Returns fresh (frames [F,Hs,Ws,3] uint8, status [F,Hs,Ws] uint8: 0 the temporal term
        is used, 1 the step failed, 2 the colour check rejected it, 3 no previous frame) CUDA tensors.  Non-uint8
        frames, processed frames of another shape, a bad strength or cuts raise ValueError before the pass."""
        from .temporal import check_strength, consistent_frame
        F, P, cuts = self._consistent_args(frames, processed, "processed frames", cuts, "consistent")
        strength = check_strength(strength, "raft_b200")
        flow_fw, flow_bw, _, _ = self.forward_sequence_bidirectional(frames, check=False)
        with torch.cuda.device(self.device):
            I, P = frames.to(self.device), P.to(self.device)
            out, status = torch.empty_like(P), torch.empty(P.shape[:3], dtype=torch.uint8, device=self.device)
            Hs, Ws = P.shape[1:3]
            ws = torch.empty(capi.size_query(capi.lib.rb_screened_poisson_workspace_bytes, Hs, Ws), dtype=torch.uint8,
                             device=self.device)  # one solver workspace for every frame
            for t in range(F):
                first = t == 0 or (t - 1) in cuts
                k = max(t - 1, 0)
                out[t], status[t] = consistent_frame(I[t], None if first else I[t - 1], P[t], out[k], flow_fw[k],
                                                     flow_bw[k], strength, self.flow_scale, ws)
            return out, status

    @torch.no_grad()
    def warp_error(self, frames: torch.Tensor, video, cuts=None):
        """Lai et al.'s (ECCV 2018) warping error of video, [F,Hs,Ws,3] uint8 frames aligned with the [F,Hs,Ws,3] uint8
        frames (sizes and input_size as for forward()), under the frames' own flow: one
        forward_sequence_bidirectional(check=False) pass and one rb_warp_error launch pair.  Returns (E_warp, E_pair):
        E_pair [F-1] float64 per pair (NaN for a scene-cut pair of cuts and a pair with no consistent pixel), E_warp
        their mean over the other pairs (raft_b200.temporal.pair_errors), in [0, 1].  Bad arguments raise ValueError
        before the pass."""
        from networks.utils import warp_error
        from .temporal import pair_errors
        F, V, cuts = self._consistent_args(frames, video, "video", cuts, "warp_error")
        flow_fw, flow_bw, _, _ = self.forward_sequence_bidirectional(frames, check=False)
        with torch.cuda.device(self.device):
            sums = warp_error(V.to(self.device), flow_fw, flow_bw, self.flow_scale, FB_ALPHA1, FB_ALPHA2)
        e_warp, e_pair, _ = pair_errors(sums.cpu().numpy(), cuts)
        return e_warp, e_pair

    @torch.no_grad()
    def interpolate(self, left: torch.Tensor, right: torch.Tensor, ts, native: bool = False) -> torch.Tensor:
        """Frames at times ts (each in [0, 1]; 0 = left, 1 = right) between B frame pairs: one bidirectional pass (as
        forward_bidirectional(check=False), from a graph of its own), then eagerly on the same stream, for as many times
        at once as REVERSE_WS_BOUND allows, rb_flow_reverse_multi(flow_fw, t) -> flow and empty mask from t to left,
        rb_flow_reverse_multi(flow_bw, 1 - t) -> from t to right, and rb_frame_synthesize_pairs on the padded frames the
        pass used.  raft-small's reference flow is in 1/8-resolution units, so its time steps are 8t and 8(1 - t) (exact:
        scaling by 8 commutes with fp32 rounding); upstream, t.  Frames as for forward().  Returns a fresh [T,B,H,W,3] fp32
        tensor, BGR in [0,1] (uint8 frames are divided by 255 first).

        native=True with input_size set blends the frames at their own size Hs x Ws instead of the resized ones the
        network saw: the reversal is unchanged, then rb_frame_synthesize_pairs_resized resizes each reversed flow to
        Hs x Ws (rb_flow_resize's bits), picks each empty mask at the network pixel holding the output pixel's centre and
        blends the raw frames, into [T,B,Hs,Ws,3].  Without input_size the frames already run at their own size and
        native changes nothing."""
        ts = _times(ts)
        self._run_frames(left, right, INTERPOLATE)
        B = self._shape[0]
        raw = self._native_frames(native, slice(None, B), slice(B, None))
        return self._synthesize(self.flow_up[:B], self.flow_up[B:], self.images[:B], self.images[B:], ts, raw=raw)

    @torch.no_grad()
    def interpolate_sequence(self, frames: torch.Tensor, ts, uint8: bool = False, bgr: bool = False,
                             native: bool = False) -> torch.Tensor:
        """Frame-rate up-conversion: the frames at times ts (each in [0, 1]) between every pair of consecutive frames of
        [T+1,H,W,3] frames, from one forward_sequence_bidirectional(check=False) pass and the per-t work of interpolate
        on its flows.  Returns a fresh [len(ts),T,H,W,3] tensor; [:, k] equals interpolate(f_k, f_(k+1), ts)[:, 0] bit for
        bit.  uint8=True quantises on the GPU as the CLI writes its PNGs (np.clip(np.rint(255 x), 0, 255), NaN -> 0), and
        bgr=True then reverses the channels (RGB frames of an upstream model written as BGR).  native as for interpolate:
        [len(ts),T,Hs,Ws,3] at the frames' own size."""
        ts = _times(ts)
        if bgr and not uint8:
            raise ValueError("raft_b200: bgr swaps the channels of uint8 output; pass uint8=True")
        self._run_sequence(frames)
        T = self._shape[0]
        raw = self._native_frames(native, slice(None, T), slice(1, None))
        return self._synthesize(self.flow_up[:T], self.flow_bw, self.images[:T], self.images[1:], ts, uint8, bgr, raw=raw)

    @torch.no_grad()
    def interpolate_sequence_at(self, frames: torch.Tensor, items, uint8: bool = False, bgr: bool = False,
                                native: bool = False) -> torch.Tensor:
        """Frame-rate conversion: the frames at per-pair times of [T+1,H,W,3] frames.  items is a list of (k, t), 0 <= k < T
        and t in [0, 1]: the frame at time t between frames k and k + 1.  One forward_sequence_bidirectional(check=False)
        pass, then per item only that item's work: rb_flow_reverse_items of flow_fw[k] by s t and of flow_bw[k] by
        s (1 - t) (s = flow_scale, as in interpolate) and rb_frame_synthesize_items, for as many items at once as
        REVERSE_WS_BOUND allows.  Returns a fresh [len(items),H,W,3] tensor; row i equals interpolate(f_k, f_(k+1), [t])[0, 0]
        bit for bit.  uint8 and bgr as for interpolate_sequence, native as for interpolate ([len(items),Hs,Ws,3], through
        rb_frame_synthesize_items_resized).  An empty list, a k outside [0, T) or a t outside [0, 1] raises ValueError
        before the pass."""
        ks, ts = _items(items, _sequence_length(frames))
        if bgr and not uint8:
            raise ValueError("raft_b200: bgr swaps the channels of uint8 output; pass uint8=True")
        self._run_sequence(frames)
        T = self._shape[0]
        raw = self._native_frames(native, slice(None, T), slice(1, None))
        return self._synthesize(self.flow_up[:T], self.flow_bw, self.images[:T], self.images[1:], ts, uint8, bgr, ks,
                                raw=raw)

    @torch.no_grad()
    def motion_blur(self, frames: torch.Tensor, shutter, fps=None, density: int = 16, cuts=None,
                    native: bool = False) -> torch.Tensor:
        """Frame-rate conversion with a camera shutter (F32): [F,H,W,3] frames converted from rate fps[0] to fps[1] (any
        ratio; fps=None keeps the rate and only blurs), every output frame the mean of m interpolated sub-frames over its
        exposure of shutter degrees, density samples per input-frame interval (raft_b200.video.shutter_schedule() states
        the times, the clamping into the clip and into shots at the scene-cut pairs cuts).  One
        forward_sequence_bidirectional(check=False) pass, then expose()'s chunks.  Returns fresh [N_out,H,W,3] uint8 in
        the frames' channel order, N_out = floor((F - 1) fps[1] / fps[0]) + 1; native as for interpolate ([N_out,Hs,Ws,3]).
        m = 1 is interpolate_sequence_at(uint8=True) at the output times byte for byte.  Bad arguments raise ValueError
        before the pass."""
        from .video import exposure, shutter_schedule
        T = _sequence_length(frames)
        try:
            fin, fout = (1, 1) if fps is None else fps
        except (TypeError, ValueError):
            raise ValueError(f"raft_b200: fps must be None or (input_fps, output_fps) (got {fps!r})") from None
        (ps,) = shutter_schedule(T + 1, fin, fout, shutter, density, T, () if cuts is None else cuts)
        return self.expose(frames, ps.samples, exposure(fin, fout, shutter, density)[1], ps.opens, ps.closes,
                           native=native)

    @torch.no_grad()
    def expose(self, frames: torch.Tensor, samples, m: int, opens, closes, bgr: bool = False,
               native: bool = False) -> torch.Tensor:
        """One pass of motion_blur on [T+1,H,W,3] frames: one forward_sequence_bidirectional(check=False) pass, then the
        samples (n, i, t) in order (raft_b200.video.ShutterPass with frame indices of these frames: pair i at t, or frame
        i with t None) of output frames of m samples each.  A frame of opens starts its sum at its first sample here; any
        other continues the sum an earlier call left in the engine's accumulator.  A frame of closes ends at its last
        sample here; any other leaves its sum for the next call.  Returns fresh [len(closes),H,W,3] uint8 in closes'
        order (bgr: channels reversed); native as for interpolate.  The sums carried between calls live in this engine,
        so while a frame is left open no other motion_blur or expose call may run on the engine: it would overwrite the
        carried sum (video_interpolate(shutter=) owns its model's engine for the whole sweep)."""
        self._run_sequence(frames)
        T = self._shape[0]
        raw = self.raw if native and self.input_size is not None else None
        with torch.cuda.device(self.device):
            return self._expose(self.flow_up[:T], self.flow_bw, samples, m, opens, closes, bgr, raw)

    def _expose(self, flow_fw, flow_bw, samples, m, opens, closes, bgr, raw):
        """expose()'s work after the pass, in chunks of at most RB_INTERP_MAX_STEPS samples whose items keep the reversal
        workspace within REVERSE_WS_BOUND: rb_flow_reverse_items of the chunk's items, then one rb_frame_expose_items
        (_resized with raw) launch.  A frame split by a chunk or pass boundary reads its sum from accumulator
        expose_slot and a frame left open stores it in the other, which the next chunk then reads."""
        T, H, W = self._shape[:3]
        lib, ptr = capi.lib, capi.ptr
        size = (H, W) if raw is None else self.src_hw
        out = torch.empty((len(closes),) + size + (3,), dtype=torch.uint8, device=self.device)
        if self.expose_acc is None or tuple(self.expose_acc.shape[1:3]) != size:
            self.expose_acc = torch.zeros((2,) + size + (3,), dtype=torch.float32, device=self.device)
        chunk = RB_INTERP_MAX_STEPS
        while chunk > 1 and capi.size_query(lib.rb_flow_reverse_multi_workspace_bytes, chunk, 1, H, W) > REVERSE_WS_BOUND:
            chunk = max(1, chunk // 2)
        first, last = {}, {}
        for g, (n, _, _) in enumerate(samples):
            first.setdefault(n, g)
            last[n] = g
        opens, out_row = set(opens), {n: r for r, n in enumerate(closes)}
        st = capi.stream()
        for c0 in range(0, len(samples), chunk):
            part = samples[c0:c0 + chunk]
            items = [(i, t) for _, i, t in part if t is not None]
            if items:
                self._reverse(flow_fw, flow_bw, [t for _, t in items], [i for i, _ in items])
            entries = (capi.ExposeEntry * len(part))()
            spans, slot = [], 0  # spans: [n, first entry, count] per output frame of the chunk
            for e, (n, i, t) in enumerate(part):
                entries[e] = capi.ExposeEntry(capi.RB_EXPOSE_FRAME, i, 0.0) if t is None else capi.ExposeEntry(slot, i, t)
                slot += t is not None
                if spans and spans[-1][0] == n:
                    spans[-1][2] += 1
                else:
                    spans.append([n, e, 1])
            rows = (capi.ExposeRow * len(spans))()
            carry = self.expose_slot
            for r, (n, e, count) in enumerate(spans):
                opened = n in opens and first[n] == c0 + e
                closed = n in out_row and last[n] == c0 + e + count - 1
                acc = self.expose_slot
                if not closed and not (not opened and r == 0):  # left open for the next chunk: the other accumulator
                    acc = carry = 1 - self.expose_slot
                flags = capi.RB_EXPOSE_OPEN * opened | capi.RB_EXPOSE_CLOSE * closed
                rows[r] = capi.ExposeRow(e, count, m, acc, out_row.get(n, 0), flags)
            self.expose_slot = carry
            flows = ((ptr(self.flow_t[0]), ptr(self.flow_t[1]), ptr(self.empty_t[0, 0]), ptr(self.empty_t[0, 1]))
                     if items else (None,) * 4)
            table = (slot, entries, len(part), rows, len(spans), ptr(self.expose_acc), 2, ptr(out), len(closes), int(bgr),
                     T)
            if raw is None:
                capi.check(lib.rb_frame_expose_items(ptr(self.images), self.Hp, self.Wp, self.pad[0], self.pad[2], *flows,
                                                     *table, H, W, st))
            else:
                capi.check(lib.rb_frame_expose_items_resized(ptr(raw), int(raw.dtype == torch.uint8), *size, *flows, H,
                                                             W, *table, st))
        return out

    def _native_frames(self, native, rows0, rows1):
        """The raw frames a native blend reads, rows rows0 and rows1 of the staging buffer at the frames' own size, or
        None: without native, and without input_size, where the network already runs at the frames' own size (and fp32
        frames that need no padding are not staged)."""
        return (self.raw[rows0], self.raw[rows1]) if native and self.input_size is not None else None

    def _synthesize(self, flow_fw, flow_bw, frames0, frames1, ts, uint8=False, bgr=False, samples=None,
                    raw=None) -> torch.Tensor:
        """The per-t work of interpolate, interpolate_sequence and interpolate_sequence_at on the B pairs of the last pass:
        per chunk, one reversal per direction (steps s t and s (1 - t), s = flow_scale) and one blend of frames0[b] and
        frames1[b].  Without samples every time applies to every pair, into a fresh [len(ts),B,H,W,3] tensor; with
        samples, time ts[i] applies to pair samples[i] alone, into a fresh [len(ts),H,W,3] tensor.  A chunk is as many
        times (items) as keep the reversal workspace within REVERSE_WS_BOUND (at least one, at most RB_INTERP_MAX_STEPS);
        each sample's bits do not depend on it.  raw = (frames0, frames1) at the frames' own size: the blend reads them
        instead, into [..., Hs,Ws,3]."""
        B, H, W = self._shape[:3]
        rows = B if samples is None else 1  # reversal samples per time
        lib = capi.lib
        size = (H, W) if raw is None else self.src_hw
        out = torch.empty((len(ts),) + ((B,) if samples is None else ()) + size + (3,),
                          dtype=torch.uint8 if uint8 else torch.float32, device=self.device)
        chunk = min(len(ts), RB_INTERP_MAX_STEPS)
        while chunk > 1 and capi.size_query(lib.rb_flow_reverse_multi_workspace_bytes, chunk, rows, H, W) > REVERSE_WS_BOUND:
            chunk = max(1, chunk // 2)
        with torch.cuda.device(self.device):
            for i in range(0, len(ts), chunk):
                self._reverse_and_blend(flow_fw, flow_bw, frames0, frames1, ts[i:i + chunk], out[i:i + chunk], uint8, bgr,
                                        None if samples is None else samples[i:i + chunk], raw)
        return out

    def _interpolate_at(self, t: float, out: torch.Tensor):
        """The per-t work of interpolate for one t on the flows of the last INTERPOLATE pass, into out [B,H,W,3] fp32."""
        B = self._shape[0]
        self._reverse_and_blend(self.flow_up[:B], self.flow_up[B:], self.images[:B], self.images[B:], [t], out[None])

    def _reverse(self, flow_fw, flow_bw, ts, samples=None):
        """The reversals of one chunk of n = len(ts) times: flow_fw by s t and flow_bw by s (1 - t) (s = flow_scale) into
        flow_t[0 | 1] and empty_t[:, 0 | 1], by rb_flow_reverse_multi on all B pairs, or with samples by
        rb_flow_reverse_items on pair samples[i].  The reversal buffers are (re)allocated for the n B (n) samples."""
        B, H, W = self._shape[:3]
        n, s, d = len(ts), self.flow_scale, self.device
        per_t = B if samples is None else 1
        rows = n * per_t
        lib, ptr = capi.lib, capi.ptr
        if self.rev_rows != rows:  # the workspace depends on the n B (n) samples alone
            self.rev_ws_bytes = capi.size_query(lib.rb_flow_reverse_multi_workspace_bytes, n, per_t, H, W)
            self.rev_ws = torch.empty(self.rev_ws_bytes, dtype=torch.uint8, device=d)
            self.flow_t = torch.empty(2, rows, H, W, 2, dtype=torch.float32, device=d)  # from t to frame 0 | to frame 1
            self.empty_t = torch.empty(2, 2, rows, H, W, dtype=torch.uint8, device=d)  # [empty | multi] x direction
            self.rev_rows = rows
        st = capi.stream()
        for k, (flow, steps) in enumerate(((flow_fw, [s * t for t in ts]), (flow_bw, [s * (1.0 - t) for t in ts]))):
            bufs = ptr(self.flow_t[k]), ptr(self.empty_t[0, k]), ptr(self.empty_t[1, k])
            if samples is None:
                capi.check(lib.rb_flow_reverse_multi(ptr(flow), _floats(steps), n, *bufs, B, H, W, ptr(self.rev_ws),
                                                     self.rev_ws_bytes, st))
            else:
                capi.check(lib.rb_flow_reverse_items(ptr(flow), B, _ints(samples), _floats(steps), n, *bufs, H, W,
                                                     ptr(self.rev_ws), self.rev_ws_bytes, st))

    def _reverse_and_blend(self, flow_fw, flow_bw, frames0, frames1, ts, out, uint8=False, bgr=False, samples=None,
                           raw=None):
        """One chunk: the reversal of flow_fw by s t and of flow_bw by s (1 - t) for the n = len(ts) times, then the blend
        into out -- rb_flow_reverse_multi and rb_frame_synthesize_pairs on all B pairs into out [n,B,H,W,3], or with
        samples rb_flow_reverse_items and rb_frame_synthesize_items on pair samples[i] at ts[i] into out [n,H,W,3].  With
        raw = (frames0, frames1) at the frames' own Hs x Ws, the *_resized blends of those into out [n,(B,)Hs,Ws,3]."""
        B, H, W = self._shape[:3]
        n = len(ts)
        lib, ptr = capi.lib, capi.ptr
        st = capi.stream()
        self._reverse(flow_fw, flow_bw, ts, samples)
        if raw is not None:
            Hs, Ws = self.src_hw
            frames = (ptr(raw[0]), ptr(raw[1]), int(raw[0].dtype == torch.uint8), Hs, Ws, ptr(self.flow_t[0]),
                      ptr(self.flow_t[1]), ptr(self.empty_t[0, 0]), ptr(self.empty_t[0, 1]), H, W)
            if samples is None:
                capi.check(lib.rb_frame_synthesize_pairs_resized(*frames, _floats(ts), n, ptr(out), int(uint8), int(bgr),
                                                                 B, st))
            else:
                capi.check(lib.rb_frame_synthesize_items_resized(*frames, _ints(samples), _floats(ts), n, ptr(out),
                                                                 int(uint8), int(bgr), B, st))
            return
        frames = (ptr(frames0), ptr(frames1), self.Hp, self.Wp, self.pad[0], self.pad[2], ptr(self.flow_t[0]),
                  ptr(self.flow_t[1]), ptr(self.empty_t[0, 0]), ptr(self.empty_t[0, 1]))
        if samples is None:
            capi.check(lib.rb_frame_synthesize_pairs(*frames, _floats(ts), n, ptr(out), int(uint8), int(bgr), B, H, W, st))
        else:
            capi.check(lib.rb_frame_synthesize_items(*frames, _ints(samples), _floats(ts), n, ptr(out), int(uint8),
                                                     int(bgr), B, H, W, st))

    def _run_sequence(self, frames: torch.Tensor):
        """One SEQUENCE_BIDIRECTIONAL pass on [T+1,H,W,3] frames."""
        T = _sequence_length(frames)
        with torch.cuda.device(self.device):
            self._ensure(T, frames.shape[1], frames.shape[2], frames.dtype == torch.uint8, SEQUENCE_BIDIRECTIONAL)
            (self.raw if self.staged else self.images).copy_(frames, non_blocking=True)
            self.run()
            if not self._range_checked:
                self._check_range()

    def _run_frames(self, left: torch.Tensor, right: torch.Tensor, mode: int, flow_init: Optional[torch.Tensor] = None):
        assert left.shape == right.shape and left.dim() == 4 and left.shape[-1] == 3 and left.dtype == right.dtype
        u8 = left.dtype == torch.uint8
        assert u8 or left.dtype == torch.float32, left.dtype
        with torch.cuda.device(self.device):
            B = left.shape[0]
            self._ensure(B, left.shape[1], left.shape[2], u8, mode)
            if mode == FORWARD_WARM:
                if flow_init is None:
                    self.flow_init.zero_()
                elif tuple(flow_init.shape) != tuple(self.flow_init.shape):
                    raise ValueError(f"raft_b200: flow_init must be [B,h,w,2] = {list(self.flow_init.shape)} on the padded "
                                     f"1/8-resolution grid (got {list(flow_init.shape)})")
                else:
                    self.flow_init.copy_(flow_init, non_blocking=True)
            dst = self.raw if self.staged else self.images
            dst[:B].copy_(left, non_blocking=True)  # H2D when the caller hands pinned host tensors
            dst[B:].copy_(right, non_blocking=True)
            self.run()
            if not self._range_checked:
                self._check_range()

    def _check_range(self):
        """Once per engine: the split-operand format (fp16 hi/lo planes) saturates beyond 65504.  The fp32 tensors at
        the boundary of that path are the feature maps, the context map and the correlation volume; a checkpoint that
        drives them (or the result) out of range must fail loudly, not return a plausible-looking wrong flow."""
        self._range_checked = True
        if os.environ.get("RAFT_B200_NO_RANGE_CHECK"):
            return
        vol = self.pyramid[:self.pyr_bytes // 4 - 64].abs().max() if self.pyramid is not None else self.fmaps.new_zeros(())
        stats = torch.stack([self.fmaps.abs().max(), self.cmap.abs().max(), vol, self.flow_up.abs().max()]).tolist()
        names = ("feature maps", "context map", "correlation volume", "flow")
        for n, v in zip(names, stats):
            if not np.isfinite(v) or (n != "flow" and v > 6.0e4):
                raise capi.RaftB200Error(f"raft_b200: {n} reach |x|max = {v:.3g}: outside the fp16 range of the "
                                         "split-operand tensor-core path (csrc/common.cuh)")

    def lowres_flow(self) -> torch.Tensor:
        g = torch.stack(torch.meshgrid(torch.arange(self.w, device=self.device),
                                       torch.arange(self.h, device=self.device), indexing="xy"), -1).float()
        return self.coords1 - g[None]


def _times(ts):
    ts = [float(t) for t in ts]
    if not ts or not all(0.0 <= t <= 1.0 for t in ts):
        raise ValueError(f"raft_b200: interpolation times must be a non-empty list in [0, 1] (got {ts})")
    return ts


def _sequence_length(frames):
    """T of [T+1,H,W,3] uint8 or float32 frames (T >= 1); anything else raises ValueError."""
    if not (isinstance(frames, torch.Tensor) and frames.dim() == 4 and frames.shape[-1] == 3
            and frames.dtype in (torch.uint8, torch.float32)):
        raise ValueError(f"raft_b200: frames must be a [N,H,W,3] uint8 or float32 tensor (got "
                         f"{getattr(frames, 'shape', None)} {getattr(frames, 'dtype', type(frames))})")
    if frames.shape[0] < 2:
        raise ValueError(f"raft_b200: a frame sequence needs two frames at least (got {frames.shape[0]})")
    return frames.shape[0] - 1


def _items(items, T):
    """The pairs and times of interpolate_sequence_at's items (k, t): a non-empty list, each k an integer in [0, T) and
    each t in [0, 1]; anything else raises ValueError."""
    items = list(items)
    if not items:
        raise ValueError("raft_b200: interpolate_sequence_at needs one (k, t) item at least")
    ks, ts = [], []
    for item in items:
        try:
            k, t = item
            ok = int(k) == k and 0 <= k < T and 0.0 <= float(t) <= 1.0
        except (TypeError, ValueError):
            ok = False
        if not ok:
            raise ValueError(f"raft_b200: item {item!r}: (k, t) needs an integer k in [0, {T}) and t in [0, 1]")
        ks.append(int(k))
        ts.append(float(t))
    return ks, ts


def track_queries(queries, F, src_hw, net_hw):
    """The query points of RaftEngine.track as kernel inputs: queries [N,3] rows (frame, x, y) in the frames' own Hs x Ws
    pixels -> (qframe [N] int32, qpos [N,2] fp32 on the network's Hn x Wn grid).  With another network size the
    positions map by cv2's pixel-centre convention, x_n = (x + 0.5) Wn / Ws - 0.5 (the ratio resize_flow applies to
    displacements), in fp64, rounded once to fp32 and clamped into [0, Wn - 1] x [0, Hn - 1]: the clamp moves only
    queries within half a source pixel of the edge, by less than half a network pixel, and keeps every query inside the
    frame the flow covers.  A frame outside [0, F), a non-integer frame, a non-finite position or one outside
    [0, Ws - 1] x [0, Hs - 1], an empty list or a wrong shape raises ValueError."""
    try:
        q = np.asarray(queries.cpu() if isinstance(queries, torch.Tensor) else queries, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError("raft_b200: queries must be an [N,3] array of (frame, x, y) rows") from None
    if q.ndim != 2 or q.shape[1] != 3 or q.shape[0] < 1:
        raise ValueError(f"raft_b200: queries must be an [N,3] array of (frame, x, y) rows, N >= 1 (got {q.shape})")
    (Hs, Ws), (Hn, Wn) = src_hw, net_hw
    frame, x, y = q[:, 0], q[:, 1], q[:, 2]
    with np.errstate(invalid="ignore"):
        bad = ~((frame >= 0) & (frame < F) & (frame == np.floor(frame)) & np.isfinite(x) & np.isfinite(y)
                & (x >= 0) & (x <= Ws - 1) & (y >= 0) & (y <= Hs - 1))
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError(f"raft_b200: query {i} = {tuple(q[i].tolist())}: needs an integer frame in [0, {F}) and a "
                         f"finite (x, y) in [0, {Ws - 1}] x [0, {Hs - 1}]")
    if (Hn, Wn) != (Hs, Ws):
        x = np.clip(((x + 0.5) * (Wn / Ws) - 0.5).astype(np.float32), np.float32(0), np.float32(Wn - 1))
        y = np.clip(((y + 0.5) * (Hn / Hs) - 0.5).astype(np.float32), np.float32(0), np.float32(Hn - 1))
    return frame.astype(np.int32), np.stack([x, y], axis=-1).astype(np.float32)


def tracks_to_frames(tracks, src_hw, net_hw):
    """Tracks [...,2] fp32 on the network's Hn x Wn grid back to the frames' own Hs x Ws pixels, the inverse of
    track_queries' map, x = (x_n + 0.5) Ws / Wn - 0.5 in fp64 rounded once to fp32 (NaN stays NaN); the tensor itself
    when the sizes agree."""
    (Hs, Ws), (Hn, Wn) = src_hw, net_hw
    if (Hn, Wn) == (Hs, Ws):
        return tracks
    scale = torch.tensor([Ws / Wn, Hs / Hn], dtype=torch.float64, device=tracks.device)
    return ((tracks.double() + 0.5) * scale - 0.5).float()


def _floats(values):
    """A host float array for the entries that copy their time steps into the kernel parameters."""
    import ctypes
    return (ctypes.c_float * len(values))(*values)


def _ints(values):
    """A host int32 array for the entries that copy their item samples into the kernel parameters."""
    import ctypes
    return (ctypes.c_int32 * len(values))(*values)
