"""Drop-in mirror of the reference's ``networks/RAFT.py``: same class name, constructor signature
``RAFT(image_shape, args)`` (only ``args.small`` is read, RAFT.py:37), same attributes, same method
names.  The TF graph is replaced by raft_b200's CUDA engine; ``build_graph`` keeps the reference's
contract (returns 0.0 and publishes the result under the name ``flow_result``, RAFT.py:136-141) and
``forward`` is the direct call.  Extensions over the reference (which hard-codes them, SURVEY fact
5): ``iters``, ``batch`` and the image shape are honoured as parameters; inputs whose H/W are not
multiples of 8 are replicate-padded and the flow cropped back (the reference itself cannot run such
shapes, SURVEY fact 6).  ``input_size=(Ho, Wo)`` gives the reference's input semantics instead: frames of any
size are resized to Ho x Wo on the GPU, bit for bit like the cv2.resize of its test dataflow.  ``mixed_precision=True``
runs every conv with fp16 operands and fp32 accumulation, like upstream RAFT's --mixed_precision (RB_MATH_TC_FP16)."""
import numpy as np
import torch

from networks import model_utils
from networks.model_utils import GetCorrPyramid, SampleCorr, BasicUpdateBlock, SmallUpdateBlock  # noqa: F401
from networks.utils import coords_grid, upflow8  # noqa: F401
from raft_b200 import capi
from raft_b200.engine import PAD_MODES, RaftEngine
from raft_b200.weights import load_npz


class RAFT(object):
    weight_decay = 1e-5          # vestigial in the reference too (RAFT.py:14)
    data_format = 'NHWC'

    def __init__(self, image_shape, args, iters=20, batch=1, device=None, volume_free=None, input_size=None, upstream=False,
                 mixed_precision=False, pad_mode='sintel'):
        self.dropout = 0.0
        self.corr_radius = 4
        self.hidden_dim = 128
        self.context_dim = 128
        self.mode = 'test'
        self.iters = iters
        self.image_shape = image_shape
        self.batch = batch
        self.small = bool(getattr(args, 'small', False))
        if self.small:
            self.hidden_dim = 96
            self.context_dim = 64
            self.corr_radius = 3
        self.device = torch.device(device if device is not None else 'cuda:0')
        self.volume_free = volume_free  # extension (SURVEY 8(f) F2): None = RAFT_B200_VOLUME_FREE env, default off
        # extension: (Ho, Wo) the frames are resized to on the GPU (test_dataflow.py:85-87), None = their own size
        self.input_size = None if input_size is None else (int(input_size[0]), int(input_size[1]))
        # extension: the numerics of princeton-vl RAFT for weights converted from its .pth checkpoints (RaftEngine upstream)
        self.upstream = bool(upstream)
        # extension: fp16 conv operands with fp32 accumulation, upstream's --mixed_precision (RaftEngine mixed_precision)
        self.mixed_precision = bool(mixed_precision)
        # extension: upstream InputPadder's padding to a multiple of 8, 'sintel' (split) or 'kitti' (bottom only)
        if pad_mode not in PAD_MODES:
            raise ValueError(f"pad_mode must be one of {PAD_MODES} (got {pad_mode!r})")
        self.pad_mode = pad_mode
        self.flow_result = None
        self._engine = None
        self._params = None

    # -- reference surface ------------------------------------------------------------------------
    def inputs(self):
        """RAFT.py:45-51: two [batch,H,W,3] fp32 inputs in [0,1] named input_left / input_right."""
        shp = (self.batch, self.image_shape[0], self.image_shape[1], self.image_shape[2])
        return [('input_left', shp, np.float32), ('input_right', shp, np.float32)]

    def input_preprocess(self, input_left, input_right):
        return 2.0 * input_left - 1.0, 2.0 * input_right - 1.0

    def initialize_flow(self, image):
        b, H, W = image.shape[0], image.shape[1], image.shape[2]
        return coords_grid(b, H // 8, W // 8, image.device), coords_grid(b, H // 8, W // 8, image.device)

    def upsample_flow(self, flow, mask):
        """RAFT.py:119-134 (convex 8x upsampling)."""
        b, h, w, _ = flow.shape
        coords1 = (flow + coords_grid(b, h, w, flow.device)).contiguous()
        out = torch.empty(b, 8 * h, 8 * w, 2, dtype=torch.float32, device=flow.device)
        with torch.cuda.device(flow.device):
            capi.check(capi.lib.rb_upsample_convex(capi.ptr(coords1), capi.ptr(mask.contiguous().float()),
                                                   capi.ptr(out), b, h, w, capi.stream()))
        return out

    def build_graph(self, input_left, input_right):
        self.flow_result = self.forward(input_left, input_right)
        return 0.0

    # -- weights (tensorpack get_model_loader(npz), infer_raft.py:77) ---------------------------
    def load(self, npz_or_params):
        self._params = load_npz(npz_or_params) if isinstance(npz_or_params, str) else dict(npz_or_params)
        model_utils.set_variables(self._params)
        self._engine = None
        return self

    def engine(self):
        if self._engine is None:
            if self._params is None:
                raise RuntimeError("RAFT.load(<npz>) must be called before inference")
            self._engine = RaftEngine(self._params, small=self.small, iters=self.iters, device=self.device,
                                      volume_free=self.volume_free, input_size=self.input_size, upstream=self.upstream,
                                      mixed_precision=self.mixed_precision, pad_mode=self.pad_mode)
        return self._engine

    # -- inference ---------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, input_left, input_right, flow_init=None, return_low=False):
        """[B,H,W,3] frames, BGR like the reference -- fp32 in [0,1] (the reference's placeholders, RAFT.py:45-51) or
        uint8 in [0,255] (extension: the /255 of test_dataflow.py:96-97 then runs on the GPU); numpy or torch, host or
        CUDA -> [B,H,W,2] torch CUDA flow (a fresh tensor per call, like a session.run result).  H, W that are not
        multiples of 8 are replicate-padded and the flow cropped back, both inside the engine's own kernels.  With
        input_size the frames may have any size: they are resized to input_size first (rb_frames_resize, in the same
        CUDA graph) and the flow is at input_size, as in the reference; flow_utils.resize_flow takes it back.

        Extension (upstream RAFT's warm start): flow_init, a [B,h,w,2] float32 flow on the padded 1/8-resolution grid
        (numpy or torch, host or CUDA), starts the loop from coords_grid + flow_init; return_low=True returns fresh
        tensors (flow_low, flow_up) like upstream's test_mode, flow_low being that grid's flow after the last iteration.
        networks.utils.forward_interpolate(flow_low) is the next frame pair's flow_init."""
        if flow_init is not None and not isinstance(flow_init, torch.Tensor):
            flow_init = torch.as_tensor(np.asarray(flow_init))
        out = self.engine().forward(_as_tensor(input_left), _as_tensor(input_right), flow_init=flow_init,
                                    return_low=return_low)
        return tuple(t.clone() for t in out) if return_low else out.clone()

    @torch.no_grad()
    def forward_sequence(self, frames, carry=False, flow_init=None, return_low=False):
        """Extension (video): the flows between consecutive frames of [T+1,H,W,3] frames (dtypes and sources as for
        ``forward``) -> fresh [T,H,W,2] flows, pair k bit-identical to ``forward(frames[k:k+1], frames[k+1:k+2])``, with
        every frame encoded once.  carry=True continues the previous call with [T,H,W,3] new frames: the first pair
        starts from that call's last frame, whose features are reused (RaftEngine.forward_sequence); it raises ValueError
        without such a call, when T, the frame size, the dtype or the upstream / mixed-precision settings differ, or when a
        call at another frame size came in between.  flow_init ([T,h,w,2]) and return_low as in ``forward``."""
        eng = self._engine
        if eng is not None and (eng.upstream, eng.mixed_precision) != (self.upstream, self.mixed_precision):
            if carry:
                raise ValueError("forward_sequence: carry=True after the upstream / mixed_precision settings changed")
            self._engine = None  # the settings changed since the engine was built: build it again
        if flow_init is not None and not isinstance(flow_init, torch.Tensor):
            flow_init = torch.as_tensor(np.asarray(flow_init))
        out = self.engine().forward_sequence(_as_tensor(frames), carry=carry, flow_init=flow_init, return_low=return_low)
        return tuple(t.clone() for t in out) if return_low else out.clone()

    @torch.no_grad()
    def forward_bidirectional(self, input_left, input_right, check=True):
        """Extension (frame interpolation needs flow both ways): the flows left -> right and right -> left of the same
        frames, each frame encoded once and both directions run as one batch.  Inputs as for ``forward``.  Returns fresh
        tensors ``(flow_fw, flow_bw, occ_fw, occ_bw)``: flow_fw equals ``forward(left, right)`` and flow_bw equals
        ``forward(right, left)`` bit for bit; the [B,H,W] uint8 masks are the forward-backward consistency check
        (networks.utils.fb_consistency with UnFlow's alpha1 = 0.01, alpha2 = 0.5; flow_scale 8 for raft-small, whose
        flow is in 1/8-resolution units): 0 consistent, 1 occluded, 2 the flow leaves the frame.  check=False skips the
        check and returns None for both masks."""
        out = self.engine().forward_bidirectional(_as_tensor(input_left), _as_tensor(input_right), check=check)
        return tuple(None if t is None else t.clone() for t in out)

    @torch.no_grad()
    def forward_sequence_bidirectional(self, frames, check=True):
        """Extension (frame interpolation over a video): the flows both ways between consecutive frames of [T+1,H,W,3]
        frames (dtypes and sources as for ``forward``), each frame encoded once and the 2T pairs run as one batch.  Returns
        fresh tensors ``(flow_fw, flow_bw, occ_fw, occ_bw)`` in pair order: flow_fw[k] equals ``forward(f_k, f_(k+1))`` and
        flow_bw[k] equals ``forward(f_(k+1), f_k)`` bit for bit ([T,H,W,2]), and the [T,H,W] uint8 masks are those of
        ``forward_bidirectional(f_k, f_(k+1))``; check=False returns None for both masks."""
        out = self.engine().forward_sequence_bidirectional(_as_tensor(frames), check=check)
        return tuple(None if t is None else t.clone() for t in out)

    @torch.no_grad()
    def track(self, frames, queries, backward=False):
        """Extension (point tracking): where each query point of [F,H,W,3] frames (dtypes and sources as for ``forward``)
        goes in the later frames, and whether it stayed visible.  queries is [N,3] rows (frame, x, y), x and y in the
        frames' own pixels (with input_size too).  One ``forward_sequence_bidirectional`` pass, then every point chained
        through the forward flows with the forward-backward test of ``forward_bidirectional`` at each step
        (RaftEngine.track).  Returns fresh (tracks [F,N,2] fp32, status [F,N] uint8) CUDA tensors: status 0 consistent, 1
        inconsistent (occluded; the position keeps integrating), 2 left the frame (NaN from then on), 3 before the query
        frame (NaN).  backward=True also tracks each point back from its frame to frame 0 through the backward flows of
        the same pass, so the rows before the query frame hold positions and status 0, 1 or 2 (never 3); the rows at and
        after it are unchanged.  A query frame outside [0, F), a non-finite position or one outside the frame, an empty
        list or a wrong shape raises ValueError."""
        return self.engine().track(_as_tensor(frames), queries, backward=bool(backward))

    @torch.no_grad()
    def propagate(self, frames, labels, frame=0, cuts=None):
        """Extension (keyframe label propagation): the [Hs,Ws] uint8 label map `labels` of frame `frame` (a segmentation
        mask, a class map, ...) carried through all of [F,Hs,Ws,3] frames (dtypes and sources as for ``forward``).  One
        ``forward_sequence_bidirectional`` pass; per pixel of every frame, the displacement back to the keyframe composed
        through the consecutive flows on the GPU, and the keyframe's label there by a vote of its four nearest pixels
        (RaftEngine.propagate).  Returns fresh (labels [F,Hs,Ws] uint8, status [F,Hs,Ws] uint8) CUDA tensors at the frames'
        own size (with input_size too): status 0 consistent at every step back to the keyframe, 1 occluded at some step,
        2 entered through the frame edge; labels[frame] equals the key.  A key that is not [Hs,Ws] uint8 or a frame
        outside [0, F) raises ValueError.

        Several keyframes (an annotation every N-th frame): labels [m,Hs,Ws] uint8 and frame a strictly increasing
        sequence of m frame indices.  Each frame takes its labels from the nearest keyframe before it and the nearest
        after it, a vote weighted toward the nearer one, and never from a keyframe on the other side of a scene cut
        (cuts: pair indices k, the cut between frames k and k + 1).  Status 3 (label 0): no keyframe reaches the frame.
        Wrong counts, orders, shapes or cuts raise ValueError before the flow pass."""
        return self.engine().propagate(_as_tensor(frames), labels, frame=frame, cuts=cuts)

    @torch.no_grad()
    def stabilize(self, frames, sigma, cuts=None, max_zoom=None, fill=False, window=None):
        """Extension (video stabilization): [F,Hs,Ws,3] uint8 frames (sources as for ``forward``) with the camera's
        shake removed.  One ``forward_sequence_bidirectional`` pass; per pair a similarity (zoom, rotation, shift) fitted
        robustly on the GPU to the flow of its consistent pixels; the camera path, restarted at every scene cut (cuts:
        pair indices k, the cut between frames k and k + 1), smoothed by a Gaussian of sigma frames; and every frame
        warped at its own size (with input_size too) by its correction and one zoom per shot that keeps the borders out
        of view, up to max_zoom (default raft_b200.stabilize.DEFAULT_MAX_ZOOM; past it the border replicates)
        (RaftEngine.stabilize).  Returns fresh (frames [F,Hs,Ws,3] uint8, transforms [F,2,3] fp64) CUDA tensors, each
        transform mapping an output pixel to its source position.  Non-uint8 frames, a bad sigma, max_zoom or cuts raise
        ValueError before the flow pass.

        fill=True gives full-frame output: max_zoom defaults to 1 (no crop) and the borders the correction uncovers are
        filled from the neighbouring frames, up to window frames each way (default raft_b200.inpaint.DEFAULT_WINDOW),
        that saw them, along the flows extended past the frame edge; what none saw is filled spatially.  Returns
        (frames, transforms, status [F,Hs,Ws] uint8): 0 the source lies in the frame, 1 filled from both sides, 2 from
        one, 3 spatially."""
        return self.engine().stabilize(_as_tensor(frames), sigma, cuts=cuts, max_zoom=max_zoom, fill=fill, window=window)

    @torch.no_grad()
    def inpaint(self, frames, masks, window=None, dilate=None, labels=None, cuts=None):
        """Extension (object removal): [F,Hs,Ws,3] uint8 frames (sources as for ``forward``) with the pixels of the
        [F,Hs,Ws] uint8 masks removed (non-zero values, or with labels those labels, dilated by `dilate` pixels).  One
        ``forward_sequence_bidirectional`` pass; each flow completed inside the holes on the GPU; every hole pixel
        followed through the completed flows up to `window` frames each way, never across a scene-cut pair of cuts, to
        the nearest frames that see behind it, and what no frame sees filled spatially (RaftEngine.inpaint).  Returns
        fresh (frames [F,Hs,Ws,3] uint8, status [F,Hs,Ws] uint8) CUDA tensors: status 0 not a hole, 1 filled from both
        sides, 2 from one, 3 spatially.  Bad masks, window, dilate, labels or cuts raise ValueError before the pass."""
        return self.engine().inpaint(_as_tensor(frames), masks, window=window, dilate=dilate, labels=labels, cuts=cuts)

    @torch.no_grad()
    def denoise(self, frames, sigma, window=None, cuts=None):
        """Extension (video denoising): [F,Hs,Ws,3] uint8 frames (sources as for ``forward``) with additive noise of
        standard deviation sigma grey levels removed (sigma="auto": estimated from the first frames).  One
        ``forward_sequence_bidirectional`` pass; every pixel followed through the flows up to `window` frames each way
        (default raft_b200.denoise.DEFAULT_WINDOW), stopping at the first step that fails the forward-backward test and
        never crossing a scene-cut pair of cuts, and merged with the patches that match it there and around it in its
        own frame (RaftEngine.denoise).  Returns fresh (frames [F,Hs,Ws,3] uint8, support [F,Hs,Ws] uint8: the frames
        matched per pixel) CUDA tensors at the frames' own size.  A bad sigma, window or cuts raise ValueError before
        the pass."""
        return self.engine().denoise(_as_tensor(frames), sigma, window=window, cuts=cuts)

    @torch.no_grad()
    def segment_motion(self, frames, window=None, tau=None, cuts=None):
        """Extension (motion segmentation): the pixels of [F,Hs,Ws,3] uint8 frames (sources as for ``forward``) whose
        motion departs from the camera's.  One ``forward_sequence_bidirectional`` pass with the occlusion check; each
        pair's camera homography fitted robustly to both of its flows; per pixel the evidence r^2 / (r^2 + tau^2) of
        its residual r (network pixels, default raft_b200.motionseg.TAU), summed over its own frame and the frames its
        chain reaches through the forward-backward test, up to `window` frames each way (default DEFAULT_WINDOW), never
        across a scene-cut pair of cuts (RaftEngine.segment_motion).  Returns fresh (masks [F,Hs,Ws] uint8 in {0, 1},
        status [F,Hs,Ws] uint8, homographies [F-1,3,3] fp64 in the frames' own pixels).  A bad window, tau or cuts
        raise ValueError before the pass."""
        return self.engine().segment_motion(_as_tensor(frames), window=window, tau=tau, cuts=cuts)

    @torch.no_grad()
    def consistent(self, frames, processed, strength, cuts=None):
        """Extension (temporal consistency): per-frame processed video made temporally consistent, guided by the flow of
        the original frames (Bonneel et al., SIGGRAPH Asia 2015).  frames, processed: [F,Hs,Ws,3] uint8 (sources as for
        ``forward``); strength > 0 (raft_b200.temporal.cutoff_wavelength gives the detail scale that keeps P's
        gradients); cuts scene-cut pairs where the output restarts from P.  Returns fresh (frames [F,Hs,Ws,3] uint8,
        status [F,Hs,Ws] uint8) CUDA tensors (RaftEngine.consistent)."""
        return self.engine().consistent(_as_tensor(frames), _as_tensor(processed), strength, cuts=cuts)

    @torch.no_grad()
    def warp_error(self, frames, video, cuts=None):
        """Extension (temporal consistency): Lai et al.'s warping error of video, [F,Hs,Ws,3] uint8 frames aligned with
        frames, under the frames' own flow: (E_warp, E_pair [F-1] float64, NaN for cut pairs and pairs with no
        consistent pixel) (RaftEngine.warp_error)."""
        return self.engine().warp_error(_as_tensor(frames), _as_tensor(video), cuts=cuts)

    @torch.no_grad()
    def interpolate_sequence(self, frames, t=0.5, uint8=False, bgr=False, native=False):
        """Extension (frame-rate up-conversion): the frames at time t (a float, or a sequence of times, each in [0, 1])
        between every pair of consecutive frames of [T+1,H,W,3] frames, from one ``forward_sequence_bidirectional`` pass.
        A float t gives a fresh [T,H,W,3] tensor, a sequence of n times [n,T,H,W,3]; pair k equals
        ``interpolate(frames[k:k+1], frames[k+1:k+2], t)`` bit for bit.  fp32 in [0,1] by default; uint8=True quantises
        on the GPU exactly as infer_raft.py writes PNGs (np.clip(np.rint(255 x), 0, 255)), and bgr=True (with uint8)
        reverses the channels, for RGB frames written by cv2.  native as for ``interpolate``.  A t outside [0, 1] raises
        ValueError."""
        scalar = np.ndim(t) == 0
        out = self.engine().interpolate_sequence(_as_tensor(frames), [t] if scalar else list(t), uint8=uint8, bgr=bgr,
                                                 native=native)
        return out[0] if scalar else out

    @torch.no_grad()
    def interpolate_sequence_at(self, frames, items, uint8=False, bgr=False, native=False):
        """Extension (frame-rate conversion to any rate): the frames at per-pair times of [T+1,H,W,3] frames (dtypes and
        sources as for ``forward``).  items is a list of (k, t) with 0 <= k < T and t in [0, 1], each the frame at time t
        between frames k and k + 1; one ``forward_sequence_bidirectional`` pass, then only the work of the listed items.
        Returns a fresh [len(items),H,W,3] tensor whose row i equals ``interpolate(frames[k:k+1], frames[k+1:k+2], t)[0]``
        bit for bit.  uint8 and bgr as for ``interpolate_sequence``, native as for ``interpolate``.  An empty list, a k
        outside [0, T) or a t outside [0, 1] raises ValueError."""
        return self.engine().interpolate_sequence_at(_as_tensor(frames), items, uint8=uint8, bgr=bgr, native=native)

    @torch.no_grad()
    def motion_blur(self, frames, shutter, fps=None, density=16, cuts=None, native=False):
        """Extension (frame-rate conversion with a camera shutter): [F,H,W,3] frames (dtypes and sources as for
        ``forward``) converted from fps[0] to fps[1] -- any ratio, down-conversion included; fps=None keeps the rate and
        only adds the blur -- each output frame the mean of interpolated sub-frames over an exposure of `shutter` degrees
        (0, 360] centred on its time, `density` samples per input-frame interval, clamped into the clip and into the shots
        between the scene-cut pairs `cuts` (Brooks & Barron, CVPR 2019).  One ``forward_sequence_bidirectional`` pass.
        Returns a fresh [floor((F - 1) fps[1] / fps[0]) + 1,H,W,3] uint8 tensor in the frames' channel order; native as
        for ``interpolate``.  Bad arguments raise ValueError (RaftEngine.motion_blur)."""
        return self.engine().motion_blur(_as_tensor(frames), shutter, fps=fps, density=density, cuts=cuts,
                                         native=native)

    @torch.no_grad()
    def interpolate(self, input_left, input_right, t=0.5, native=False):
        """Extension (the reference computes the flow for frame interpolation and projects it to time t with
        flow_utils.py:166 on the CPU): the frames at time t between left (t = 0) and right (t = 1).  One bidirectional
        pass, then per t the flows from time t to both frames by the reference's flow reversal (rb_flow_reverse, bit for
        bit) and a blend of both frames warped by them (rb_frame_synthesize; a frame whose reversed flow is empty at a
        pixel gets weight 0 there).  Inputs as for ``forward``.  A float t in [0, 1] gives a fresh [B,H,W,3] fp32 tensor,
        BGR in [0,1] (uint8 frames are divided by 255); a sequence of T times gives [T,B,H,W,3] from one pass.  t = 0
        and t = 1 return the frames themselves exactly.  A t outside [0, 1] raises ValueError.

        native=True (with input_size) returns the frames at the inputs' own size rather than input_size: the flow is
        estimated and reversed at input_size as always, then resized to the frames' size inside the blend, which warps
        the frames as given (not their resized copies).  Without input_size it changes nothing."""
        scalar = np.ndim(t) == 0
        out = self.engine().interpolate(_as_tensor(input_left), _as_tensor(input_right), [t] if scalar else list(t),
                                        native=native)
        return out[0] if scalar else out


def _as_tensor(x):
    t = torch.as_tensor(x)
    return t if t.dtype == torch.uint8 else t.to(torch.float32)
