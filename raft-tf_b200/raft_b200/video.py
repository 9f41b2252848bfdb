"""F11: optical flow over a video -- upstream RAFT's demo.py (a directory of frames in, one flow visualisation per
consecutive pair out) on RaftEngine.forward_sequence, with the colour coding on the GPU (rb_flow_to_color).

    from raft_b200.video import video
    video(RAFT((432, 1024, 3), args, input_size=(432, 1024)).load("raft-things.npz"), "frames/", "out/")

writes out/flow_000000.png (frame 0 -> 1), out/flow_000001.png, ...; BGR like the single-pair CLI's PNG.

video_interpolate(model, "frames/", "out/", ts=[0.5]) is frame-rate up-conversion on RaftEngine.interpolate_sequence: the
input frames and, between every consecutive pair, the frames at times ts, written as one numbered sequence
out/frame_<n:06d>.png.  Each pass is a fresh call on batch + 1 frames (interp_schedule()), the frames quantised to uint8
on the GPU.  video_interpolate(model, "frames/", "out/", fps=(24, 60)) converts to another frame rate instead: output
frame n sits at input time n 24 / 60, so every pair gets its own times (fps_schedule()), and each pass runs
RaftEngine.interpolate_sequence_at on the (pair, time) items of its pairs alone.

Schedule (schedule()): the first pass is a fresh forward_sequence on batch + 1 frames, every later pass a carry call on
batch new frames, so every frame is decoded, uploaded and encoded once.  A short last pass is padded by repeating the last
frame; its extra rows are idle and their flows discarded, so one pair of CUDA graphs serves the whole video.  warm_start
runs T = 1 carry passes, each started from forward_interpolate of the previous pass's flow_low (upstream's warm start).

Pipeline (_Pipeline, shared by every sweep here): worker threads decode the frames of the next passes (cv2 releases the
GIL) into two pinned slots used in turn, each refilled only after the event behind its pass has completed; each pass's
outputs (colour images and flows, interpolated frames, track rows, label maps, filled frames) are copied to two pinned
output slots and encoded and written by writer threads (_FrameWriter for frames).  The files are the same bytes for
every workers value.  A sweep whose GPU work reads the frames from device memory copies each pass to one reused device
buffer (_Upload), and scores that copy for scene cuts.  The windowed sweeps (video_stabilize(fill=True), video_inpaint,
video_denoise, video_segment_motion) keep a sliding window of frames and flows on the GPU (_Window): frame t is finished
once the data up to frame min(t + window, F - 1) is complete, and frames no later frame reaches are dropped.

video_track(model, "frames/", "out/", queries=[[0, 120.0, 64.5], ...]) tracks points through the clip (grid=STEP: a point
at every STEP-th pixel of one frame): interp_schedule()'s passes of forward_sequence_bidirectional, each followed by one
rb_track_points launch that carries the points' positions and states on the GPU, the rows streamed into out/tracks.npy and
out/status.npy.

video_propagate(model, "frames/", "out/", "key.png", frame=K) carries frame K's label map to every frame: the same passes,
each followed by rb_flow_accumulate (and, before the key frame, rb_flow_accumulate_backward) launches that carry the
per-pixel displacement to the key frame on the GPU and one rb_labels_propagate launch, written as out/label_<i:06d>.png.
With several keyframes (frame=[K_0, K_1, ...]) every frame votes between the nearest keys on either side
(keyframe_rows(), KeyframeSweep, rb_labels_propagate_keys), and scene_cut keeps labels from crossing a cut.

video_stabilize(model, "frames/", "out/", sigma=10) removes the camera's shake: a motion sweep of interp_schedule()'s
passes fits each pair's camera motion on the GPU (rb_global_motion), the host smooths the camera path per shot
(raft_b200.stabilize), and a warp sweep decodes every frame again and warps it at its own size (rb_frames_warp_affine),
written as out/frame_<i:06d>.png with out/transforms.npy.

video_stabilize(..., fill=True) keeps the frames whole instead of zooming: the fill sweep reruns the flow passes, extends
each pass's flows past the frame edge (rb_flow_extend_residual / rb_masked_fill / rb_flow_extend_finish) and fills each
uncovered border pixel from the neighbouring frames that saw it (rb_frames_warp_affine_fill).

video_inpaint(model, "frames/", "out/", "masks/") removes the masked objects: one sweep of interp_schedule()'s passes,
each pass's flows completed inside the holes on the GPU (rb_masked_fill), every frame filled from the nearest frames that
see behind its holes (rb_inpaint_propagate) once the pairs it may reach have run, and the rest filled spatially; written
as out/frame_<i:06d>.png.

video_denoise(model, "frames/", "out/", sigma=20) removes additive noise: the same sweep, every frame merged with its
patch matches in the neighbouring frames the chained flows reach consistently (rb_denoise_merge) once the pairs it may
reach have run; written as out/frame_<i:06d>.png.

Scene cuts (scene_cut=<threshold in [0, 1]>, video_interpolate, video_stabilize, video_inpaint, video_denoise and
warm-started video): each pass's
decoded frames are copied to the GPU once and scored there (networks.utils.scene_cut_scores: one minus the intersection
of consecutive frames' colour histograms); a pair whose score exceeds the threshold is a cut.  Frame-rate conversion
copies the nearer input frame instead of blending two shots (cut_copy(), split_cut_items()), warm-started flow restarts
its chain (cold_start()) and stabilization restarts the camera path.  Without a threshold none of this runs.
"""
from __future__ import annotations

import glob
import math
import os
import threading
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor
from fractions import Fraction
from functools import partial

import numpy as np
import torch

from .evaluate import _imread

# one forward_sequence call: carry or fresh, the frame indices it uploads (T + 1 fresh, T carry; a short last pass repeats
# the last frame), and per flow row the pair index k (frame k -> k + 1) or None for an idle row
Pass = namedtuple("Pass", "carry frames pairs")
# one interpolate_sequence_at call of frame-rate conversion (fps_schedule()): the frames and pairs of its Pass, the output
# frames it interpolates as (n, k, t) (output index, pair, time) and the input frames it copies as (n, i)
FpsPass = namedtuple("FpsPass", "frames pairs items copies")
# one pass of frame-rate conversion with a shutter (shutter_schedule()): the frames and pairs of its Pass, its samples in
# run order as (n, i, t) -- output frame n's blend of pair i at time t, or with t None input frame i -- and the output
# frames whose first / last sample it runs
ShutterPass = namedtuple("ShutterPass", "frames pairs samples opens closes")


def list_frames(frames):
    """The frame paths of a video: a directory's *.png and *.jpg files in sorted order (upstream demo.py's glob), or a list
    of paths as given.  Fewer than two frames raise ValueError."""
    if isinstance(frames, (str, os.PathLike)):
        root = os.fspath(frames)
        if not os.path.isdir(root):
            raise FileNotFoundError(f"video: no directory {root}")
        paths = sorted(glob.glob(os.path.join(root, "*.png")) + glob.glob(os.path.join(root, "*.jpg")))
    else:
        paths = [os.fspath(p) for p in frames]
    if len(paths) < 2:
        raise ValueError(f"video: a flow needs two frames at least (got {len(paths)})")
    return paths


def schedule(n_frames, batch, warm_start=False):
    """The passes over n_frames frames with T = batch pairs per pass (T = 1 with warm_start): pass j covers the pairs
    j T .. j T + T - 1, a fresh call on frames 0 .. T for j = 0 and a carry call on frames j T + 1 .. j T + T after it.
    Frame indices past the last frame repeat it; their rows are idle (None)."""
    if int(n_frames) < 2:
        raise ValueError(f"video: a flow needs two frames at least (got {n_frames})")
    if int(batch) < 1:
        raise ValueError(f"video: batch must be >= 1 (got {batch})")
    if warm_start and int(batch) != 1:
        raise ValueError(f"video: warm_start runs one pair per pass, each warm-started from the one before; batch must be 1 "
                         f"(got {batch})")
    T, n_pairs, last = int(batch), int(n_frames) - 1, int(n_frames) - 1
    passes = []
    for j in range(-(-n_pairs // T)):
        first = j * T + (1 if j else 0)
        frames = [min(i, last) for i in range(first, j * T + T + 1)]
        passes.append(Pass(j > 0, frames, [k if k < n_pairs else None for k in range(j * T, j * T + T)]))
    return passes


def check_times(ts):
    """The interpolation times of video_interpolate as floats: strictly increasing inside (0, 1), at least one (the input
    frames themselves are the times 0 and 1 of the output sequence).  Anything else raises ValueError."""
    ts = [float(t) for t in ts]
    if not ts or not all(0.0 < t < 1.0 for t in ts) or any(b <= a for a, b in zip(ts, ts[1:])):
        raise ValueError(f"video_interpolate: the times must be strictly increasing inside (0, 1) (got {ts})")
    return ts


def interp_schedule(n_frames, batch):
    """The passes of video_interpolate over n_frames frames with T = batch pairs per pass: pass j is a fresh call on the
    frames j T .. j T + T and covers the pairs j T .. j T + T - 1.  Frame indices past the last frame repeat it; their
    rows are idle (None), so every pass has the same T."""
    if int(n_frames) < 2:
        raise ValueError(f"video: interpolation needs two frames at least (got {n_frames})")
    if int(batch) < 1:
        raise ValueError(f"video: batch must be >= 1 (got {batch})")
    T, n_pairs, last = int(batch), int(n_frames) - 1, int(n_frames) - 1
    return [Pass(False, [min(i, last) for i in range(j * T, j * T + T + 1)],
                 [k if k < n_pairs else None for k in range(j * T, j * T + T)]) for j in range(-(-n_pairs // T))]


def parse_rate(rate):
    """A frame rate as a Fraction: anything Fraction parses ("60", "59.94", "60000/1001", 24, Fraction(...)); a float by its
    shortest decimal repr (59.94 is 2997/50, not the nearest binary fraction).  Not positive raises ValueError."""
    try:
        r = Fraction(repr(rate)) if isinstance(rate, float) else Fraction(rate)
    except (TypeError, ValueError, ZeroDivisionError, OverflowError):
        raise ValueError(f"video: a frame rate must be a positive finite number (got {rate!r})") from None
    if r <= 0:
        raise ValueError(f"video: a frame rate must be a positive finite number (got {rate!r})")
    return r


def fps_schedule(n_frames, input_fps, output_fps, batch):
    """The passes of video_interpolate(fps=(input_fps, output_fps)) over n_frames frames: interp_schedule()'s passes, each
    with the output frames it writes.  Output frame n sits at input time s = n input_fps / output_fps, for n = 0 ..
    floor((n_frames - 1) output_fps / input_fps), computed exactly in Fractions.  An integer s is a copy of input frame s
    (written by the pass that holds pair min(s, n_frames - 2)); any other s is the item (k, t) = (floor(s), float(s - k))
    of the pass that holds pair k.  Returns a list of FpsPass(frames, pairs, items, copies): items are (n, k, t) and
    copies (n, i), both with global frame indices.  Needs output_fps > input_fps (up-conversion); anything else raises
    ValueError."""
    fin, fout = parse_rate(input_fps), parse_rate(output_fps)
    if fout <= fin:
        raise ValueError(f"video: frame-rate conversion goes up: the output rate must exceed the input rate "
                         f"(got {fin} -> {fout})")
    passes = interp_schedule(n_frames, batch)
    T, last = int(batch), int(n_frames) - 1
    items, copies = [[] for _ in passes], [[] for _ in passes]
    for n in range(last * fout // fin + 1):
        s = n * fin / fout
        k = s.numerator // s.denominator
        if s.denominator == 1:
            copies[min(k, last - 1) // T].append((n, k))
        else:
            items[k // T].append((n, k, float(s - k)))
    return [FpsPass(p.frames, p.pairs, i, c) for p, i, c in zip(passes, items, copies)]


def check_shutter(shutter):
    """A shutter angle in degrees as a Fraction in (0, 360] (parse_rate()'s parsing: a float by its shortest repr).  360 is
    an exposure as long as the output frame interval, 180 half of it.  Anything else raises ValueError."""
    try:
        a = Fraction(repr(shutter)) if isinstance(shutter, float) else Fraction(shutter)
    except (TypeError, ValueError, ZeroDivisionError, OverflowError):
        a = None
    if isinstance(shutter, bool) or a is None or not 0 < a <= 360:
        raise ValueError(f"video: the shutter angle must be a number of degrees in (0, 360] (got {shutter!r})")
    return a


def check_density(density):
    """The samples per input-frame interval of a shutter as an int >= 1.  Anything else raises ValueError."""
    try:
        ok = not isinstance(density, bool) and int(density) == density and density >= 1
    except (TypeError, ValueError, OverflowError):
        ok = False
    if not ok:
        raise ValueError(f"video: the shutter density must be an integer >= 1 (got {density!r})")
    return int(density)


def exposure(input_fps, output_fps, shutter, density):
    """The exposure of one output frame in input frames and its sample count: (e, m) = ((shutter / 360) input_fps /
    output_fps as a Fraction, max(1, ceil(density e)))."""
    e = check_shutter(shutter) / 360 * parse_rate(input_fps) / parse_rate(output_fps)
    return e, max(1, math.ceil(check_density(density) * e))


def shot_range(i, last, cuts):
    """The first and last frame of the shot holding frame i: a cut pair k ends a shot at frame k."""
    return (max([c + 1 for c in cuts if c < i], default=0), min([c for c in cuts if c >= i], default=last))


def shutter_schedule(n_frames, input_fps, output_fps, shutter, density, batch, cuts=()):
    """The passes of video_interpolate(fps=(input_fps, output_fps), shutter=, density=) over n_frames frames:
    interp_schedule()'s passes, each with the samples it runs.  Output frame n sits at s = n input_fps / output_fps, n = 0
    .. floor((n_frames - 1) output_fps / input_fps), at any rate ratio (down-conversion and equal rates included).  Its
    exposure [s - e/2, s + e/2] holds m samples (exposure()), u_j = s - e/2 + (j + 1/2) e / m, exact in Fractions, each
    clamped into the frames [a, b] of the shot holding s (shot_range(); inside a cut pair k, the shot of cut_copy(k, t)).
    An integer u_j is input frame u_j, run by the pass that holds pair min(u_j, n_frames - 2); any other is the item
    (k, t) = (floor(u_j), float(u_j - k)) of the pass that holds pair k.  A frame's samples run in order, so they may
    span passes.  Returns a list of ShutterPass(frames, pairs, samples, opens, closes): samples (n, i, t) with global
    frame indices in run order (t None: input frame i, else pair i at t), opens / closes the output frames whose first /
    last sample the pass runs.  cuts: the scene-cut pairs (check_cuts())."""
    fin, fout = parse_rate(input_fps), parse_rate(output_fps)
    e, m = exposure(fin, fout, shutter, density)
    passes = interp_schedule(n_frames, batch)
    T, last = int(batch), int(n_frames) - 1
    cuts = check_cuts(cuts, n_frames, "shutter_schedule")
    samples, opens, closes = [[] for _ in passes], [[] for _ in passes], [[] for _ in passes]
    for n in range(last * fout // fin + 1):
        s = n * fin / fout
        k = math.floor(s)
        a, b = shot_range(cut_copy(k, s - k) if k in cuts and s != k else k, last, cuts)
        for j in range(m):
            u = min(max(s - e / 2 + (j + Fraction(1, 2)) * e / m, Fraction(a)), Fraction(b))
            i = math.floor(u)
            p = min(i, last - 1) // T if u == i else i // T
            samples[p].append((n, i, None if u == i else float(u - i)))
            if j == 0:
                opens[p].append(n)
            if j == m - 1:
                closes[p].append(n)
    return [ShutterPass(p.frames, p.pairs, sm, o, c) for p, sm, o, c in zip(passes, samples, opens, closes)]


def check_scene_cut(scene_cut):
    """A scene-cut threshold as a float in [0, 1]: pair k (frame k -> k + 1) is a cut when its score (networks.utils.
    scene_cut_scores) exceeds it, so 1.0 finds none.  Anything else raises ValueError."""
    try:
        thr = float(scene_cut)
    except (TypeError, ValueError):
        thr = None
    if thr is None or not 0.0 <= thr <= 1.0:
        raise ValueError(f"video: scene_cut must be a threshold in [0, 1] (got {scene_cut!r})")
    return thr


def pass_cuts(pairs, scores, thr):
    """The cut pairs of one pass, in order: the pair k of row r is a cut when float(scores[r]) > thr; idle rows (None)
    are ignored."""
    return [k for r, k in enumerate(pairs) if k is not None and float(scores[r]) > thr]


def print_cuts(cuts):
    """Prints the number of scene-cut pairs and their indices (pair k: frame k -> k + 1), as the sweeps and the CLI
    report them."""
    print(f"scene cuts: {len(cuts)}" + (" at pairs " + " ".join(str(k) for k in cuts) if cuts else ""))


def cut_copy(k, t):
    """The input frame that stands in for the frame at time t of pair k when the pair is a scene cut: the nearer one, k
    for t <= 0.5 and k + 1 after it (blending two shots would give a ghosted cross-dissolve)."""
    return k if t <= 0.5 else k + 1


def split_cut_items(items, cuts):
    """The (n, k, t) items of an fps pass (fps_schedule()) split by the cut pairs: (the items of pairs that are not cuts,
    in order; the copies (n, cut_copy(k, t)) that replace the others)."""
    return ([it for it in items if it[1] not in cuts],
            [(n, cut_copy(k, t)) for n, k, t in items if k in cuts])


def cold_start(k, cuts):
    """Whether pair k of a warm-started video runs cold: the first pair, a cut pair (it spans two shots) and the pair
    after a cut (the first of a shot), so each shot runs the chain it would run alone."""
    return k == 0 or k in cuts or k - 1 in cuts


def frame_number(k, m, j=None):
    """The output index of input frame k (j None), or of the j-th of the m frames interpolated between frames k and k + 1:
    k (m + 1) and k (m + 1) + j + 1.  N input frames give (N - 1)(m + 1) + 1 outputs."""
    return k * (m + 1) + (0 if j is None else j + 1)


class _Slot:
    """Pinned host staging (frames in, or a pass's outputs) and the event behind the last pass that used it; futures:
    the writer tasks that still read it."""

    def __init__(self, **shapes):
        for name, (shape, dtype) in shapes.items():
            setattr(self, name, torch.zeros(*shape, dtype=dtype).pin_memory())
        self.event = None
        self.futures = []

    def wait(self):
        for f in self.futures:
            f.result()
        self.futures = []
        if self.event is not None:
            self.event.synchronize()


def _workers(workers):
    """The decode and write threads of a _Pipeline as an int (0: none); a negative count raises ValueError."""
    workers = int(workers)
    if workers < 0:
        raise ValueError(f"video: workers must be >= 0 (got {workers})")
    return workers


class _Pipeline:
    """The passes of a video on the host, on `device`'s current stream:

        with _Pipeline(paths, passes, rgb, batch, workers, device) as pipe:
            for j, ps, imgs, frames in pipe:  # pass j = passes[j]: its decoded frames, and the pinned rows holding them
                ...                           # the GPU work of the pass
                pipe.emit(write, rows, name=device_output, ...)

    The frames of passes[j].frames (paths, decoded RGB with rgb, else BGR) are decoded depth passes ahead by `workers`
    threads (workers = 0: on this thread when the pass is due) into two pinned input slots of batch + 1 rows used in
    turn; every frame needs the size of paths[0].  emit() copies the pass's device outputs into two pinned output slots
    used in turn (allocated on first use with `rows` rows, default the output's own) and records one event behind them
    and the pass's work; write(slot) then runs on a writer thread (workers = 0: inline) and calls slot.event.synchronize()
    before it reads the slot (slot None: the pass had no outputs).  A slot is refilled only once its event has completed
    and its writers have returned, so a writer's exception reaches the caller there or when the pipeline exits.

    extra (a list of paths aligned with paths, each of paths[0]'s size) is decoded alongside by the same threads into a
    second pinned buffer of each input slot; pipe.extra holds the current pass's rows of it."""

    def __init__(self, paths, passes, rgb, batch, workers, device, extra=None):
        self.paths, self.passes, self.rgb, self.T, self.workers, self.device = paths, passes, rgb, batch, workers, device
        self.extra_paths, self.extra = extra, None
        self.depth = max(1, -(-workers // batch))  # passes decoded ahead of the one the GPU is given
        self.ins = self.outs = None
        self.loose = []  # the writes of passes without outputs

    def __enter__(self):
        self.decoders = ThreadPoolExecutor(self.workers) if self.workers > 0 else None
        self.writers = ThreadPoolExecutor(self.workers) if self.workers > 0 else None
        self.on_device = torch.cuda.device(self.device)
        self.on_device.__enter__()
        self.stream = torch.cuda.current_stream(self.device)
        return self

    def __exit__(self, exc_type, exc, tb):
        try:
            if exc_type is None:
                for o in self.outs or ():
                    o.wait()
                for f in self.loose:
                    f.result()
        finally:
            self.on_device.__exit__(None, None, None)
            for pool in (self.decoders, self.writers):
                if pool is not None:
                    pool.shutdown(wait=True, cancel_futures=True)

    def _load(self, paths, i):
        if paths is None:
            return None
        if self.decoders is None:
            return lambda: _imread(paths[i], self.rgb)
        return self.decoders.submit(_imread, paths[i], self.rgb).result

    def _submit(self, j):
        return [(i, self._load(self.paths, i), self._load(self.extra_paths, i)) for i in self.passes[j].frames]

    def __iter__(self):
        paths, depth, shape = self.paths, self.depth, None
        ahead = [self._submit(j) for j in range(min(depth, len(self.passes)))]
        for j, ps in enumerate(self.passes):
            loads = ahead.pop(0)
            if j + depth < len(self.passes):
                ahead.append(self._submit(j + depth))
            imgs, extra = [], []
            for i, load, xload in loads:
                img = load()
                if shape is None:
                    shape = img.shape
                elif img.shape != shape:
                    raise ValueError(f"video: {paths[i]} is a {img.shape[0]}x{img.shape[1]} frame, {paths[0]} is "
                                     f"{shape[0]}x{shape[1]}: every frame needs one size")
                imgs.append(img)
                if xload is not None:
                    x = xload()
                    if x.shape != shape:
                        raise ValueError(f"video: {self.extra_paths[i]} is a {x.shape[0]}x{x.shape[1]} frame, "
                                         f"{paths[0]} is {shape[0]}x{shape[1]}: the frames must be aligned")
                    extra.append(x)
            if self.ins is None:
                rows = ((self.T + 1,) + shape, torch.uint8)
                self.ins = [_Slot(frames=rows, **({} if self.extra_paths is None else {"extra": rows}))
                            for _ in range(2)]
            self.j, self.slot = j, self.ins[j % 2]
            self.slot.wait()
            frames = self.slot.frames[:len(imgs)]
            for r, img in enumerate(imgs):
                frames[r].numpy()[...] = img
            if self.extra_paths is not None:
                self.extra = self.slot.extra[:len(extra)]
                for r, x in enumerate(extra):
                    self.extra[r].numpy()[...] = x
            yield j, ps, imgs, frames

    def emit(self, write, rows=None, **outputs):
        """Ends the current pass: stages its device outputs (those not None) and hands write the slot."""
        outputs = {name: t for name, t in outputs.items() if t is not None}
        o = None
        if outputs:
            if self.outs is None:
                self.outs = [_Slot(**{name: ((rows or len(t),) + tuple(t.shape[1:]), t.dtype)
                                      for name, t in outputs.items()}) for _ in range(2)]
            o = self.outs[self.j % 2]
            o.wait()
            for name, t in outputs.items():
                getattr(o, name)[:len(t)].copy_(t, non_blocking=True)
        event = torch.cuda.Event()  # behind the pass's reads of its input slot and its copies to o
        event.record(self.stream)
        self.slot.event = event
        if o is not None:
            o.event = event
        if self.writers is None:
            write(o)
        else:
            (self.loose if o is None else o.futures).append(self.writers.submit(write, o))


class _Upload:
    """A device copy of each pass's pinned rows, in one buffer allocated on the first pass (later passes may be
    shorter), and the pass's scene cuts scored on that copy."""

    def __init__(self, device):
        self.device, self.buf = device, None

    def __call__(self, src, pairs, thr=None):
        """Copies src to the buffer.  Returns (the device rows, the cut pairs of the pass with the pair indices pairs:
        pass_cuts of networks.utils.scene_cut_scores on the device rows with a threshold thr, else [])."""
        from networks.utils import scene_cut_scores
        if self.buf is None:
            self.buf = torch.empty(src.shape, dtype=src.dtype, device=self.device)
        rows = self.buf[:len(src)]
        rows.copy_(src, non_blocking=True)
        return rows, ([] if thr is None else pass_cuts(pairs, scene_cut_scores(rows).cpu(), thr))


class _FrameWriter:
    """The write callback of a pass's finished frames (_Pipeline.emit, bound to first and n): slot.frames[r] written
    as names[first + r] for r < n, BGR (converted when rgb), then with tally total += tally(slot, n) (0 before any
    slot; the sums of the writer threads, taken under a lock)."""

    def __init__(self, names, rgb, tally=None):
        self.names, self.rgb, self.tally, self.total = names, rgb, tally, 0
        self.lock = threading.Lock()

    def __call__(self, slot, first, n):
        import cv2
        if slot is None:
            return
        slot.event.synchronize()
        for r in range(n):
            img = slot.frames[r].numpy()
            if not cv2.imwrite(self.names[first + r], cv2.cvtColor(img, cv2.COLOR_RGB2BGR) if self.rgb else img):
                raise OSError(f"cannot write {self.names[first + r]}")
        if self.tally is not None:
            c = self.tally(slot, n)
            with self.lock:
                self.total = self.total + c


class _Window:
    """The frames a windowed sweep (video_stabilize(fill=True), video_inpaint, video_denoise, video_segment_motion)
    keeps on the GPU over interp_schedule(F, batch)'s passes.  Frame t is finished once the sweep's data is complete up
    to frame min(t + window, F - 1), and reaches back to frame t - window, so at most cap = min(F, 2 window + batch + 2)
    frames are kept.  Row r of a frame store holds frame base + r, row r of a pair store (flows) pair base + r; frames
    base .. base + have - 1 are kept and the frames before done are finished.

        win = _Window(F, window, batch, device)
        for each pass, on the frames first .. first + n:
            s = win.alloc(frames=((Hs, Ws, 3), torch.uint8), fw=((Hn, Wn, 2), torch.float32), ...)  # allocates once
            new = win.admit(first + n)  # the store rows of the pass's frames not kept yet
            ...                         # those frames into s[name][new], the pass's pairs from row win.row(first) on
            t0, m, rows = win.finish(complete, table)  # frames t0 .. t0 + m - 1 are due: their table rows, rebased
            ...                         # the sweep's kernel on win.kept(name), win.kept_pairs(name) and rows

    It does no GPU work beyond allocating the stores and shifting their rows when frames are dropped."""

    def __init__(self, F, window, batch, device):
        self.F, self.window, self.device = int(F), int(window), device
        self.cap = min(self.F, 2 * self.window + int(batch) + 2)
        self.base = self.have = self.done = 0
        self.store = None

    def alloc(self, **rows):
        """On the first call, allocates store[name] with cap rows of each name=(row shape, dtype); later calls do
        nothing.  Returns the stores."""
        if self.store is None:
            self.store = {name: torch.empty(self.cap, *shape, dtype=dtype, device=self.device)
                          for name, (shape, dtype) in rows.items()}
        return self.store

    def admit(self, last):
        """Keeps the frames up to `last`: returns the store rows of those not kept yet.  When they would not fit, the
        frames no frame still to be finished reaches (those before done - window) are dropped first; if they still
        do not fit, RuntimeError."""
        new = last + 1 - self.base - self.have
        if self.have + new > self.cap:
            drop = max(self.done - self.window, self.base) - self.base
            if self.have - drop + new > self.cap:
                raise RuntimeError(f"video: frames {self.base + self.have} .. {last} do not fit beside the frames a "
                                   f"window of {self.window} keeps ({self.cap} at most)")
            for t in self.store.values():
                t[:self.have - drop].copy_(t[drop:self.have].clone())
            self.base, self.have = self.base + drop, self.have - drop
        self.have += new
        return slice(self.have - new, self.have)

    def row(self, t):
        """The store row of frame (or pair) t."""
        return t - self.base

    def kept(self, name):
        """The rows of frame store `name` that hold the kept frames."""
        return self.store[name][:self.have]

    def kept_pairs(self, name):
        """The rows of pair store `name` that hold the pairs between the kept frames."""
        return self.store[name][:self.have - 1]

    def finish(self, complete, table):
        """Finishes the frames from done on, in order, while min(t + window, F - 1) <= complete (the last frame whose
        inputs are complete).  Returns (t0, m, table[t0:t0 + m] with column 0, the frame, as its store row)."""
        t0 = last = self.done
        while last < self.F and min(last + self.window, self.F - 1) <= complete:
            last += 1
        rows = table[t0:last].copy()
        rows[:, 0] -= self.base
        self.done = last
        return t0, last - t0, rows


def video(model, frames, out, batch=8, workers=4, warm_start=False, flo=None, npy=None, native_flow=False,
          scene_cut=None):
    """The flow between every pair of consecutive frames of a loaded networks.RAFT.RAFT model, written as
    <out>/flow_<k:06d>.png for pair k (frame k -> k + 1; the GPU colour coding of networks.utils.flow_to_color, BGR), and
    with flo / npy (directories) also as flow_<k:06d>.flo / .npy.  frames: a directory (its sorted *.png and *.jpg) or a
    list of paths; all frames must have one size (a mismatch raises ValueError naming the first such file).  Frames go in
    RGB with model.upstream and BGR otherwise, like the CLI.  batch pairs run per pass (schedule()); warm_start warm-starts
    every pair from the previous one (batch must be 1).  native_flow resizes the flows of a model with input_size back to
    the frames' size (networks.utils.resize_flow) before they are coloured or saved.  Each flow equals the model's
    forward(f_k, f_(k+1)) (warm_start: the chain forward(..., flow_init=forward_interpolate(flow_low))) bit for bit.

    scene_cut (warm_start only; a threshold in [0, 1]) restarts the chain at scene cuts: every pair is scored on the GPU
    (networks.utils.scene_cut_scores of the decoded frames k and k + 1, the previous one kept on the device), pair k is a
    cut when its score exceeds scene_cut, and it runs cold when cold_start(k, cuts) -- so each shot's flows equal those of
    video(warm_start=True) on that shot's frames alone, and a cut pair's flow is the cold forward(f_k, f_(k+1)).
    Returns the written paths, pair by pair; with scene_cut the tuple (paths, cuts), cuts the increasing cut pairs."""
    import cv2
    from flow_utils import write_flo
    from networks.utils import flow_to_color, forward_interpolate, resize_flow, scene_cut_scores

    paths = list_frames(frames)
    batch, workers = int(batch), _workers(workers)
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    if thr is not None and not warm_start:
        raise ValueError("video: scene_cut restarts the warm-start chain at cuts; without warm_start every pair runs cold, "
                         "so a cut changes nothing")
    passes = schedule(len(paths), batch, warm_start)
    dirs = {"png": os.fspath(out), "flo": None if flo is None else os.fspath(flo),
            "npy": None if npy is None else os.fspath(npy)}
    for d in dirs.values():
        if d is not None:
            os.makedirs(d, exist_ok=True)
    keep_flow = flo is not None or npy is not None
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device

    def name(k, ext):
        return os.path.join(dirs[ext], f"flow_{k:06d}.{ext}")

    def write(slot, rows):  # writer thread: the files of one pass, once its copies have landed
        slot.event.synchronize()
        for r, k in rows:
            if not cv2.imwrite(name(k, "png"), slot.color[r].numpy()):
                raise OSError(f"cannot write {name(k, 'png')}")
            if flo is not None:
                write_flo(name(k, "flo"), slot.flow[r].numpy())
            if npy is not None:
                np.save(name(k, "npy"), slot.flow[r].numpy())

    written, init = [], None
    on_dev, cuts = None, []  # scene_cut: frames k and k + 1 in rows k % 2 and (k + 1) % 2 (the score is symmetric)
    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for j, ps, imgs, host in pipe:
            shape = imgs[0].shape
            if thr is not None:  # one pair per pass: score it, then hand the engine the device rows
                k = ps.pairs[0]
                if on_dev is None:
                    on_dev = torch.empty((2,) + shape, dtype=torch.uint8, device=dev)
                if ps.carry:
                    on_dev[(k + 1) % 2].copy_(host[0], non_blocking=True)
                    host = on_dev[(k + 1) % 2][None]
                else:
                    on_dev.copy_(host, non_blocking=True)
                    host = on_dev
                cuts += pass_cuts(ps.pairs, scene_cut_scores(on_dev).cpu(), thr)
                if cold_start(k, cuts):
                    init = None
            if warm_start:
                low, flow = engine.forward_sequence(host, carry=ps.carry, flow_init=init, return_low=True)
                init = forward_interpolate(low)  # before the next pass overwrites flow_low
            else:
                flow = engine.forward_sequence(host, carry=ps.carry)
            if native_flow and tuple(flow.shape[1:3]) != tuple(shape[:2]):
                flow = resize_flow(flow, shape[:2])
            rows = [(r, k) for r, k in enumerate(ps.pairs) if k is not None]
            pipe.emit(partial(write, rows=rows), color=flow_to_color(flow, convert_to_bgr=True),
                      flow=flow if keep_flow else None)
            for _, k in rows:
                written += [name(k, e) for e in ("png", "flo", "npy") if dirs[e] is not None]
    return written if thr is None else (written, cuts)


def video_interpolate(model, frames, out, ts=None, batch=8, workers=4, fps=None, scene_cut=None, native=False,
                      shutter=None, density=16):
    """Frame-rate up-conversion with a loaded networks.RAFT.RAFT model of the frames (a directory's sorted *.png / *.jpg,
    or a list of paths, all of one size), written as one numbered sequence <out>/frame_<n:06d>.png.  Give exactly one of:

    - ts: the m = len(ts) frames at times ts (strictly increasing inside (0, 1)) between every consecutive pair, n =
      frame_number(k, m[, j]).  Every pass runs interpolate_sequence on batch + 1 frames (interp_schedule()), so an
      interpolated frame equals the single-pair CLI's PNG of model.interpolate(f_k, f_(k+1), ts) byte for byte.
    - fps = (input_fps, output_fps): the sequence at output_fps > input_fps (rates as parse_rate() takes them), output
      frame n at input time s = n input_fps / output_fps (fps_schedule()).  Every pass runs interpolate_sequence_at on
      batch + 1 frames with the (pair, time) items of its pairs alone, so a frame at a fractional s equals the single-pair
      CLI's PNG of model.interpolate(f_k, f_(k+1), float(s - k)) byte for byte; an integer s is input frame s.

    Both quantise on the GPU.  The input frames are written as the network saw them: the decoded bytes, or with
    model.input_size exactly the bytes of cv2.resize of them (which the GPU resize reproduces).  Frames go in RGB with
    model.upstream and BGR otherwise, like the CLI; the files are BGR.  The files do not depend on batch or workers.

    native=True (a model with input_size) writes every frame at the decoded size: the flows are estimated and reversed at
    input_size, and the interpolated frames blended from the decoded frames (RaftEngine's native blend), so each equals
    the single-pair CLI's --native-frames PNG byte for byte; input frames and scene-cut copies are the decoded frames
    (only converted to BGR).

    scene_cut (a threshold in [0, 1]) stops interpolation at scene cuts: each pass's frames are copied to the GPU once and
    scored there (networks.utils.scene_cut_scores of the decoded frames), and pair k is a cut when its score exceeds
    scene_cut.  Every frame of a cut pair at time t is then a copy of the nearer input frame (cut_copy(): k for t <= 0.5,
    else k + 1), written like the input frames; only the other pairs' frames are interpolated, and a pass with none of
    them makes no engine call.  The other files are the bytes of the run without scene_cut.

    shutter (degrees in (0, 360], with fps; any rate ratio, down-conversion included) gives the conversion a camera
    shutter: every output frame is the mean of the sub-frames over its exposure, density samples per input-frame
    interval (shutter_schedule(), RaftEngine.expose), in one sweep of interp_schedule()'s passes.  The fp32 sums of the
    output frames whose exposure spans two passes stay on the GPU between them, so the files do not depend on batch or
    workers: they are the frames of model.motion_blur on the whole clip, byte for byte (BGR).  With scene_cut a first
    sweep decodes and scores every pair (no flow), so the exposures are clamped at every cut before any is summed.
    Returns the written paths in output order; with scene_cut the tuple (paths, cuts), cuts the increasing cut pairs."""
    import cv2

    paths = list_frames(frames)
    if (ts is None) == (fps is None):
        raise ValueError("video_interpolate: give the times ts or the rates fps = (input_fps, output_fps), exactly one")
    batch, workers = int(batch), _workers(workers)
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    if shutter is not None:
        if fps is None:
            raise ValueError("video_interpolate: a shutter needs the rates fps = (input_fps, output_fps)")
        return _video_shutter(model, paths, out, fps, shutter, density, batch, workers, thr, native)
    last = len(paths) - 1
    if fps is None:
        ts = check_times(ts)
        m = len(ts)
        passes = interp_schedule(len(paths), batch)
        n_out = frame_number(last, m) + 1
        rows = m * batch  # output rows of one pass
    else:
        passes = fps_schedule(len(paths), *fps, batch)
        n_out = sum(len(p.items) + len(p.copies) for p in passes)
        rows = max(len(p.items) for p in passes)
    T = batch
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    engine = model.engine()
    rgb = bool(model.upstream)
    size = model.input_size
    dev = engine.device

    def name(n):
        return os.path.join(out, f"frame_{n:06d}.png")

    def original(img):  # the frame as the network saw it, BGR
        if size is not None and not native:
            img = cv2.resize(img, dsize=(size[1], size[0]))
        return cv2.cvtColor(img, cv2.COLOR_RGB2BGR) if rgb else img

    def write(slot, made, copies):  # writer thread: the files of one pass, once its copies have landed (slot None: none)
        for n, img in copies:
            if not cv2.imwrite(name(n), original(img)):
                raise OSError(f"cannot write {name(n)}")
        if slot is None:
            return
        slot.event.synchronize()
        for n, r in made:
            if not cv2.imwrite(name(n), slot.frames[r].numpy()):
                raise OSError(f"cannot write {name(n)}")

    upload, cuts = _Upload(dev), []
    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for j, ps, imgs, src in pipe:
            first = ps.frames[0]  # frame i is row i - first of the pass
            cut = []
            if thr is not None:  # score the pass on the GPU; the engine then reads the frames from there too
                src, cut = upload(src, ps.pairs, thr)
                cuts += cut
            res = None
            if fps is None:  # row j T + r: pair r of the pass at ts[j]
                pairs = [(r, k) for r, k in enumerate(ps.pairs) if k is not None]
                live = [(r, k) for r, k in pairs if k not in cut]
                if live:
                    res = engine.interpolate_sequence(src, ts, uint8=True, bgr=rgb, native=native).flatten(0, 1)
                made = [(frame_number(k, m, jt), jt * T + r) for r, k in live for jt in range(m)]
                copies = [(frame_number(k, m), k) for _, k in pairs] + ([(n_out - 1, last)]
                                                                        if j == len(passes) - 1 else [])
                copies += [(frame_number(k, m, jt), cut_copy(k, t)) for k in cut for jt, t in enumerate(ts)]
            else:  # row i: item i of the pass
                items, cut_copies = split_cut_items(ps.items, cut)
                if items:
                    res = engine.interpolate_sequence_at(src, [(k - first, t) for _, k, t in items], uint8=True,
                                                         bgr=rgb, native=native)
                made = [(n, i) for i, (n, _, _) in enumerate(items)]
                copies = ps.copies + cut_copies
            copies = [(n, imgs[i - first]) for n, i in copies]
            pipe.emit(partial(write, made=made, copies=copies), rows, frames=res)
    paths = [name(n) for n in range(n_out)]
    return paths if thr is None else (paths, cuts)


def _video_shutter(model, paths, out, fps, shutter, density, batch, workers, thr, native):
    """video_interpolate(fps=, shutter=, density=) after its argument checks: the optional scoring sweep, then one sweep of
    shutter_schedule()'s passes, each one RaftEngine.expose call whose closed frames are written."""
    import cv2

    try:
        fin, fout = fps
    except (TypeError, ValueError):
        raise ValueError(f"video_interpolate: fps must be (input_fps, output_fps) (got {fps!r})") from None
    _, m = exposure(fin, fout, shutter, density)
    n_out = (len(paths) - 1) * parse_rate(fout) // parse_rate(fin) + 1
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    engine = model.engine()
    rgb, dev = bool(model.upstream), engine.device

    def name(n):
        return os.path.join(out, f"frame_{n:06d}.png")

    def write(slot, made):  # writer thread: the frames one pass closed, once its copies have landed
        if slot is None:
            return
        slot.event.synchronize()
        for n, r in made:
            if not cv2.imwrite(name(n), slot.frames[r].numpy()):
                raise OSError(f"cannot write {name(n)}")

    cuts = []
    if thr is not None:  # every cut is known before any exposure is summed
        upload = _Upload(dev)
        with _Pipeline(paths, interp_schedule(len(paths), batch), rgb, batch, workers, dev) as pipe:
            for _, ps, _, src in pipe:
                cuts += upload(src, ps.pairs, thr)[1]
                pipe.emit(lambda slot: None)
    passes = shutter_schedule(len(paths), fin, fout, shutter, density, batch, cuts)
    rows = max(1, max(len(p.closes) for p in passes))
    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for _, ps, _, src in pipe:
            first = ps.frames[0]
            res = None
            if ps.samples:
                res = engine.expose(src, [(n, i - first, t) for n, i, t in ps.samples], m, ps.opens, ps.closes,
                                    bgr=rgb, native=native)
            pipe.emit(partial(write, made=[(n, r) for r, n in enumerate(ps.closes)]), rows, frames=res)
    paths = [name(n) for n in range(n_out)]
    return paths if thr is None else (paths, cuts)


def read_queries(path):
    """The query points of a text file, one `frame x y` line per point (frame an integer, x and y pixels of the frames'
    own size); blank lines and text after '#' are skipped.  Returns an [N,3] float64 array; a malformed line or a file
    without points raises ValueError."""
    rows = []
    with open(path) as f:
        for n, line in enumerate(f, 1):
            parts = line.split("#", 1)[0].split()
            if not parts:
                continue
            try:
                if len(parts) != 3:
                    raise ValueError
                rows.append((int(parts[0]), float(parts[1]), float(parts[2])))
            except ValueError:
                raise ValueError(f"video: {path}:{n}: expected `frame x y` with an integer frame "
                                 f"(got {line.strip()!r})") from None
    if not rows:
        raise ValueError(f"video: {path} holds no query points")
    return np.array(rows, dtype=np.float64)


def track_grid(H, W, step, frame=0):
    """The queries of a grid on frame `frame` of H x W frames: a point at every step-th pixel, x in {0, step, ...} <= W - 1
    and y likewise, row by row.  Returns an [N,3] float64 array of (frame, x, y); step = 1 is every pixel.  A step below
    1 raises ValueError."""
    if int(step) != step or int(step) < 1:
        raise ValueError(f"video: the grid step must be an integer >= 1 (got {step!r})")
    ys, xs = np.meshgrid(np.arange(0, int(H), int(step)), np.arange(0, int(W), int(step)), indexing="ij")
    return np.stack([np.full(xs.size, int(frame)), xs.ravel(), ys.ravel()], axis=-1).astype(np.float64)


def track_colors(N):
    """The fixed BGR colour of each of N query points in video_track's drawings (a seeded draw, so every run and every
    batch paints a point alike)."""
    return np.random.default_rng(0).integers(40, 256, size=(N, 3)).astype(np.uint8)


def video_track(model, frames, out, queries=None, grid=None, grid_frame=0, batch=8, workers=4, vis=None, backward=False):
    """Point tracking through a video of any length with a loaded networks.RAFT.RAFT model: the frames (a directory's
    sorted *.png / *.jpg, or a list of paths, all of one size) and the query points as `queries` ([N,3] rows (frame, x,
    y) in the frames' own pixels) or `grid` = STEP (track_grid() on frame grid_frame; give exactly one).  Every pass runs
    forward_sequence_bidirectional(check=False) on batch + 1 frames (interp_schedule()) and one rb_track_points launch
    (networks.utils.track_points), the points' positions and states carried from pass to pass on the GPU.  Writes
    <out>/tracks.npy [F,N,2] fp32 and <out>/status.npy [F,N] uint8 (RaftEngine.track's outputs), each pass's rows
    streamed into them through memory maps, so host memory does not grow with F.  vis (a directory) also writes every
    frame at its own size as <vis>/frame_<i:06d>.png with each point of status 0 drawn as a dot in its own colour
    (track_colors()).  The files are the same bytes for every batch and workers value, and equal RAFT.track on the whole
    clip.  Frames go in RGB with model.upstream and BGR otherwise, like the CLI.  Returns (tracks path, status path).

    backward=True also tracks every point back from its frame to frame 0 (RAFT.track(backward=True)).  After the forward
    sweep a reverse sweep runs the same passes again, last to first, each followed by one rb_track_points_backward launch
    (networks.utils.track_points_backward) that carries the points from later passes to earlier ones; only the passes
    whose first frame lies before the largest query frame run, so a grid on frame 0 costs nothing more.  The entries
    (f, i) with f before point i's frame are merged into the memory maps, and with vis the frames before the largest
    query frame are drawn in the reverse sweep from the merged rows.  The flow passes of the reverse sweep are computed a
    second time: that is the price of streaming a clip of any length without keeping its flows."""
    import cv2
    from networks.utils import track_points, track_points_backward
    from .engine import FB_ALPHA1, FB_ALPHA2, track_queries, tracks_to_frames

    paths = list_frames(frames)
    if (queries is None) == (grid is None):
        raise ValueError("video_track: give the query points or a grid step, exactly one")
    batch, workers = int(batch), _workers(workers)
    passes = interp_schedule(len(paths), batch)
    F, T = len(paths), batch
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    if vis is not None:
        vis = os.fspath(vis)
        os.makedirs(vis, exist_ok=True)
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device
    files = (os.path.join(out, "tracks.npy"), os.path.join(out, "status.npy"))
    kw = dict(flow_scale=engine.flow_scale, alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)

    def draw(f, img, tr, st):  # frame f with the points of status 0 of its rows tr, st
        img = cv2.cvtColor(img, cv2.COLOR_RGB2BGR) if rgb else img.copy()
        seen = np.flatnonzero(st == 0)
        xy = np.rint(tr[seen]).astype(np.int64)
        for i, (x, y) in zip(seen, xy):
            cv2.circle(img, (int(x), int(y)), 2, colors[i].tolist(), -1)
        name = os.path.join(vis, f"frame_{f:06d}.png")
        if not cv2.imwrite(name, img):
            raise OSError(f"cannot write {name}")

    def write(slot, first, rows, imgs):  # writer thread: the rows of one pass, once its copies have landed
        slot.event.synchronize()
        tracks_mm[first + rows.start:first + rows.stop] = slot.tracks[rows.start:rows.stop].numpy()
        status_mm[first + rows.start:first + rows.stop] = slot.status[rows.start:rows.stop].numpy()
        if vis is None:
            return
        for r in rows:
            if first + r >= vis_from:  # with backward, the frames before vis_from are drawn by the reverse sweep
                draw(first + r, imgs[r], slot.tracks[r].numpy(), slot.status[r].numpy())

    def merge(slot, first, rows, imgs):  # writer thread, reverse sweep: the entries before each point's frame
        slot.event.synchronize()
        for r in rows:
            f = first + r
            before = f < qf
            tr, st = tracks_mm[f], status_mm[f]
            tr[before] = slot.tracks[r].numpy()[before]
            st[before] = slot.status[r].numpy()[before]
            if vis is not None:
                draw(f, imgs[r], tr, st)

    state = tracks_mm = status_mm = None
    vis_from = 0
    try:
        with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
            for j, ps, imgs, frames in pipe:
                if j == 0:  # the queries, now that the frame size is known
                    src_hw = tuple(frames.shape[1:3])
                    net_hw = engine.input_size if engine.input_size is not None else src_hw
                    q = track_grid(*src_hw, grid, grid_frame) if grid is not None else queries
                    qf, qp = track_queries(q, F, src_hw, net_hw)
                    qframe, qpos = torch.from_numpy(qf).to(dev), torch.from_numpy(qp).to(dev)
                    N = len(qf)
                    vis_from = int(qf.max()) if backward else 0
                    colors = track_colors(N) if vis is not None else None
                    tracks_mm = np.lib.format.open_memmap(files[0], mode="w+", dtype=np.float32, shape=(F, N, 2))
                    status_mm = np.lib.format.open_memmap(files[1], mode="w+", dtype=np.uint8, shape=(F, N))
                flow_fw, flow_bw, _, _ = engine.forward_sequence_bidirectional(frames, check=False)
                n_steps = sum(k is not None for k in ps.pairs)
                first = ps.frames[0]
                tracks, status, state = track_points(flow_fw, flow_bw, qframe, qpos, state=state, first_frame=first,
                                                     n_steps=n_steps, **kw)
                rows = range(0 if j == 0 else 1, n_steps + 1)  # row 0 of a later pass is the last row of the one before
                pipe.emit(partial(write, first=first, rows=rows, imgs=imgs), T + 1,
                          tracks=tracks_to_frames(tracks, src_hw, net_hw), status=status)
        # the reverse sweep: the passes before the largest query frame, last to first; each owns its rows below its last
        # (the row of the last frame of the latest such pass lies at or after every query frame: nothing to merge there)
        reverse = [ps for ps in passes if ps.frames[0] < vis_from][::-1]
        if reverse:
            state = None
            with _Pipeline(paths, reverse, rgb, batch, workers, dev) as pipe:
                for j, ps, imgs, frames in pipe:
                    flow_fw, flow_bw, _, _ = engine.forward_sequence_bidirectional(frames, check=False)
                    n_steps = sum(k is not None for k in ps.pairs)
                    first = ps.frames[0]
                    tracks, status, state = track_points_backward(flow_fw, flow_bw, qframe, qpos, state=state,
                                                                  first_frame=first, n_steps=n_steps, **kw)
                    rows = range(0, min(n_steps, vis_from - first))
                    pipe.emit(partial(merge, first=first, rows=rows, imgs=imgs), T + 1,
                              tracks=tracks_to_frames(tracks, src_hw, net_hw), status=status)
    finally:
        for mm in (tracks_mm, status_mm):
            if mm is not None:
                mm.flush()
    return files


def read_labels(path):
    """A label map from a PNG: palette (mode P) images give their indices, 8-bit grey (mode L) images their values.
    Returns (labels [H,W] uint8, palette [n,3] uint8 or None for grey).  Any other image raises ValueError (an RGB mask
    holds colours, not label ids).  Needs Pillow: cv2 expands a palette PNG to colours and loses the indices."""
    from PIL import Image
    with Image.open(os.fspath(path)) as im:
        if im.mode not in ("P", "L"):
            raise ValueError(f"video: {path} is a mode {im.mode} image; label maps are palette (P) or 8-bit grey (L) PNGs")
        labels = np.array(im, dtype=np.uint8)
        palette = None
        if im.mode == "P":
            palette = np.array(im.getpalette() or [], dtype=np.uint8).reshape(-1, 3)
    return labels, palette


def write_labels(path, labels, palette=None):
    """Writes an [H,W] uint8 label map as a PNG: with the [n,3] palette as a palette image (DAVIS's annotation format),
    without one as 8-bit grey."""
    from PIL import Image
    arr = np.ascontiguousarray(labels, dtype=np.uint8)
    im = Image.frombytes("L" if palette is None else "P", (arr.shape[1], arr.shape[0]), arr.tobytes())
    if palette is not None:
        im.putpalette(np.asarray(palette, dtype=np.uint8).reshape(-1).tolist())
    im.save(os.fspath(path), format="PNG")


def check_keyframes(frames, F, what="video_propagate"):
    """The keyframe indices as a list of ints: one int, or a strictly increasing sequence of at least one index, each in
    [0, F).  Anything else raises ValueError."""
    seq = [frames] if isinstance(frames, (int, np.integer)) else frames
    try:
        keys = list(seq)
    except TypeError:
        keys = None
    if not keys or not all(isinstance(k, (int, np.integer)) and not isinstance(k, bool) for k in keys):
        raise ValueError(f"{what}: the key frames must be an integer or a sequence of integers (got {frames!r})")
    keys = [int(k) for k in keys]
    if not all(0 <= k < F for k in keys) or any(b <= a for a, b in zip(keys, keys[1:])):
        raise ValueError(f"{what}: the key frames must be strictly increasing integers in [0, {F}) (got {keys})")
    return keys


def check_cuts(cuts, F, what="video_propagate"):
    """Scene-cut pairs as a sorted list of distinct ints in [0, F - 1) (pair k: frames k and k + 1).  Anything else
    raises ValueError."""
    try:
        cuts = list(cuts)
        cs = [int(c) for c in cuts if not isinstance(c, bool) and int(c) == c]
        ok = len(cs) == len(cuts)
    except (TypeError, ValueError):
        ok = False
    if not ok or not all(0 <= c < F - 1 for c in cs):
        raise ValueError(f"{what}: the cuts must be integer pair indices in [0, {F - 1}) (got {cuts!r})")
    return sorted(set(cs))


def keyframe_rows(F, frames, cuts=()):
    """The per-frame table of several-keyframe propagation (rb_labels_propagate_keys' rows): [F,4] int32, row t =
    (slot_a, slot_b, w_a, w_b).  With keyframes K_0 < ... < K_(m-1) (frames) and the cut pairs `cuts` (pair k between
    frames k and k + 1):
      side A = i, the latest key K_i <= t, when no cut lies among pairs K_i .. t - 1, else -1;
      side B = j, the earliest key K_j > t, when no cut lies among pairs t .. K_j - 1, else -1;
      a keyframe row t = K_i has side A only (its key, bit for bit);
      w_a = K_j - t and w_b = t - K_i when both sides are present (the nearer key weighs more), else 0.
    A row without sides (only possible with cuts) gets label 0 and status 3."""
    keys = np.asarray(check_keyframes(frames, F, "keyframe_rows"), dtype=np.int64)
    cuts = np.asarray(check_cuts(cuts, F, "keyframe_rows"), dtype=np.int64)
    t = np.arange(int(F), dtype=np.int64)
    i = np.searchsorted(keys, t, side="right") - 1  # latest K_i <= t
    j = i + 1  # earliest K_j > t
    has_a = i >= 0
    has_b = j < len(keys)
    ka = keys[np.clip(i, 0, None)]
    kb = keys[np.clip(j, None, len(keys) - 1)]
    n_cuts_before = np.searchsorted(cuts, t, side="left")  # cuts < t, i.e. pairs .. t - 1
    has_a &= np.searchsorted(cuts, ka, side="left") == n_cuts_before  # no cut in [K_i, t)
    has_b &= np.searchsorted(cuts, kb, side="left") == n_cuts_before  # no cut in [t, K_j)
    has_b &= ~np.isin(t, keys)
    both = has_a & has_b
    return np.stack([np.where(has_a, i, -1), np.where(has_b, j, -1), np.where(both, kb - t, 0),
                     np.where(both, t - ka, 0)], axis=1).astype(np.int32)


class KeyframeSweep:
    """The GPU side of streaming keyframe propagation over interp_schedule(F, T) passes (video_propagate and
    raft_b200.davis.propagate_clip): the labels of every frame with the bits of RaftEngine.propagate on the whole clip.

        sweep = KeyframeSweep(engine, keys, K, F, T, cuts)
        for ps in sweep.forward_passes(passes):  # flows of each: forward_sequence_bidirectional(check=False)
            chunks = sweep.forward(ps, flow_fw, flow_bw)
        for ps in sweep.reverse_passes(passes):  # the passes before the first key's, last to first
            chunks = sweep.reverse(ps, flow_fw, flow_bw)

    Each call returns the frames it completes as chunks (first frame, labels [n,Hs,Ws], status [n,Hs,Ws]) of device
    tensors, valid until the next call.  `cuts` is a list the caller extends with each pass's cut pairs before the call.
    - Frames before the first key K_0 take side B from K_0 alone: the pass holding K_0 chains back from it, and the
      reverse sweep carries that chain to frame 0 (as video_track(backward=True) does).
    - Frames from the last key K_(m-1) on take side A from it alone: a forward chain carried from pass to pass.
    - Between K_0 and K_(m-1) the flows of the current keyframe interval are copied to the device as their passes arrive;
      when the next key is reached, both chains run over the interval, one rb_labels_propagate_keys launch labels its
      frames, and the store is reused.  Memory therefore grows with the longest keyframe interval L, not the clip: 16 B
      per network pixel per pair for the two flows and 18 B per pixel per frame for the two chains, about 15 MB per
      interval frame at 432x1024 (by arithmetic).
    With one key and no scene-cut detection (simple) this is the single-key path: one chain buffer per pass and
    rb_labels_propagate."""

    def __init__(self, engine, keys, K, F, T, cuts, simple):
        from .engine import FB_ALPHA1, FB_ALPHA2
        self.keys, self.K, self.F, self.T, self.cuts, self.simple = keys, list(K), int(F), int(T), cuts, simple
        self.kw = dict(flow_scale=engine.flow_scale, alpha1=FB_ALPHA1, alpha2=FB_ALPHA2)
        self.dev = engine.device
        self.L = max((b - a for a, b in zip(self.K, self.K[1:])), default=0)  # the longest interval
        self.acc = self.store = None
        self.cur, self.next_pair = 0, self.K[0]  # the interval being stored, the next pair it needs
        self.carry_fw = self.carry_bw = None

    def first_pass(self, n_passes):
        """The pass the forward sweep starts at: the one holding K_0 (the last pass when K_0 is the last frame)."""
        return min(self.K[0] // self.T, n_passes - 1)

    def _buffers(self, H, W):
        if self.acc is None:
            self.acc = torch.empty(self.T + 1, H, W, 2, dtype=torch.float32, device=self.dev)
            self.status = torch.empty(self.T + 1, H, W, dtype=torch.uint8, device=self.dev)
            if self.L:
                self.store = torch.empty(2, self.L, H, W, 2, dtype=torch.float32, device=self.dev)  # flow_fw, flow_bw
                self.ia = torch.empty(2, self.L + 1, H, W, 2, dtype=torch.float32, device=self.dev)  # side A, side B
                self.ist = torch.empty(2, self.L + 1, H, W, dtype=torch.uint8, device=self.dev)

    def _one_sided(self, first, n, acc, status):
        """Labels of the pass rows first .. first + n (one chain buffer, the head's and the tail's rows): the table of
        keyframe_rows with the rows between K_0 and K_(m-1) absent (the intervals label those)."""
        from networks.utils import propagate_labels, propagate_labels_keys
        if self.simple:
            return propagate_labels(acc, status, self.keys[0])
        rows = keyframe_rows(self.F, self.K, self.cuts)[first:first + n + 1].copy()
        t = np.arange(first, first + n + 1)
        rows[(t >= self.K[0]) & (t < self.K[-1])] = (-1, -1, 0, 0)
        return propagate_labels_keys(acc, status, acc, status, self.keys, rows)

    def forward(self, ps, flow_fw, flow_bw):
        from networks.utils import accumulate_flow, accumulate_flow_backward
        n = sum(k is not None for k in ps.pairs)
        first, K0, Kl = ps.frames[0], self.K[0], self.K[-1]
        self._buffers(*flow_fw.shape[1:3])
        acc, status, kw = self.acc[:n + 1], self.status[:n + 1], self.kw
        chunks, pass_rows = [], []
        if self.carry_bw is None:  # the pass holding K_0: side B of the frames before it
            acc[K0 - first].zero_()
            status[K0 - first].zero_()
            accumulate_flow_backward(flow_fw, flow_bw, acc, status, start=K0 - first, n_steps=n, **kw)
            self.carry_bw = (acc[0].clone(), status[0].clone())
            pass_rows.append((first, K0))
        if self.carry_fw is not None:  # past K_(m-1): row 0 is the last row of the pass before
            acc[0].copy_(self.carry_fw[0])
            status[0].copy_(self.carry_fw[1])
            accumulate_flow(flow_fw, flow_bw, acc, status, start=0, n_steps=n, **kw)
            pass_rows.append((first + 1, first + n + 1))
        elif first <= Kl <= first + n:  # the pass holding K_(m-1): side A from it
            acc[Kl - first].zero_()
            status[Kl - first].zero_()
            accumulate_flow(flow_fw, flow_bw, acc, status, start=Kl - first, n_steps=n, **kw)
            pass_rows.append((Kl, first + n + 1))
        if any(a < b for a, b in pass_rows):
            self.carry_fw = (acc[n].clone(), status[n].clone()) if pass_rows[-1][1] == first + n + 1 else None
            labels, st = self._one_sided(first, n, acc, status)
            chunks += [(a, labels[a - first:b - first], st[a - first:b - first]) for a, b in pass_rows if a < b]
        p = max(first, self.next_pair)  # the interval store: pairs K_0 .. K_(m-1) - 1
        while p < min(first + n, Kl):
            Ki, Kj = self.K[self.cur], self.K[self.cur + 1]
            end = min(first + n, Kj)
            self.store[0, p - Ki:end - Ki].copy_(flow_fw[p - first:end - first])
            self.store[1, p - Ki:end - Ki].copy_(flow_bw[p - first:end - first])
            p = end
            if end == Kj:
                chunks.append(self._interval(Ki, Kj))
                self.cur += 1
        self.next_pair = p
        return sorted(chunks, key=lambda c: c[0])

    def _interval(self, Ki, Kj):
        """Both chains over the stored flows of pairs Ki .. Kj - 1 and the labels of frames Ki .. Kj - 1."""
        from networks.utils import accumulate_flow, accumulate_flow_backward, propagate_labels_keys
        L = Kj - Ki
        fw, bw = self.store[0, :L], self.store[1, :L]
        self.ia[:, 0].zero_()  # side A of frames Ki .. Kj - 1 in rows 0 .. L - 1
        self.ist[:, 0].zero_()
        self.ia[1, L].zero_()  # side B of frames Ki + 1 .. Kj in rows 1 .. L
        self.ist[1, L].zero_()
        if L > 1:
            accumulate_flow(fw, bw, self.ia[0, :L], self.ist[0, :L], start=0, n_steps=L - 1, **self.kw)
            accumulate_flow_backward(fw[1:], bw[1:], self.ia[1, 1:L + 1], self.ist[1, 1:L + 1], start=L - 1,
                                     **self.kw)
        rows = keyframe_rows(self.F, self.K, self.cuts)[Ki:Kj]
        labels, st = propagate_labels_keys(self.ia[0, :L], self.ist[0, :L], self.ia[1, :L], self.ist[1, :L],
                                           self.keys, rows)
        return Ki, labels, st

    def reverse(self, ps, flow_fw, flow_bw):
        from networks.utils import accumulate_flow_backward
        n = sum(k is not None for k in ps.pairs)
        first = ps.frames[0]
        acc, status = self.acc[:n + 1], self.status[:n + 1]
        acc[n].copy_(self.carry_bw[0])  # the last row is the first row of the pass after this one
        status[n].copy_(self.carry_bw[1])
        accumulate_flow_backward(flow_fw, flow_bw, acc, status, start=n, n_steps=n, **self.kw)
        self.carry_bw = (acc[0].clone(), status[0].clone())
        labels, st = self._one_sided(first, n, acc, status)
        return [(first, labels[:n], st[:n])]


def _read_keys(labels, frame, F, what):
    """video_propagate's keys: (K, [m,Hs,Ws] uint8 array, palette of the first PNG or None)."""
    several = not isinstance(frame, (int, np.integer))
    K = check_keyframes(frame, F, what)
    items = list(labels) if several and not isinstance(labels, (str, os.PathLike)) else [labels]
    if len(items) != len(K):
        raise ValueError(f"{what}: {len(items)} key label maps for {len(K)} key frames")
    keys, palette = [], None
    for i, item in enumerate(items):
        if isinstance(item, (str, os.PathLike)):
            key, pal = read_labels(item)
            palette = pal if i == 0 else palette
        else:
            key = np.asarray(item)
            if key.ndim != 2 or key.dtype != np.uint8:
                raise ValueError(f"{what}: labels must be PNG paths or [Hs,Ws] uint8 maps (got {key.shape} {key.dtype})")
        if keys and key.shape != keys[0].shape:
            raise ValueError(f"{what}: the key label maps differ in size ({keys[0].shape} and {key.shape})")
        keys.append(key)
    return K, np.stack(keys), palette


def video_propagate(model, frames, out, labels, frame=0, batch=8, workers=4, scene_cut=None):
    """Keyframe label propagation through a video of any length with a loaded networks.RAFT.RAFT model: the label map of
    frame `frame` (`labels`: a palette or grey PNG path, or an [Hs,Ws] uint8 array at the frames' size) carried to every
    frame (a directory's sorted *.png / *.jpg, or a list of paths, all of one size).  Writes <out>/label_<i:06d>.png for
    every frame, in the key's palette when it has one and grey otherwise.  Returns (the paths, the [Hs,Ws] uint8 status
    of the last frame: 0 consistent at every step back to the key frame, 1 occluded at some step, 2 entered through the
    frame edge).

    Passes come from interp_schedule(): forward_sequence_bidirectional(check=False) on batch + 1 frames.  The forward
    sweep starts at the pass holding `frame`: a zero row there, one rb_flow_accumulate launch to the pass's last frame and
    one rb_flow_accumulate_backward launch to its first; each later pass starts from the last row of the one before.  A
    reverse sweep then runs the passes before that one again, last to first, each with one rb_flow_accumulate_backward
    launch from the first row of the pass after it (as video_track(backward=True) does), so frame = 0 costs nothing
    more.  Every row's labels come from one rb_labels_propagate launch at the frames' own size.  The files are the same
    bytes for every batch and workers value, and equal RAFT.propagate on the whole clip.  Frames go in RGB with
    model.upstream and BGR otherwise, like the CLI.

    Several keyframes: `labels` a list of PNG paths or maps (or an [m,Hs,Ws] array) and `frame` the strictly increasing
    list of their frames; the files are in the first PNG's palette.  Each frame votes between the nearest keyframes
    before and after it (RAFT.propagate with a list; KeyframeSweep streams it).  The flows of one keyframe interval are
    kept on the GPU until the next key is reached, so memory is bounded by the longest interval, not the clip: 16 B per
    network pixel per pair plus 18 B per pixel per frame, about 15 MB per interval frame at 432x1024 (by arithmetic).

    scene_cut (a threshold in [0, 1]) scores each pass's decoded frames on the GPU (networks.utils.scene_cut_scores; the
    reverse sweep scores its own passes), and no frame takes labels from a keyframe across a cut pair: the files are
    RAFT.propagate(..., cuts=<the cuts found>)'s, status 3 (label 0) where no keyframe reaches a frame.  It then returns
    (paths, last status, cuts), cuts the increasing cut pairs."""
    paths = list_frames(frames)
    F = len(paths)
    K, keys_np, palette = _read_keys(labels, frame, F, "video_propagate")
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    batch, workers = int(batch), _workers(workers)
    passes = interp_schedule(F, batch)
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device
    names = [os.path.join(out, f"label_{i:06d}.png") for i in range(F)]
    cuts, last = [], None
    with torch.cuda.device(dev):
        keys = torch.from_numpy(np.ascontiguousarray(keys_np)).to(dev)
    sweep = KeyframeSweep(engine, keys, K, F, batch, cuts, simple=len(K) == 1 and thr is None)
    j0 = sweep.first_pass(len(passes))
    rows = batch + 1 + sweep.L  # the most frames one pass completes

    def write(slot, spans):  # writer thread: the label maps a pass completed, once its copies have landed
        if slot is None:
            return
        slot.event.synchronize()
        r = 0
        for a, n in spans:
            for f in range(a, a + n):
                write_labels(names[f], slot.labels[r].numpy(), palette)
                r += 1

    def run(sweep_passes, step):
        nonlocal last
        upload = _Upload(dev)
        with _Pipeline(paths, sweep_passes, rgb, batch, workers, dev) as pipe:
            for j, ps, imgs, src in pipe:
                if j == 0 and tuple(src.shape[1:3]) != keys_np.shape[1:]:
                    raise ValueError(f"video_propagate: the key is {keys_np.shape[1]}x{keys_np.shape[2]}, the frames "
                                     f"{src.shape[1]}x{src.shape[2]}")
                if thr is not None:  # score the pass on the GPU; the engine then reads the frames from there too
                    src, cut = upload(src, ps.pairs, thr)
                    cuts.extend(cut)
                    cuts.sort()
                flow_fw, flow_bw, _, _ = engine.forward_sequence_bidirectional(src, check=False)
                chunks = step(ps, flow_fw, flow_bw)
                spans = [(a, len(lab)) for a, lab, _ in chunks]
                for a, lab, st in chunks:
                    if a + len(lab) == F:
                        last = st[-1].clone()
                labels_out = (None if not chunks else chunks[0][1] if len(chunks) == 1
                              else torch.cat([lab for _, lab, _ in chunks]))
                pipe.emit(partial(write, spans=spans), rows, labels=labels_out)

    run(passes[j0:], sweep.forward)
    if j0 > 0:
        run(passes[:j0][::-1], sweep.reverse)
    last = last.cpu().numpy()
    return (names, last) if thr is None else (names, last, cuts)


def video_stabilize(model, frames, out, sigma, batch=8, workers=4, scene_cut=None, max_zoom=None, fill=False,
                    window=None):
    """Video stabilization of a clip of any length with a loaded networks.RAFT.RAFT model: the frames (a directory's
    sorted *.png / *.jpg, or a list of paths, all of one size) written as <out>/frame_<i:06d>.png at their own size with
    the camera's shake removed, equal byte for byte to RAFT.stabilize on the whole clip.  Two sweeps:

    - motion: interp_schedule()'s passes of forward_sequence_bidirectional (with the occlusion check) and one
      rb_global_motion launch each (networks.utils.global_motion); only the F x 4 motion parameters stay, so host and
      device memory do not grow with F.  scene_cut (a threshold in [0, 1]) scores each pass's decoded frames on the GPU
      (networks.utils.scene_cut_scores), and a pair above it is a cut: its motion is the identity and the camera path
      restarts after it.
    - warp: the host path of raft_b200.stabilize (sigma frames, max_zoom, default DEFAULT_MAX_ZOOM), then every frame
      decoded and uploaded again, batch at a time, and warped at its own size (networks.utils.warp_frames).

    Also writes <out>/transforms.npy [F,2,3] fp64 (RAFT.stabilize's transforms) and prints the zoom of every shot, the
    cuts and the number of unreliable pairs.  Frames go in RGB with model.upstream and BGR otherwise, like the CLI; the
    files are BGR and do not depend on batch or workers.  Returns (paths, info), info a dict of "zooms" (per shot),
    "capped" (the shots whose zoom hit max_zoom), "cuts" and "unreliable" (pair indices).

    fill=True writes full-frame output, the bytes of RAFT.stabilize(fill=True) (max_zoom then defaults to 1.0; window
    to raft_b200.inpaint.DEFAULT_WINDOW): the motion sweep and the transforms as above, then the canvas margin of the
    whole clip (raft_b200.stabilize.fill_margin) and a fill sweep instead of the warp sweep -- interp_schedule()'s passes
    again with check=False, each pass's flows extended past the frame edge as one batch (networks.utils.extend_flows).
    A window of the clip stays on the GPU: the frames and extended flows from t - window to the newest, at most
    2 window + batch + 2 frames of 3 Hs Ws + 16 Hc Wc bytes each (Hc x Wc the canvas).  For 1080x1920 frames and
    432x1024 flows that is 17.3 MB per frame at a margin of 12.5 % of the grid per side and 34.5 MB at the cap (half the
    grid per side), by arithmetic: 0.52 GB and 1.04 GB at window 10, batch 8.  Frame t is filled (raft_b200.stabilize.
    fill_warp over inpaint_rows(F, window, cuts)) and written once the pairs up to min(t + window, F - 1) have run.  It
    also prints the pixel counts of status 1 / 2 / 3, and info gains "counts" (pixels filled from both sides, one side,
    spatially) and "margin" ((my, mx) network pixels)."""
    from networks.utils import global_motion, warp_frames
    from .inpaint import DEFAULT_WINDOW, check_window
    from .stabilize import DEFAULT_MAX_ZOOM, camera_transforms, check_max_zoom, check_sigma

    paths = list_frames(frames)
    sigma = check_sigma(sigma, "video_stabilize")
    max_zoom = check_max_zoom((1.0 if fill else DEFAULT_MAX_ZOOM) if max_zoom is None else max_zoom, "video_stabilize")
    if window is not None and not fill:
        raise ValueError("video_stabilize: window is the reach of fill=True")
    if fill:
        window = check_window(DEFAULT_WINDOW if window is None else window, "video_stabilize")
    batch, workers = int(batch), _workers(workers)
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    F = len(paths)
    passes = interp_schedule(F, batch)
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device
    motions = np.zeros((F - 1, 4))
    reliable = np.ones(F - 1, dtype=bool)
    hw = None

    def keep(slot, pairs):  # writer thread: the motions of one pass, once its copies have landed
        slot.event.synchronize()
        for r, k in pairs:
            motions[k] = slot.params[r].numpy()
            reliable[k] = bool(slot.reliable[r])

    upload, cuts = _Upload(dev), []
    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for j, ps, imgs, src in pipe:
            hw = tuple(src.shape[1:3])
            if thr is not None:  # score the pass on the GPU; the engine then reads the frames from there too
                src, cut = upload(src, ps.pairs, thr)
                cuts += cut
            flow_fw, _, occ_fw, _ = engine.forward_sequence_bidirectional(src, check=True)
            params, _, rel = global_motion(flow_fw, occ_fw, hw, flow_scale=engine.flow_scale)
            pipe.emit(partial(keep, pairs=[(r, k) for r, k in enumerate(ps.pairs) if k is not None]), batch,
                      params=params, reliable=rel)
    motions[cuts] = (1.0, 0.0, 0.0, 0.0)
    transforms, zooms, capped = camera_transforms(motions, hw, sigma, cuts, max_zoom)
    np.save(os.path.join(out, "transforms.npy"), transforms)

    names = [os.path.join(out, f"frame_{i:06d}.png") for i in range(F)]
    A = torch.from_numpy(transforms).to(dev)
    if fill:
        counts, margin = _stabilize_fill_sweep(engine, paths, passes, rgb, batch, workers, hw, motions, transforms, A,
                                               sorted(cuts), window, names)
    else:
        chunks = [Pass(False, list(range(i, min(i + batch, F))), []) for i in range(0, F, batch)]
        write, upload = _FrameWriter(names, rgb), _Upload(dev)
        with _Pipeline(paths, chunks, rgb, batch, workers, dev) as pipe:
            for j, ps, imgs, src in pipe:
                n, first = len(ps.frames), ps.frames[0]
                res = warp_frames(upload(src, ps.pairs)[0], A[first:first + n])
                pipe.emit(partial(write, first=first, n=n), batch, frames=res)
    unreliable = [k for k in np.flatnonzero(~reliable).tolist() if k not in cuts]
    print("stabilize: zoom per shot " + " ".join(f"{z:.4f}" for z in zooms)
          + (f" (shots {' '.join(map(str, capped))} capped at {max_zoom:g})" if capped else ""))
    print_cuts(cuts)
    print(f"unreliable pairs (identity motion): {len(unreliable)}")
    info = {"zooms": zooms, "capped": capped, "cuts": cuts, "unreliable": unreliable}
    if fill:
        print(f"stabilize fill: pixels filled from both sides {counts[1]}, from one side {counts[2]}, spatially "
              f"{counts[3]}")
        info.update(counts=counts[1:].tolist(), margin=margin)
    return names, info


def _status_counts(slot, n):
    """The [4] int64 pixel counts of each status in the first n rows of slot.status (a _FrameWriter tally)."""
    return np.bincount(slot.status[:n].numpy().reshape(-1), minlength=4)[:4]


def _stabilize_fill_sweep(engine, paths, passes, rgb, batch, workers, hw, motions, transforms, A, cuts, window, names):
    """video_stabilize's fill sweep: writes every frame, full-frame stabilized, as names[i].  Returns (counts [4] int64
    of each status, margin)."""
    from networks.utils import extend_flows
    from .inpaint import inpaint_rows
    from .stabilize import fill_margin, fill_warp
    F, dev = len(paths), engine.device
    win, upload, write = _Window(F, window, batch, dev), _Upload(dev), _FrameWriter(names, rgb, _status_counts)
    table = inpaint_rows(F, window, cuts)
    margin = None
    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for j, ps, imgs, src in pipe:
            src, _ = upload(src, ps.pairs)
            flow_fw, flow_bw, _, _ = engine.forward_sequence_bidirectional(src, check=False)
            n = sum(k is not None for k in ps.pairs)
            first = ps.frames[0]
            if margin is None:
                net_hw = tuple(flow_fw.shape[1:3])
                margin = fill_margin(transforms, hw, net_hw)
                canvas = (net_hw[0] + 2 * margin[0], net_hw[1] + 2 * margin[1], 2)
            s = win.alloc(frames=(hw + (3,), torch.uint8), fw=(canvas, torch.float32), bw=(canvas, torch.float32))
            new = win.admit(first + n)
            r = win.row(first)
            s["frames"][new].copy_(src[new.start - r:n + 1])
            # copies out of the engine's views, which the next pass overwrites
            fw, bw = extend_flows(flow_fw[:n], flow_bw[:n], motions[first:first + n], hw, margin, engine.flow_scale)
            s["fw"][r:r + n].copy_(fw)
            s["bw"][r:r + n].copy_(bw)
            t0, m, rows = win.finish(first + n, table)  # pairs 0 .. first + n - 1 have run
            res = None
            if m:
                res = fill_warp(win.kept("frames"), win.kept_pairs("fw"), win.kept_pairs("bw"), net_hw, margin,
                                A[t0:t0 + m], rows, engine.flow_scale)
            pipe.emit(partial(write, first=t0, n=m), win.cap, frames=None if res is None else res[0],
                      status=None if res is None else res[1])
    return write.total, margin


def list_masks(masks, F, what="video_inpaint"):
    """The mask paths of video_inpaint: a directory's *.png files in sorted order (one per frame), or a list of paths.
    A count other than F raises ValueError."""
    if isinstance(masks, (str, os.PathLike)):
        root = os.fspath(masks)
        if not os.path.isdir(root):
            raise FileNotFoundError(f"{what}: no directory {root}")
        paths = sorted(glob.glob(os.path.join(root, "*.png")))
    else:
        paths = [os.fspath(p) for p in masks]
    if len(paths) != F:
        raise ValueError(f"{what}: {len(paths)} masks for {F} frames: one mask PNG per frame")
    return paths


def video_inpaint(model, frames, out, masks, window=None, dilate=None, labels=None, batch=8, workers=4, scene_cut=None):
    """Object removal from a clip of any length with a loaded networks.RAFT.RAFT model, in one sweep: the frames (a
    directory's sorted *.png / *.jpg, or a list of paths, all of one size) with the pixels of their masks (a directory
    of one palette or grey PNG per frame in sorted order, read_labels(), at the frames' size; non-zero values are
    removed, or with labels those labels) filled from the nearest frames that see behind them, written as
    <out>/frame_<i:06d>.png, equal byte for byte to RAFT.inpaint on the whole clip for every batch and workers value.

    Passes come from interp_schedule(): forward_sequence_bidirectional(check=False) on batch + 1 frames, the pass's
    masks read on the host and turned into holes on the GPU (rb_inpaint_masks), and its flows completed inside the holes
    as one rb_masked_fill batch.  A window of the clip stays on the GPU: the uploaded frames, their holes and the
    completed flows of the frames from t - window to the newest.  Frame t is filled (rb_inpaint_propagate, the spatial
    fill and the rounding) and written once the pairs up to min(t + window, F - 1) have run, and the frames no later
    frame reaches are dropped, so memory is bounded by the window, not the clip: 4 Hs Ws bytes (frame and hole) plus
    Hn Wn (grid hole) plus 16 Hn Wn (the two completed flows) per kept frame, at most 2 window + batch + 2 of them --
    about 15.8 MB per frame for 1080x1920 frames and 432x1024 flows (by arithmetic), 0.47 GB at window 10, batch 8.
    scene_cut (a threshold in [0, 1]) scores each pass's frames on the GPU (networks.utils.scene_cut_scores); no side
    crosses a cut pair.  Prints the pixel counts of status 1 / 2 / 3 and the cuts.  Frames go in RGB with model.upstream
    and BGR otherwise, like the CLI; the files are BGR.  Returns (paths, info), info a dict of "counts" (pixels filled
    from both sides, one side, spatially) and "cuts"."""
    from networks.utils import inpaint_masks
    from .inpaint import (DEFAULT_DILATE, DEFAULT_WINDOW, check_dilate, check_window, complete_flows, fill_frames,
                          inpaint_rows, selection_table)

    paths = list_frames(frames)
    F = len(paths)
    mask_paths = list_masks(masks, F)
    window = check_window(DEFAULT_WINDOW if window is None else window, "video_inpaint")
    dilate = check_dilate(DEFAULT_DILATE if dilate is None else dilate, "video_inpaint")
    selection_table(labels, "video_inpaint")
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    batch, workers = int(batch), _workers(workers)
    passes = interp_schedule(F, batch)
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device
    names = [os.path.join(out, f"frame_{i:06d}.png") for i in range(F)]
    win, upload, write = _Window(F, window, batch, dev), _Upload(dev), _FrameWriter(names, rgb, _status_counts)
    cuts = []
    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for j, ps, imgs, src in pipe:
            Hs, Ws = src.shape[1:3]
            src, cut = upload(src, ps.pairs, thr)
            cuts += cut
            flow_fw, flow_bw, _, _ = engine.forward_sequence_bidirectional(src, check=False)
            n = sum(k is not None for k in ps.pairs)
            first = ps.frames[0]
            Hn, Wn = flow_fw.shape[1:3]
            s = win.alloc(frames=((Hs, Ws, 3), torch.uint8), hole=((Hs, Ws), torch.uint8),
                          hole_net=((Hn, Wn), torch.uint8), fw=((Hn, Wn, 2), torch.float32),
                          bw=((Hn, Wn, 2), torch.float32))
            new = win.admit(first + n)
            r = win.row(first)
            lab = []
            for i in range(first + new.start - r, first + n + 1):
                mask, _ = read_labels(mask_paths[i])
                if mask.shape != (Hs, Ws):
                    raise ValueError(f"video_inpaint: {mask_paths[i]} is {mask.shape[0]}x{mask.shape[1]}, the frames "
                                     f"{Hs}x{Ws}")
                lab.append(mask)
            s["frames"][new].copy_(src[new.start - r:n + 1])
            h, hn = inpaint_masks(torch.from_numpy(np.stack(lab)).to(dev), (Hn, Wn), dilate, labels)
            s["hole"][new].copy_(h)
            s["hole_net"][new].copy_(hn)
            fw, bw = complete_flows(flow_fw[:n], flow_bw[:n], s["hole_net"][r:r + n + 1])
            s["fw"][r:r + n].copy_(fw)
            s["bw"][r:r + n].copy_(bw)
            t0, m, rows = win.finish(first + n, inpaint_rows(F, window, sorted(cuts)))  # pairs .. first + n - 1 ran
            res = None
            if m:
                res = fill_frames(win.kept("frames"), win.kept("hole"), win.kept_pairs("fw"), win.kept_pairs("bw"),
                                  rows, engine.flow_scale)
            pipe.emit(partial(write, first=t0, n=m), win.cap, frames=None if res is None else res[0],
                      status=None if res is None else res[1])
    cuts, counts = sorted(cuts), write.total
    print(f"inpaint: pixels filled from both sides {counts[1]}, from one side {counts[2]}, spatially {counts[3]}")
    print_cuts(cuts)
    return names, {"counts": counts[1:].tolist(), "cuts": cuts}


def video_denoise(model, frames, out, sigma, window=None, batch=8, workers=4, scene_cut=None):
    """Video denoising of a clip of any length with a loaded networks.RAFT.RAFT model, in one sweep: the frames (a
    directory's sorted *.png / *.jpg, or a list of paths, all of one size) with additive noise of standard deviation
    sigma grey levels removed (sigma="auto": estimated from frames 0 .. 7, raft_b200.denoise.estimate_sigma), written as
    <out>/frame_<i:06d>.png, equal byte for byte to RAFT.denoise on the whole clip for every batch and workers value.

    Passes come from interp_schedule(): forward_sequence_bidirectional(check=False) on batch + 1 frames.  A window of the
    clip stays on the GPU: the uploaded frames and the flows of the frames from t - window to the newest.  Frame t is
    merged (rb_denoise_merge) and written once the pairs up to min(t + window, F - 1) have run, and the frames no later
    frame reaches are dropped, so memory is bounded by the window, not the clip: 3 Hs Ws bytes (the frame) plus 16 Hn Wn
    (the two flows) per kept frame, at most 2 window + batch + 2 of them -- about 13.3 MB per frame for 1080x1920 frames
    and 432x1024 flows (by arithmetic), 0.21 GB at window 3, batch 8.  scene_cut (a threshold in [0, 1]) scores each
    pass's frames on the GPU (networks.utils.scene_cut_scores); no side crosses a cut pair.  Prints the sigma used, the
    mean support (matched frames per pixel) and the cuts.  Frames go in RGB with model.upstream and BGR otherwise, like
    the CLI; the files are BGR.  Returns (paths, info), info a dict of "sigma", "support" (the mean) and "cuts"."""
    from .denoise import DEFAULT_WINDOW, ESTIMATE_FRAMES, check_sigma, check_window, estimate_sigma, merge_frames
    from .inpaint import inpaint_rows

    paths = list_frames(frames)
    F = len(paths)
    sigma = check_sigma(sigma, "video_denoise")
    window = check_window(DEFAULT_WINDOW if window is None else window, "video_denoise")
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    batch, workers = int(batch), _workers(workers)
    passes = interp_schedule(F, batch)
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device
    if sigma == "auto":
        with torch.cuda.device(dev):
            sigma = estimate_sigma(torch.from_numpy(np.stack([_imread(p, rgb) for p in paths[:ESTIMATE_FRAMES]])).to(dev))
    names = [os.path.join(out, f"frame_{i:06d}.png") for i in range(F)]
    win, upload = _Window(F, window, batch, dev), _Upload(dev)
    write = _FrameWriter(names, rgb, lambda slot, n: int(slot.support[:n].numpy().sum(dtype=np.int64)))
    cuts = []
    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for j, ps, imgs, src in pipe:
            Hs, Ws = src.shape[1:3]
            src, cut = upload(src, ps.pairs, thr)
            cuts += cut
            flow_fw, flow_bw, _, _ = engine.forward_sequence_bidirectional(src, check=False)
            n = sum(k is not None for k in ps.pairs)
            first = ps.frames[0]
            Hn, Wn = flow_fw.shape[1:3]
            s = win.alloc(frames=((Hs, Ws, 3), torch.uint8), fw=((Hn, Wn, 2), torch.float32),
                          bw=((Hn, Wn, 2), torch.float32))
            new = win.admit(first + n)
            r = win.row(first)
            s["frames"][new].copy_(src[new.start - r:n + 1])
            s["fw"][r:r + n].copy_(flow_fw[:n])
            s["bw"][r:r + n].copy_(flow_bw[:n])
            t0, m, rows = win.finish(first + n, inpaint_rows(F, window, sorted(cuts)))  # pairs .. first + n - 1 ran
            res = None
            if m:
                res = merge_frames(win.kept("frames"), win.kept_pairs("fw"), win.kept_pairs("bw"), rows, sigma,
                                   engine.flow_scale)
            pipe.emit(partial(write, first=t0, n=m), win.cap, frames=None if res is None else res[0],
                      support=None if res is None else res[1])
    cuts = sorted(cuts)
    mean = write.total / (F * Hs * Ws)
    print(f"denoise: sigma {sigma:.4g}, mean support {mean:.3f} frames")
    print_cuts(cuts)
    return names, {"sigma": float(sigma), "support": mean, "cuts": cuts}


MASK_PALETTE = [[0, 0, 0], [128, 0, 0]]  # background, moving: DAVIS's colours for labels 0 and 1


def video_segment_motion(model, frames, out, window=None, tau=None, batch=8, workers=4, scene_cut=None):
    """Motion segmentation of a clip of any length with a loaded networks.RAFT.RAFT model, in one sweep: the frames (a
    directory's sorted *.png / *.jpg, or a list of paths, all of one size) segmented into the pixels that move on their
    own (1) and the rest (0), written as palette PNGs <out>/mask_<i:06d>.png (write_labels; --inpaint reads them as they
    are) and the forward pairs' homographies in the frames' own pixels as <out>/homographies.npy [F-1,3,3] fp64, equal
    byte for byte to RAFT.segment_motion on the whole clip for every batch and workers value.

    Passes come from interp_schedule(): forward_sequence_bidirectional(check=True) on batch + 1 frames, the pass's 2n
    fields fitted as one batch (global_motion, rb_homography_motion: a field's bits do not depend on the batch) and one
    rb_motion_evidence launch on them.  The frame two passes share gets its forward field from the later pass and its
    backward field from the earlier one: its (N, C) is the sum of the two launches' rows, the same bits as one launch,
    since each launch starts from +0 and fp32 addition commutes.  A window of the clip stays on the GPU: the evidence
    and the flows of the frames from t - window to the newest.  Frame t is segmented (rb_motion_segment) and written
    once the evidence of frames up to min(t + window, F - 1) is complete, and the frames no later frame reaches are
    dropped, so memory is bounded by the window, not the clip: 24 Hn Wn bytes per kept frame (evidence and two flows),
    at most 2 window + batch + 2 of them.  scene_cut (a threshold in [0, 1]) scores each pass's frames on the GPU
    (networks.utils.scene_cut_scores); a cut pair adds no evidence and no chain crosses it.  Prints the pairs with an
    unreliable similarity (a field flagged 2) and with a singular fit (a field flagged 1), the mean moving fraction and
    the cuts.  Returns (paths, info), info a dict of "unreliable", "fallback", "moving" and "cuts"."""
    from networks.utils import motion_evidence
    from .motionseg import (DEFAULT_WINDOW, SINGULAR, TAU, UNRELIABLE, check_tau, check_window, cut_flags, fit_fields,
                            segment_frames, segment_rows, to_pixels)

    paths = list_frames(frames)
    F = len(paths)
    if F < 2:
        raise ValueError(f"video_segment_motion: motion needs at least 2 frames (got {F})")
    window = check_window(DEFAULT_WINDOW if window is None else window, "video_segment_motion")
    tau = check_tau(TAU if tau is None else tau, "video_segment_motion")
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    batch, workers = int(batch), _workers(workers)
    passes = interp_schedule(F, batch)
    out = os.fspath(out)
    os.makedirs(out, exist_ok=True)
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device
    names = [os.path.join(out, f"mask_{i:06d}.png") for i in range(F)]
    moving, lock = [0], threading.Lock()
    homs, field_flags = np.zeros((F - 1, 3, 3)), np.zeros((2, F - 1), np.uint8)
    win, upload, cuts = _Window(F, window, batch, dev), _Upload(dev), []

    def write(slot, first, n):  # writer thread: the masks of one pass, once its copies have landed
        if slot is None:
            return
        slot.event.synchronize()
        for r in range(n):
            write_labels(names[first + r], slot.mask[r].numpy(), MASK_PALETTE)
        s = int(slot.mask[:n].numpy().sum(dtype=np.int64))
        with lock:
            moving[0] += s

    with _Pipeline(paths, passes, rgb, batch, workers, dev) as pipe:
        for j, ps, imgs, src in pipe:
            Hs, Ws = src.shape[1:3]
            src, cut = upload(src, ps.pairs, thr)
            cuts += cut
            flow_fw, flow_bw, occ_fw, occ_bw = engine.forward_sequence_bidirectional(src, check=True)
            n = sum(k is not None for k in ps.pairs)
            first = ps.frames[0]
            Hn, Wn = flow_fw.shape[1:3]
            s = win.alloc(ev=((Hn, Wn, 2), torch.float32), fw=((Hn, Wn, 2), torch.float32),
                          bw=((Hn, Wn, 2), torch.float32))
            fw, bw, ofw, obw = flow_fw[:n], flow_bw[:n], occ_fw[:n], occ_bw[:n]
            H, flags = fit_fields(torch.cat([fw, bw]), torch.cat([ofw, obw]), (Hs, Ws), engine.flow_scale)
            ev = motion_evidence(fw, bw, ofw, obw, H, flags, (Hs, Ws), cut_flags(cuts, range(first, first + n), dev),
                                 engine.flow_scale, tau)
            homs[first:first + n] = to_pixels(H[:n].cpu().numpy(), (Hs, Ws))
            field_flags[:, first:first + n] = flags.cpu().numpy().reshape(2, n)
            new = win.admit(first + n)
            r = win.row(first)
            k0 = new.start - r  # 1 when frame `first` holds the previous pass's half of its evidence
            if k0:
                s["ev"][r].add_(ev[0])
            s["ev"][new].copy_(ev[k0:])
            s["fw"][r:r + n].copy_(fw)
            s["bw"][r:r + n].copy_(bw)
            ran = first + n  # pairs 0 .. ran - 1 have run: the evidence of frames < ran is complete (all at the end)
            t0, m, rows = win.finish(F - 1 if ran == F - 1 else ran - 1, segment_rows(F, window, sorted(cuts)))
            res = None
            if m:
                res = segment_frames(win.kept("ev"), win.kept_pairs("fw"), win.kept_pairs("bw"), (Hs, Ws), rows,
                                     engine.flow_scale)
            pipe.emit(partial(write, first=t0, n=m), win.cap, mask=None if res is None else res[0])
    cuts = sorted(cuts)
    np.save(os.path.join(out, "homographies.npy"), homs)
    unreliable = int((field_flags == UNRELIABLE).any(0).sum())
    fallback = int((field_flags == SINGULAR).any(0).sum())
    frac = moving[0] / (F * Hs * Ws)
    print(f"segment motion: {unreliable} pairs with an unreliable similarity, {fallback} with a singular homography "
          f"fit, moving fraction {frac:.4f}")
    print_cuts(cuts)
    return names, {"unreliable": unreliable, "fallback": fallback, "moving": frac, "cuts": cuts}


def _aligned(frames, other, what):
    """The frame paths of frames and of other, which must hold as many frames; anything else raises ValueError."""
    paths, opaths = list_frames(frames), list_frames(other)
    if len(opaths) != len(paths):
        raise ValueError(f"{what}: {len(opaths)} frames in {other!r} for {len(paths)} original frames: the frames must "
                         f"be aligned with the originals")
    if len(paths) < 2:
        raise ValueError(f"{what}: a sequence needs two frames at least (got {len(paths)})")
    return paths, opaths


def _temporal_sweep(model, frames, other, what, batch, workers, scene_cut, strength=None, out=None):
    """The one sweep behind video_consistent (strength given) and video_warp_error: per pass the originals and the other
    frames, one forward_sequence_bidirectional(check=False), and each frame whose pair ran in order; the per-pair
    warping-error sums of the originals, of other and (with strength) of the output stay on the GPU until the end."""
    from networks.utils import warp_error
    from .engine import FB_ALPHA1, FB_ALPHA2
    from .temporal import check_strength, consistent_frame

    paths, opaths = _aligned(frames, other, what)
    F = len(paths)
    if strength is not None:
        strength = check_strength(strength, what)
    thr = None if scene_cut is None else check_scene_cut(scene_cut)
    batch, workers = int(batch), _workers(workers)
    passes = interp_schedule(F, batch)
    names = None
    if out is not None:
        out = os.fspath(out)
        os.makedirs(out, exist_ok=True)
        names = [os.path.join(out, f"frame_{i:06d}.png") for i in range(F)]
    engine = model.engine()
    rgb = bool(model.upstream)
    dev = engine.device
    cuts = []
    prev_out = None  # O of the frame before the pass's next frame
    upload_I, upload_P, write = _Upload(dev), _Upload(dev), _FrameWriter(names, rgb)
    sums = torch.zeros(3, F - 1, 2, dtype=torch.float64, device=dev)
    counts = torch.zeros(4, dtype=torch.int64, device=dev)
    with _Pipeline(paths, passes, rgb, batch, workers, dev, extra=opaths) as pipe:
        for j, ps, imgs, src in pipe:
            I_dev, cut = upload_I(src, ps.pairs, thr)
            P_dev, _ = upload_P(pipe.extra, ps.pairs)
            cuts += cut
            n = sum(k is not None for k in ps.pairs)
            first = ps.frames[0]
            fw, bw, _, _ = engine.forward_sequence_bidirectional(I_dev, check=False)
            fw, bw = fw[:n], bw[:n]
            sums[0, first:first + n] = warp_error(I_dev[:n + 1], fw, bw, engine.flow_scale, FB_ALPHA1, FB_ALPHA2)
            sums[1, first:first + n] = warp_error(P_dev[:n + 1], fw, bw, engine.flow_scale, FB_ALPHA1, FB_ALPHA2)
            res = None
            if strength is not None:
                rows = list(range(0 if first == 0 else 1, n + 1))  # the pass's frames whose pair has run
                O = torch.empty((n + 1,) + tuple(src.shape[1:]), dtype=torch.uint8, device=dev)
                if first > 0:
                    O[0] = prev_out
                for r in rows:
                    t = first + r
                    restart = t == 0 or (t - 1) in cuts
                    O[r], st = consistent_frame(I_dev[r], None if restart else I_dev[r - 1], P_dev[r], O[max(r - 1, 0)],
                                                fw[max(r - 1, 0)], bw[max(r - 1, 0)], strength, engine.flow_scale)
                    counts += torch.bincount(st.reshape(-1), minlength=4)
                sums[2, first:first + n] = warp_error(O, fw, bw, engine.flow_scale, FB_ALPHA1, FB_ALPHA2)
                prev_out = O[n].clone()
                res = O[rows[0]:]
            pipe.emit(partial(write, first=first + (0 if first == 0 else 1), n=0 if res is None else len(res)),
                      frames=res)
    from .temporal import pair_errors
    cuts = sorted(cuts)
    s = sums.cpu().numpy()
    info = {"cuts": cuts}
    for k, name in enumerate(("original", "input", "output")[:3 if strength is not None else 2]):
        e, per, excluded = pair_errors(s[k], cuts)
        info[name] = {"E_warp": e, "E_pair": per.tolist(), "excluded": excluded}
    if strength is not None:
        info["status"] = counts.cpu().tolist()
    return names, info


def video_consistent(model, frames, processed, out, strength, batch=8, workers=4, scene_cut=None):
    """Temporal consistency of a processed clip of any length with a loaded networks.RAFT.RAFT model, in one sweep:
    processed (a directory's sorted *.png / *.jpg, or a list of paths) holds per-frame processed versions of frames,
    as many and of the same size.  Every output frame is written as <out>/frame_<i:06d>.png, equal byte for byte to
    RAFT.consistent on the whole clip (with the cuts found here) for every batch and workers value.

    Passes come from interp_schedule(): the pass's originals and processed frames, both decoded by the pipeline's
    workers, and one forward_sequence_bidirectional(check=False).  Frames are corrected in order
    (raft_b200.temporal.consistent_frame); only the pass's frames and the output of the frame before it stay on the GPU.
    scene_cut (a threshold in [0, 1]) scores each pass's originals on the GPU; the frame after a cut pair restarts from
    P.  Prints E_warp of the originals, of the processed frames and of the output, all from the sweep's flows, the
    status counts and the cuts.  Frames go in RGB with model.upstream and BGR otherwise, like the CLI; the files are BGR.
    Returns (paths, info), info a dict of "cuts", "status" (counts of statuses 0-3) and per video ("original", "input",
    "output") its "E_warp", "E_pair" (NaN: excluded) and "excluded" pairs."""
    names, info = _temporal_sweep(model, frames, processed, "video_consistent", batch, workers, scene_cut,
                                  strength=strength, out=out)
    print("consistent: E_warp original {:.6g}, processed {:.6g}, output {:.6g}".format(
        info["original"]["E_warp"], info["input"]["E_warp"], info["output"]["E_warp"]))
    print("status: used {} / step failed {} / rejected {} / no previous frame {}".format(*info["status"]))
    print_cuts(info["cuts"])
    return names, info


def video_warp_error(model, frames, video, batch=8, workers=4, scene_cut=None):
    """Lai et al.'s warping error of video (a directory or list of frames aligned with frames: as many, the same size)
    under the flow of frames, in one sweep like video_consistent's without the solve: the same values as
    RAFT.warp_error on the whole clip (with the cuts found here).  Prints E_warp of video and of the originals and the
    cuts.  Returns info: "cuts" and per video ("original", "input") its "E_warp", "E_pair" and "excluded" pairs."""
    _, info = _temporal_sweep(model, frames, video, "video_warp_error", batch, workers, scene_cut)
    print("warp error: E_warp {:.6g} (original frames {:.6g}) over {} pairs, {} excluded".format(
        info["input"]["E_warp"], info["original"]["E_warp"], len(info["input"]["E_pair"]),
        len(info["input"]["excluded"])))
    print_cuts(info["cuts"])
    return info
