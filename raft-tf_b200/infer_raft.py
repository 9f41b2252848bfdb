#!/usr/bin/env python
"""Drop-in for the reference's ``infer_raft.py`` (same flags and defaults, infer_raft.py:51-67) on the
raft_b200 CUDA engine -- no TensorFlow, no tensorpack.

    python infer_raft.py --im1 frame_0016.png --im2 frame_0017.png --load release_weight/raft-things.npz [--small]

Like the reference it decodes BGR with OpenCV, resizes both frames to 432x1024 (bilinear cv2.resize,
dataflow/test_dataflow.py:85-87; here on the GPU from the uint8 frames, bit for bit), scales to [0,1], runs 20 iterations and writes the colour-coded flow
to ``raft_flow_raft-things.png`` in the working directory (regardless of --small, infer_raft.py:44).
Flags the reference parses but ignores (--gpu, -o) are accepted; --data, --out and --batch are read by -m val only.
Extensions: --iters, --keep-size (replicate-pad to a multiple of 8 instead of resizing), --npy, --flo, and
--bidirectional: also the flow im2 -> im1 (``raft_flow_raft-things_bw.png``, ``<npy>_bw.npy``, ``<flo>_bw.flo``) and the
forward-backward occlusion masks ``raft_occ_fw.png`` / ``raft_occ_bw.png`` (0 consistent, 128 occluded, 255 leaves the
frame), from one pass that encodes each frame once, and --interpolate T [T ...]: the frames at times T in [0, 1] between
im1 (0) and im2 (1), written as ``raft_interp_<k>.png`` (k = position in the list), and --native-flow: the written
flow(s) resized back to im1's size with the reference's flow_utils.resize_flow (no effect with --keep-size), and
--mixed_precision (upstream RAFT's spelling): every conv with fp16 operands and fp32 accumulation, the correlation in fp32.

-m val (declared by the reference, implemented here): upstream RAFT's validation on a Sintel or KITTI-2015 training tree,

    python infer_raft.py -m val --dataset sintel --data datasets/Sintel --load raft-things.npz --upstream [--batch 8]

prints upstream's lines (``Validation (clean) EPE: ...``, ``Validation KITTI: <epe>, <f1>``) and writes the aggregates and
per-pair records to ``<--out>/val_<dataset>.json`` (raft_b200.evaluate).  --warm-start runs each Sintel scene as a chain,
every pair after the first warm-started from the previous pair's flow (upstream's forward_interpolate; an extension of
the validation, which upstream runs cold).  --split test writes upstream's test-split submission under --out instead:

    python infer_raft.py -m val --split test --dataset sintel --data datasets/Sintel --out submission --load ... [--warm-start]

Sintel: ``<out>/<dstype>/<scene>/frameNNNN.flo``; KITTI (no --warm-start): ``<out>/<id>_10.png``, 16-bit PNGs
(raft_b200.evaluate.submit).  --dataset vimeo scores frame interpolation on a Vimeo-90K triplet tree instead:

    python infer_raft.py -m val --dataset vimeo --data datasets/vimeo_triplet --load raft-things.npz [--batch 8]

im2 of every triplet in <data>/tri_testlist.txt is interpolated from im1 and im3 at t = 0.5 (20 iterations, like the
reference), and the mean PSNR and SSIM of the 8-bit frames against im2 are printed (``Validation Vimeo-90K: PSNR: ...,
SSIM: ...``) and written with the per-triplet records to ``<--out>/val_vimeo.json`` (no --split test, no --warm-start).
--dataset gopro scores the --shutter conversion's motion blur on GOPRO_Large_all (raft_b200.gopro): every --stride S
(8) frame of each 240 fps sequence is an input, converted at its own rate and size with shutter 360 M / S and density S
(--blur-frames M, 7), each blurred frame scored against np.rint of the mean of its M true frames, the sharp input's
scores beside it; ``Validation GoPro motion blur (...)`` and ``<--out>/val_gopro.json`` (--split test: <data>/test,
otherwise <data>/train):

    python infer_raft.py -m val --dataset gopro --data datasets/GOPRO_Large_all --split test --load raft-things.npz

--dataset tapvid scores point tracking on TAP-Vid instead (raft_b200.tapvid):

    python infer_raft.py -m val --dataset tapvid --data tapvid_davis.pkl --load raft-things.npz [--query-mode strided]

--data is a .pkl file or a directory of .pkl shards; the frames run at 256x256 with 20 iterations, and the mean Average
Jaccard, fraction of points within 1-16 px and occlusion accuracy are printed (``Validation TAP-Vid (first): AJ: ...``)
and written with the per-video records to ``<--out>/val_tapvid.json``.  --query-mode first (default) tracks each point
from its first visible frame, strided from every 5th frame, backward too (no --split test, no --warm-start).

--path DIR (upstream demo.py's flag): the flow of every consecutive pair of DIR's sorted *.png / *.jpg frames, written as
``<--out>/flow_<k:06d>.png`` (and ``flow_<k:06d>.flo`` / ``.npy`` under the directories --flo / --npy name), each frame
encoded once, --batch pairs per pass, coloured on the GPU (raft_b200.video):

    python infer_raft.py --path frames/ --out flows/ --load raft-things.npz [--batch 8 | --warm-start]

--path DIR --interpolate T [T ...] is frame-rate up-conversion instead: DIR's frames and, between every consecutive pair,
the frames at times T (strictly increasing inside (0, 1)), written as one sequence ``<--out>/frame_<n:06d>.png`` (input
frame k is n = k (m + 1) for m times), --batch pairs per pass, each frame encoded once per pass (raft_b200.video):

    python infer_raft.py --path frames/ --out slow/ --interpolate 0.25 0.5 0.75 --load raft-things.npz [--batch 8]

--path DIR --input-fps IN --fps OUT converts DIR's frames from IN to OUT frames per second (OUT > IN; rates such as 24,
59.94 or 24000/1001): output frame n, at input time s = n IN / OUT, is input frame s where s is an integer and otherwise
the frame interpolated at time s - floor(s) between frames floor(s) and floor(s) + 1, written as
``<--out>/frame_<n:06d>.png`` (raft_b200.video):

    python infer_raft.py --path film/ --out tv/ --input-fps 24 --fps 60 --load raft-things.npz [--batch 8]

--shutter ANGLE (with --input-fps/--fps) gives the conversion a camera shutter of ANGLE degrees in (0, 360]: every
output frame is the mean of frames interpolated across its exposure, --shutter-density D (default 16) samples per input
frame interval, and OUT may be at most IN, so 60p -> 24p does not strobe (raft_b200.video.shutter_schedule):

    python infer_raft.py --path clip60/ --out clip24/ --input-fps 60 --fps 24 --shutter 180 --load raft-things.npz

--scene-cut THRESH (with --path and --interpolate, --input-fps/--fps or --warm-start) scores every consecutive pair on the
GPU (one minus the intersection of the frames' colour histograms, in [0, 1]); a pair above THRESH is a scene cut.  There
interpolated frames are copies of the nearer input frame, and warm-started flow restarts cold.  The run prints
``scene cuts: <count> at pairs <k> ...``.  No default: pick the threshold for the footage.

--path DIR --track POINTS.txt tracks points through DIR's frames (one `frame x y` line per point, in the frames' own
pixels; --track-grid STEP [--track-frame K] puts one at every STEP-th pixel of frame K instead): every point is chained
through the consecutive flows with a forward-backward check at each step, and ``<--out>/tracks.npy`` [F,N,2] and
``<--out>/status.npy`` [F,N] (0 consistent, 1 occluded, 2 left the frame, 3 before the query frame) are written;
--track-vis DIR also draws the visible points on every frame (raft_b200.video.video_track):

    python infer_raft.py --path frames/ --out tracks/ --track points.txt --load raft-things.npz [--track-vis vis/]

--track-backward also follows every point back from its frame to frame 0, so the rows before a query frame hold positions
and status 0 / 1 / 2 instead of 3; the flow passes over the frames before the last query frame run a second time, in
reverse order.

--path DIR --propagate KEY.png [--propagate-frame K] carries the label map of frame K (default 0; a palette or 8-bit
grey PNG at the frames' own size: a segmentation mask, a class map) to every frame of DIR: per pixel of every frame, the
displacement back to frame K is composed through the consecutive flows on the GPU and the key's label there taken by a
vote of its four nearest pixels.  ``<--out>/label_<i:06d>.png`` is written for every frame, in the key's palette
(raft_b200.video.video_propagate):

    python infer_raft.py --path frames/ --out labels/ --propagate key.png --load raft-things.npz [--batch 8]

Several keyframes: --propagate K0.png K1.png ... --propagate-frame 0 8 ... (one frame per map, strictly increasing); each
frame votes between the nearest keys before and after it.  With keyframes, --scene-cut THRESH stops propagation at scene
cuts (the cuts are printed; pixels that no key reaches get label 0, and the final line counts them in the last frame).
The single-key form is unchanged and refuses --scene-cut; video_propagate(..., scene_cut=THRESH) takes one key too.

--path DIR --inpaint MASKDIR removes objects: MASKDIR holds one palette or grey label PNG per frame (sorted), and the
pixels with a non-zero label (--inpaint-labels L ...: those labels), grown by --inpaint-dilate R pixels (default 2), are
filled from the nearest frames, at most --inpaint-window N (default 10) each way and never across a --scene-cut, that see
behind them through the completed flow; what no frame sees is filled spatially (raft_b200.video.video_inpaint).  Annotate
one frame, then remove the object from the whole clip:

    python infer_raft.py --path frames/ --out masks/ --propagate key.png --load raft-things.npz
    python infer_raft.py --path frames/ --out clean/ --inpaint masks/ --load raft-things.npz [--batch 8]

--path DIR --stabilize SIGMA removes the camera's shake from DIR's frames: each consecutive pair's camera motion (a
similarity: zoom, rotation, shift) is fitted robustly on the GPU to the flow of its consistent pixels, the camera path is
smoothed by a Gaussian of SIGMA frames (no default: pick it for the footage; larger is steadier), and every frame is
warped at its own size by its correction, zoomed just enough to hide the borders up to --stabilize-zoom Z (default 1.25).
``<--out>/frame_<i:06d>.png`` and ``<--out>/transforms.npy`` [F,2,3] are written, and the zoom per shot, the cuts and the
number of unreliable pairs printed; with --scene-cut THRESH the path restarts at every cut (raft_b200.video.
video_stabilize):

    python infer_raft.py --path frames/ --out stable/ --stabilize 10 --load raft-things.npz [--batch 8]

--stabilize-fill keeps the whole frame instead: --stabilize-zoom defaults to 1, and the borders the correction uncovers
are filled from the neighbouring frames, at most --stabilize-window N (default 10) each way and never across a
--scene-cut, that saw them along the flow extended past the frame edge; what none saw is filled spatially.  The pixel
counts filled from both sides, one side and spatially are printed:

    python infer_raft.py --path frames/ --out stable/ --stabilize 10 --stabilize-fill --load raft-things.npz

--path DIR --denoise SIGMA removes additive noise of standard deviation SIGMA grey levels ('auto': estimated from the
first 8 frames): each pixel is followed through the flow, at most --denoise-window N (default 3) frames each way, never
across a --scene-cut and only while the forward-backward test holds, and merged with the patches that match it there
and around it in its own frame (raft_b200.video.video_denoise).  The sigma used and the mean number of matched frames are
printed:

    python infer_raft.py --path noisy/ --out clean/ --denoise 20 --load raft-things.npz [--batch 8]

--path DIR --segment-motion writes <--out>/mask_<i:06d>.png, 1 where a pixel moves on its own rather than with the
camera: each pair's camera homography is fitted robustly to its flow, each pixel's residual r (network pixels) gives
evidence r^2 / (r^2 + tau^2), and the evidence is averaged along the flow, at most --segment-window N (default 3)
frames each way, never across a --scene-cut and only while the forward-backward test holds (raft_b200.video.
video_segment_motion).  --segment-tau PX sets tau (default 1 network pixel; not tuned).  The masks are palette PNGs
that --inpaint reads as they are; <--out>/homographies.npy holds the forward pairs' homographies in the frames' pixels:

    python infer_raft.py --path frames/ --out masks/ --segment-motion --load raft-things.npz [--batch 8]

-m val --dataset davis --segment-motion scores it on DAVIS-2016's val sequences, unsupervised (raft_b200.davis.
evaluate_motion): the flow at the frames' own size with 20 iterations, the union of the object labels as ground truth,
J&F printed (``Validation DAVIS-2016 motion segmentation (val): ...``) and written to ``<--out>/val_davis_motion.json``.

--path ORIG --consistent PROC_DIR --consistent-strength L makes per-frame processed frames (PROC_DIR: as many as ORIG,
the same size) temporally consistent, guided by the flow of the original frames (Bonneel et al. 2015;
raft_b200.video.video_consistent); frames after a --scene-cut restart from the processed frame.  E_warp of the
originals, the processed frames and the output, and the per-pixel status counts are printed:

    python infer_raft.py --path orig/ --consistent styled/ --consistent-strength 0.1 --out stable/ --load raft-things.npz

--path ORIG --warp-error VIDEO_DIR prints Lai et al.'s warping error of VIDEO_DIR under the flow of ORIG
(raft_b200.video.video_warp_error) and writes the per-pair values to <--out>/warp_error.json.

-m val --dataset davis --denoise SIGMA scores it on DAVIS-2017 test-dev (raft_b200.davis.evaluate_denoise): seeded
Gaussian noise of SIGMA added to every frame, the flow at the frames' own size with 20 iterations, PSNR and SSIM of the
output and of the noisy input printed (``Validation DAVIS-2017 denoising (test-dev, sigma S): ...``) and written to
``<--out>/val_davis_denoise.json``.

-m val --dataset davis scores it on DAVIS-2017's val split (raft_b200.davis): frame 0's annotation of every sequence
propagated at 480p with 20 iterations, J&F printed (``Validation DAVIS-2017 (val): J&F: ...``) and written to
``<--out>/val_davis.json``, the predicted masks to ``<--out>/davis_val/<seq>/`` in DAVIS's results layout.
--keyframe-step N uses the annotations of frames 0, N, 2N, ... as keyframes and scores the other frames.

--native-frames (with --interpolate, or --path with --interpolate or --input-fps/--fps) writes the interpolated frames,
and with --path the copied input frames, at the input's own size: the flow is estimated and reversed at the network size,
then resized inside the blend, which warps the decoded frames.  --flow-size H W sets that network size in place of
432x1024 wherever the CLI resizes (e.g. --flow-size 544 960 keeps 16:9 footage's aspect ratio):

    python infer_raft.py --path film/ --out tv/ --input-fps 24 --fps 60 --native-frames --flow-size 544 960 --load ...
"""
import glob
import argparse
import math
import os
import sys
from fractions import Fraction

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _decode(path, rgb=False):
    import cv2
    with open(path, "rb") as f:
        img = cv2.imdecode(np.asarray(bytearray(f.read()), dtype="uint8"), cv2.IMREAD_COLOR)  # BGR
    if img is None:
        raise FileNotFoundError(path)
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB) if rgb else img


def read_pair(im1, im2, size, rgb=False):
    import cv2
    out = []
    for path in (im1, im2):
        img = _decode(path, rgb)
        if size is not None:
            img = cv2.resize(img, dsize=(size[1], size[0]))
        out.append(np.float32(img) / 255.0)
    return out[0][None], out[1][None]


def decode_pair(im1, im2, rgb=False):
    """Both frames as decoded (BGR uint8, or RGB with rgb, their own size), [1,H,W,3] each: the engine resizes and scales
    them."""
    return tuple(_decode(path, rgb)[None] for path in (im1, im2))


def parser():
    p = argparse.ArgumentParser()
    p.add_argument('--gpu', default='1', help='comma separated list of GPU(s) to use (ignored, as in the reference)')
    p.add_argument('--data', default='', help='-m val: dataset root (reference flag)')
    p.add_argument('--load', default='release_weight/raft-things.npz', help='npz checkpoint keyed by TF variable names')
    p.add_argument('-m', '--mode', default='test', choices=['train', 'val', 'test', 'export', 'flops'])
    p.add_argument('--out', default='./log', help='-m val: where val_<dataset>.json is written')
    p.add_argument('--batch', default=1, type=int,
                   help='-m val and --path: frame pairs per engine pass (test mode runs one pair)')
    p.add_argument('-o', '--optimizer', default='adam', choices=['adam', 'adamw', 'sgd', 'sgd_cyclic', 'sgd_1cycle'])
    p.add_argument('--im1', default='frame_0010.png')
    p.add_argument('--im2', default='frame_0011.png')
    p.add_argument('--small', action='store_true')
    p.add_argument('--iters', type=int, default=None,
                   help='extension: GRU iterations (test mode: 20 like the reference; -m val: the protocol\'s 32 / 24)')
    p.add_argument('--dataset', default=None, choices=['sintel', 'kitti', 'vimeo', 'tapvid', 'davis', 'gopro'],
                   help='-m val: which dataset --data holds (Sintel / KITTI-2015 training sets: flow; Vimeo-90K '
                        'triplets: frame interpolation; TAP-Vid .pkl file or directory of .pkl shards: point tracking; '
                        'DAVIS-2017 tree: label propagation; GOPRO_Large_all tree: motion blur of a shutter)')
    p.add_argument('--stride', type=int, default=None, metavar='S',
                   help='-m val --dataset gopro: every S-th 240 fps frame is an input (default 8)')
    p.add_argument('--blur-frames', type=int, default=None, metavar='M',
                   help='-m val --dataset gopro: the true frames averaged per blurred frame, odd and <= S (default 7)')
    p.add_argument('--query-mode', default=None, choices=['first', 'strided'],
                   help="-m val --dataset tapvid: TAP-Vid's query mode (default first: each track from its first visible "
                        "frame; strided: from every 5th frame, tracked forward and backward)")
    p.add_argument('--dstype', nargs='+', default=['clean', 'final'], choices=['clean', 'final'],
                   help='-m val, Sintel: the passes to evaluate')
    p.add_argument('--workers', type=int, default=4, help='-m val and --path: frame-decoding (and writing) threads')
    p.add_argument('--split', default='training', choices=['training', 'test'],
                   help='-m val: validate on the training split, or write the test-split submission under --out')
    p.add_argument('--warm-start', action='store_true',
                   help="-m val, Sintel, and --path: warm-start each pair from the previous pair's flow (in its scene; "
                        "upstream's warm_start=True)")
    p.add_argument('--keep-size', action='store_true', help='extension: pad to a multiple of 8 instead of resizing to 432x1024')
    p.add_argument('--npy', default=None, help='extension: also save the raw [H,W,2] flow (--path: a directory)')
    p.add_argument('--flo', default=None, help='extension: also save the flow as a Middlebury .flo file (--path: a directory)')
    p.add_argument('--path', default=None,
                   help="extension (upstream demo.py): a directory of frames; the flow of every consecutive pair is "
                        "written as <--out>/flow_<k:06d>.png")
    p.add_argument('--bidirectional', action='store_true',
                   help='extension: also the backward flow and the forward-backward occlusion masks')
    p.add_argument('--interpolate', type=float, nargs='+', default=None, metavar='T',
                   help='extension: also write the frames at times T in [0, 1] between im1 and im2 (raft_interp_<k>.png); '
                        'with --path, the up-converted sequence <--out>/frame_<n:06d>.png (T strictly increasing inside '
                        '(0, 1))')
    p.add_argument('--input-fps', default=None, metavar='IN',
                   help='extension, with --path and --fps: the frame rate of the --path frames (24, 25, 23.976, '
                        '24000/1001, ...)')
    p.add_argument('--fps', default=None, metavar='OUT',
                   help='extension, with --path and --input-fps: convert the frames to OUT frames per second (above IN), '
                        'written as <--out>/frame_<n:06d>.png')
    p.add_argument('--shutter', type=float, default=None, metavar='ANGLE',
                   help='extension, with --path --input-fps/--fps: a camera shutter of ANGLE degrees in (0, 360]: every '
                        'output frame is the mean of interpolated sub-frames over its exposure, and OUT may be at most '
                        'IN (down-conversion)')
    p.add_argument('--shutter-density', type=int, default=None, metavar='D',
                   help='extension, with --shutter: samples per input-frame interval (default 16)')
    p.add_argument('--scene-cut', type=float, default=None, metavar='THRESH',
                   help='extension, with --path and one of --interpolate, --input-fps/--fps, --warm-start, '
                        '--stabilize or two or more --propagate maps: a threshold in [0, 1] on the colour-histogram '
                        'score of each frame pair; a pair above it is a scene cut, where interpolation copies the nearer '
                        'frame, warm-started flow restarts cold, the stabilized camera path restarts and no label '
                        'crosses from a keyframe')
    p.add_argument('--native-flow', action='store_true',
                   help="extension: resize the written flow(s) back to im1's size (flow_utils.resize_flow)")
    p.add_argument('--native-frames', action='store_true',
                   help="extension, with --interpolate or --path --input-fps/--fps: write the interpolated (and, with "
                        "--path, the copied input) frames at the input's own size, from flow estimated at the network size")
    p.add_argument('--flow-size', type=int, nargs=2, default=None, metavar=('H', 'W'),
                   help='extension: the network size frames are resized to, in place of 432x1024 (test mode and --path)')
    p.add_argument('--track', default=None, metavar='POINTS.txt',
                   help="extension, with --path: track the points of a text file (one `frame x y` line per point, in "
                        "the frames' own pixels) through the frames; writes <--out>/tracks.npy and status.npy")
    p.add_argument('--track-grid', type=int, default=None, metavar='STEP',
                   help='extension, with --path: track a point at every STEP-th pixel of frame --track-frame (1: dense)')
    p.add_argument('--track-frame', type=int, default=0, metavar='K',
                   help='extension, with --track-grid: the frame the grid is laid on (default 0)')
    p.add_argument('--track-vis', default=None, metavar='DIR',
                   help='extension, with --track or --track-grid: also write every frame with the visible points drawn')
    p.add_argument('--track-backward', action='store_true',
                   help='extension, with --track or --track-grid: also track every point back from its frame to frame 0 '
                        '(a second flow sweep over the frames before the last query frame)')
    p.add_argument('--propagate', default=None, nargs='+', metavar='KEY.png',
                   help="extension, with --path: carry the label map KEY.png (palette or 8-bit grey, the frames' size) "
                        "of frame --propagate-frame to every frame; writes <--out>/label_<i:06d>.png.  Several maps are "
                        "keyframes, one per --propagate-frame: each frame votes between the nearest two")
    p.add_argument('--propagate-frame', type=int, nargs='+', default=None, metavar='K',
                   help='extension, with --propagate: the frame each key label map belongs to (default 0; strictly '
                        'increasing)')
    p.add_argument('--keyframe-step', type=int, default=None, metavar='N',
                   help='extension, -m val --dataset davis: the annotations of frames 0, N, 2N, ... are keyframes, the '
                        'other frames are scored')
    p.add_argument('--stabilize', type=float, default=None, metavar='SIGMA',
                   help="extension, with --path: stabilize the frames, smoothing the camera path with a Gaussian of "
                        "SIGMA frames (no default); writes <--out>/frame_<i:06d>.png at the frames' own size and "
                        "<--out>/transforms.npy")
    p.add_argument('--stabilize-zoom', type=float, default=None, metavar='Z',
                   help='extension, with --stabilize: the largest zoom per shot that hides the borders (default 1.25; '
                        'past it the border replicates)')
    p.add_argument('--stabilize-fill', action='store_true',
                   help='extension, with --stabilize: keep the whole frame -- fill the borders the correction uncovers '
                        'from the neighbouring frames that saw them (what none saw spatially) instead of zooming '
                        '(--stabilize-zoom then defaults to 1)')
    p.add_argument('--stabilize-window', type=int, default=None, metavar='N',
                   help='extension, with --stabilize-fill: the frames each side may look ahead or back (default 10; not '
                        'tuned)')
    p.add_argument('--inpaint', default=None, metavar='MASKDIR',
                   help="extension, with --path: remove the masked objects -- MASKDIR holds one palette or grey PNG "
                        "label map per frame (sorted; e.g. what --propagate key.png --out MASKDIR wrote); each hole is "
                        "filled from the nearest frames that see behind it, the rest spatially; writes "
                        "<--out>/frame_<i:06d>.png at the frames' own size")
    p.add_argument('--inpaint-labels', type=int, nargs='+', default=None, metavar='L',
                   help='extension, with --inpaint: remove only these labels (default: every non-zero label)')
    p.add_argument('--inpaint-window', type=int, default=None, metavar='N',
                   help='extension, with --inpaint: the frames each side may look ahead or back (default 10; not tuned)')
    p.add_argument('--inpaint-dilate', type=int, default=None, metavar='R',
                   help='extension, with --inpaint: grow the masks by R pixels (default 2; not tuned)')
    p.add_argument('--denoise', default=None, metavar='SIGMA',
                   help="extension, with --path: remove additive noise of standard deviation SIGMA grey levels (0-255) "
                        "or 'auto' (estimated from the first frames) -- each pixel is merged with its patch matches in "
                        "the neighbouring frames the flow reaches consistently; writes <--out>/frame_<i:06d>.png at the "
                        "frames' own size.  With -m val --dataset davis: score denoising on DAVIS-2017 test-dev at "
                        "noise SIGMA")
    p.add_argument('--denoise-window', type=int, default=None, metavar='N',
                   help='extension, with --denoise: the frames each side may look ahead or back (default 3, at most '
                        '16; not tuned)')
    p.add_argument('--segment-motion', action='store_true',
                   help="extension, with --path: write <--out>/mask_<i:06d>.png, 1 where a pixel moves on its own "
                        "rather than with the camera, and <--out>/homographies.npy.  With -m val --dataset davis: "
                        "score it on DAVIS-2016 val (unsupervised)")
    p.add_argument('--segment-window', type=int, default=None, metavar='N',
                   help='extension, with --segment-motion: the frames each side may look ahead or back (default 3, at '
                        'most 16; not tuned)')
    p.add_argument('--segment-tau', type=float, default=None, metavar='PX',
                   help='extension, with --segment-motion: the residual in network pixels at which a field votes 1/2 '
                        'for motion (default 1; not tuned)')
    p.add_argument('--consistent', default=None, metavar='PROC_DIR',
                   help="extension, with --path: make the per-frame processed frames of PROC_DIR (as many as --path, "
                        "the same size) temporally consistent, guided by the flow of the --path frames (needs "
                        "--consistent-strength); writes <--out>/frame_<i:06d>.png")
    p.add_argument('--consistent-strength', type=float, default=None, metavar='L',
                   help='extension, with --consistent: the strength lambda > 0 (no default); detail finer than about '
                        '2 pi / sqrt(L) pixels keeps the processed frames\' gradients')
    p.add_argument('--warp-error', default=None, metavar='VIDEO_DIR',
                   help="extension, with --path: Lai et al.'s warping error E_warp of the frames of VIDEO_DIR (as many "
                        "as --path, the same size) under the flow of the --path frames; with --out also writes "
                        "<--out>/warp_error.json")
    p.add_argument('--upstream', action='store_true',
                   help='extension: weights converted from an official princeton-vl RAFT .pth (raft_b200.convert): RGB '
                        'frames and the upstream numerics (RAFT(..., upstream=True))')
    p.add_argument('--mixed_precision', action='store_true',
                   help="extension: upstream RAFT's mixed precision -- fp16 conv operands, fp32 accumulation and "
                        "correlation (RAFT(..., mixed_precision=True)); the flow differs from the default by ~1e-2 px")
    return p


def _temporal_refusals(p, args, flag, what):
    """The refusals shared by --consistent and --warp-error."""
    if args.path is None or args.mode != 'test':
        p.error(f'{flag} works on a frame directory: it needs --path DIR (and no -m val)')
    for other, given in (('--consistent', flag != '--consistent' and args.consistent is not None),
                         ('--warp-error', flag != '--warp-error' and args.warp_error is not None),
                         ('--denoise', args.denoise is not None), ('--inpaint', args.inpaint is not None),
                         ('--stabilize', args.stabilize is not None), ('--stabilize-fill', args.stabilize_fill),
                         ('--propagate', args.propagate is not None), ('--track', args.track is not None),
                         ('--track-grid', args.track_grid is not None), ('--interpolate', args.interpolate),
                         ('--fps', args.fps), ('--input-fps', args.input_fps), ('--warm-start', args.warm_start),
                         ('--bidirectional', args.bidirectional), ('--native-flow', args.native_flow),
                         ('--native-frames', args.native_frames), ('--flo', args.flo), ('--npy', args.npy),
                         ('--keyframe-step', args.keyframe_step is not None)):
        if given:
            p.error(f'{flag} {what}: it cannot be combined with {other}')
    if args.scene_cut is not None and not 0.0 <= args.scene_cut <= 1.0:
        p.error(f'--scene-cut: {args.scene_cut} is not a threshold in [0, 1]')
    if args.flow_size is not None and args.keep_size:
        p.error('--flow-size sets the size frames are resized to; --keep-size runs them at their own size')
    if args.batch < 1 or args.workers < 0:
        p.error('--path needs --batch >= 1 and --workers >= 0')
    from raft_b200.video import list_frames
    other = args.consistent if flag == '--consistent' else args.warp_error
    try:
        a, b = list_frames(args.path), list_frames(other)
    except (OSError, ValueError) as e:
        p.error(f'{flag}: {e}')
    if len(a) != len(b):
        p.error(f'{flag}: {other} holds {len(b)} frames, --path {len(a)}: the frames must be aligned')
    if len(a) < 2:
        p.error(f'{flag}: a sequence needs two frames at least')
    import cv2
    sa, sb = cv2.imread(a[0]), cv2.imread(b[0])
    if sa is None or sb is None or sa.shape != sb.shape:
        p.error(f'{flag}: {b[0]} and {a[0]} differ in size (or cannot be read): the frames must be aligned')


def main(argv=None):
    p = parser()
    args = p.parse_args(argv)
    if args.shutter_density is not None and args.shutter is None:
        p.error('--shutter-density goes with --shutter')
    if args.shutter is not None:
        if args.fps is None or args.input_fps is None or args.path is None or args.mode != 'test':
            p.error('--shutter exposes the frames of a frame-rate conversion: it needs --path DIR --input-fps IN --fps OUT')
        if not 0.0 < args.shutter <= 360.0:
            p.error(f'--shutter: ANGLE must be in (0, 360] degrees (got {args.shutter})')
        if args.shutter_density is not None and args.shutter_density < 1:
            p.error(f'--shutter-density: D must be >= 1 (got {args.shutter_density})')
    if args.consistent_strength is not None and args.consistent is None:
        p.error('--consistent-strength goes with --consistent')
    if args.consistent is not None:
        L = args.consistent_strength
        if L is None:
            p.error('--consistent needs --consistent-strength L (no default)')
        from raft_b200.temporal import check_strength
        try:
            check_strength(L)
        except ValueError:
            p.error(f'--consistent-strength: L must be a finite number > 0 (got {L})')
        _temporal_refusals(p, args, '--consistent', 'writes consistent frames')
        return run_consistent(args, L)
    if args.warp_error is not None:
        _temporal_refusals(p, args, '--warp-error', 'scores a video')
        return run_warp_error(args)
    if args.segment_motion:
        return _segment_motion(p, args)
    if args.segment_window is not None or args.segment_tau is not None:
        p.error('--segment-window and --segment-tau go with --segment-motion')
    if args.denoise is not None:
        sigma = args.denoise
        if sigma != 'auto':
            try:
                sigma = float(sigma)
            except ValueError:
                sigma = None
            if sigma is None or not (math.isfinite(sigma) and sigma > 0):
                p.error(f"--denoise: SIGMA must be a number > 0 (grey levels) or 'auto' (got {args.denoise})")
        if args.denoise_window is not None and not 1 <= args.denoise_window <= 16:
            p.error(f'--denoise-window: N must be in [1, 16] (got {args.denoise_window})')
        if args.mode == 'val':
            if args.dataset != 'davis':
                p.error('-m val --denoise scores video denoising on DAVIS-2017 test-dev: it needs --dataset davis')
            if sigma == 'auto':
                p.error('-m val --denoise adds noise of a known level: give SIGMA, not auto')
            if args.warm_start:
                p.error('--warm-start warm-starts flow validation; denoising merges along cold flows')
            if args.split == 'test':
                p.error('--split test writes a flow submission; -m val --denoise scores the test-dev frames')
            for other, given in (('--keyframe-step', args.keyframe_step is not None),
                                 ('--scene-cut', args.scene_cut is not None), ('--path', args.path is not None)):
                if given:
                    p.error(f'-m val --denoise cannot be combined with {other}')
            if not args.data:
                p.error('-m val needs --data <dataset root>')
            return validate_denoise(args, sigma)
        if args.path is None or args.mode != 'test':
            p.error('--denoise removes noise from a frame directory: it needs --path DIR (or -m val --dataset davis)')
        for other, given in (('--inpaint', args.inpaint is not None),
                             ('--inpaint-labels', args.inpaint_labels is not None),
                             ('--inpaint-window', args.inpaint_window is not None),
                             ('--inpaint-dilate', args.inpaint_dilate is not None),
                             ('--stabilize', args.stabilize is not None),
                             ('--stabilize-zoom', args.stabilize_zoom is not None),
                             ('--stabilize-fill', args.stabilize_fill),
                             ('--stabilize-window', args.stabilize_window is not None),
                             ('--propagate', args.propagate is not None),
                             ('--propagate-frame', args.propagate_frame is not None),
                             ('--track', args.track is not None), ('--track-grid', args.track_grid is not None),
                             ('--track-frame', args.track_frame != 0), ('--track-vis', args.track_vis is not None),
                             ('--track-backward', args.track_backward), ('--interpolate', args.interpolate),
                             ('--fps', args.fps), ('--input-fps', args.input_fps), ('--warm-start', args.warm_start),
                             ('--bidirectional', args.bidirectional), ('--native-flow', args.native_flow),
                             ('--native-frames', args.native_frames), ('--flo', args.flo), ('--npy', args.npy),
                             ('--keyframe-step', args.keyframe_step is not None)):
            if given:
                p.error(f'--denoise writes denoised frames: it cannot be combined with {other}')
        if args.scene_cut is not None and not 0.0 <= args.scene_cut <= 1.0:
            p.error(f'--scene-cut: {args.scene_cut} is not a threshold in [0, 1]')
        if args.flow_size is not None and args.keep_size:
            p.error('--flow-size sets the size frames are resized to; --keep-size runs them at their own size')
        if args.batch < 1 or args.workers < 0:
            p.error('--path needs --batch >= 1 and --workers >= 0')
        return run_denoise(args, sigma)
    if args.denoise_window is not None:
        p.error('--denoise-window goes with --denoise')
    if args.inpaint is not None:
        if args.path is None or args.mode != 'test':
            p.error('--inpaint removes objects from a frame directory: it needs --path DIR (and no -m val)')
        for other, given in (('--stabilize', args.stabilize is not None),
                             ('--stabilize-zoom', args.stabilize_zoom is not None),
                             ('--stabilize-fill', args.stabilize_fill),
                             ('--stabilize-window', args.stabilize_window is not None),
                             ('--propagate', args.propagate is not None),
                             ('--propagate-frame', args.propagate_frame is not None),
                             ('--track', args.track is not None), ('--track-grid', args.track_grid is not None),
                             ('--track-frame', args.track_frame != 0), ('--track-vis', args.track_vis is not None),
                             ('--track-backward', args.track_backward), ('--interpolate', args.interpolate),
                             ('--fps', args.fps), ('--input-fps', args.input_fps), ('--warm-start', args.warm_start),
                             ('--bidirectional', args.bidirectional), ('--native-flow', args.native_flow),
                             ('--native-frames', args.native_frames), ('--flo', args.flo), ('--npy', args.npy)):
            if given:
                p.error(f'--inpaint writes frames with the objects removed: it cannot be combined with {other}')
        if args.inpaint_window is not None and args.inpaint_window < 1:
            p.error(f'--inpaint-window: N must be >= 1 (got {args.inpaint_window})')
        if args.inpaint_dilate is not None and not 0 <= args.inpaint_dilate <= 32:
            p.error(f'--inpaint-dilate: R must be in [0, 32] (got {args.inpaint_dilate})')
        if args.inpaint_labels is not None and not all(0 <= v <= 255 for v in args.inpaint_labels):
            p.error(f'--inpaint-labels: labels are in [0, 255] (got {args.inpaint_labels})')
        if args.scene_cut is not None and not 0.0 <= args.scene_cut <= 1.0:
            p.error(f'--scene-cut: {args.scene_cut} is not a threshold in [0, 1]')
        if args.flow_size is not None and args.keep_size:
            p.error('--flow-size sets the size frames are resized to; --keep-size runs them at their own size')
        if args.batch < 1 or args.workers < 0:
            p.error('--path needs --batch >= 1 and --workers >= 0')
        return run_inpaint(args)
    for sub in ('labels', 'window', 'dilate'):
        if getattr(args, f'inpaint_{sub}') is not None:
            p.error(f'--inpaint-{sub} goes with --inpaint')
    if args.stabilize is not None:
        if args.path is None or args.mode != 'test':
            p.error('--stabilize stabilizes a frame directory: it needs --path DIR (and no -m val)')
        for other, given in (('--propagate', args.propagate is not None),
                             ('--propagate-frame', args.propagate_frame is not None),
                             ('--track', args.track is not None), ('--track-grid', args.track_grid is not None),
                             ('--track-frame', args.track_frame != 0), ('--track-vis', args.track_vis is not None),
                             ('--track-backward', args.track_backward), ('--interpolate', args.interpolate),
                             ('--fps', args.fps), ('--input-fps', args.input_fps), ('--warm-start', args.warm_start),
                             ('--bidirectional', args.bidirectional), ('--native-flow', args.native_flow),
                             ('--native-frames', args.native_frames), ('--flo', args.flo), ('--npy', args.npy)):
            if given:
                p.error(f'--stabilize writes stabilized frames: it cannot be combined with {other}')
        if not (math.isfinite(args.stabilize) and args.stabilize > 0):
            p.error(f'--stabilize: SIGMA must be a number of frames > 0 (got {args.stabilize})')
        if args.stabilize_zoom is not None and not (math.isfinite(args.stabilize_zoom) and args.stabilize_zoom >= 1):
            p.error(f'--stabilize-zoom: Z must be a zoom >= 1 (got {args.stabilize_zoom})')
        if args.stabilize_window is not None and not args.stabilize_fill:
            p.error('--stabilize-window goes with --stabilize-fill')
        if args.stabilize_window is not None and args.stabilize_window < 1:
            p.error(f'--stabilize-window: N must be >= 1 (got {args.stabilize_window})')
        if args.scene_cut is not None and not 0.0 <= args.scene_cut <= 1.0:
            p.error(f'--scene-cut: {args.scene_cut} is not a threshold in [0, 1]')
        if args.flow_size is not None and args.keep_size:
            p.error('--flow-size sets the size frames are resized to; --keep-size runs them at their own size')
        if args.batch < 1 or args.workers < 0:
            p.error('--path needs --batch >= 1 and --workers >= 0')
        return run_stabilize(args)
    for flag, given in (('zoom', args.stabilize_zoom is not None), ('fill', args.stabilize_fill),
                        ('window', args.stabilize_window is not None)):
        if given:
            p.error(f'--stabilize-{flag} goes with --stabilize')
    if args.propagate is not None:
        if args.path is None or args.mode != 'test':
            p.error('--propagate carries labels through a frame directory: it needs --path DIR (and no -m val)')
        for other, given in (('--track', args.track is not None), ('--track-grid', args.track_grid is not None),
                             ('--track-frame', args.track_frame != 0), ('--track-vis', args.track_vis is not None),
                             ('--track-backward', args.track_backward), ('--interpolate', args.interpolate),
                             ('--fps', args.fps), ('--input-fps', args.input_fps), ('--warm-start', args.warm_start),
                             ('--bidirectional', args.bidirectional),
                             ('--native-flow', args.native_flow), ('--native-frames', args.native_frames),
                             ('--flo', args.flo), ('--npy', args.npy)):
            if given:
                p.error(f'--propagate writes label maps: it cannot be combined with {other}')
        if args.scene_cut is not None and len(args.propagate) == 1:  # the single-key form is kept as it was
            p.error('--propagate with one key map cannot be combined with --scene-cut: scene cuts go with keyframes '
                    '(two or more key maps and their --propagate-frame); for one key, video_propagate(..., '
                    'scene_cut=THRESH) stops it at cuts')
        if args.batch < 1 or args.workers < 0:
            p.error('--path needs --batch >= 1 and --workers >= 0')
        if args.scene_cut is not None and not 0.0 <= args.scene_cut <= 1.0:
            p.error(f'--scene-cut: {args.scene_cut} is not a threshold in [0, 1]')
        return run_propagate(args, p)
    if args.propagate_frame is not None:
        p.error('--propagate-frame goes with --propagate')
    if args.track is not None or args.track_grid is not None:
        if args.track is not None and args.track_grid is not None:
            p.error('--track and --track-grid are two ways to give the points: pass one')
        flag = '--track' if args.track is not None else '--track-grid'
        if args.path is None or args.mode != 'test':
            p.error(f'{flag} tracks points through a frame directory: it needs --path DIR (and no -m val)')
        for other, given in (('--interpolate', args.interpolate), ('--fps', args.fps), ('--input-fps', args.input_fps),
                             ('--warm-start', args.warm_start), ('--scene-cut', args.scene_cut is not None),
                             ('--bidirectional', args.bidirectional), ('--native-flow', args.native_flow),
                             ('--native-frames', args.native_frames), ('--flo', args.flo), ('--npy', args.npy)):
            if given:
                p.error(f'{flag} writes point tracks: it cannot be combined with {other}')
        if args.track_grid is not None and args.track_grid < 1:
            p.error(f'--track-grid: the step must be >= 1 (got {args.track_grid})')
        if args.batch < 1 or args.workers < 0:
            p.error('--path needs --batch >= 1 and --workers >= 0')
        return run_track(args, p)
    for flag, given in (('--track-frame', args.track_frame != 0), ('--track-vis', args.track_vis is not None),
                        ('--track-backward', args.track_backward)):
        if given:
            p.error(f'{flag} goes with --track-grid' + (' or --track' if flag != '--track-frame' else ''))
    fps = None
    if args.fps is not None or args.input_fps is not None:
        if args.fps is None or args.input_fps is None:
            p.error('--fps OUT and --input-fps IN go together: frame-rate conversion needs both rates')
        if args.path is None:
            p.error('--fps / --input-fps convert the frame rate of a frame directory: they need --path DIR')
        for flag, given in (('--interpolate', args.interpolate), ('--warm-start', args.warm_start),
                            ('--native-flow', args.native_flow), ('--flo', args.flo), ('--npy', args.npy),
                            ('--bidirectional', args.bidirectional)):
            if given:
                p.error(f'--fps writes the frames of one output rate: it cannot be combined with {flag}')
        fps = (_rate(p, '--input-fps', args.input_fps), _rate(p, '--fps', args.fps))
        if fps[1] <= fps[0] and args.shutter is None:
            p.error(f'--fps {args.fps} must exceed --input-fps {args.input_fps}: frame-rate conversion goes up only')
    if args.native_frames:
        if args.keep_size:
            p.error('--native-frames resizes the flow of a smaller network size to the frames; with --keep-size the '
                    'network already runs at their size')
        if args.mode == 'val':
            p.error('--native-frames writes interpolated frames: it has no effect with -m val')
        if not (args.interpolate or fps is not None):
            p.error('--native-frames needs an interpolation mode: --interpolate, or --path with --input-fps/--fps')
    if args.flow_size is not None:
        if args.keep_size:
            p.error('--flow-size sets the size frames are resized to; --keep-size runs them at their own size')
        if args.mode == 'val':
            p.error('--flow-size: -m val runs the validation protocol at the datasets\' own sizes')
        least = 121 if args.upstream else 57
        if min(args.flow_size) < least:
            p.error(f'--flow-size {args.flow_size[0]} {args.flow_size[1]}: each side must be at least {least} (the '
                    f'4-level correlation pyramid{" of --upstream" if args.upstream else ""})')
    if args.interpolate and not all(0.0 <= t <= 1.0 for t in args.interpolate):
        p.error('--interpolate: every T must be in [0, 1]')
    if args.scene_cut is not None:
        if not 0.0 <= args.scene_cut <= 1.0:
            p.error(f'--scene-cut: {args.scene_cut} is not a threshold in [0, 1]')
        if args.mode != 'test' or args.path is None:
            p.error('--scene-cut finds the cuts of a frame directory: it needs --path DIR (and no -m val)')
        if not (args.interpolate or fps is not None or args.warm_start):
            p.error('--scene-cut needs --interpolate, --input-fps/--fps or --warm-start: cold flows over --path do not '
                    'depend on neighbouring pairs, so a cut changes nothing')
    if args.mode == 'val':
        if not args.data or not args.dataset:
            p.error('-m val needs --data <dataset root> and --dataset {sintel,kitti,vimeo,tapvid}')
        if args.warm_start and args.dataset == 'kitti':
            p.error("--warm-start needs frame sequences: KITTI's pairs are not sequences")
        if args.dataset == 'vimeo' and args.split == 'test':
            p.error('--split test writes a flow submission; Vimeo-90K has no hidden-ground-truth split (-m val scores '
                    'its test list)')
        if args.dataset == 'vimeo' and args.warm_start:
            p.error("--warm-start needs frame sequences: Vimeo-90K's triplets are not chains")
        if args.dataset == 'tapvid' and args.split == 'test':
            p.error('--split test writes a flow submission; TAP-Vid has no hidden-ground-truth split (-m val scores its '
                    'videos)')
        if args.dataset == 'tapvid' and args.warm_start:
            p.error('--warm-start warm-starts flow validation; TAP-Vid tracks points through cold flows')
        if args.dataset == 'davis' and args.split == 'test':
            p.error('--split test writes a flow submission; DAVIS-2017 test-dev submissions are not supported (-m val '
                    'scores the val split)')
        if args.dataset == 'davis' and args.warm_start:
            p.error('--warm-start warm-starts flow validation; DAVIS propagates labels through cold flows')
    if (args.stride is not None or args.blur_frames is not None) and (args.mode != 'val' or args.dataset != 'gopro'):
        p.error('--stride and --blur-frames go with -m val --dataset gopro')
    if args.mode == 'val' and args.dataset == 'gopro':
        if args.warm_start:
            p.error('--warm-start warm-starts flow validation; the GoPro protocol runs cold bidirectional flows')
        from raft_b200.gopro import DEFAULT_BLUR_FRAMES, DEFAULT_STRIDE, check_window
        try:
            check_window(DEFAULT_STRIDE if args.stride is None else args.stride,
                         DEFAULT_BLUR_FRAMES if args.blur_frames is None else args.blur_frames)
        except ValueError:
            p.error(f'--stride {args.stride} --blur-frames {args.blur_frames}: S must be >= 1 and M odd with '
                    '1 <= M <= S')
        if args.batch < 1:
            p.error('--batch must be >= 1')
    if args.query_mode is not None and (args.mode != 'val' or args.dataset != 'tapvid'):
        p.error('--query-mode goes with -m val --dataset tapvid')
    if args.keyframe_step is not None:
        if args.mode != 'val' or args.dataset != 'davis':
            p.error('--keyframe-step goes with -m val --dataset davis')
        if args.keyframe_step < 1:
            p.error(f'--keyframe-step: the step must be >= 1 (got {args.keyframe_step})')
    if args.mode == 'val':
        return validate_gopro(args) if args.dataset == 'gopro' else validate(args)
    if args.mode != 'test':
        print(f"mode '{args.mode}' has no implementation in the reference either (infer_raft.py:71-95); nothing to do")
        return 0
    if args.path is not None:
        if args.bidirectional:
            p.error('--path runs forward flow or frame interpolation over a frame sequence; it cannot be combined with '
                    '--bidirectional')
        if args.interpolate:
            for flag, given in (('--warm-start', args.warm_start), ('--native-flow', args.native_flow),
                                ('--flo', args.flo), ('--npy', args.npy)):
                if given:
                    p.error(f'--path --interpolate writes frames, not flows: it cannot be combined with {flag}')
            ts = args.interpolate
            if not all(0.0 < t < 1.0 for t in ts) or any(b <= a for a, b in zip(ts, ts[1:])):
                p.error('--path --interpolate: the times T must be strictly increasing inside (0, 1) (the input frames '
                        'are the times 0 and 1)')
        if args.interpolate or fps is not None:
            if args.batch < 1 or args.workers < 0:
                p.error('--path needs --batch >= 1 and --workers >= 0')
            n = len(glob.glob(os.path.join(args.path, '*.png')) + glob.glob(os.path.join(args.path, '*.jpg')))
            if n < 2:
                p.error(f'--path {"--fps" if fps else "--interpolate"}: {args.path} holds {n} *.png / *.jpg frames; '
                        'interpolation needs two')
            return run_video_interpolate(args, fps)
        if args.warm_start and args.batch != 1:
            p.error('--path --warm-start warm-starts each pair from the one before: it runs one pair per pass (--batch 1)')
        if args.batch < 1 or args.workers < 0:
            p.error('--path needs --batch >= 1 and --workers >= 0')
        return run_video(args)
    from networks import RAFT
    import cv2
    from flow_utils import flow_to_color, resize_flow, write_flo
    rgb = args.upstream  # the official checkpoints expect RGB frames; the reference's expect BGR
    args.iters = 20 if args.iters is None else args.iters
    if args.keep_size:
        left, right = read_pair(args.im1, args.im2, None, rgb)
        model = RAFT.RAFT(left.shape[1:], args, iters=args.iters, upstream=args.upstream,
                          mixed_precision=args.mixed_precision).load(args.load)
    else:  # the reference's 432x1024 (infer_raft.py:69,76) or --flow-size, resized and scaled on the GPU
        size = _flow_size(args)
        left, right = decode_pair(args.im1, args.im2, rgb)
        native = left.shape[1:3]
        if left.shape != right.shape:  # one engine pass takes one frame size: resize such a pair on the host, as before
            if args.native_frames:
                p.error(f'--native-frames: {args.im1} is {left.shape[1]}x{left.shape[2]} and {args.im2} '
                               f'{right.shape[1]}x{right.shape[2]}; frames at their own size need one size')
            left, right = read_pair(args.im1, args.im2, size, rgb)
        model = RAFT.RAFT(size + (3,), args, iters=args.iters, input_size=size,
                          upstream=args.upstream, mixed_precision=args.mixed_precision).load(args.load)
    if args.bidirectional:
        flow, flow_bw, occ_fw, occ_bw = (t.cpu().numpy() for t in model.forward_bidirectional(left, right))
    else:
        flow = model.forward(left, right).cpu().numpy()
    if args.native_flow and not args.keep_size:
        H, W = native
        flow = resize_flow(flow[0], W, H)[None]
        if args.bidirectional:
            flow_bw = resize_flow(flow_bw[0], W, H)[None]
    print(0, flow.shape)
    cv2.imwrite("raft_flow_raft-things.png", flow_to_color(flow[0], convert_to_bgr=True))
    if args.npy:
        np.save(args.npy, flow[0])
    if args.flo:
        write_flo(args.flo, flow[0])
    if args.bidirectional:
        cv2.imwrite("raft_flow_raft-things_bw.png", flow_to_color(flow_bw[0], convert_to_bgr=True))
        grey = np.array([0, 128, 255], dtype=np.uint8)  # consistent / occluded / leaves the frame
        cv2.imwrite("raft_occ_fw.png", grey[occ_fw[0]])
        cv2.imwrite("raft_occ_bw.png", grey[occ_bw[0]])
        if args.npy:
            np.save(_bw_path(args.npy), flow_bw[0])
        if args.flo:
            write_flo(_bw_path(args.flo), flow_bw[0])
    if args.interpolate:
        frames = model.interpolate(left, right, args.interpolate, native=args.native_frames).cpu().numpy()
        for k, frame in enumerate(frames):
            img = np.clip(np.rint(255.0 * frame[0]), 0, 255).astype(np.uint8)
            cv2.imwrite(f"raft_interp_{k}.png", cv2.cvtColor(img, cv2.COLOR_RGB2BGR) if rgb else img)
    return 0


def run_video(args):
    """--path: raft_b200.video over the frames of --path, at 432x1024 (or --flow-size) like test mode (or their own size
    with --keep-size)."""
    from raft_b200.video import video
    model = _video_model(args)
    files = video(model, args.path, args.out, batch=args.batch, workers=args.workers, warm_start=args.warm_start,
                  flo=args.flo, npy=args.npy, native_flow=args.native_flow, scene_cut=args.scene_cut)
    if args.scene_cut is not None:
        files = _print_cuts(*files)
    print(f"{len(files)} files written under {args.out}" + (" and the --flo / --npy directories" if args.flo or args.npy
                                                            else ""))
    return 0


def run_video_interpolate(args, fps=None):
    """--path --interpolate, or --path --input-fps --fps (fps = the two rates): raft_b200.video.video_interpolate over the
    frames of --path, at 432x1024 (or --flow-size) like test mode (or their own size with --keep-size); --native-frames
    writes the frames at their own size."""
    from raft_b200.video import video_interpolate
    model = _video_model(args)
    files = video_interpolate(model, args.path, args.out, args.interpolate, batch=args.batch, workers=args.workers,
                              fps=fps, scene_cut=args.scene_cut, native=args.native_frames,
                              **({} if args.shutter is None else {"shutter": args.shutter,
                                                                  "density": args.shutter_density or 16}))
    if args.scene_cut is not None:
        files = _print_cuts(*files)
    print(f"{len(files)} frames written under {args.out}")
    return 0


def run_track(args, p):
    """--path --track / --track-grid: raft_b200.video.video_track over the frames of --path, at 432x1024 (or --flow-size)
    like test mode (or their own size with --keep-size); the points are given and tracked in the frames' own pixels.
    Prints the point count, the frame count and how many points are consistent (status 0) in the last frame."""
    from raft_b200.video import read_queries, video_track
    queries = None
    if args.track is not None:
        try:
            queries = read_queries(args.track)
        except (OSError, ValueError) as e:
            p.error(f'--track: {e}')
    model = _video_model(args)
    tracks, status = video_track(model, args.path, args.out, queries=queries, grid=args.track_grid,
                                 grid_frame=args.track_frame, batch=args.batch, workers=args.workers, vis=args.track_vis,
                                 backward=args.track_backward)
    st = np.load(status, mmap_mode='r')
    F, N = st.shape
    print(f"{N} points tracked through {F} frames: {int((st[-1] == 0).sum())} consistent (status 0) in the last frame; "
          f"{tracks} and {status} written")
    return 0


def run_propagate(args, p):
    """--path --propagate: raft_b200.video.video_propagate over the frames of --path, at 432x1024 (or --flow-size) like
    test mode (or their own size with --keep-size); the keys and the written label maps are at the frames' own size.
    Prints the frame count and how many pixels of the last frame are consistent (status 0) all the way to a key, and
    with --scene-cut the cuts and how many of its pixels no key reaches (status 3)."""
    import cv2
    from raft_b200.video import list_frames, read_labels, video_propagate
    frames = [0] if args.propagate_frame is None else args.propagate_frame
    if len(frames) != len(args.propagate):
        p.error(f'--propagate gives {len(args.propagate)} key label maps and --propagate-frame {len(frames)} frames: '
                'the counts must match')
    if any(b <= a for a, b in zip(frames, frames[1:])):
        p.error(f'--propagate-frame {" ".join(map(str, frames))}: the key frames must be strictly increasing')
    try:
        keys = [read_labels(k)[0] for k in args.propagate]
        paths = list_frames(args.path)
    except (OSError, ValueError) as e:
        p.error(f'--propagate: {e}')
    for frame in frames:
        if not 0 <= frame < len(paths):
            p.error(f'--propagate-frame {frame}: {args.path} holds {len(paths)} frames')
    first = cv2.imread(paths[0], cv2.IMREAD_COLOR)
    for name, key in zip(args.propagate, keys):
        if first is not None and first.shape[:2] != key.shape:
            p.error(f'--propagate: {name} is {key.shape[0]}x{key.shape[1]}, the frames of {args.path} are '
                    f'{first.shape[0]}x{first.shape[1]}; the key labels need the frames\' size')
    model = _video_model(args)
    single = len(frames) == 1
    res = video_propagate(model, paths, args.out, args.propagate[0] if single else args.propagate,
                          frame=frames[0] if single else frames, batch=args.batch, workers=args.workers,
                          scene_cut=args.scene_cut)
    if args.scene_cut is not None:
        files, last, cuts = res
        _print_cuts(files, cuts)
    else:
        files, last = res
    which = f"frame {frames[0]}" if single else f"frames {', '.join(map(str, frames))}"
    unreached = f", {int((last == 3).sum())} reached by no key (status 3)" if args.scene_cut is not None else ""
    print(f"labels of {which} propagated through {len(files)} frames: {int((last == 0).sum())} of {last.size} "
          f"pixels of the last frame consistent (status 0){unreached}; written under {args.out}")
    return 0


def run_stabilize(args):
    """--path --stabilize: raft_b200.video.video_stabilize over the frames of --path, the flow at 432x1024 (or
    --flow-size) like test mode (or the frames' own size with --keep-size), the frames written at their own size."""
    from raft_b200.video import video_stabilize
    model = _video_model(args)
    files, _ = video_stabilize(model, args.path, args.out, args.stabilize, batch=args.batch, workers=args.workers,
                               scene_cut=args.scene_cut, max_zoom=args.stabilize_zoom, fill=args.stabilize_fill,
                               window=args.stabilize_window)
    print(f"{len(files)} stabilized frames and transforms.npy written under {args.out}")
    return 0


def run_inpaint(args):
    """--path --inpaint: raft_b200.video.video_inpaint over the frames of --path and the masks of --inpaint, the flow at
    432x1024 (or --flow-size) like test mode (or the frames' own size with --keep-size), the frames written at their own
    size."""
    from raft_b200.video import video_inpaint
    model = _video_model(args)
    files, _ = video_inpaint(model, args.path, args.out, args.inpaint, window=args.inpaint_window,
                             dilate=args.inpaint_dilate, labels=args.inpaint_labels, batch=args.batch,
                             workers=args.workers, scene_cut=args.scene_cut)
    print(f"{len(files)} frames with the masked objects removed written under {args.out}")
    return 0


def run_denoise(args, sigma):
    """--path --denoise: raft_b200.video.video_denoise over the frames of --path, the flow at 432x1024 (or --flow-size)
    like test mode (or the frames' own size with --keep-size), the frames written at their own size."""
    from raft_b200.video import video_denoise
    model = _video_model(args)
    files, _ = video_denoise(model, args.path, args.out, sigma, window=args.denoise_window, batch=args.batch,
                             workers=args.workers, scene_cut=args.scene_cut)
    print(f"{len(files)} denoised frames written under {args.out}")
    return 0


def _segment_motion(p, args):
    """--segment-motion: the checks, then -m val --dataset davis (validate_motion) or --path (run_segment_motion)."""
    from raft_b200.motionseg import MAX_WINDOW, check_tau
    if args.segment_window is not None and not 0 <= args.segment_window <= MAX_WINDOW:
        p.error(f'--segment-window: N must be in [0, {MAX_WINDOW}] (got {args.segment_window})')
    if args.segment_tau is not None:
        try:
            check_tau(args.segment_tau)
        except ValueError:
            p.error(f'--segment-tau: PX must be a finite number > 0 (got {args.segment_tau})')
    others = (('--denoise', args.denoise is not None), ('--inpaint', args.inpaint is not None),
              ('--stabilize', args.stabilize is not None), ('--stabilize-fill', args.stabilize_fill),
              ('--propagate', args.propagate is not None), ('--track', args.track is not None),
              ('--track-grid', args.track_grid is not None), ('--interpolate', args.interpolate),
              ('--fps', args.fps), ('--input-fps', args.input_fps), ('--warm-start', args.warm_start),
              ('--bidirectional', args.bidirectional), ('--native-flow', args.native_flow),
              ('--native-frames', args.native_frames), ('--flo', args.flo), ('--npy', args.npy),
              ('--keyframe-step', args.keyframe_step is not None), ('--consistent', args.consistent is not None),
              ('--warp-error', args.warp_error is not None))
    if args.mode == 'val':
        if args.dataset != 'davis':
            p.error('-m val --segment-motion scores motion segmentation on DAVIS-2016 val: it needs --dataset davis')
        if args.split == 'test':
            p.error('--split test writes a flow submission; -m val --segment-motion scores the val sequences')
        for other, given in others + (('--scene-cut', args.scene_cut is not None), ('--path', args.path is not None)):
            if given:
                p.error(f'-m val --segment-motion cannot be combined with {other}')
        if not args.data:
            p.error('-m val needs --data <dataset root>')
        return validate_motion(args)
    if args.path is None or args.mode != 'test':
        p.error('--segment-motion segments a frame directory: it needs --path DIR (or -m val --dataset davis)')
    for other, given in others:
        if given:
            p.error(f'--segment-motion writes masks: it cannot be combined with {other}')
    if args.scene_cut is not None and not 0.0 <= args.scene_cut <= 1.0:
        p.error(f'--scene-cut: {args.scene_cut} is not a threshold in [0, 1]')
    if args.flow_size is not None and args.keep_size:
        p.error('--flow-size sets the size frames are resized to; --keep-size runs them at their own size')
    if args.batch < 1 or args.workers < 0:
        p.error('--path needs --batch >= 1 and --workers >= 0')
    return run_segment_motion(args)


def run_segment_motion(args):
    """--path --segment-motion: raft_b200.video.video_segment_motion over the frames of --path, the flow at 432x1024 (or
    --flow-size) like test mode (or the frames' own size with --keep-size), the masks written at the frames' own size."""
    from raft_b200.video import video_segment_motion
    model = _video_model(args)
    files, _ = video_segment_motion(model, args.path, args.out, window=args.segment_window, tau=args.segment_tau,
                                    batch=args.batch, workers=args.workers, scene_cut=args.scene_cut)
    print(f"{len(files)} motion masks written under {args.out}")
    return 0


def validate_motion(args):
    """-m val --dataset davis --segment-motion: raft_b200.davis.evaluate_motion on --data, the summary line on stdout,
    the per-sequence records in <--out>/val_davis_motion.json, the masks in DAVIS's results layout under
    <--out>/davis_motion."""
    import json
    from networks import RAFT
    from raft_b200.davis import evaluate_motion, motion_summary
    model = RAFT.RAFT(None, args, upstream=args.upstream, mixed_precision=args.mixed_precision).load(args.load)
    res = evaluate_motion(model, args.data, window=args.segment_window, tau=args.segment_tau, batch=args.batch,
                          iters=args.iters, masks_out=os.path.join(args.out, 'davis_motion'))
    print(motion_summary(res))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "val_davis_motion.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


def run_consistent(args, strength):
    """--path --consistent PROC_DIR: raft_b200.video.video_consistent, the flow of the --path frames at 432x1024 (or
    --flow-size, or their own size with --keep-size), the frames written at their own size."""
    from raft_b200.video import video_consistent
    model = _video_model(args)
    files, _ = video_consistent(model, args.path, args.consistent, args.out, strength, batch=args.batch,
                                workers=args.workers, scene_cut=args.scene_cut)
    print(f"{len(files)} consistent frames written under {args.out}")
    return 0


def run_warp_error(args):
    """--path --warp-error VIDEO_DIR: raft_b200.video.video_warp_error; the summary line on stdout, the per-pair values
    in <--out>/warp_error.json."""
    from raft_b200.video import video_warp_error
    model = _video_model(args)
    info = video_warp_error(model, args.path, args.warp_error, batch=args.batch, workers=args.workers,
                            scene_cut=args.scene_cut)
    import json
    for v in ("original", "input"):  # excluded pairs (NaN) as null
        info[v]["E_pair"] = [None if e != e else e for e in info[v]["E_pair"]]
        info[v]["E_warp"] = None if info[v]["E_warp"] != info[v]["E_warp"] else info[v]["E_warp"]
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "warp_error.json"), "w") as f:
        json.dump(info, f, indent=1)
    return 0


def validate_denoise(args, sigma):
    """-m val --dataset davis --denoise SIGMA: raft_b200.davis.evaluate_denoise on --data, the summary line on stdout,
    the per-sequence records in <--out>/val_davis_denoise.json."""
    import json
    from networks import RAFT
    from raft_b200.davis import evaluate_denoise, denoise_summary
    model = RAFT.RAFT(None, args, upstream=args.upstream, mixed_precision=args.mixed_precision).load(args.load)
    res = evaluate_denoise(model, args.data, sigma, window=args.denoise_window, batch=args.batch,
                           iters=args.iters)
    print(denoise_summary(res))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "val_davis_denoise.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


def _video_model(args):
    """The model of --path: at 432x1024 (or --flow-size) like test mode, or at the frames' own size with --keep-size."""
    from networks import RAFT
    size = None if args.keep_size else _flow_size(args)
    return RAFT.RAFT(None if size is None else size + (3,), args, iters=20 if args.iters is None else args.iters,
                     input_size=size, upstream=args.upstream, mixed_precision=args.mixed_precision).load(args.load)


def _flow_size(args):
    """The network size of test mode and --path: --flow-size H W, or the reference's 432x1024."""
    return (432, 1024) if args.flow_size is None else tuple(args.flow_size)


def _print_cuts(files, cuts):
    """--scene-cut: the number of cut pairs and their indices (raft_b200.video.print_cuts); returns files."""
    from raft_b200.video import print_cuts
    print_cuts(cuts)
    return files


def validate(args):
    """-m val: raft_b200.evaluate on --data, upstream's summary lines on stdout, everything in <--out>/val_<dataset>.json;
    with --split test, raft_b200.evaluate.submit's files under --out."""
    import json
    from networks import RAFT
    from raft_b200.evaluate import evaluate, submit, summary_lines
    model = RAFT.RAFT(None, args, upstream=args.upstream, mixed_precision=args.mixed_precision).load(args.load)
    if args.split == 'test':
        files = submit(model, args.data, args.dataset, args.out, dstypes=tuple(args.dstype), batch=args.batch,
                       workers=args.workers, iters=args.iters, warm_start=args.warm_start)
        print(f"{len(files)} flows written under {args.out}")
        return 0
    res = evaluate(model, args.data, args.dataset, dstypes=tuple(args.dstype), batch=args.batch, workers=args.workers,
                   iters=args.iters, warm_start=args.warm_start, query_mode=args.query_mode,
                   masks_out=os.path.join(args.out, 'davis_val') if args.dataset == 'davis' else None,
                   keyframe_step=args.keyframe_step)
    for line in summary_lines(res):
        print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, f"val_{args.dataset}.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


def validate_gopro(args):
    """-m val --dataset gopro: raft_b200.gopro.evaluate on --data at the frames' own size (20 iterations), the summary
    line on stdout and everything in <--out>/val_gopro.json.  --split test scores <data>/test, the default <data>/train."""
    import json
    from networks import RAFT
    from raft_b200.gopro import DEFAULT_BLUR_FRAMES, DEFAULT_STRIDE, evaluate, summary_line
    model = RAFT.RAFT(None, args, iters=20 if args.iters is None else args.iters, upstream=args.upstream,
                      mixed_precision=args.mixed_precision).load(args.load)
    res = evaluate(model, args.data, "test" if args.split == "test" else "train",
                   DEFAULT_STRIDE if args.stride is None else args.stride,
                   DEFAULT_BLUR_FRAMES if args.blur_frames is None else args.blur_frames, batch=args.batch)
    print(summary_line(res))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "val_gopro.json"), "w") as f:
        json.dump(res, f, indent=1)
    return 0


def _rate(p, flag, text):
    """A frame-rate flag as a Fraction ("24", "59.94", "24000/1001"); anything else, zero or negative is a usage error."""
    try:
        rate = Fraction(text)
    except (ValueError, ZeroDivisionError):
        rate = None
    if rate is None or rate <= 0:
        p.error(f'{flag}: {text!r} is not a frame rate (a positive number such as 24, 59.94 or 24000/1001)')
    return rate


def _bw_path(path):
    stem, ext = os.path.splitext(path)
    return stem + "_bw" + ext


if __name__ == '__main__':
    sys.exit(main())
