"""F9: upstream RAFT's validation protocol (evaluate.py: validate_sintel, validate_kitti) with the metrics on the GPU.

    from raft_b200.evaluate import evaluate
    res = evaluate(RAFT(None, args, upstream=True).load("raft-things.npz"), "datasets/Sintel", "sintel")

Sintel: every frame of <root>/training/{clean,final}/<scene>/ paired with the next one, ground truth
<root>/training/flow/<scene>/frame_NNNN.flo, 32 iterations, InputPadder 'sintel' padding, every pixel counted.  KITTI-2015:
<root>/training/image_2/<id>_10.png and <id>_11.png, ground truth <root>/training/flow_occ/<id>_10.png (16-bit PNG with a
valid flag), 24 iterations, 'kitti' padding (bottom only), valid pixels counted.  Frames run at their own size.

submit writes upstream's test-split submissions (create_sintel_submission, create_kitti_submission) the same way, and
warm_start runs each Sintel scene as a chain warm-started by forward_interpolate (upstream's warm_start=True).

Vimeo-90K (F12): the triplets <root>/sequences/<entry>/im1.png, im2.png, im3.png of <root>/tri_testlist.txt, in list
order; im2 is interpolated from im1 and im3 at t = 0.5 (RaftEngine.interpolate, 20 iterations like the reference) and
scored by rb_frame_metrics against the uploaded im2 on the same stream -- the predicted frame never leaves the GPU -- into
per-triplet PSNR and SSIM, reported as their means over the list.

TAP-Vid (F17, raft_b200.tapvid): point tracking scored by Average Jaccard, the fraction of points within 1-16 pixels and
occlusion accuracy, at 256 x 256 with 20 iterations, in the 'first' or 'strided' query mode.

DAVIS-2017 (F20, raft_b200.davis): keyframe label propagation from each sequence's first annotation, scored by region
similarity J and boundary accuracy F (davis2017-evaluation's semi-supervised protocol) at 480p with 20 iterations.

Pipeline: pairs are grouped by frame size (one CUDA graph per size) and run in batches through RaftEngine.forward, whose
flow stays on the GPU: rb_flow_metrics scores it against the uploaded ground truth on the same stream and writes per-pair
stats into one device buffer, read back once per split.  Worker threads decode the next batches (cv2 releases the GIL)
while the GPU runs the current one, into two pinned staging slots used in turn; a slot is refilled only after the event
recorded behind its batch's work has completed.  Every kernel is batch-invariant, so the results are the same bits for
every batch size and worker count.  Aggregates are computed on the host in fp64 from the per-pair stats.
"""
from __future__ import annotations

import os
import re
import struct
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import capi
from .engine import RaftEngine

# dataset -> (iterations, pad_mode): upstream's validate_sintel / validate_kitti
PROTOCOLS = {"sintel": (32, "sintel"), "kitti": (24, "kitti"), "vimeo": (20, "sintel"), "tapvid": (20, "sintel"),
             "davis": (20, "sintel")}
DSTYPES = ("clean", "final")
QUERY_MODES = ("first", "strided")  # TAP-Vid's (raft_b200.tapvid)
STATS = 6  # RB_FLOW_STATS: n, sum of EPE, #(EPE < 1), #(EPE < 3), #(EPE < 5), #outliers
FRAME_STATS = 2  # RB_FRAME_STATS: SSE, SSIM

Pair = namedtuple("Pair", "image1 image2 gt")
# Vimeo-90K: image1 = im1, image2 = im3 (the frames the engine reads), gt = im2; dir = the list entry
Triplet = namedtuple("Triplet", "image1 image2 gt dir")


# ---- dataset enumeration ----------------------------------------------------------------------------
def _listdir(path, what):
    if not os.path.isdir(path):
        raise FileNotFoundError(f"{what}: no directory {path}")
    return sorted(os.listdir(path))


def sintel_pairs(root, dstype="clean"):
    """MPI-Sintel training pairs of one pass (dstype 'clean' or 'final'), scene by scene in sorted order: frame k with
    frame k + 1 of the same scene and the ground truth of frame k.  Frame numbers must be consecutive within a scene, and
    every frame but the last needs its .flo and every .flo its frame: otherwise FileNotFoundError names the file."""
    if dstype not in DSTYPES:
        raise ValueError(f"Sintel dstype must be one of {DSTYPES} (got {dstype!r})")
    img_root, flow_root = os.path.join(root, "training", dstype), os.path.join(root, "training", "flow")
    pairs = []
    for scene in _listdir(img_root, "Sintel"):
        sdir = os.path.join(img_root, scene)
        if not os.path.isdir(sdir):
            continue
        frames = [f for f in sorted(os.listdir(sdir)) if f.endswith(".png")]
        fdir = os.path.join(flow_root, scene)
        flos = set(f for f in _listdir(fdir, "Sintel ground truth") if f.endswith(".flo"))
        for a, b in zip(frames[:-1], frames[1:]):
            ma, mb = re.fullmatch(r"frame_(\d+)\.png", a), re.fullmatch(r"frame_(\d+)\.png", b)
            if not (ma and mb and int(mb.group(1)) == int(ma.group(1)) + 1):
                raise FileNotFoundError(f"Sintel: {os.path.join(sdir, b)} does not follow {os.path.join(sdir, a)} "
                                        "(frames must be frame_NNNN.png, numbered consecutively)")
            flo = a[:-4] + ".flo"
            if flo not in flos:
                raise FileNotFoundError(f"Sintel: ground truth {os.path.join(fdir, flo)} of {os.path.join(sdir, a)} is "
                                        "missing")
            flos.discard(flo)
            pairs.append(Pair(os.path.join(sdir, a), os.path.join(sdir, b), os.path.join(fdir, flo)))
        if flos:
            raise FileNotFoundError(f"Sintel: ground truth {os.path.join(fdir, sorted(flos)[0])} has no frame pair")
    if not pairs:
        raise FileNotFoundError(f"Sintel: no frame pairs under {img_root}")
    return pairs


def kitti_pairs(root):
    """KITTI-2015 training pairs in sorted id order: image_2/<id>_10.png, image_2/<id>_11.png, flow_occ/<id>_10.png.  A
    missing second frame or ground truth, or a ground truth without frames, raises FileNotFoundError naming the file."""
    img_root, flow_root = os.path.join(root, "training", "image_2"), os.path.join(root, "training", "flow_occ")
    images = set(_listdir(img_root, "KITTI"))
    gts = set(f for f in _listdir(flow_root, "KITTI ground truth") if f.endswith("_10.png"))
    pairs = []
    for f in sorted(images):
        if not f.endswith("_10.png"):
            continue
        second = f[:-len("_10.png")] + "_11.png"
        if second not in images:
            raise FileNotFoundError(f"KITTI: second frame {os.path.join(img_root, second)} is missing")
        if f not in gts:
            raise FileNotFoundError(f"KITTI: ground truth {os.path.join(flow_root, f)} is missing")
        gts.discard(f)
        pairs.append(Pair(os.path.join(img_root, f), os.path.join(img_root, second), os.path.join(flow_root, f)))
    if gts:
        raise FileNotFoundError(f"KITTI: ground truth {os.path.join(flow_root, sorted(gts)[0])} has no frame pair")
    if not pairs:
        raise FileNotFoundError(f"KITTI: no frame pairs under {img_root}")
    return pairs


def vimeo_triplets(root):
    """Vimeo-90K triplets in the order of <root>/tri_testlist.txt (one '00001/0389'-style entry per line; blank lines and
    surrounding whitespace are ignored): <root>/sequences/<entry>/im1.png, im2.png, im3.png.  A missing list, a missing
    frame or an empty list raises FileNotFoundError naming the path."""
    lst = os.path.join(root, "tri_testlist.txt")
    if not os.path.isfile(lst):
        raise FileNotFoundError(f"Vimeo-90K: no triplet list {lst}")
    with open(lst) as f:
        entries = [e.strip() for e in f if e.strip()]
    trips = []
    for e in entries:
        im1, im2, im3 = (os.path.join(root, "sequences", e, f"im{k}.png") for k in (1, 2, 3))
        for p in (im1, im2, im3):
            if not os.path.isfile(p):
                raise FileNotFoundError(f"Vimeo-90K: frame {p} of triplet {e} is missing")
        trips.append(Triplet(im1, im3, im2, e))
    if not trips:
        raise FileNotFoundError(f"Vimeo-90K: {lst} lists no triplets")
    return trips


# ---- decoding (worker threads) ------------------------------------------------------------------------
def _png_size(path):
    """(H, W) from the PNG header, without decoding the image."""
    with open(path, "rb") as f:
        head = f.read(24)
    if len(head) < 24 or head[:8] != b"\x89PNG\r\n\x1a\n" or head[12:16] != b"IHDR":
        raise ValueError(f"{path}: not a PNG file")
    w, h = struct.unpack(">II", head[16:24])
    return int(h), int(w)


def _imread(path, rgb):
    import cv2
    img = cv2.imread(path, cv2.IMREAD_COLOR)  # BGR uint8
    if img is None:
        raise FileNotFoundError(f"cannot read {path}")
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB) if rgb else img


def _decode_frames(pair, rgb):
    left, right = _imread(pair.image1, rgb), _imread(pair.image2, rgb)
    if right.shape != left.shape:
        raise ValueError(f"{pair.image2}: {right.shape[:2]} frame, {pair.image1} is {left.shape[:2]}")
    return left, right


def _decode_triplet(trip, rgb):
    left, right = _decode_frames(trip, rgb)
    mid = _imread(trip.gt, rgb)
    if mid.shape != left.shape:
        raise ValueError(f"{trip.gt}: {mid.shape[:2]} frame, {trip.image1} is {left.shape[:2]}")
    return left, right, mid


def _decode(pair, kitti, rgb):
    from flow_utils import read_flo, read_kitti_flow
    left, right = _decode_frames(pair, rgb)
    gt, valid = read_kitti_flow(pair.gt) if kitti else (read_flo(pair.gt), None)
    if gt.shape[:2] != left.shape[:2]:
        raise ValueError(f"{pair.gt}: {gt.shape[:2]} ground truth for {left.shape[:2]} frames ({pair.image1})")
    return left, right, gt, valid


class _Slot:
    """Pinned host staging of one batch (frames, and ground truth and mask when scored; with gt_frame the ground truth
    is a uint8 [B,H,W,3] frame instead of a flow) and the event behind the last batch that used it."""

    def __init__(self, B, H, W, kitti, scored=True, gt_frame=False):
        self.left = torch.zeros(B, H, W, 3, dtype=torch.uint8).pin_memory()
        self.right = torch.zeros_like(self.left).pin_memory()
        gt_shape, gt_dtype = ((B, H, W, 3), torch.uint8) if gt_frame else ((B, H, W, 2), torch.float32)
        self.gt = torch.zeros(*gt_shape, dtype=gt_dtype).pin_memory() if scored else None
        self.valid = torch.zeros(B, H, W, dtype=torch.uint8).pin_memory() if kitti and scored else None
        self.event = None


# ---- scheduling ---------------------------------------------------------------------------------------
def chains_of(pairs, warm):
    """The chains _steps runs: with warm, the pairs of each scene (consecutive pairs whose first frames share a
    directory) as one chain of pair indices; otherwise every pair on its own."""
    if not warm:
        return [[i] for i in range(len(pairs))]
    chains, last = [], None
    for i, p in enumerate(pairs):
        d = os.path.dirname(p.image1)
        if d != last:
            chains.append([])
            last = d
        chains[-1].append(i)
    return chains


def warm_schedule(lengths, batch):
    """Lockstep steps of chains with the given lengths on B = min(batch, len(lengths)) slots: each step is a list of B
    entries, (chain, k) = pair k of that chain, or None for an idle slot.  A slot runs its chain's pairs in order, one per
    step, then takes the first pair of the next chain not yet started (chains start in index order), so (chain, k > 0)
    always runs in the slot that ran (chain, k - 1) one step before -- the pair whose flow warm-starts it."""
    B = min(int(batch), len(lengths))
    cur, nxt, steps = [None] * B, 0, []
    while True:
        for i in range(B):
            c = cur[i]
            if c is not None and c[1] + 1 < lengths[c[0]]:
                cur[i] = (c[0], c[1] + 1)
                continue
            while nxt < len(lengths) and lengths[nxt] == 0:
                nxt += 1
            cur[i] = (nxt, 0) if nxt < len(lengths) else None
            nxt += cur[i] is not None
        if all(c is None for c in cur):
            return steps
        steps.append(list(cur))


# ---- the run ------------------------------------------------------------------------------------------
def _steps(engine, pairs, chains, decode, batch, workers, warm, scored, kitti=False, run=None, gt_frame=False):
    """Runs every pair of chains (lists of indices into pairs) through engine.forward and yields (row, flow, slot) per
    batch: row[i] = the pair index in batch row i (None: idle, its flow is not meaningful), flow = the engine's flow
    buffer, slot = the pinned staging that holds the batch's decoded frames (and ground truth when scored).  run (not
    with warm): the engine call per batch instead, run(left, right) -> what is yielded in place of the flow; gt_frame:
    the ground truth is a uint8 frame (_Slot).

    Chains are grouped by frame size (one CUDA graph per size), each group run by warm_schedule.  With warm, pair k > 0
    of a chain starts from forward_interpolate of the flow_low of pair k - 1 (computed on the device from the engine's
    buffer, in the same row of the previous batch) and pair 0 from a zero init: grid + 0.0 is the cold start, bit for bit.
    Worker threads decode the next batches (cv2 releases the GIL) into two pinned slots used in turn; a slot is refilled
    only after the event recorded behind its batch's work (the consumer's included) has completed."""
    from networks.utils import forward_interpolate
    groups = {}  # (H, W) -> chain indices; sizes in the order they first appear
    for c, chain in enumerate(chains):
        groups.setdefault(_png_size(pairs[chain[0]].image1), []).append(c)
    steps = []
    for hw, cidx in groups.items():
        for row in warm_schedule([len(chains[c]) for c in cidx], batch):
            steps.append((hw, len(row), [None if e is None else chains[cidx[e[0]]][e[1]] for e in row],
                          [e is not None and e[1] > 0 for e in row]))
    dev = engine.device
    pool = ThreadPoolExecutor(workers) if workers > 0 else None
    # decode this many batches ahead of the one the GPU is given (workers=0: the main thread decodes batch j + 1 while the
    # GPU runs batch j)
    depth = max(1, -(-workers // batch))

    def submit(j):
        ents = [(k, pairs[i]) for k, i in enumerate(steps[j][2]) if i is not None]
        if pool is None:
            return [(k, lambda p=p: decode(p)) for k, p in ents]
        return [(k, pool.submit(decode, p).result) for k, p in ents]

    try:
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            ahead = [submit(j) for j in range(min(depth, len(steps)))]
            shape, init = None, None
            for j, ((H, W), B, row, cont) in enumerate(steps):
                loads = ahead.pop(0)
                if j + depth < len(steps):
                    ahead.append(submit(j + depth))  # workers start on it now
                if shape != (B, H, W):
                    shape, init = (B, H, W), None
                    slots = [_Slot(B, H, W, kitti, scored, gt_frame), _Slot(B, H, W, kitti, scored, gt_frame)]
                slot = slots[j % 2]
                if slot.event is not None:
                    slot.event.synchronize()  # its last batch's copies (and work) are done
                lft, rgt = slot.left.numpy(), slot.right.numpy()
                for k, load in loads:
                    got = load()
                    lft[k], rgt[k] = got[0], got[1]
                    if scored:
                        slot.gt.numpy()[k] = got[2]
                        if kitti:
                            slot.valid.numpy()[k] = got[3]
                if warm:
                    if init is not None:
                        for k, c in enumerate(cont):
                            if not c:
                                init[k].zero_()  # a chain starts (or the row is idle): cold
                    low, flow = engine.forward(slot.left, slot.right, flow_init=init, return_low=True)
                elif run is not None:
                    flow = run(slot.left, slot.right)
                else:
                    flow = engine.forward(slot.left, slot.right)
                yield row, flow, slot
                if warm:
                    init = forward_interpolate(low)  # before the next batch overwrites flow_low
                slot.event = torch.cuda.Event()
                slot.event.record(stream)
    finally:
        if pool is not None:
            pool.shutdown(wait=True, cancel_futures=True)


def _run(engine, pairs, kitti, batch, workers, rgb, warm=False):
    """Per-pair stats [N, STATS] fp64 (host, dataset order) of engine.forward on every pair (warm: scene by scene,
    warm-started as in _steps), scored by rb_flow_metrics against the uploaded ground truth on the same stream."""
    dev = engine.device
    with torch.cuda.device(dev):
        stats = torch.empty(len(pairs), STATS, dtype=torch.float64, device=dev)
        shape = None
        for row, flow, slot in _steps(engine, pairs, chains_of(pairs, warm), lambda p: _decode(p, kitti, rgb), batch,
                                      workers, warm, True, kitti):
            B, H, W = flow.shape[:3]
            if shape != (B, H, W):
                shape = (B, H, W)
                gt = torch.empty(B, H, W, 2, dtype=torch.float32, device=dev)
                valid = torch.empty(B, H, W, dtype=torch.uint8, device=dev) if kitti else None
                ws_bytes = capi.size_query(capi.lib.rb_flow_metrics_workspace_bytes, B, H, W)
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                part = torch.empty(B, STATS, dtype=torch.float64, device=dev)
            gt.copy_(slot.gt, non_blocking=True)
            if kitti:
                valid.copy_(slot.valid, non_blocking=True)
            # every row is scored (idle rows too: the kernel is batch-invariant), the pairs' rows are kept
            capi.check(capi.lib.rb_flow_metrics(capi.ptr(flow), float(engine.flow_scale), capi.ptr(gt), capi.ptr(valid),
                                                B, H, W, None, capi.ptr(part), capi.ptr(ws), ws_bytes, capi.stream()))
            rows = [k for k, i in enumerate(row) if i is not None]
            stats.index_copy_(0, torch.tensor([row[k] for k in rows], device=dev), part[rows])
        return stats.cpu().numpy()


def _run_vimeo(engine, trips, batch, workers, rgb):
    """Per-triplet stats [N, 3] fp64 (host, list order): {values 3HW, SSE, SSIM} of engine.interpolate(im1, im3, [0.5])
    against im2, scored by rb_frame_metrics on the same stream."""
    dev = engine.device
    with torch.cuda.device(dev):
        stats = torch.empty(len(trips), FRAME_STATS, dtype=torch.float64, device=dev)
        values = np.zeros(len(trips), dtype=np.float64)
        shape = None
        for row, pred, slot in _steps(engine, trips, chains_of(trips, False), lambda t: _decode_triplet(t, rgb), batch,
                                      workers, False, True, run=lambda l, r: engine.interpolate(l, r, [0.5])[0],
                                      gt_frame=True):
            B, H, W = pred.shape[:3]
            if shape != (B, H, W):
                shape = (B, H, W)
                gt = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev)
                ws_bytes = capi.size_query(capi.lib.rb_frame_metrics_workspace_bytes, B, H, W)
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                part = torch.empty(B, FRAME_STATS, dtype=torch.float64, device=dev)
            gt.copy_(slot.gt, non_blocking=True)
            # every row is scored (idle rows too: the kernel is batch-invariant), the triplets' rows are kept
            capi.check(capi.lib.rb_frame_metrics(capi.ptr(pred), 0, capi.ptr(gt), B, H, W, capi.ptr(part), capi.ptr(ws),
                                                 ws_bytes, capi.stream()))
            rows = [k for k, i in enumerate(row) if i is not None]
            idx = [row[k] for k in rows]
            stats.index_copy_(0, torch.tensor(idx, device=dev), part[rows])
            values[idx] = 3.0 * H * W
        return np.concatenate([values[:, None], stats.cpu().numpy()], axis=1)


def psnr(sse, values):
    """10 log10(255^2 * values / sse) in fp64: inf for sse = 0."""
    with np.errstate(divide="ignore"):
        return 10.0 * np.log10(255.0 ** 2 * np.asarray(values, np.float64) / np.asarray(sse, np.float64))


def aggregate_vimeo(trips, stats):
    """fp64 aggregates of the per-triplet stats [N, 3] {values, SSE, SSIM}: psnr = the mean of the per-triplet PSNRs and
    ssim = the mean of the per-triplet SSIMs (as interpolation papers report them), and one record per triplet in list
    order with its mse = SSE / values."""
    s = np.asarray(stats, dtype=np.float64).reshape(-1, 3)
    n, sse, ssim = s.T
    p = psnr(sse, n)
    return {"psnr": float(p.mean()), "ssim": float(ssim.mean()), "n_triplets": len(s),
            "triplets": [{"dir": t.dir, "psnr": float(pi), "ssim": float(si), "mse": float(e / v)}
                         for t, pi, si, e, v in zip(trips, p, ssim, sse, n)]}


def aggregate(pairs, stats, kitti):
    """fp64 aggregates of the per-pair stats [N, STATS]: epe pooled over all counted pixels (Sintel) or the mean of the
    per-pair means (KITTI, as upstream's validate_kitti); 1px / 3px / 5px pooled fractions; f1 = 100 * outliers / pixels;
    and one record per pair in dataset order."""
    s = np.asarray(stats, dtype=np.float64).reshape(-1, STATS)
    n, se, c1, c3, c5, out = s.T
    tot = n.sum()
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = se / n
        res = {"epe": float(mean.mean() if kitti else se.sum() / tot), "1px": float(c1.sum() / tot),
               "3px": float(c3.sum() / tot), "5px": float(c5.sum() / tot), "f1": float(100.0 * out.sum() / tot),
               "pixels": int(tot), "n_pairs": len(s)}
        res["pairs"] = [{"image1": p.image1, "image2": p.image2, "gt": p.gt, "n": int(r[0]), "epe": float(r[1] / r[0]),
                         "1px": float(r[2] / r[0]), "3px": float(r[3] / r[0]), "5px": float(r[4] / r[0]),
                         "f1": float(100.0 * r[5] / r[0])} for p, r in zip(pairs, np.asarray(s))]
    return res


def _setup(model, dataset, dstypes, batch, workers, iters, warm_start, what):
    """Argument checks shared by evaluate and submit -> (kitti, splits, iterations, pad_mode)."""
    if dataset not in PROTOCOLS:
        raise ValueError(f"dataset must be one of {tuple(PROTOCOLS)} (got {dataset!r})")
    if getattr(model, "input_size", None) is not None:
        if dataset == "tapvid":
            raise ValueError(f"{what}: TAP-Vid runs its frames at 256x256 by its protocol; build the model without "
                             "input_size")
        raise ValueError(f"{what}: frames run at their own size; build the model without input_size")
    if int(batch) < 1 or int(workers) < 0:
        raise ValueError(f"{what}: batch must be >= 1 and workers >= 0 (got {batch}, {workers})")
    kitti, vimeo = dataset == "kitti", dataset == "vimeo"
    if kitti and warm_start:
        raise ValueError(f"{what}: warm_start needs frame sequences; KITTI's pairs are not sequences")
    if vimeo and warm_start:
        raise ValueError(f"{what}: warm_start needs frame sequences; Vimeo-90K's triplets are not chains")
    if dataset == "tapvid" and warm_start:
        raise ValueError(f"{what}: warm_start warm-starts flow validation; TAP-Vid tracks points through cold flows")
    if dataset == "davis" and warm_start:
        raise ValueError(f"{what}: warm_start warm-starts flow validation; DAVIS propagates labels through cold flows")
    if model._params is None:
        raise RuntimeError(f"RAFT.load(<npz>) must be called before {what}")
    splits = ("kitti",) if kitti else ("vimeo",) if vimeo else (dataset,) if dataset in ("tapvid", "davis") \
        else tuple(dstypes)
    if dataset == "sintel" and (not splits or any(d not in DSTYPES for d in splits)):
        raise ValueError(f"Sintel dstypes must be a non-empty subset of {DSTYPES} (got {dstypes!r})")
    n_iters, pad_mode = PROTOCOLS[dataset]
    return kitti, splits, n_iters if iters is None else int(iters), pad_mode


def _engine(model, n_iters, pad_mode, input_size=None):
    return RaftEngine(model._params, small=model.small, iters=n_iters, device=model.device, volume_free=model.volume_free,
                      upstream=model.upstream, mixed_precision=model.mixed_precision, pad_mode=pad_mode,
                      input_size=input_size)


def evaluate(model, root, dataset="sintel", dstypes=DSTYPES, batch=1, workers=4, iters=None, warm_start=False,
             query_mode=None, masks_out=None, keyframe_step=None):
    """Upstream RAFT's validation of a loaded networks.RAFT.RAFT model on a Sintel or KITTI-2015 training tree, or the
    interpolation quality on a Vimeo-90K triplet tree (dataset 'vimeo').

    The engine is built from the model's configuration (small, upstream, mixed_precision, volume_free, device, weights)
    with the protocol's iterations (iters overrides them) and padding.  Frames go in RGB with upstream=True and BGR
    otherwise, like the CLI.  A model with input_size is refused: validation runs frames at their own size.  Returns
    {"dataset", "iters", "pad_mode", "splits": {name: aggregate(...)}} with the splits 'clean' / 'final' (Sintel, those in
    dstypes) or 'kitti'; the same for every batch and workers.

    warm_start (Sintel only; an extension, upstream validates cold): every scene runs as a chain, each pair after the
    first starting from forward_interpolate of the previous pair's 1/8-resolution flow, as in upstream's
    create_sintel_submission(warm_start=True) -- the way to measure what the warm start does against ground truth.

    vimeo: im2 of every triplet of vimeo_triplets(root) interpolated from im1 and im3 at t = 0.5 and scored on the GPU
    (rb_frame_metrics: PSNR of the 8-bit frame the CLI would write, SSIM as skimage's Gaussian-window form); the split
    'vimeo' holds aggregate_vimeo(...).  dstypes is ignored and warm_start raises ValueError.

    tapvid: root is a TAP-Vid .pkl file or a directory of .pkl shards, scored in query_mode 'first' (the default) or
    'strided' at 256 x 256 (raft_b200.tapvid: the engine resizes the frames on the GPU); returns {"dataset", "iters",
    "query_mode", "resolution": [256, 256], "splits": {"tapvid": aggregate_tapvid(...)}}.  dstypes and workers are
    ignored, warm_start raises ValueError, and query_mode is refused for the other datasets.

    davis: root is a DAVIS-2017 tree; frame 0's annotation of every sequence of ImageSets/2017/val.txt is propagated
    through the sequence at its own size and scored by J and F (raft_b200.davis); returns {"dataset", "iters",
    "pad_mode", "splits": {"val": aggregate_davis(...)}}.  masks_out (a directory) also receives the predicted masks in
    DAVIS's results layout.  dstypes and workers are ignored and warm_start raises ValueError; masks_out is refused for
    the other datasets.  keyframe_step N (an integer >= 1) propagates the annotations of frames 0, N, 2N, ... as
    keyframes instead and scores the other frames (raft_b200.davis.run); the result then records "keyframe_step"."""
    if masks_out is not None and dataset != "davis":
        raise ValueError(f"evaluate: masks_out writes DAVIS-2017 predictions (got dataset {dataset!r})")
    if query_mode is not None and dataset != "tapvid":
        raise ValueError(f"evaluate: query_mode belongs to TAP-Vid's point tracking (got dataset {dataset!r})")
    if dataset == "tapvid" and query_mode not in (None,) + QUERY_MODES:
        raise ValueError(f"evaluate: query_mode must be one of {QUERY_MODES} (got {query_mode!r})")
    if keyframe_step is not None:
        if dataset != "davis":
            raise ValueError(f"evaluate: keyframe_step belongs to DAVIS-2017 label propagation (got dataset {dataset!r})")
        if isinstance(keyframe_step, bool) or int(keyframe_step) != keyframe_step or int(keyframe_step) < 1:
            raise ValueError(f"evaluate: keyframe_step must be an integer >= 1 (got {keyframe_step!r})")
        keyframe_step = int(keyframe_step)
    kitti, splits, n_iters, pad_mode = _setup(model, dataset, dstypes, batch, workers, iters, warm_start, "evaluate")
    if dataset == "tapvid":
        from . import tapvid
        mode = "first" if query_mode is None else query_mode
        tapvid.tapvid_files(root)  # the files checked up front
        engine = _engine(model, n_iters, pad_mode, input_size=tapvid.SIZE)
        records = tapvid.run(engine, root, mode, int(batch), model.upstream)
        return {"dataset": dataset, "iters": n_iters, "query_mode": mode, "resolution": list(tapvid.SIZE),
                "splits": {"tapvid": tapvid.aggregate_tapvid(records)}}
    if dataset == "davis":
        from . import davis
        seqs = davis.davis_sequences(root)  # every file checked up front
        engine = _engine(model, n_iters, pad_mode)
        records = davis.run(engine, seqs, int(batch), model.upstream, masks_out, keyframe_step)
        res = {"dataset": dataset, "iters": n_iters, "pad_mode": pad_mode}
        if keyframe_step is not None:
            res["keyframe_step"] = keyframe_step
        return {**res, "splits": {"val": davis.aggregate_davis(records)}}
    if dataset == "vimeo":
        trips = vimeo_triplets(root)  # every file checked up front
        engine = _engine(model, n_iters, pad_mode)
        stats = _run_vimeo(engine, trips, int(batch), int(workers), model.upstream)
        return {"dataset": dataset, "iters": n_iters, "pad_mode": pad_mode,
                "splits": {"vimeo": aggregate_vimeo(trips, stats)}}
    lists = {s: kitti_pairs(root) if kitti else sintel_pairs(root, s) for s in splits}  # every file checked up front
    engine = _engine(model, n_iters, pad_mode)
    res = {"dataset": dataset, "iters": n_iters, "pad_mode": pad_mode, "splits": {}}
    for s, pairs in lists.items():
        stats = _run(engine, pairs, kitti, int(batch), int(workers), model.upstream, warm=bool(warm_start))
        res["splits"][s] = aggregate(pairs, stats, kitti)
    return res


# ---- test-split submissions ---------------------------------------------------------------------------------------
TestPair = namedtuple("TestPair", "image1 image2 out")


def sintel_test_pairs(root, dstype="clean"):
    """MPI-Sintel test pairs of one pass, scene by scene in sorted order: the k-th frame (sorted) of
    <root>/test/<dstype>/<scene>/ with the next one, written to <dstype>/<scene>/frame%04d.flo % (k + 1) (upstream's
    create_sintel_submission)."""
    if dstype not in DSTYPES:
        raise ValueError(f"Sintel dstype must be one of {DSTYPES} (got {dstype!r})")
    img_root = os.path.join(root, "test", dstype)
    pairs = []
    for scene in _listdir(img_root, "Sintel test"):
        sdir = os.path.join(img_root, scene)
        if not os.path.isdir(sdir):
            continue
        frames = [f for f in sorted(os.listdir(sdir)) if f.endswith(".png")]
        for k, (a, b) in enumerate(zip(frames[:-1], frames[1:])):
            pairs.append(TestPair(os.path.join(sdir, a), os.path.join(sdir, b),
                                  os.path.join(dstype, scene, "frame%04d.flo" % (k + 1))))
    if not pairs:
        raise FileNotFoundError(f"Sintel: no frame pairs under {img_root}")
    return pairs


def kitti_test_pairs(root):
    """KITTI-2015 test pairs in sorted id order: <root>/testing/image_2/<id>_10.png with <id>_11.png, written to
    <id>_10.png (upstream's create_kitti_submission).  A missing second frame raises FileNotFoundError naming it."""
    img_root = os.path.join(root, "testing", "image_2")
    images = set(_listdir(img_root, "KITTI test"))
    pairs = []
    for f in sorted(images):
        if not f.endswith("_10.png"):
            continue
        second = f[:-len("_10.png")] + "_11.png"
        if second not in images:
            raise FileNotFoundError(f"KITTI: second frame {os.path.join(img_root, second)} is missing")
        pairs.append(TestPair(os.path.join(img_root, f), os.path.join(img_root, second), f))
    if not pairs:
        raise FileNotFoundError(f"KITTI: no frame pairs under {img_root}")
    return pairs


def submit(model, root, dataset, out, dstypes=DSTYPES, batch=1, workers=4, iters=None, warm_start=False):
    """Upstream RAFT's create_sintel_submission / create_kitti_submission for a loaded networks.RAFT.RAFT model: the flow
    of every test pair, at the frames' own size, in pixels (raft-small's reference-semantics flow is scaled by 8, exactly),
    with the protocol's iterations and padding as in evaluate.  Sintel: <out>/<dstype>/<scene>/frame%04d.flo (write_flo);
    KITTI: <out>/<id>_10.png (write_kitti_flow, upstream's 16-bit PNG).  warm_start (Sintel only): each scene as a chain
    warm-started by forward_interpolate, as upstream's warm_start=True.  The files are the same bytes for every batch and
    workers.  Returns the paths written, in dataset order."""
    from flow_utils import write_flo, write_kitti_flow
    if dataset == "vimeo":
        raise ValueError("submit: Vimeo-90K has no test split with hidden ground truth; evaluate scores its test list")
    if dataset == "tapvid":
        raise ValueError("submit: TAP-Vid has no test split with hidden ground truth; evaluate scores its videos")
    if dataset == "davis":
        raise ValueError("submit: DAVIS-2017 test-dev submissions are not supported; evaluate scores the val split")
    kitti, splits, n_iters, pad_mode = _setup(model, dataset, dstypes, batch, workers, iters, warm_start, "submit")
    lists = {s: kitti_test_pairs(root) if kitti else sintel_test_pairs(root, s) for s in splits}
    engine = _engine(model, n_iters, pad_mode)
    rgb, scale, written = model.upstream, np.float32(engine.flow_scale), []
    for s, pairs in lists.items():
        for row, flow, _ in _steps(engine, pairs, chains_of(pairs, warm_start), lambda p: _decode_frames(p, rgb),
                                   int(batch), int(workers), bool(warm_start), False):
            host = flow.cpu().numpy()
            for k, i in enumerate(row):
                if i is None:
                    continue
                path = os.path.join(out, pairs[i].out)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                (write_kitti_flow if kitti else write_flo)(path, host[k] * scale)
        written += [os.path.join(out, p.out) for p in pairs]
    return written


def summary_lines(res):
    """upstream evaluate.py's lines: 'Validation (clean) EPE: ..., 1px: ..., 3px: ..., 5px: ...' per Sintel pass,
    'Validation KITTI: <epe>, <f1>'; for Vimeo-90K 'Validation Vimeo-90K: PSNR: ..., SSIM: ...'; and for TAP-Vid
    'Validation TAP-Vid (<query mode>): AJ: ..., <δ_avg>: ..., OA: ...'; for DAVIS-2017
    'Validation DAVIS-2017 (val): J&F: ..., J: ..., F: ...' ('(val, a keyframe every N)' with keyframe_step N)."""
    if res["dataset"] == "davis":
        r = res["splits"]["val"]
        split = "val" if res.get("keyframe_step") is None else f"val, a keyframe every {res['keyframe_step']}"
        return ["Validation DAVIS-2017 (%s): J&F: %f, J: %f, F: %f" % (split, r["J&F-Mean"], r["J-Mean"], r["F-Mean"])]
    if res["dataset"] == "tapvid":
        r = res["splits"]["tapvid"]
        return ["Validation TAP-Vid (%s): AJ: %f, <δ_avg>: %f, OA: %f" % (res["query_mode"], r["average_jaccard"],
                                                                          r["average_pts_within_thresh"],
                                                                          r["occlusion_accuracy"])]
    if res["dataset"] == "vimeo":
        r = res["splits"]["vimeo"]
        return ["Validation Vimeo-90K: PSNR: %f, SSIM: %f" % (r["psnr"], r["ssim"])]
    if res["dataset"] == "kitti":
        r = res["splits"]["kitti"]
        return ["Validation KITTI: %f, %f" % (r["epe"], r["f1"])]
    return ["Validation (%s) EPE: %f, 1px: %f, 3px: %f, 5px: %f" % (s, r["epe"], r["1px"], r["3px"], r["5px"])
            for s, r in res["splits"].items()]
