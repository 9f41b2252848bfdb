"""Synthetic inputs and seeded random weights (reference npz key scheme).

There is no network access, so neither Sintel/KITTI frames nor the reference's pretrained
``release_weight/*.npz`` (readme.md:28, git-ignored) exist here.  ``make_pair`` builds smooth
textured frame pairs related by a smooth flow (SURVEY 8(d)); ``make_weights`` builds an
``.npz``-style dict keyed exactly like the TF variables the reference creates
(``<scope>/W`` HWIO, ``<scope>/b``, BN ``gamma``/``beta``/``mean/EMA``/``variance/EMA``).
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np


def _blur(a: np.ndarray, sigma: float) -> np.ndarray:
    from scipy.ndimage import gaussian_filter
    return gaussian_filter(a, sigma=(sigma, sigma, 0), mode="wrap")


def make_pair(H: int, W: int, seed: int = 1000, amp: float = 12.0, return_flow: bool = False):
    """One synthetic frame pair, float32 [H,W,3] in [0,1]; with return_flow also the [H,W,2] float32 flow (u, v) that
    warped the first frame into the second (frame 2 at p samples frame 1 at p - flow(p))."""
    from scipy.ndimage import map_coordinates
    rng = np.random.default_rng(seed)
    base = rng.random((H + 64, W + 64, 3), dtype=np.float32)
    base = 0.6 * _blur(base, 3.0) + 0.4 * _blur(base, 1.0)
    base -= base.min()
    base /= max(base.max(), 1e-6)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    ph = rng.uniform(0, 2 * np.pi, size=6)
    u = amp * (0.5 * np.sin(2 * np.pi * xs / W + ph[0]) + 0.3 * np.sin(2 * np.pi * ys / H * 2 + ph[1])
               + 0.2 * np.sin(2 * np.pi * (xs + ys) / (W + H) * 3 + ph[2]))
    v = amp * 0.5 * (0.5 * np.sin(2 * np.pi * ys / H + ph[3]) + 0.3 * np.sin(2 * np.pi * xs / W * 2 + ph[4])
                     + 0.2 * np.sin(2 * np.pi * (xs - ys) / (W + H) * 3 + ph[5]))
    f1 = base[32:32 + H, 32:32 + W].copy()
    f2 = np.stack([map_coordinates(base[..., c], [ys + 32 - v, xs + 32 - u], order=1, mode="nearest")
                   for c in range(3)], axis=-1)
    f2 = f2 + rng.normal(0, 0.01, f2.shape).astype(np.float32)
    frames = (f1.astype(np.float32), np.clip(f2, 0, 1).astype(np.float32))
    return frames + (np.stack([u, v], -1).astype(np.float32),) if return_flow else frames


def write_sintel_tree(root: str, scenes: int, frames: int, H: int, W: int, seed: int = 2000,
                      dstypes: Tuple[str, ...] = ("clean", "final")) -> int:
    """A dataset in MPI-Sintel's training layout under root (training/<dstype>/scene_<i>/frame_NNNN.png as 8-bit PNG,
    training/flow/scene_<i>/frame_NNNN.flo) from make_pair: frames 2j+1 and 2j+2 of a scene are one synthetic pair and the
    ground truth of frame 2j+1 is the flow that made it; frame 2j+2 and the next pair's first frame are unrelated and get a
    zero ground truth.  'final' holds the 'clean' frames at lower contrast, so both share the ground truth, as in Sintel.
    Returns the number of pairs per dstype."""
    import os

    import cv2
    from flow_utils import write_flo
    for i in range(scenes):
        fdir = os.path.join(root, "training", "flow", f"scene_{i}")
        os.makedirs(fdir, exist_ok=True)
        for j in range(0, frames, 2):
            f1, f2, flow = make_pair(H, W, seed + 100 * i + j, return_flow=True)
            gts = ((j, flow), (j + 1, np.zeros_like(flow)))
            for k, g in gts:
                if k < frames - 1:
                    write_flo(os.path.join(fdir, f"frame_{k + 1:04d}.flo"), g)
            for dstype in dstypes:
                sdir = os.path.join(root, "training", dstype, f"scene_{i}")
                os.makedirs(sdir, exist_ok=True)
                for k, f in ((j, f1), (j + 1, f2)):
                    if k < frames:
                        f = f if dstype == "clean" else 0.8 * f + 0.1
                        cv2.imwrite(os.path.join(sdir, f"frame_{k + 1:04d}.png"), np.round(255 * f).astype(np.uint8))
    return scenes * (frames - 1)


def write_vimeo_tree(root: str, sizes, seed: int = 4000, shift: int = 4):
    """A dataset in Vimeo-90K's triplet layout under root: one triplet per (H, W) of sizes, <root>/sequences/<entry>/im1.png,
    im2.png, im3.png (8-bit PNGs) cropped from one textured image that moves by a seeded (dx, dy), |dx|, |dy| <= shift, per
    frame -- so im2 is the true middle frame -- and <root>/tri_testlist.txt listing the entries in order.  Returns them."""
    import os

    import cv2
    rng = np.random.default_rng(seed)
    entries = []
    for i, (H, W) in enumerate(sizes):
        m = 2 * shift
        base = rng.random((H + 2 * m, W + 2 * m, 3), dtype=np.float32)
        base = 0.6 * _blur(base, 3.0) + 0.4 * _blur(base, 1.0)
        base = (base - base.min()) / max(float(base.max() - base.min()), 1e-6)
        dy, dx = (int(v) for v in rng.integers(-shift, shift + 1, 2))
        entry = f"{i // 7 + 1:05d}/{i % 7 + 1:04d}"
        d = os.path.join(root, "sequences", entry)
        os.makedirs(d, exist_ok=True)
        for k in range(3):
            y0, x0 = m + (k - 1) * dy, m + (k - 1) * dx
            cv2.imwrite(os.path.join(d, f"im{k + 1}.png"), np.round(255 * base[y0:y0 + H, x0:x0 + W]).astype(np.uint8))
        entries.append(entry)
    with open(os.path.join(root, "tri_testlist.txt"), "w") as f:
        f.write("\n".join(entries) + "\n")
    return entries


def write_highfps_tree(root: str, split: str, sequences, H: int, W: int, seed: int = 6000, speed=(1, 0)):
    """A dataset in GOPRO_Large_all's layout under root: <root>/<split>/<name>/<i:06d>.png for each (name, n_frames) of
    sequences, 8-bit crops of one smooth seeded texture that pans by speed = (dx, dy) whole pixels per frame, as a
    240 fps camera would see it.  Returns {name: [F,H,W,3] uint8 BGR frames as written}."""
    import os

    import cv2
    rng = np.random.default_rng(seed)
    out = {}
    for name, n in sequences:
        dx, dy = speed
        m = 2 + max(abs(dx), abs(dy)) * n
        base = rng.random((H + 2 * m, W + 2 * m, 3), dtype=np.float32)
        base = 0.6 * _blur(base, 3.0) + 0.4 * _blur(base, 1.0)
        base = np.round(255 * (base - base.min()) / max(float(base.max() - base.min()), 1e-6)).astype(np.uint8)
        d = os.path.join(root, split, name)
        os.makedirs(d, exist_ok=True)
        frames = []
        for i in range(n):
            y0, x0 = m + i * dy, m + i * dx
            frames.append(base[y0:y0 + H, x0:x0 + W])
            cv2.imwrite(os.path.join(d, f"{i:06d}.png"), frames[-1])
        out[name] = np.stack(frames)
    return out


# PASCAL VOC's first colours, as DAVIS's annotations use them
DAVIS_PALETTE = np.array([[0, 0, 0], [128, 0, 0], [0, 128, 0], [128, 128, 0], [0, 0, 128], [128, 0, 128],
                          [0, 128, 128], [128, 128, 128], [64, 0, 0], [192, 0, 0], [64, 128, 0], [192, 128, 0],
                          [64, 0, 128]] + [[i, i, i] for i in range(13, 256)], dtype=np.uint8)


def write_davis_tree(root: str, sequences, H: int = 480, W: int = 854, objects: int = 2, seed: int = 5000,
                     shift: int = 3):
    """A dataset in DAVIS-2017's layout under root: per (name, n_frames) of sequences, <root>/JPEGImages/480p/<name>/
    NNNNN.jpg frames and <root>/Annotations/480p/<name>/NNNNN.png palette annotations, and <root>/ImageSets/2017/val.txt
    listing the names in order.  Each frame is a textured background with `objects` textured ellipses (labels 1..objects,
    drawn in label order, so a later one occludes an earlier one) moving by seeded whole-pixel steps of at most `shift`
    per frame; the annotations are the exact label maps.  Returns the names."""
    import os

    import cv2
    from PIL import Image
    rng = np.random.default_rng(seed)
    names = []
    for name, n in sequences:
        fdir = os.path.join(root, "JPEGImages", "480p", name)
        adir = os.path.join(root, "Annotations", "480p", name)
        os.makedirs(fdir, exist_ok=True)
        os.makedirs(adir, exist_ok=True)
        tex = [_blur(rng.random((H, W, 3), dtype=np.float32), 2.0) for _ in range(objects + 1)]
        tex = [(t - t.min()) / max(float(t.max() - t.min()), 1e-6) for t in tex]
        ys, xs = np.mgrid[0:H, 0:W]
        centre = rng.uniform([0.25 * W, 0.25 * H], [0.75 * W, 0.75 * H], (objects, 2))
        radii = rng.uniform(0.06, 0.16, (objects, 2)) * np.array([W, H])
        step = rng.integers(-shift, shift + 1, (objects, 2))
        for k in range(n):
            img = tex[0].copy()
            lab = np.zeros((H, W), np.uint8)
            for o in range(objects):
                cx, cy = centre[o] + k * step[o]
                inside = ((xs - cx) / radii[o, 0]) ** 2 + ((ys - cy) / radii[o, 1]) ** 2 <= 1.0
                lab[inside] = o + 1
                img[inside] = np.roll(tex[o + 1], (int(k * step[o, 1]), int(k * step[o, 0])), (0, 1))[inside]
            cv2.imwrite(os.path.join(fdir, f"{k:05d}.jpg"), np.round(255 * img).astype(np.uint8),
                        [cv2.IMWRITE_JPEG_QUALITY, 95])
            im = Image.frombytes("P", (W, H), lab.tobytes())
            im.putpalette(DAVIS_PALETTE.reshape(-1).tolist())
            im.save(os.path.join(adir, f"{k:05d}.png"))
        names.append(name)
    os.makedirs(os.path.join(root, "ImageSets", "2017"), exist_ok=True)
    with open(os.path.join(root, "ImageSets", "2017", "val.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    return names


def make_batch(B: int, H: int, W: int, seed0: int = 1000):
    pairs = [make_pair(H, W, seed0 + i) for i in range(B)]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


# ------------------------------------------------------------------------------------
def _encoder_shapes(name: str, small: bool, out_dim: int, norm_fn: str):
    convs, norms = {}, []
    if not small:  # BasicEncoder, model_utils.py:61-82
        convs[f"{name}/conv1"] = (7, 7, 3, 64)
        norms.append((f"{name}/norm1", 64))
        cin = 64
        for lname, dim, stride in (("layer1", 64, 1), ("layer2", 96, 2), ("layer3", 128, 2)):
            for blk, (ci, st) in enumerate(((cin, stride), (dim, 1))):
                s = f"{name}/{lname}/{blk}"
                convs[s + "/conv1"] = (3, 3, ci, dim)
                convs[s + "/conv2"] = (3, 3, dim, dim)
                norms += [(s + "/norm1", dim), (s + "/norm2", dim)]
                if st != 1:
                    convs[s + "/downsample.0"] = (1, 1, ci, dim)
                    norms.append((s + "/downsample.1", dim))
            cin = dim
        convs[f"{name}/conv2"] = (1, 1, 128, out_dim)
    else:  # SmallEncoder, model_utils.py:84-105
        convs[f"{name}/conv1"] = (7, 7, 3, 32)
        norms.append((f"{name}/norm1", 32))
        cin = 32
        for lname, dim, stride in (("layer1", 32, 1), ("layer2", 64, 2), ("layer3", 96, 2)):
            for blk, (ci, st) in enumerate(((cin, stride), (dim, 1))):
                s = f"{name}/{lname}/{blk}"
                convs[s + "/conv1"] = (1, 1, ci, dim // 4)
                convs[s + "/conv2"] = (3, 3, dim // 4, dim // 4)
                convs[s + "/conv3"] = (1, 1, dim // 4, dim)
                norms += [(s + "/norm1", dim // 4), (s + "/norm2", dim // 4), (s + "/norm3", dim)]
                if st != 1:
                    convs[s + "/downsample.0"] = (1, 1, ci, dim)
                    norms.append((s + "/downsample.1", dim))
            cin = dim
        convs[f"{name}/conv2"] = (1, 1, 96, out_dim)
    return convs, (norms if norm_fn == "batch" else [])


def update_block_shapes(small: bool) -> Dict[str, tuple]:
    """Hot-path conv shapes (SURVEY 8(a) 'Hot-path weights')."""
    u = "update_block"
    if not small:
        return {
            f"{u}/encoder/convc1": (1, 1, 324, 256), f"{u}/encoder/convc2": (3, 3, 256, 192),
            f"{u}/encoder/convf1": (7, 7, 2, 128), f"{u}/encoder/convf2": (3, 3, 128, 64),
            f"{u}/encoder/conv": (3, 3, 256, 126),
            f"{u}/gru/convz1": (1, 5, 384, 128), f"{u}/gru/convr1": (1, 5, 384, 128),
            f"{u}/gru/convq1": (1, 5, 384, 128),
            f"{u}/gru/convz2": (5, 1, 384, 128), f"{u}/gru/convr2": (5, 1, 384, 128),
            f"{u}/gru/convq2": (5, 1, 384, 128),
            f"{u}/flow_head/conv1": (3, 3, 128, 256), f"{u}/flow_head/conv2": (3, 3, 256, 2),
            f"{u}/mask/0": (3, 3, 128, 256), f"{u}/mask/2": (1, 1, 256, 576),
        }
    return {
        f"{u}/encoder/convc1": (1, 1, 196, 96), f"{u}/encoder/convf1": (7, 7, 2, 64),
        f"{u}/encoder/convf2": (3, 3, 64, 32), f"{u}/encoder/conv": (3, 3, 128, 80),
        f"{u}/gru/convz": (3, 3, 242, 96), f"{u}/gru/convr": (3, 3, 242, 96),
        f"{u}/gru/convq": (3, 3, 242, 96),
        f"{u}/flow_head/conv1": (3, 3, 96, 128), f"{u}/flow_head/conv2": (3, 3, 128, 2),
    }


def make_weights(small: bool = False, seed: int = 7, gain: float = 1.0) -> Dict[str, np.ndarray]:
    """Seeded random weights in the reference's variable naming.

    He-normal conv kernels (std = gain*sqrt(2/fan_in)), small non-zero biases (so a dropped
    bias is caught), ``flow_head/conv2`` scaled by 0.05 and ``mask/2`` by 0.5 so that the
    recurrence moves the flow by a fraction of a pixel per iteration instead of exploding;
    BN statistics are non-trivial (gamma~U(.8,1.2), beta~N(0,.05), mean~N(0,.05), var~U(.8,1.2)).
    """
    rng = np.random.default_rng(seed)
    p: Dict[str, np.ndarray] = {}
    convs: Dict[str, tuple] = {}
    norms = []
    hidden, ctx, fdim = (96, 64, 128) if small else (128, 128, 256)
    c, n = _encoder_shapes("fnet", small, fdim, "instance")
    convs.update(c)
    c, n2 = _encoder_shapes("cnet", small, hidden + ctx, "none" if small else "batch")
    convs.update(c)
    norms += n + n2
    convs.update(update_block_shapes(small))
    for k, shp in convs.items():
        fan_in = shp[0] * shp[1] * shp[2]
        std = gain * np.sqrt(2.0 / fan_in)
        if k.endswith("flow_head/conv2"):
            std *= 0.05
        if k.endswith("mask/2"):
            std *= 0.5
        p[k + "/W"] = rng.normal(0, std, shp).astype(np.float32)
        p[k + "/b"] = rng.normal(0, 0.02, (shp[3],)).astype(np.float32)
    for s, ch in norms:
        p[s + "/gamma"] = rng.uniform(0.8, 1.2, ch).astype(np.float32)
        p[s + "/beta"] = rng.normal(0, 0.05, ch).astype(np.float32)
        p[s + "/mean/EMA"] = rng.normal(0, 0.05, ch).astype(np.float32)
        p[s + "/variance/EMA"] = rng.uniform(0.8, 1.2, ch).astype(np.float32)
    return p
