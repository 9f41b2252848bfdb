#!/usr/bin/env python
"""Golden vectors for the resize at the input/output edge (SURVEY 8(f) F3): cv2.resize (the call of the reference's
test dataflow, dataflow/test_dataflow.py:85-87) on uint8 and float32 frames, and the UNMODIFIED reference function
flow_utils.py:resize_flow (lines 277-284 of gonglixue/RAFT-tf; numpy + cv2 only) on float32 flows, including NaN and
+-inf.  Writes tests/golden/resize.npz; tests/test_resize.py holds tests/resize_oracle.py to it bit for bit and
tests/test_gpu_resize.py the kernels.  Generated with OpenCV 4.13 (bundled Intel IPP) and numpy 2.3.  Inputs are
integer formulas (no RNG, no libm), so any machine regenerates them; outputs above DIGEST_ABOVE values are stored as the
SHA-256 of their bytes (with their shape), which keeps the file small and the comparison bit for bit.  Test infrastructure;
the reference checkout is only read here:
    RAFT_REFERENCE=<reference checkout> python oracle/make_resize_golden.py"""
import hashlib
import importlib.util
import os

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIGEST_ABOVE = 20000

# (H, W, Ho, Wo): down / up / identity on each axis independently, odd sizes, 1-pixel sources, the CLI's frame sizes
# to 432x1024, an output that is not a multiple of 8
FRAME_CASES = [
    (40, 50, 20, 50), (40, 50, 40, 25), (20, 30, 45, 30), (20, 30, 20, 71), (40, 50, 40, 50), (40, 50, 17, 83),
    (37, 53, 61, 29), (1, 9, 5, 7), (9, 1, 6, 4), (1, 1, 3, 4), (50, 70, 45, 69),
    (436, 1024, 432, 1024), (1080, 1920, 432, 1024), (375, 1242, 432, 1024), (64, 96, 432, 1024),
]
# flows: the CLI's 432x1024 back to the frame sizes, and small shapes of each kind
FLOW_CASES = [
    (432, 1024, 436, 1024), (432, 1024, 375, 1242), (432, 1024, 64, 96), (54, 128, 135, 240),
    (43, 61, 80, 33), (30, 40, 30, 40), (30, 40, 30, 57), (1, 12, 7, 5), (12, 1, 5, 7),
]


def frames_u8(B, H, W):
    """Deterministic uint8 frames with edges, ramps and fine texture."""
    b, y, x, c = np.meshgrid(np.arange(B), np.arange(H), np.arange(W), np.arange(3), indexing="ij")
    v = (x * x * 3 + y * 7 + x * y + 41 * c + 97 * b) % 256
    return np.where((x // 5 + y // 3) % 2 == 0, v, 255 - v).astype(np.uint8)


def frames_f32(B, H, W):
    """Deterministic float32 frames in [0,1]: the uint8 frames over 255 plus an offset that is not a multiple of 1/255."""
    y = np.arange(H).reshape(1, H, 1, 1)
    return (frames_u8(B, H, W).astype(np.float32) * np.float32(0.99) + (y % 3).astype(np.float32)) / np.float32(257)


def flow_f32(H, W, special):
    y, x = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    u = ((x * 37 + y * 11) % 997).astype(np.float32) / np.float32(16) - np.float32(30)
    v = ((x * 13 + y * y * 5) % 613).astype(np.float32) / np.float32(8) - np.float32(40)
    f = np.stack([u, v], -1).astype(np.float32)
    if special:  # NaN and +-inf inside, on the border and in a corner
        for k, val in enumerate((np.nan, np.inf, -np.inf)):
            f[(7 * k + 3) % H, (11 * k + 5) % W, k % 2] = val
            f[0, (5 * k + 2) % W, (k + 1) % 2] = val
            f[(3 * k + 1) % H, W - 1, k % 2] = val
        f[0, 0, 0] = np.inf
        f[H - 1, W - 1, 1] = np.nan
    return f


def store(out, key, arr):
    if arr.dtype == np.float32:  # one NaN bit pattern: payloads are platform detail (tests compare NaNs as one)
        arr = arr.copy()
        arr[np.isnan(arr)] = np.float32(np.nan)
    if arr.size > DIGEST_ABOVE:
        out[key + "/sha256"] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(arr).tobytes()).digest(), np.uint8)
        out[key + "/shape"] = np.array(arr.shape)
    else:
        out[key] = arr


def main():
    spec = importlib.util.spec_from_file_location("ref_flow_utils",
                                                  os.path.join(os.environ["RAFT_REFERENCE"], "flow_utils.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    out = {}
    for H, W, Ho, Wo in FRAME_CASES:
        for kind, make in (("u8", frames_u8), ("f32", frames_f32)):
            src = make(1, H, W)[0]
            store(out, f"frames/{kind}/{H}x{W}->{Ho}x{Wo}", cv2.resize(src, dsize=(Wo, Ho)))
    for H, W, Ho, Wo in FLOW_CASES:
        for special in (False, True):
            flow = flow_f32(H, W, special)
            with np.errstate(invalid="ignore"):
                store(out, f"flow/{int(special)}/{H}x{W}->{Ho}x{Wo}", ref.resize_flow(flow.copy(), Wo, Ho))
    path = os.path.join(ROOT, "tests", "golden", "resize.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; cv2", cv2.__version__, "numpy", np.__version__)


if __name__ == "__main__":
    main()
