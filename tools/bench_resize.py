#!/usr/bin/env python
"""Time the resize at the input edge (rb_frames_resize, csrc/resize.cu) at 1080x1920 -> 432x1024, B = 1 and 8:

- the kernel alone (uint8 and fp32 frames): CUDA events around --reps back-to-back launches, with the bytes the
  algorithm must move (read once every source pixel a tap touches -- a 2.5x bilinear downscale skips some rows and
  columns -- and write every fp32 output) over that time;
- the two ways to get resized frames onto the GPU: the reference's host path (cv2.resize + np.float32(x) / 255 on the
  CPU, then a pinned fp32 host-to-device copy) against a pinned uint8 host-to-device copy of the native frames plus the
  kernel.  Host clock around each, ending in a device synchronise; the arms alternate.

The card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/bench_resize.py [--reps 200] [--steps 30]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

SRC, DST = (1080, 1920), (432, 1024)


def power_limit_w(index):
    try:  # read-only query
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def taps(src, dst):
    """Distinct source indices the two bilinear taps of dst outputs touch along one axis."""
    import numpy as np
    s = np.floor((np.arange(dst) + 0.5) * (src / dst) - 0.5).astype(np.int64)
    return len(np.unique(np.clip(np.concatenate([s, s + 1]), 0, src - 1)))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200, help="kernel launches per event-timed span (at least 100)")
    ap.add_argument("--steps", type=int, default=30, help="timed transfers per arm (at least 10)")
    args = ap.parse_args(argv)
    if args.reps < 100 or args.steps < 10:
        ap.error("--reps >= 100, --steps >= 10")

    import cv2
    import numpy as np
    import torch
    from networks.utils import resize_frames

    if not torch.cuda.is_available():
        raise SystemExit("bench_resize needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    (H, W), (Ho, Wo) = SRC, DST
    rng = np.random.default_rng(0)
    result = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "src": [H, W], "dst": [Ho, Wo]}
    for B in (1, 8):
        frames_u8 = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
        row = {}
        # --- the kernel alone
        for kind, host in (("u8", frames_u8), ("f32", frames_u8.astype(np.float32) / np.float32(255))):
            src = torch.from_numpy(host).to(dev)
            resize_frames(src, DST)  # warm-up: module load
            torch.cuda.synchronize()
            spans = []
            for _ in range(5):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    resize_frames(src, DST)
                e1.record()
                torch.cuda.synchronize()
                spans.append(e0.elapsed_time(e1) / args.reps)
            ms = statistics.median(spans)
            nbytes = B * taps(H, Ho) * taps(W, Wo) * 3 * src.element_size() + B * Ho * Wo * 3 * 4
            row[f"kernel_{kind}_us"] = round(ms * 1e3, 2)
            row[f"kernel_{kind}_GBps"] = round(nbytes / (ms * 1e-3) / 1e9, 1)
            row[f"kernel_{kind}_bytes"] = nbytes
        # --- host path against the GPU path, end to end
        pin_u8 = torch.from_numpy(frames_u8).pin_memory()
        pin_f32 = torch.empty(B, Ho, Wo, 3, dtype=torch.float32).pin_memory()
        out_np = pin_f32.numpy()

        def host_path():
            for b in range(B):
                out_np[b] = np.float32(cv2.resize(frames_u8[b], dsize=(Wo, Ho))) / 255.0
            d = pin_f32.to(dev, non_blocking=True)
            torch.cuda.synchronize()
            return d

        def gpu_path():
            d = resize_frames(pin_u8.to(dev, non_blocking=True), DST)
            torch.cuda.synchronize()
            return d

        assert torch.equal(host_path(), gpu_path())  # same frames either way
        times = {"host": [], "gpu": []}
        for step in range(args.steps):
            order = (("host", host_path), ("gpu", gpu_path)) if step % 2 == 0 else (("gpu", gpu_path), ("host", host_path))
            for name, fn in order:
                t0 = time.perf_counter()
                fn()
                times[name].append(time.perf_counter() - t0)
        row["host_resize_plus_f32_h2d_ms"] = round(statistics.median(times["host"]) * 1e3, 3)
        row["u8_h2d_plus_kernel_ms"] = round(statistics.median(times["gpu"]) * 1e3, 3)
        row["cv2_threads"] = cv2.getNumThreads()
        result[f"B{B}"] = row
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
