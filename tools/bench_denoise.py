#!/usr/bin/env python
"""Video denoising (rb_denoise_merge, rb_noise_sums, video_denoise), one JSON line per measurement, each with the card's
name and power limit:

1. rb_denoise_merge per output frame at 480x854 and 1080x1920 from 432x1024 flows, at window 1 / 3 / 5, on seeded frames
   and flows whose steps all pass the forward-backward test (every pixel merges the whole window: the costliest case).
   CUDA events around `--reps` back-to-back calls of the C entry on preallocated buffers, median of 5 windows.  Each
   line carries the model below: the fp32 operations and the DRAM bytes one output frame needs at the least.
2. rb_noise_sums per 1080x1920 frame (8 frames per call).
3. video_denoise end to end (decode, upload, bidirectional flow, merge, PNG writes) on a seeded synthetic 24-frame
   1080x1920 PNG clip, raft-things at 432x1024, 20 iterations, batch 8, window 3, 4 workers, sigma 20, against
   forward_sequence_bidirectional(check=False) alone on the same passes (frames already on the GPU); host clock, median
   of `--steps` runs.  The seeded weights' flows fail the forward-backward test almost everywhere, so the chains stop
   early: the merge's share here is a lower bound.

Seeded random weights; everything is written to a temporary directory.

    python tools/bench_denoise.py [--reps 20] [--steps 3]
"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

T, N_CLIP, ITERS, WINDOW, SIGMA = 8, 24, 20, 3, 20.0


def merge_model(Hs, Ws, Hn, Wn, window):
    """(fp32 operations, least DRAM bytes) of one output frame that merges 2 window + 1 frames at every pixel.
    Per pixel and merged frame: 6 x 5 x 3 horizontal and 5 x 5 x 3 vertical bilinear passes (3 operations each), 9
    candidates x 27 squared differences (3 each: subtract, multiply, add) and the weight and sums (about 12 each); per
    chain step two bilinear flow samples and the forward-backward test (about 40).  Bytes: every frame of the window and
    its two flows read once, the output and support written once."""
    n = 2 * window + 1
    per_frame = 3 * (6 * 5 * 3 + 5 * 5 * 3) + 9 * (27 * 3 + 12)
    ops = Hs * Ws * (n * per_frame + 2 * window * 40)
    dram = n * 3 * Hs * Ws + 2 * window * 2 * 8 * Hn * Wn + 4 * Hs * Ws
    return ops, dram


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="calls per kernel timing window (at least 5)")
    ap.add_argument("--steps", type=int, default=3, help="timed whole-clip runs (at least 3)")
    args = ap.parse_args(argv)
    if args.reps < 5 or args.steps < 3:
        ap.error("--reps >= 5, --steps >= 3")

    import cv2
    import numpy as np
    import torch
    from types import SimpleNamespace
    from networks.RAFT import RAFT
    from raft_b200 import capi, synth
    from raft_b200.engine import FB_ALPHA1, FB_ALPHA2
    from raft_b200.inpaint import inpaint_rows
    from raft_b200.video import interp_schedule, video_denoise

    if not torch.cuda.is_available():
        raise SystemExit("bench_denoise needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ctx = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(call, reps):
        for _ in range(3):
            call()
        windows = []
        for _ in range(5):
            torch.cuda.synchronize()
            a_ev.record()
            for _ in range(reps):
                call()
            b_ev.record()
            torch.cuda.synchronize()
            windows.append(a_ev.elapsed_time(b_ev) / 1e3 / reps)
        return statistics.median(windows), windows

    # 1. rb_denoise_merge, one output row per call
    rng = np.random.default_rng(0)
    Hn, Wn = 432, 1024
    F = 11
    fw = torch.full((F - 1, Hn, Wn, 2), 0.0, dtype=torch.float32, device=dev)
    fw[..., 0], fw[..., 1] = 1.5, 0.5  # a pan: every step stays on the grid away from the edges and is consistent
    bw = (-fw).contiguous()
    for Hs, Ws in ((480, 854), (1080, 1920)):
        frames = torch.from_numpy(rng.integers(0, 256, (F, Hs, Ws, 3), dtype=np.uint8)).to(dev)
        out = torch.empty(1, Hs, Ws, 3, dtype=torch.uint8, device=dev)
        support = torch.empty(1, Hs, Ws, dtype=torch.uint8, device=dev)
        for window in (1, 3, 5):
            rows = torch.from_numpy(inpaint_rows(F, window)[5:6].copy()).to(dev)
            a = (capi.ptr(frames), F, Hs, Ws, capi.ptr(fw), capi.ptr(bw), Hn, Wn, 1.0, FB_ALPHA1, FB_ALPHA2,
                 capi.ptr(rows), 1, SIGMA, capi.ptr(out), capi.ptr(support), capi.stream())
            t, w = timed(lambda: capi.check(capi.lib.rb_denoise_merge(*a)), args.reps)
            ops, dram = merge_model(Hs, Ws, Hn, Wn, window)
            print(json.dumps({"benchmark": "denoise_merge", "frame_hw": [Hs, Ws], "flow_hw": [Hn, Wn], "window": window,
                              "mean_support": float(support.float().mean()), "ms_per_frame": t * 1e3,
                              "model_fp32_ops": ops, "model_dram_bytes": dram, "tflops": ops / t / 1e12,
                              "dram_gb_s": dram / t / 1e9, "windows_ms": [x * 1e3 for x in w], **ctx}), flush=True)
        del frames, out, support
    del fw, bw

    # 2. rb_noise_sums on 8 frames of 1080x1920
    N, Hs, Ws = 8, 1080, 1920
    frames = torch.from_numpy(rng.integers(0, 256, (N, Hs, Ws, 3), dtype=np.uint8)).to(dev)
    sums = torch.empty(N, 3, dtype=torch.int64, device=dev)
    t, w = timed(lambda: capi.check(capi.lib.rb_noise_sums(capi.ptr(frames), N, Hs, Ws, capi.ptr(sums),
                                                           capi.stream())), args.reps)
    print(json.dumps({"benchmark": "noise_sums", "frame_hw": [Hs, Ws], "frames_per_call": N,
                      "us_per_frame": t * 1e6 / N, "dram_gb_s": N * 3 * Hs * Ws / t / 1e9,
                      "windows_us": [x * 1e6 for x in w], **ctx}), flush=True)
    del frames

    # 3. video_denoise against the flow passes alone
    model = RAFT((Hn, Wn, 3), SimpleNamespace(small=False), iters=ITERS, device=dev,
                 input_size=(Hn, Wn)).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, 540 + 2 * N_CLIP + 16, 960 + 3 * N_CLIP + 16, seed0=4321)
    tmp = tempfile.mkdtemp(prefix="bench_denoise_")
    try:
        d = os.path.join(tmp, "frames")
        os.makedirs(d)
        clip = []
        for k in range(N_CLIP):
            img = base[0, 2 * k:2 * k + 540, 3 * k:3 * k + 960]
            img = cv2.resize(np.clip(np.rint(img * 255), 0, 255).astype(np.uint8), (1920, 1080))
            img = np.clip(np.rint(img + SIGMA * rng.standard_normal(img.shape)), 0, 255).astype(np.uint8)
            clip.append(img)
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
        times = []
        for i in range(args.steps + 1):
            out = os.path.join(tmp, "out")
            shutil.rmtree(out, ignore_errors=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, info = video_denoise(model, d, out, SIGMA, window=WINDOW, batch=T, workers=4)
            torch.cuda.synchronize()
            if i:  # the first run captures the CUDA graph
                times.append(time.perf_counter() - t0)
        engine = model.engine()
        passes = [torch.from_numpy(np.stack([clip[f] for f in ps.frames])).to(dev) for ps in interp_schedule(N_CLIP, T)]
        flow_times = []
        for i in range(args.steps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for p in passes:
                engine.forward_sequence_bidirectional(p, check=False)
            torch.cuda.synchronize()
            if i:
                flow_times.append(time.perf_counter() - t0)
        t, tf = statistics.median(times), statistics.median(flow_times)
        print(json.dumps({"benchmark": "video_denoise",
                          "workload": f"video_denoise, raft-things {Hn}x{Wn}, {ITERS} iterations, {N_CLIP}-frame seeded "
                                      f"synthetic 1080x1920 pan with sigma {SIGMA:g} noise as PNG files, window "
                                      f"{WINDOW}, batch {T}, 4 workers, seeded weights",
                          "mean_support": info["support"], "s_per_clip": t, "ms_per_frame": t * 1e3 / N_CLIP,
                          "flow_passes_s": tf, "flow_ms_per_frame": tf * 1e3 / N_CLIP, "clip_over_flow_passes": t / tf,
                          "runs_s": times, "flow_runs_s": flow_times, **ctx}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
