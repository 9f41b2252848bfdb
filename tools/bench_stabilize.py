#!/usr/bin/env python
"""Video stabilization (rb_global_motion, rb_frames_warp_affine, video_stabilize), one JSON line per measurement, each
with the card's name and power limit:

1. rb_global_motion per pass over B = 1 and 8 pairs of 436x1024 flows (frames 436x1024), with the default rounds: a
   seeded similarity flow with noise and 15% occluded pixels.  CUDA events around `--reps` back-to-back calls of the C
   entry on preallocated buffers, median of 5 windows.
2. rb_frames_warp_affine per frame at 1080x1920 and 2160x3840 (8 frames per call, 3 channels, a small rotation and
   zoom), against its byte model (one frame read, one written: 2 H W 3 bytes) and against torch's affine_grid +
   grid_sample (bilinear, border padding, align_corners=True) on the same frames with the uint8 -> fp32 -> uint8
   conversions and layout changes included.
3. video_stabilize end to end (decode, upload, bidirectional flow with the occlusion check, global motion, host path,
   second decode, warp, PNG writes) on a seeded synthetic 24-frame 436x1024 PNG clip, raft-things, 20 iterations,
   batch 8, 4 workers, against the flow passes alone (forward_sequence_bidirectional with the check on the same
   passes, frames already on the GPU); host clock, median of `--steps` runs.

Seeded random weights; everything is written to a temporary directory.

    python tools/bench_stabilize.py [--reps 100] [--steps 3]
"""
import argparse
import json
import math
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

T, N_CLIP, ITERS, N_WARP = 8, 24, 20, 8


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100, help="calls per kernel timing window (at least 20)")
    ap.add_argument("--steps", type=int, default=3, help="timed whole-clip runs (at least 3)")
    args = ap.parse_args(argv)
    if args.reps < 20 or args.steps < 3:
        ap.error("--reps >= 20, --steps >= 3")

    import cv2
    import numpy as np
    import torch
    import torch.nn.functional as Fn
    from types import SimpleNamespace
    from networks.RAFT import RAFT
    from raft_b200 import capi, synth
    from raft_b200.stabilize import MOTION_CAUCHY, MOTION_MIN_WEIGHT, MOTION_ROUNDS
    from raft_b200.video import interp_schedule, video_stabilize
    import stabilize_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("bench_stabilize needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ctx = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(call):
        for _ in range(5):
            call()
        windows = []
        for _ in range(5):
            torch.cuda.synchronize()
            a_ev.record()
            for _ in range(args.reps):
                call()
            b_ev.record()
            torch.cuda.synchronize()
            windows.append(a_ev.elapsed_time(b_ev) / 1e3 / args.reps)
        return statistics.median(windows), windows

    # 1. rb_global_motion
    rng = np.random.default_rng(0)
    H, W = 436, 1024
    for B in (1, 8):
        flow = np.stack([O.similarity_flow((1.001, 0.002, 3.0, -1.5), H, W, H, W) for _ in range(B)])
        flow += rng.normal(0, 0.2, flow.shape).astype(np.float32)
        f = torch.from_numpy(flow).to(dev)
        occ = torch.from_numpy((rng.random((B, H, W)) < 0.15).astype(np.uint8)).to(dev)
        params = torch.empty(B, 4, dtype=torch.float64, device=dev)
        weight = torch.empty(B, dtype=torch.float64, device=dev)
        flags = torch.empty(B, dtype=torch.uint8, device=dev)
        nbytes = capi.size_query(capi.lib.rb_global_motion_workspace_bytes, B, H, W)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        a = (capi.ptr(f), capi.ptr(occ), B, H, W, H, W, 1.0, MOTION_ROUNDS, MOTION_CAUCHY, MOTION_MIN_WEIGHT,
             capi.ptr(params), capi.ptr(weight), capi.ptr(flags), None, capi.ptr(ws), nbytes, capi.stream())
        t, w = timed(lambda: capi.check(capi.lib.rb_global_motion(*a)))
        print(json.dumps({"benchmark": "global_motion", "flow_hw": [H, W], "B": B, "rounds": MOTION_ROUNDS,
                          "launches": 2 * (MOTION_ROUNDS + 1), "us_per_pass": t * 1e6, "us_per_pair": t * 1e6 / B,
                          "windows_us": [x * 1e6 for x in w], **ctx}), flush=True)
        del f, occ, ws

    # 2. rb_frames_warp_affine against its byte model and torch's affine_grid + grid_sample
    th, s = 0.01, 1.05
    for Hs, Ws in ((1080, 1920), (2160, 3840)):
        frames = torch.from_numpy(rng.integers(0, 256, (N_WARP, Hs, Ws, 3)).astype(np.uint8)).to(dev)
        out = torch.empty_like(frames)
        cx, cy = 0.5 * (Ws - 1), 0.5 * (Hs - 1)
        L = np.array([[s * math.cos(th), -s * math.sin(th)], [s * math.sin(th), s * math.cos(th)]])
        A = np.concatenate([L, (np.array([cx, cy]) - L @ np.array([cx, cy]))[:, None]], 1)
        At = torch.from_numpy(np.tile(A, (N_WARP, 1, 1))).to(dev)
        a = (capi.ptr(frames), capi.ptr(At), N_WARP, Hs, Ws, 3, capi.ptr(out), capi.stream())
        t, w = timed(lambda: capi.check(capi.lib.rb_frames_warp_affine(*a)))
        # the same map for affine_grid (align_corners=True: -1 / +1 are the centres of the edge pixels)
        N = np.diag([2.0 / (Ws - 1), 2.0 / (Hs - 1), 1.0])
        N[:2, 2] = -1.0
        theta = (N @ np.vstack([A, [0, 0, 1]]) @ np.linalg.inv(N))[:2]
        theta_t = torch.from_numpy(np.tile(theta, (N_WARP, 1, 1))).float().to(dev)

        def torch_warp():
            x = frames.permute(0, 3, 1, 2).float()
            grid = Fn.affine_grid(theta_t, list(x.shape), align_corners=True)
            y = Fn.grid_sample(x, grid, mode="bilinear", padding_mode="border", align_corners=True)
            return y.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
        tt, wt = timed(torch_warp)
        nbytes = 2 * Hs * Ws * 3
        diff = (torch_warp().int() - out.int()).abs()
        print(json.dumps({"benchmark": "warp_affine", "frame_hw": [Hs, Ws], "frames_per_call": N_WARP,
                          "us_per_frame": t * 1e6 / N_WARP, "GB_per_s": nbytes * N_WARP / t / 1e9,
                          "share_of_3350_GBps": nbytes * N_WARP / t / 3.35e12,
                          "torch_affine_grid_sample_us_per_frame": tt * 1e6 / N_WARP, "torch_over_kernel": tt / t,
                          "max_byte_diff_vs_torch": int(diff.max()), "windows_us": [x * 1e6 / N_WARP for x in w],
                          "torch_windows_us": [x * 1e6 / N_WARP for x in wt], **ctx}), flush=True)
        del frames, out

    # 3. video_stabilize against the flow passes alone
    Hc, Wc = 436, 1024
    model = RAFT((Hc, Wc, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, Hc + 2 * N_CLIP + 16, Wc + 3 * N_CLIP + 16, seed0=4321)
    jit = rng.integers(0, 8, (N_CLIP, 2))
    clip = [np.clip(np.rint(base[0, 2 * k + jit[k, 0]:2 * k + jit[k, 0] + Hc, 3 * k + jit[k, 1]:3 * k + jit[k, 1] + Wc]
                            * 255), 0, 255).astype(np.uint8) for k in range(N_CLIP)]
    tmp = tempfile.mkdtemp(prefix="bench_stabilize_")
    try:
        d = os.path.join(tmp, "frames")
        os.makedirs(d)
        for k, img in enumerate(clip):
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
        times = []
        for i in range(args.steps + 1):
            out = os.path.join(tmp, "out")
            shutil.rmtree(out, ignore_errors=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            video_stabilize(model, d, out, 10.0, batch=T, workers=4)
            torch.cuda.synchronize()
            if i:  # the first run captures the CUDA graph
                times.append(time.perf_counter() - t0)
        engine = model.engine()
        passes = [torch.from_numpy(np.stack([clip[f] for f in ps.frames])).to(dev)
                  for ps in interp_schedule(N_CLIP, T)]
        flow_times = []
        for i in range(args.steps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for p in passes:
                engine.forward_sequence_bidirectional(p, check=True)
            torch.cuda.synchronize()
            if i:
                flow_times.append(time.perf_counter() - t0)
        t, tf = statistics.median(times), statistics.median(flow_times)
        print(json.dumps({"benchmark": "video_stabilize",
                          "workload": f"video_stabilize, raft-things {Hc}x{Wc}, {ITERS} iterations, {N_CLIP}-frame "
                                      f"seeded synthetic jittered pan as PNG files, sigma 10, batch {T}, 4 workers, "
                                      "seeded weights",
                          "s_per_clip": t, "ms_per_frame": t * 1e3 / N_CLIP, "flow_passes_s": tf,
                          "clip_over_flow_passes": t / tf, "runs_s": times, "flow_runs_s": flow_times, **ctx}),
              flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
