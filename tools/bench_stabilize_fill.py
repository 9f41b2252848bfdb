#!/usr/bin/env python
"""Full-frame stabilization (F26), one JSON line per measurement, each with the card's name and power limit:

1. The flow extension of one batch-8 pass (8 forward and 8 backward 432x1024 flows of 1080x1920 frames, one batch of 16
   canvases): rb_flow_extend_residual + rb_masked_fill + rb_flow_extend_finish (networks.utils.extend_flows) at margins
   of 5, 12.5 and 25 % of the grid per side.  CUDA events around `--reps` calls, median of 5 windows.
2. rb_frames_warp_affine_fill per 1080x1920 frame at window 10 under a pan (similarity flows of a 6 px per frame pan on
   extended 432x1024 flows, 8 rows per call, a correction that uncovers a 40 px border), against rb_frames_warp_affine.
3. video_stabilize with and without fill on a seeded synthetic 24-frame PNG clip at 436x1024 and at 1080x1920 (flow at
   432x1024 there), raft-things, 20 iterations, sigma 10, batch 8, 4 workers; host clock, median of `--steps` runs.

Seeded random weights; everything is written to a temporary directory.

    python tools/bench_stabilize_fill.py [--reps 20] [--steps 3]
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
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

T, N_CLIP, ITERS = 8, 24, 20


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="calls per kernel timing window (at least 10)")
    ap.add_argument("--steps", type=int, default=3, help="timed whole-clip runs (at least 3)")
    args = ap.parse_args(argv)
    if args.reps < 10 or args.steps < 3:
        ap.error("--reps >= 10, --steps >= 3")

    import cv2
    import numpy as np
    import torch
    from types import SimpleNamespace
    from networks.RAFT import RAFT
    from networks.utils import extend_flows, warp_frames, warp_frames_fill
    from raft_b200 import synth
    from raft_b200.inpaint import inpaint_rows
    from raft_b200.video import video_stabilize
    import stabilize_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("bench_stabilize_fill needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ctx = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(call):
        for _ in range(3):
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

    rng = np.random.default_rng(0)
    hw, net = (1080, 1920), (432, 1024)
    pan = (1.0, 0.0, 6.0, 0.0)  # 6 frame pixels per frame
    mot = np.tile(pan, (T, 1))
    inv = (1.0, 0.0, -pan[2], 0.0)
    fw = torch.from_numpy(np.stack([O.similarity_flow(pan, *net, *hw)] * T)
                          + rng.normal(0, 0.2, (T,) + net + (2,)).astype(np.float32)).to(dev)
    bw = torch.from_numpy(np.stack([O.similarity_flow(inv, *net, *hw)] * T)).to(dev)

    # 1. the extension
    for frac in (0.05, 0.125, 0.25):
        margin = (int(round(frac * net[0])), int(round(frac * net[1])))
        t, w = timed(lambda: extend_flows(fw, bw, mot, hw, margin))
        print(json.dumps({"benchmark": "extend_flows", "flow_hw": list(net), "fields": 2 * T, "margin": list(margin),
                          "margin_fraction": frac, "ms_per_pass": t * 1e3, "windows_ms": [x * 1e3 for x in w], **ctx}),
              flush=True)

    # 2. the fill warp against the plain warp, window 10, under the pan
    F = 2 * 10 + T
    margin = (24, 48)
    efw, ebw = extend_flows(fw[:1].expand(F - 1, -1, -1, -1).contiguous(), bw[:1].expand(F - 1, -1, -1, -1).contiguous(),
                            np.tile(pan, (F - 1, 1)), hw, margin)
    frames = torch.from_numpy(rng.integers(0, 256, (F,) + hw + (3,)).astype(np.uint8)).to(dev)
    rows = inpaint_rows(F, 10)[10:10 + T]
    A = np.tile(np.array([[1.0, 0, -40.0], [0, 1, 0]]), (T, 1, 1))
    At = torch.from_numpy(A).to(dev)
    tf, wf = timed(lambda: warp_frames_fill(frames, efw, ebw, net, margin, At, rows))
    _, st = warp_frames_fill(frames, efw, ebw, net, margin, At, rows)
    sub = frames[10:10 + T].contiguous()
    tw, ww = timed(lambda: warp_frames(sub, At))
    print(json.dumps({"benchmark": "warp_affine_fill", "frame_hw": list(hw), "flow_hw": list(net), "window": 10,
                      "rows_per_call": T, "border_fraction": float((st > 0).float().mean()),
                      "status_counts": torch.bincount(st.reshape(-1).long(), minlength=4).tolist(),
                      "us_per_frame": tf * 1e6 / T, "warp_affine_us_per_frame": tw * 1e6 / T, "fill_over_warp": tf / tw,
                      "windows_us": [x * 1e6 / T for x in wf], **ctx}), flush=True)
    del efw, ebw, frames

    # 3. video_stabilize with and without fill
    for size in ((436, 1024), (1080, 1920)):
        Hs, Ws = size
        model = RAFT((436, 1024, 3) if size == (436, 1024) else (432, 1024, 3), SimpleNamespace(small=False),
                     iters=ITERS, device=dev, input_size=None if size == (436, 1024) else (432, 1024)).load(
                         synth.make_weights(False))
        base, _ = synth.make_batch(1, Hs + 2 * N_CLIP + 16, Ws + 3 * N_CLIP + 16, seed0=4321)
        jit = rng.integers(0, 8, (N_CLIP, 2))
        clip = [np.clip(np.rint(base[0, 2 * k + jit[k, 0]:2 * k + jit[k, 0] + Hs,
                                     3 * k + jit[k, 1]:3 * k + jit[k, 1] + Ws] * 255), 0, 255).astype(np.uint8)
                for k in range(N_CLIP)]
        tmp = tempfile.mkdtemp(prefix="bench_stabilize_fill_")
        try:
            d = os.path.join(tmp, "frames")
            os.makedirs(d)
            for k, img in enumerate(clip):
                cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
            res = {}
            for fill in (False, True):
                times = []
                for i in range(args.steps + 1):
                    out = os.path.join(tmp, "out")
                    shutil.rmtree(out, ignore_errors=True)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    _, info = video_stabilize(model, d, out, 10.0, batch=T, workers=4, fill=fill)
                    torch.cuda.synchronize()
                    if i:  # the first run captures the CUDA graphs
                        times.append(time.perf_counter() - t0)
                res[fill] = (statistics.median(times), times, info)
            print(json.dumps({"benchmark": "video_stabilize_fill",
                              "workload": f"video_stabilize, raft-things, {Hs}x{Ws} frames, {ITERS} iterations, "
                                          f"{N_CLIP}-frame seeded synthetic jittered pan as PNG files, sigma 10, batch "
                                          f"{T}, 4 workers, seeded weights",
                              "s_per_clip_plain": res[False][0], "s_per_clip_fill": res[True][0],
                              "fill_over_plain": res[True][0] / res[False][0], "runs_plain_s": res[False][1],
                              "runs_fill_s": res[True][1], "margin": list(res[True][2]["margin"]),
                              "counts": res[True][2]["counts"], **ctx}), flush=True)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
