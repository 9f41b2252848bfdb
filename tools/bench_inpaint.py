#!/usr/bin/env python
"""Object removal (rb_masked_fill, rb_inpaint_propagate, video_inpaint), one JSON line per measurement, each with the
card's name and power limit:

1. rb_masked_fill on 16 fields of 432x1024 flows (the 2T completed fields of a batch-8 pass) with seeded elliptic holes
   covering about 5 / 15 / 30 % of the frame, and on 8 fields of 1080x1920 colours with 5 % holes.  CUDA events around
   `--reps` back-to-back calls of the C entry on preallocated buffers (each call refills the same holes from the same
   known data), median of 5 windows.  Also the launches one call makes.
2. One rb_inpaint_propagate row at 1080x1920 from 432x1024 flows, window 15, a 15 % hole moving 60 px a frame and flows
   that keep the chains inside the grid.
3. video_inpaint end to end (decode, mask PNG reads, upload, bidirectional flow, masks, flow completion, temporal and
   spatial fill, PNG writes) on a seeded synthetic 24-frame 1080x1920 PNG clip with a moving elliptic mask, raft-things
   at 432x1024, 20 iterations, batch 8, window 10, 4 workers, against forward_sequence_bidirectional(check=False) alone
   on the same passes (frames already on the GPU); host clock, median of `--steps` runs.  The seeded weights' flows fail
   the forward-backward test, so every hole pixel goes to the spatial fill: the costlier path.

Seeded random weights; everything is written to a temporary directory.

    python tools/bench_inpaint.py [--reps 20] [--steps 3]
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

T, N_CLIP, ITERS, WINDOW = 8, 24, 20, 10


def ellipses(rng, n, H, W, frac):
    """n [H,W] uint8 masks of random ellipses covering about frac of the frame each."""
    import numpy as np
    yy, xx = np.mgrid[0:H, 0:W]
    out = np.zeros((n, H, W), np.uint8)
    for i in range(n):
        while out[i].mean() < frac:
            cy, cx = rng.uniform(0, H), rng.uniform(0, W)
            ry, rx = rng.uniform(0.05, 0.2) * H, rng.uniform(0.05, 0.2) * W
            out[i][((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1] = 1
    return out


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
    from raft_b200.video import interp_schedule, video_inpaint, write_labels

    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint needs a CUDA device")
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

    # 1. rb_masked_fill
    rng = np.random.default_rng(0)
    for (B, H, W, C), fracs in (((2 * T, 432, 1024, 2), (0.05, 0.15, 0.30)), ((T, 1080, 1920, 3), (0.05,))):
        vals = torch.from_numpy(rng.normal(0, 5, (B, H, W, C)).astype(np.float32)).to(dev)
        work = torch.empty_like(vals)
        nbytes = capi.size_query(capi.lib.rb_masked_fill_workspace_bytes, B, H, W, C)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        for frac in fracs:
            hole = torch.from_numpy(ellipses(rng, B, H, W, frac)).to(dev)

            def call():
                work.copy_(vals)
                capi.check(capi.lib.rb_masked_fill(capi.ptr(work), capi.ptr(hole), B, H, W, C, None, capi.ptr(ws),
                                                   nbytes, capi.stream()))
            tc, _ = timed(lambda: work.copy_(vals), args.reps)
            capi.lib.rb_launch_count_reset()
            call()
            launches = capi.lib.rb_launch_count()
            t, w = timed(call, args.reps)
            print(json.dumps({"benchmark": "masked_fill", "field_hw": [H, W], "C": C, "fields": B,
                              "hole_fraction": float(hole.float().mean()), "launches_per_call": launches,
                              "ms_per_call": (t - tc) * 1e3, "ms_per_field": (t - tc) * 1e3 / B,
                              "copy_ms_subtracted": tc * 1e3, "windows_ms": [x * 1e3 for x in w], **ctx}), flush=True)
        del vals, work, ws

    # 2. one rb_inpaint_propagate row at 1080x1920 from 432x1024 flows, window 15
    F, Hs, Ws, Hn, Wn = 31, 1080, 1920, 432, 1024
    frames = torch.from_numpy(rng.integers(0, 256, (F, Hs, Ws, 3), dtype=np.uint8)).to(dev)
    e = ellipses(rng, 1, Hs, Ws, 0.15)[0]
    hole = torch.from_numpy(np.stack([np.roll(e, 60 * f, axis=1) for f in range(F)])).to(dev)  # moves 60 px a frame
    fw = torch.from_numpy((rng.normal(0, 0.5, (F - 1, Hn, Wn, 2)) + [1.5, 0.5]).astype(np.float32)).to(dev)
    bw = (-fw).contiguous()
    rows = torch.from_numpy(inpaint_rows(F, 15)[15:16].copy()).to(dev)
    colour = torch.empty(1, Hs, Ws, 3, dtype=torch.float32, device=dev)
    status = torch.empty(1, Hs, Ws, dtype=torch.uint8, device=dev)
    a = (capi.ptr(frames), capi.ptr(hole), F, Hs, Ws, capi.ptr(fw), capi.ptr(bw), Hn, Wn, 1.0, FB_ALPHA1, FB_ALPHA2,
         capi.ptr(rows), 1, capi.ptr(colour), capi.ptr(status), capi.stream())
    t, w = timed(lambda: capi.check(capi.lib.rb_inpaint_propagate(*a)), args.reps)
    st = torch.bincount(status.flatten(), minlength=4).tolist()
    print(json.dumps({"benchmark": "inpaint_propagate_row", "frame_hw": [Hs, Ws], "flow_hw": [Hn, Wn], "window": 15,
                      "hole_fraction": float(hole[0].float().mean()), "status_counts": st[:4], "us_per_row": t * 1e6,
                      "windows_us": [x * 1e6 for x in w], **ctx}), flush=True)
    del frames, hole, fw, bw

    # 3. video_inpaint against the flow passes alone
    model = RAFT((Hn, Wn, 3), SimpleNamespace(small=False), iters=ITERS, device=dev,
                 input_size=(Hn, Wn)).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, 540 + 2 * N_CLIP + 16, 960 + 3 * N_CLIP + 16, seed0=4321)
    tmp = tempfile.mkdtemp(prefix="bench_inpaint_")
    try:
        d, md = os.path.join(tmp, "frames"), os.path.join(tmp, "masks")
        os.makedirs(d)
        os.makedirs(md)
        yy, xx = np.mgrid[0:Hs, 0:Ws]
        clip = []
        for k in range(N_CLIP):
            img = base[0, 2 * k:2 * k + 540, 3 * k:3 * k + 960]
            img = cv2.resize(np.clip(np.rint(img * 255), 0, 255).astype(np.uint8), (Ws, Hs))
            clip.append(img)
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
            m = (((yy - Hs / 2) / 200.0) ** 2 + ((xx - 400 - 40 * k) / 150.0) ** 2 < 1).astype(np.uint8)
            write_labels(os.path.join(md, f"mask_{k:04d}.png"), m)
        times = []
        for i in range(args.steps + 1):
            out = os.path.join(tmp, "out")
            shutil.rmtree(out, ignore_errors=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, info = video_inpaint(model, d, out, md, window=WINDOW, batch=T, workers=4)
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
        print(json.dumps({"benchmark": "video_inpaint",
                          "workload": f"video_inpaint, raft-things {Hn}x{Wn}, {ITERS} iterations, {N_CLIP}-frame seeded "
                                      f"synthetic {Hs}x{Ws} pan as PNG files with a moving elliptic mask, window "
                                      f"{WINDOW}, batch {T}, 4 workers, seeded weights",
                          "status_counts": info["counts"], "s_per_clip": t, "ms_per_frame": t * 1e3 / N_CLIP,
                          "flow_passes_s": tf, "flow_ms_per_frame": tf * 1e3 / N_CLIP, "clip_over_flow_passes": t / tf,
                          "runs_s": times, "flow_runs_s": flow_times, **ctx}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
