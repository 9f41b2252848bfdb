#!/usr/bin/env python
"""Motion segmentation (rb_homography_motion, rb_motion_evidence, rb_motion_segment), one JSON line per measurement,
each with the card's name and power limit:

1. the homography fit of one batch-8 pass: 16 fields at 432x1024 from 1080x1920 frames, 8 rounds, against
   rb_global_motion (8 rounds) on the same fields;
2. the evidence launch of that pass (9 frames at 432x1024);
3. rb_motion_segment per output frame at 480x854 and 1080x1920 from 432x1024 flows, at window 0 / 3 / 8, on seeded
   flows whose steps all pass the forward-backward test (every chain runs the whole window: the costliest case), the C
   entry called directly on a device rows table (no host copy or check in the timed loop);
4. video_segment_motion end to end (decode, upload, bidirectional flow with the occlusion check, fit, evidence,
   segmentation, PNG writes) on a seeded synthetic 24-frame 1080x1920 PNG clip, raft-things at 432x1024, 20 iterations,
   batch 8, window 3, 4 workers, against forward_sequence_bidirectional(check=True) alone on the same passes (frames
   already on the GPU); host clock, median of `--steps` runs.

1-3: CUDA events around `--reps` back-to-back calls on preallocated inputs, median of 5 windows.  Seeded data and
weights; files go to a temporary directory.

    python tools/bench_motionseg.py [--reps 20] [--steps 3]
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


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="calls per timing window (at least 5)")
    ap.add_argument("--steps", type=int, default=3, help="timed whole-clip runs (at least 3)")
    args = ap.parse_args(argv)
    if args.reps < 5 or args.steps < 3:
        ap.error("--reps >= 5, --steps >= 3")
    import torch
    from networks import utils as U
    from raft_b200 import motionseg as M
    if not torch.cuda.is_available():
        raise SystemExit("bench_motionseg: needs a CUDA device")
    dev = torch.device("cuda:0")
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(0)}

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                fn()
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b) / args.reps)
        return statistics.median(ms)

    g = torch.Generator(device=dev).manual_seed(0)
    T, Hn, Wn, src = 8, 432, 1024, (1080, 1920)
    fw = torch.randn(T, Hn, Wn, 2, device=dev, generator=g) * 0.3 + 1.0
    bw = -fw
    flow = torch.cat([fw, bw])
    occ = torch.zeros(2 * T, Hn, Wn, dtype=torch.uint8, device=dev)
    params, _, reliable = U.global_motion(flow, occ, src)
    gm = timed(lambda: U.global_motion(flow, occ, src, rounds=M.ROUNDS - 1))
    hm = timed(lambda: U.homography_motion(flow, occ, src, params, reliable, rounds=M.ROUNDS))
    print(json.dumps(dict(card, what="fit per batch-8 pass", fields=2 * T, net=[Hn, Wn], rounds=M.ROUNDS,
                          homography_ms=round(hm, 4), global_motion_ms=round(gm, 4))))
    H, flags = U.homography_motion(flow, occ, src, params, reliable)
    ev_ms = timed(lambda: U.motion_evidence(fw, bw, occ[:T], occ[T:], H, flags, src))
    print(json.dumps(dict(card, what="evidence per batch-8 pass", frames=T + 1, net=[Hn, Wn], ms=round(ev_ms, 4))))
    F = 17
    fw2 = torch.full((F - 1, Hn, Wn, 2), 0.25, device=dev)
    bw2 = -fw2
    ev = torch.rand(F, Hn, Wn, 2, device=dev, generator=g)
    from raft_b200 import capi
    from raft_b200.engine import FB_ALPHA1, FB_ALPHA2
    for hw in ((480, 854), (1080, 1920)):
        mask = torch.empty(1, *hw, dtype=torch.uint8, device=dev)
        status = torch.empty_like(mask)
        for window in (0, 3, 8):
            rows = torch.from_numpy(M.segment_rows(F, window)[8:9].copy()).to(dev)  # the middle frame: whole window
            a = (capi.ptr(ev), F, Hn, Wn, capi.ptr(fw2), capi.ptr(bw2), hw[0], hw[1], 1.0, FB_ALPHA1, FB_ALPHA2,
                 capi.ptr(rows), 1, capi.ptr(mask), capi.ptr(status), capi.stream())
            ms = timed(lambda: capi.check(capi.lib.rb_motion_segment(*a)))
            print(json.dumps(dict(card, what="rb_motion_segment per frame", frame=list(hw), net=[Hn, Wn],
                                  window=window, ms=round(ms, 4))))
    del ev, fw2, bw2, fw, bw, flow

    # 4. video_segment_motion against the flow passes alone
    import cv2
    import numpy as np
    from types import SimpleNamespace
    from networks.RAFT import RAFT
    from raft_b200 import synth
    from raft_b200.video import interp_schedule, video_segment_motion
    n_clip, batch = 24, 8
    model = RAFT((Hn, Wn, 3), SimpleNamespace(small=False), iters=20, device=dev,
                 input_size=(Hn, Wn)).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, 540 + 2 * n_clip + 16, 960 + 3 * n_clip + 16, seed0=4321)
    tmp = tempfile.mkdtemp(prefix="bench_motionseg_")
    try:
        d = os.path.join(tmp, "frames")
        os.makedirs(d)
        clip = []
        for k in range(n_clip):
            img = base[0, 2 * k:2 * k + 540, 3 * k:3 * k + 960]
            img = cv2.resize(np.clip(np.rint(img * 255), 0, 255).astype(np.uint8), (1920, 1080))
            clip.append(img)
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
        times = []
        for i in range(args.steps + 1):
            out = os.path.join(tmp, "out")
            shutil.rmtree(out, ignore_errors=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            video_segment_motion(model, d, out, window=3, batch=batch, workers=4)
            torch.cuda.synchronize()
            if i:  # the first run captures the CUDA graph
                times.append(time.perf_counter() - t0)
        engine = model.engine()
        passes = [torch.from_numpy(np.stack([clip[f] for f in ps.frames])).to(dev)
                  for ps in interp_schedule(n_clip, batch)]
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
        print(json.dumps(dict(card, what="video_segment_motion per frame",
                              workload=f"raft-things {Hn}x{Wn}, 20 iterations, {n_clip}-frame seeded synthetic "
                                       f"1080x1920 pan as PNG files, window 3, batch {batch}, 4 workers, seeded weights",
                              ms_per_frame=round(t * 1e3 / n_clip, 3), flow_ms_per_frame=round(tf * 1e3 / n_clip, 3),
                              clip_over_flow_passes=round(t / tf, 4), runs_s=times, flow_runs_s=flow_times)),
              flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)

if __name__ == "__main__":
    main()
