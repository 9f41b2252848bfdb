#!/usr/bin/env python
"""Point tracking (rb_track_points and video_track), one JSON line per measurement:

1. kernel: rb_track_points over T = 8 steps of 436x1024 flows, for 1 024 sparse queries (random positions on frame 0)
   and a dense grid (every pixel of frame 0, 446 464 queries).  The flows are a seeded smooth random field (a few
   pixels of motion) with bw = -fw plus noise, so most tracks stay inside and the gathers have a video's locality.  CUDA
   events around `--reps` back-to-back calls of the C entry on preallocated buffers, median of 5 such windows (the state
   carries from call to call, so later windows step points that have already moved).  Bytes: the model's per query and
   step -- 8 float2 gathers (64 B, mostly served by the L2) and 9 B written -- next to the HBM bytes a cold read of both
   flow fields would take.
   The first launch is checked against tests/track_oracle.py bit for bit.
2. video_track: end to end (decode, upload, bidirectional flow, tracking, memory-mapped writes) on a seeded synthetic
   24-frame 436x1024 pan as PNG files, batch 8, 4 workers, 1 024 sparse queries and a grid of every 4th pixel; host clock
   around each call, which returns after its last write; median of `--steps` runs per query set.  The cost of
   video_track(backward=True): 1 024 sparse queries on random frames, the largest query frame the last one, so the reverse
   sweep re-runs every flow pass; timed like the others with backward=False and backward=True, in alternation.
3. flow only: forward_sequence_bidirectional(check=False) alone on the same clip's passes (frames already on the
   device), the same passes video_track runs; CUDA events around all passes, median of `--steps`.

raft-things, 20 iterations, seeded random weights, frames at their own 436x1024 size.  Frames are written to a temporary
directory.

    python tools/bench_track.py [--reps 200] [--steps 3]
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

H_IMG, W_IMG, T, N_SPARSE, N_CLIP, ITERS = 436, 1024, 8, 1024, 24, 20


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200, help="launches per kernel timing window (at least 50)")
    ap.add_argument("--steps", type=int, default=3, help="timed whole-clip runs per query set (at least 3)")
    args = ap.parse_args(argv)
    if args.reps < 50 or args.steps < 3:
        ap.error("--reps >= 50, --steps >= 3")

    import cv2
    import numpy as np
    import torch
    from scipy.ndimage import gaussian_filter
    from types import SimpleNamespace
    import track_oracle as O
    from networks.RAFT import RAFT
    from networks.utils import track_points
    from raft_b200 import capi, synth
    from raft_b200.video import interp_schedule, track_grid, video_track

    if not torch.cuda.is_available():
        raise SystemExit("bench_track needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    gpu, watts = torch.cuda.get_device_name(dev), power_limit_w(dev.index or 0)
    ctx = {"gpu": gpu, "power_limit_w": watts}
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    # 1. the kernel
    rng = np.random.default_rng(0)
    f = gaussian_filter(rng.normal(0, 1, (T, H_IMG, W_IMG, 2)), sigma=(0, 24, 24, 0), mode="wrap")
    fw = (4.0 * f / np.abs(f).max()).astype(np.float32)
    bw = (-fw + rng.normal(0, 0.3, fw.shape)).astype(np.float32)
    fw_d, bw_d = torch.from_numpy(fw).to(dev), torch.from_numpy(bw).to(dev)
    sparse = np.stack([rng.uniform(0, W_IMG - 1, N_SPARSE), rng.uniform(0, H_IMG - 1, N_SPARSE)], -1).astype(np.float32)
    dense = track_grid(H_IMG, W_IMG, 1)[:, 1:].astype(np.float32)
    for kind, qpos in (("sparse", sparse), ("dense", dense)):
        N = len(qpos)
        qframe = torch.zeros(N, dtype=torch.int32, device=dev)
        qp = torch.from_numpy(qpos).to(dev)
        tracks, status, state = track_points(fw_d, bw_d, qframe, qp)
        if kind == "sparse":
            want_t, want_s, _ = O.track(fw, bw, np.zeros(N), qpos)
            assert O.same_bits(tracks.cpu().numpy(), want_t) and np.array_equal(status.cpu().numpy(), want_s)
        final = status[-1].cpu().numpy()
        pos, st = state
        launch = (capi.ptr(fw_d), capi.ptr(bw_d), T, H_IMG, W_IMG, T, 1.0, 0.01, 0.5, capi.ptr(qframe), capi.ptr(qp), N, 0,
                  capi.ptr(pos), capi.ptr(st), capi.ptr(tracks), capi.ptr(status), capi.stream())

        def call():  # the C entry on preallocated buffers: no allocation in the timed window
            capi.check(capi.lib.rb_track_points(*launch))

        for _ in range(20):
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
        t = statistics.median(windows)
        model_bytes = N * T * (64 + 9)
        print(json.dumps({"benchmark": "track_kernel", "queries": kind, "N": N, "T": T, "H": H_IMG, "W": W_IMG,
                          "us_per_launch": t * 1e6, "ns_per_query_step": t * 1e9 / (N * T),
                          "gather_and_store_bytes": model_bytes, "flow_field_bytes": fw.nbytes + bw.nbytes,
                          "status_counts_last_frame": [int((final == k).sum()) for k in range(4)],
                          "reps": args.reps, "windows_us": [w * 1e6 for w in windows], **ctx}),
              flush=True)

    # 2. and 3. end to end and the flow alone
    model = RAFT((H_IMG, W_IMG, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, H_IMG + 2 * N_CLIP, W_IMG + 3 * N_CLIP, seed0=4321)
    pan = [np.clip(np.rint(base[0, 2 * k:2 * k + H_IMG, 3 * k:3 * k + W_IMG] * 255), 0, 255).astype(np.uint8)
           for k in range(N_CLIP)]
    tmp = tempfile.mkdtemp(prefix="bench_track_")
    try:
        d = os.path.join(tmp, "frames")
        os.makedirs(d)
        for k, img in enumerate(pan):
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
        queries = np.concatenate([np.zeros((N_SPARSE, 1)), sparse.astype(np.float64)], -1)
        for kind, kw in (("sparse", {"queries": queries}), ("grid4", {"grid": 4})):
            times = []
            for i in range(args.steps + 1):
                out = os.path.join(tmp, "out")
                shutil.rmtree(out, ignore_errors=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                video_track(model, d, out, batch=T, workers=4, **kw)
                torch.cuda.synchronize()
                if i:  # the first run captures the CUDA graph
                    times.append(time.perf_counter() - t0)
            st = np.load(os.path.join(tmp, "out", "status.npy"))
            t = statistics.median(times)
            print(json.dumps({"benchmark": "video_track", "queries": kind, "N": int(st.shape[1]),
                              "workload": f"video_track, raft-things {H_IMG}x{W_IMG}, {ITERS} iterations, {N_CLIP}-frame "
                                          f"seeded synthetic pan as PNG files, batch {T}, 4 workers, seeded random weights",
                              "s_per_clip": t, "ms_per_frame": t * 1e3 / N_CLIP, "runs_s": times,
                              "status_counts_last_frame": [int((st[-1] == k).sum()) for k in range(4)], **ctx}),
                  flush=True)
        spread = np.concatenate([rng.integers(0, N_CLIP, (N_SPARSE, 1)), sparse.astype(np.float64)], -1)
        spread[-1, 0] = N_CLIP - 1  # the largest query frame is the last frame: the reverse sweep runs every pass
        times = {False: [], True: []}
        for i in range(args.steps + 1):
            for backward in (False, True):
                out = os.path.join(tmp, "out")
                shutil.rmtree(out, ignore_errors=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                video_track(model, d, out, queries=spread, batch=T, workers=4, backward=backward)
                torch.cuda.synchronize()
                if i:
                    times[backward].append(time.perf_counter() - t0)
        st = np.load(os.path.join(tmp, "out", "status.npy"))
        fwd, both = statistics.median(times[False]), statistics.median(times[True])
        print(json.dumps({"benchmark": "video_track_backward", "queries": "spread", "N": N_SPARSE,
                          "largest_query_frame": N_CLIP - 1,
                          "workload": f"video_track with and without backward=True, raft-things {H_IMG}x{W_IMG}, "
                                      f"{ITERS} iterations, {N_CLIP}-frame seeded synthetic pan as PNG files, batch {T}, "
                                      f"4 workers, queries on random frames",
                          "s_per_clip_forward": fwd, "s_per_clip_backward": both, "ratio": both / fwd,
                          "runs_forward_s": times[False], "runs_backward_s": times[True],
                          "status_counts_first_frame": [int((st[0] == k).sum()) for k in range(4)], **ctx}),
              flush=True)
        engine = model.engine()
        passes = interp_schedule(N_CLIP, T)
        clips = [torch.from_numpy(np.stack([pan[i] for i in p.frames])).to(dev) for p in passes]
        for c in clips:
            engine.forward_sequence_bidirectional(c, check=False)
        runs = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            a_ev.record()
            for c in clips:
                engine.forward_sequence_bidirectional(c, check=False)
            b_ev.record()
            torch.cuda.synchronize()
            runs.append(a_ev.elapsed_time(b_ev) / 1e3)
        t = statistics.median(runs)
        print(json.dumps({"benchmark": "flow_only", "workload": f"forward_sequence_bidirectional(check=False) on the "
                          f"{len(passes)} passes of batch {T} over the same {N_CLIP}-frame clip, frames on the device",
                          "s_per_clip": t, "ms_per_frame": t * 1e3 / N_CLIP, "runs_s": runs, **ctx}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
