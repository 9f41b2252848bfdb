#!/usr/bin/env python
"""TAP-Vid evaluation cost (raft_b200.tapvid), one JSON line per measurement:

1. kernels: rb_track_points and rb_track_points_backward over one 50-frame 256x256 clip's flows (49 steps) for the
   1 000 queries of TAP-Vid's strided mode (100 tracks, query frames 0, 5, ..., 45).  CUDA events around `--reps`
   back-to-back calls of each C entry on preallocated buffers, median of 5 such windows.  The first launches are checked
   against tests/track_oracle.py and tests/track_backward_oracle.py bit for bit.
2. end to end: raft_b200.tapvid.run (unpickling, the flow passes, the launches, the metrics) over a pickle of `--videos`
   such clips in strided mode, at batch 1 and batch 8, with the flow passes per video; host clock around each run after
   one untimed run per batch (CUDA graph capture), median of `--steps` runs.

raft-things, 20 iterations (the protocol's), seeded random weights; the clips are seeded synthetic pans already at
256x256, the points follow the pan.  The pickle goes to a temporary directory.

    python tools/bench_tapvid.py [--reps 200] [--steps 3] [--videos 4]
"""
import argparse
import json
import os
import pickle
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

F, N_TRACKS, ITERS = 50, 100, 20


def _clip(seed):
    import numpy as np
    from raft_b200 import synth
    base, _ = synth.make_batch(1, 256 + 2 * F, 256 + 3 * F, seed0=seed)
    video = np.stack([np.clip(np.rint(base[0, 2 * k:2 * k + 256, 3 * k:3 * k + 256] * 255), 0, 255).astype(np.uint8)
                      for k in range(F)])
    rng = np.random.default_rng(seed)
    start = rng.uniform(0.3, 0.95, (N_TRACKS, 1, 2))
    points = start - np.arange(F)[None, :, None] * np.array([3 / 256, 2 / 256])  # the content moves left and up
    return {"video": video, "points": points.astype(np.float32), "occluded": np.zeros((N_TRACKS, F), bool)}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200, help="launches per kernel timing window (at least 50)")
    ap.add_argument("--steps", type=int, default=3, help="timed end-to-end runs per batch (at least 3)")
    ap.add_argument("--videos", type=int, default=4, help="clips in the end-to-end pickle")
    args = ap.parse_args(argv)
    if args.reps < 50 or args.steps < 3 or args.videos < 1:
        ap.error("--reps >= 50, --steps >= 3, --videos >= 1")

    import numpy as np
    import torch
    from types import SimpleNamespace
    import track_backward_oracle as B
    import track_oracle as O
    from networks.RAFT import RAFT
    from networks.utils import track_points, track_points_backward
    from raft_b200 import capi, synth, tapvid
    from raft_b200.evaluate import PROTOCOLS, _engine
    from raft_b200.video import interp_schedule

    if not torch.cuda.is_available():
        raise SystemExit("bench_tapvid needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ctx = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    model = RAFT(None, SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    engine = _engine(model, ITERS, PROTOCOLS["tapvid"][1], input_size=tapvid.SIZE)

    # 1. the kernels on one clip's flows
    clip = _clip(7)
    track, frame = tapvid.sample_queries(clip["occluded"], "strided")
    qframe, qpos = tapvid.query_inputs(clip["points"], track, frame)
    N = len(qframe)
    frames = torch.from_numpy(clip["video"][..., ::-1].copy()).to(dev)
    fw, bw, _, _ = engine.forward_sequence_bidirectional(frames, check=False)
    fw, bw = fw.clone(), bw.clone()
    qf, qp = torch.from_numpy(qframe).to(dev), torch.from_numpy(qpos).to(dev)
    tracks, status, (pos, st) = track_points(fw, bw, qf, qp)
    want_t, want_s, _ = O.track(fw.cpu().numpy(), bw.cpu().numpy(), qframe, qpos)
    assert O.same_bits(tracks.cpu().numpy(), want_t) and np.array_equal(status.cpu().numpy(), want_s)
    track_points_backward(fw, bw, qf, qp, tracks, status)
    want_t, want_s, _ = B.track_backward(fw.cpu().numpy(), bw.cpu().numpy(), qframe, qpos, want_t, want_s)
    assert O.same_bits(tracks.cpu().numpy(), want_t) and np.array_equal(status.cpu().numpy(), want_s)
    T = F - 1
    launch = (capi.ptr(fw), capi.ptr(bw), T, 256, 256, T, 1.0, 0.01, 0.5, capi.ptr(qf), capi.ptr(qp), N, 0,
              capi.ptr(pos), capi.ptr(st), capi.ptr(tracks), capi.ptr(status), capi.stream())
    for name, fn in (("forward", capi.lib.rb_track_points), ("backward", capi.lib.rb_track_points_backward)):
        for _ in range(20):
            capi.check(fn(*launch))
        windows = []
        for _ in range(5):
            torch.cuda.synchronize()
            a_ev.record()
            for _ in range(args.reps):
                capi.check(fn(*launch))
            b_ev.record()
            torch.cuda.synchronize()
            windows.append(a_ev.elapsed_time(b_ev) / 1e3 / args.reps)
        t = statistics.median(windows)
        print(json.dumps({"benchmark": "tapvid_track_kernel", "direction": name, "N": N, "steps": T, "H": 256, "W": 256,
                          "us_per_launch": t * 1e6, "reps": args.reps, "windows_us": [w * 1e6 for w in windows],
                          **ctx}), flush=True)

    # 2. end to end
    tmp = tempfile.mkdtemp(prefix="bench_tapvid_")
    try:
        path = os.path.join(tmp, "synth.pkl")
        with open(path, "wb") as f:
            pickle.dump({f"clip{i}": _clip(100 + i) for i in range(args.videos)}, f)
        for batch in (1, 8):
            times, records = [], None
            for i in range(args.steps + 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                records = tapvid.run(engine, path, "strided", batch)
                torch.cuda.synchronize()
                if i:
                    times.append(time.perf_counter() - t0)
            t = statistics.median(times)
            agg = tapvid.aggregate_tapvid(records)
            print(json.dumps({"benchmark": "tapvid_end_to_end", "query_mode": "strided", "batch": batch,
                              "videos": args.videos, "frames_per_video": F, "queries_per_video": N,
                              "flow_passes_per_video": len(interp_schedule(F, batch)),
                              "workload": f"raft_b200.tapvid.run, raft-things at 256x256, {ITERS} iterations, seeded "
                                          f"random weights, {args.videos} seeded synthetic {F}-frame pans",
                              "videos_per_s": args.videos / t, "s_per_video": t / args.videos, "runs_s": times,
                              "average_jaccard": agg["average_jaccard"], **ctx}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
