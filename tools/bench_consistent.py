#!/usr/bin/env python
"""Temporal consistency (rb_tcons_terms, rb_screened_poisson, rb_warp_error), one JSON line per measurement, each with
the card's name and power limit:

1. rb_tcons_terms + rb_screened_poisson per frame at 480x854 and 1080x1920 from 432x1024 flows, at lambda 1e-3 and 1e-1,
   on seeded frames and flows whose steps all pass the forward-backward test (every pixel carries a temporal term), with
   the solver's launches and copies per frame.  CUDA events around `--reps` back-to-back frames on preallocated
   buffers, median of 5 windows.
2. rb_warp_error per pair at the same sizes (8 pairs per call).
3. video_consistent end to end (decode of both clips, upload, bidirectional flow, terms, solve, E_warp of three videos,
   PNG writes) on a seeded synthetic 24-frame 1080x1920 PNG clip and a flickering 'processed' copy, raft-things at
   432x1024, 20 iterations, batch 8, 4 workers, lambda 0.1, against forward_sequence_bidirectional(check=False) alone on
   the same passes (frames already on the GPU); host clock, median of `--steps` runs.

Seeded data and weights; everything is written to a temporary directory.

    python tools/bench_consistent.py [--reps 20] [--steps 3]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

NET = (432, 1024)


def solver_launches(H, W):
    """Launches and device copies of one rb_screened_poisson call (include/raft_b200.h F30): 61 L + 12 for L levels."""
    from raft_b200.inpaint import fill_levels
    return 61 * len(fill_levels(H, W)) + 12


def _timed(torch, fn, reps):
    times = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / reps)
    return statistics.median(times)


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--steps", type=int, default=3)
    args = p.parse_args(argv)
    import torch
    from networks.utils import screened_poisson, tcons_terms, warp_error
    from raft_b200 import capi
    assert torch.cuda.is_available(), "bench_consistent measures on the GPU"
    dev = torch.device("cuda:0")
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(0)}
    g = torch.Generator(device=dev).manual_seed(0)
    Hn, Wn = NET
    fw = torch.full((8, Hn, Wn, 2), 0.5, device=dev)
    bw = -fw
    for Hs, Ws in ((480, 854), (1080, 1920)):
        fr = torch.randint(0, 256, (9, Hs, Ws, 3), dtype=torch.uint8, device=dev, generator=g)
        I1, I0 = fr[1], fr[1].clone()  # the originals match, so the colour check passes everywhere
        P, O = fr[2], fr[3]
        ws = torch.empty(capi.size_query(capi.lib.rb_screened_poisson_workspace_bytes, Hs, Ws), dtype=torch.uint8,
                         device=dev)
        for lam in (1e-3, 1e-1):
            def frame():
                c, r, _ = tcons_terms(I1, I0, P, O, fw[0], bw[0], lam)
                return screened_poisson(c, r, workspace=ws)
            frame()
            ms = _timed(torch, frame, args.reps)
            c, r, _ = tcons_terms(I1, I0, P, O, fw[0], bw[0], lam)
            ms_terms = _timed(torch, lambda: tcons_terms(I1, I0, P, O, fw[0], bw[0], lam), args.reps)
            print(json.dumps({"what": "terms+solve per frame", "size": [Hs, Ws], "net": [Hn, Wn], "lambda": lam,
                              "ms": round(ms, 4), "terms_ms": round(ms_terms, 4),
                              "solver_launches": solver_launches(Hs, Ws), **card}), flush=True)
        warp_error(fr, fw, bw)
        ms = _timed(torch, lambda: warp_error(fr, fw, bw), args.reps) / 8
        print(json.dumps({"what": "warp_error per pair", "size": [Hs, Ws], "net": [Hn, Wn], "ms": round(ms, 4),
                          **card}), flush=True)
    del fr
    video_bench(torch, dev, card, args.steps)


def video_bench(torch, dev, card, steps, n_clip=24, batch=8, iters=20, lam=0.1):
    import shutil
    import tempfile
    import time
    from types import SimpleNamespace
    import cv2
    import numpy as np
    from networks.RAFT import RAFT
    from raft_b200 import synth
    from raft_b200.video import interp_schedule, video_consistent
    Hn, Wn = NET
    model = RAFT((Hn, Wn, 3), SimpleNamespace(small=False), iters=iters, device=dev,
                 input_size=(Hn, Wn)).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, 540 + 2 * n_clip + 16, 960 + 3 * n_clip + 16, seed0=4321)
    rng = np.random.default_rng(7)
    tmp = tempfile.mkdtemp(prefix="bench_consistent_")
    try:
        d, q = os.path.join(tmp, "frames"), os.path.join(tmp, "processed")
        os.makedirs(d)
        os.makedirs(q)
        clip = []
        for k in range(n_clip):
            img = base[0, 2 * k:2 * k + 540, 3 * k:3 * k + 960]
            img = cv2.resize(np.clip(np.rint(img * 255), 0, 255).astype(np.uint8), (1920, 1080))
            clip.append(img)
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
            proc = np.clip(np.rint(img * rng.uniform(0.85, 1.15) + rng.uniform(-12, 12, 3)), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(q, f"frame_{k:04d}.png"), proc)
        times = []
        for i in range(steps + 1):
            out = os.path.join(tmp, "out")
            shutil.rmtree(out, ignore_errors=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, info = video_consistent(model, d, q, out, lam, batch=batch, workers=4)
            torch.cuda.synchronize()
            if i:  # the first run captures the CUDA graph
                times.append(time.perf_counter() - t0)
        engine = model.engine()
        passes = [torch.from_numpy(np.stack([clip[f] for f in ps.frames])).to(dev)
                  for ps in interp_schedule(n_clip, batch)]
        flow_times = []
        for i in range(steps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for p in passes:
                engine.forward_sequence_bidirectional(p, check=False)
            torch.cuda.synchronize()
            if i:
                flow_times.append(time.perf_counter() - t0)
        t, tf = statistics.median(times), statistics.median(flow_times)
        print(json.dumps({"what": "video_consistent", "workload": f"raft-things {Hn}x{Wn}, {iters} iterations, "
                          f"{n_clip}-frame seeded synthetic 1080x1920 PNG clip and a flickering copy, batch {batch}, "
                          f"4 workers, lambda {lam}, seeded weights", "status": info["status"],
                          "s_per_clip": t, "ms_per_frame": t * 1e3 / n_clip, "flow_passes_s": tf,
                          "flow_ms_per_frame": tf * 1e3 / n_clip, "clip_over_flow_passes": t / tf, "runs_s": times,
                          "flow_runs_s": flow_times, **card}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
