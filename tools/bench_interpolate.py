#!/usr/bin/env python
"""Time RAFT.interpolate(L, R, [0.5]) against forward_bidirectional(L, R, check=False) on the same model, the per-t work
on its own (two flow reversals and the blend), and the worst case of the reversal (every source on one pixel).
raft-things, 436x1024, 32 iterations, B = 1, frames resident on the GPU, L2 flushed before every timed span (outside
it).  The two arms alternate step by step (ABBA order); every span ends in a device synchronise.  Prints one JSON line.

    python tools/bench_interpolate.py [--steps 30] [--warmup 5] [--reps 200] [--worst-reps 10]
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

H_IMG, W_IMG, ITERS, B = 436, 1024, 32, 1


def power_limit_w(index):
    try:  # read-only query
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per arm (at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=200, help="launch sequences per per-t timing (at least 100)")
    ap.add_argument("--worst-reps", type=int, default=10, help="launches of the single-target reversal")
    args = ap.parse_args(argv)
    if args.steps < 20 or args.reps < 100 or args.worst_reps < 1:
        ap.error("--steps >= 20, --reps >= 100, --worst-reps >= 1")

    import numpy as np
    import torch
    from types import SimpleNamespace
    from raft_b200 import capi, synth
    from networks.RAFT import RAFT

    if not torch.cuda.is_available():
        raise SystemExit("bench_interpolate needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = RAFT((H_IMG, W_IMG, 3), SimpleNamespace(small=False), iters=ITERS, batch=B, device=dev).load(
        synth.make_weights(False))
    l_np, r_np = synth.make_batch(B, H_IMG, W_IMG)
    l, r = torch.from_numpy(l_np).to(dev), torch.from_numpy(r_np).to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)  # > 50 MB L2 (H100)

    def bidirectional():
        return model.forward_bidirectional(l, r, check=False)

    def interpolate():
        return model.interpolate(l, r, [0.5])

    def span(fn):
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for _ in range(args.warmup):
        span(bidirectional)
        span(interpolate)
    t_bi, t_in = [], []
    for i in range(args.steps):
        if i % 2 == 0:
            t_in.append(span(interpolate))
            t_bi.append(span(bidirectional))
        else:
            t_bi.append(span(bidirectional))
            t_in.append(span(interpolate))

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def events(fn, reps):
        torch.cuda.synchronize()
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / 1e3 / reps

    # per t: the engine's own calls on the flows of the last interpolate pass
    mid = interpolate()[0]
    eng = model.engine()
    out = torch.empty(B, H_IMG, W_IMG, 3, dtype=torch.float32, device=dev)
    for _ in range(10):
        eng._interpolate_at(0.5, out)
    t_per_t = events(lambda: eng._interpolate_at(0.5, out), args.reps)
    assert torch.equal(out, mid)

    # worst case: every source of the frame on pixel (0, 0), summed in raster order by one thread
    lib, st, ptr = capi.lib, capi.stream(), capi.ptr
    yy, xx = np.mgrid[0:H_IMG, 0:W_IMG].astype(np.float32)
    worst = torch.from_numpy(np.stack([-(xx + 0.75), -(yy + 0.75)], -1)[None].astype(np.float32)).to(dev)
    flow_t = torch.empty_like(worst)
    masks = torch.empty(2, B, H_IMG, W_IMG, dtype=torch.uint8, device=dev)
    nbytes = capi.size_query(lib.rb_flow_reverse_workspace_bytes, B, H_IMG, W_IMG)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)

    def reverse(flow):
        capi.check(lib.rb_flow_reverse(ptr(flow), None, None, 0, 0, 1.0, ptr(flow_t), ptr(masks[0]), ptr(masks[1]), None,
                                       None, B, H_IMG, W_IMG, ptr(ws), nbytes, st))

    reverse(worst)
    t_worst = events(lambda: reverse(worst), args.worst_reps)
    assert int(masks[0].sum()) == H_IMG * W_IMG - 1
    fw = model.forward_bidirectional(l, r, check=False)[0]
    for _ in range(10):
        reverse(fw)
    t_typical = events(lambda: reverse(fw), args.reps)

    med_bi, med_in = statistics.median(t_bi), statistics.median(t_in)
    line = {
        "benchmark": "interpolate",
        "workload": f"raft-things {H_IMG}x{W_IMG} (padded to 440x1024), {ITERS} iterations, B={B}, resident frames, "
                    "L2 flushed before each span, seeded random weights",
        "steps_per_arm": args.steps,
        "interpolate_ms": {"median": med_in * 1e3, "min": min(t_in) * 1e3, "max": max(t_in) * 1e3},
        "bidirectional_ms": {"median": med_bi * 1e3, "min": min(t_bi) * 1e3, "max": max(t_bi) * 1e3},
        "overhead_ms": (med_in - med_bi) * 1e3,
        "per_t_us": {"launches": args.reps, "two_reversals_and_blend": t_per_t * 1e6},
        "reversal_us": {"raft_flow": t_typical * 1e6, "all_sources_on_one_pixel": t_worst * 1e6,
                        "worst_launches": args.worst_reps},
        "gpu": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(dev.index or 0),
    }
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
