#!/usr/bin/env python
"""Time RAFT.forward_bidirectional against forward(L, R) + forward(R, L) on the same model, and the consistency-check
kernel on its own.  raft-things, 436x1024, 32 iterations, B = 1, frames resident on the GPU, L2 flushed before every
timed span (outside it).  The two arms alternate step by step (ABBA order); every span ends in a device synchronise.
Prints one JSON line.

    python tools/bench_bidirectional.py [--steps 30] [--warmup 5] [--check-reps 200]
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
    ap.add_argument("--check-reps", type=int, default=200, help="launches of rb_flow_fb_check per timing (at least 100)")
    args = ap.parse_args(argv)
    if args.steps < 20 or args.check_reps < 100:
        ap.error("--steps >= 20 and --check-reps >= 100")

    import torch
    from types import SimpleNamespace
    from raft_b200 import capi, synth
    from networks.RAFT import RAFT

    if not torch.cuda.is_available():
        raise SystemExit("bench_bidirectional needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = RAFT((H_IMG, W_IMG, 3), SimpleNamespace(small=False), iters=ITERS, batch=B, device=dev).load(
        synth.make_weights(False))
    l_np, r_np = synth.make_batch(B, H_IMG, W_IMG)
    l, r = torch.from_numpy(l_np).to(dev), torch.from_numpy(r_np).to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)  # > 50 MB L2 (H100)

    def two_forwards():
        return model.forward(l, r), model.forward(r, l)

    def bidirectional():
        return model.forward_bidirectional(l, r)

    def span(fn):
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for _ in range(args.warmup):
        span(two_forwards)
        span(bidirectional)
    fw_ref, bw_ref = two_forwards()
    fw, bw, occ_fw, occ_bw = bidirectional()
    identical = bool(torch.equal(fw, fw_ref) and torch.equal(bw, bw_ref))

    t_bi, t_two = [], []
    for i in range(args.steps):
        if i % 2 == 0:
            t_bi.append(span(bidirectional))
            t_two.append(span(two_forwards))
        else:
            t_two.append(span(two_forwards))
            t_bi.append(span(bidirectional))

    # the check kernel alone, on the flows just computed
    lib, st = capi.lib, capi.stream()
    occ = torch.empty(2, B, H_IMG, W_IMG, dtype=torch.uint8, device=dev)

    def check():
        capi.check(lib.rb_flow_fb_check(capi.ptr(fw), capi.ptr(bw), capi.ptr(occ[0]), capi.ptr(occ[1]), B, H_IMG, W_IMG,
                                        1.0, 0.01, 0.5, st))

    for _ in range(10):
        check()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(args.check_reps):
        check()
    b.record()
    torch.cuda.synchronize()
    t_check_warm = a.elapsed_time(b) / 1e3 / args.check_reps
    cold = []
    for _ in range(args.check_reps):
        flush.zero_()
        a.record()
        check()
        b.record()
        torch.cuda.synchronize()
        cold.append(a.elapsed_time(b) / 1e3)
    t_check_cold = statistics.median(cold)
    assert torch.equal(occ[0], occ_fw) and torch.equal(occ[1], occ_bw)
    nbytes = B * H_IMG * W_IMG * (2 * 8 + 2 * 1)  # each flow read once, each mask written once

    med_bi, med_two = statistics.median(t_bi), statistics.median(t_two)
    line = {
        "benchmark": "bidirectional",
        "workload": f"raft-things {H_IMG}x{W_IMG} (padded to 440x1024), {ITERS} iterations, B={B}, resident frames, "
                    "L2 flushed before each span, seeded random weights",
        "steps_per_arm": args.steps,
        "bidirectional_ms": {"median": med_bi * 1e3, "min": min(t_bi) * 1e3, "max": max(t_bi) * 1e3},
        "two_forwards_ms": {"median": med_two * 1e3, "min": min(t_two) * 1e3, "max": max(t_two) * 1e3},
        "speedup": med_two / med_bi,
        "flows_bit_identical": identical,
        "fb_check": {
            "launches": args.check_reps,
            "us_l2_warm": t_check_warm * 1e6,
            "us_l2_flushed": t_check_cold * 1e6,
            "algorithmic_bytes": nbytes,
            "gbs_l2_warm": nbytes / t_check_warm / 1e9,
            "gbs_l2_flushed": nbytes / t_check_cold / 1e9,
            "note": "bytes = B*H*W*(2*8 + 2*1): each flow read once, each mask written once",
        },
        "gpu": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(dev.index or 0),
    }
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
