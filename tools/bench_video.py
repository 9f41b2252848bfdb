#!/usr/bin/env python
"""Time video flow: RaftEngine.forward_sequence (carry calls at T = 1 and T = 8, and the warm-started T = 1 stream)
against forward at B = 1 and B = 8 on the same resident frames, in pairs per second; rb_flow_to_color against the host
flow_utils.flow_to_color plus the flow's device-to-host copy; and raft_b200.video end to end on synthetic PNG frames.
raft-things, 436x1024, 32 iterations, seeded random weights.  Each arm runs on a model of its own (so no arm evicts
another's CUDA graphs); the arms alternate step by step (ABBA order), the L2 is flushed before every timed span (outside
it) and every span ends in a device synchronise.  Prints one JSON line.

    python tools/bench_video.py [--steps 10] [--warmup 2] [--color-reps 200] [--frames 64]
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

H_IMG, W_IMG, ITERS, N = 436, 1024, 32, 8  # N pairs per timed step


def power_limit_w(index):
    try:  # read-only query
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def _ms(ts):
    return {"median": statistics.median(ts) * 1e3, "min": min(ts) * 1e3, "max": max(ts) * 1e3}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help=f"timed steps per arm ({N} pairs each)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--color-reps", type=int, default=200, help="launches of rb_flow_to_color per timing")
    ap.add_argument("--host-reps", type=int, default=5, help="runs of the host colour coding per timing")
    ap.add_argument("--frames", type=int, default=64, help="PNG frames of the end-to-end video() run")
    args = ap.parse_args(argv)

    import numpy as np
    import torch
    from types import SimpleNamespace
    from raft_b200 import synth
    from raft_b200.video import video
    from networks.RAFT import RAFT
    from networks.utils import flow_to_color, forward_interpolate
    import flow_utils

    if not torch.cuda.is_available():
        raise SystemExit("bench_video needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    params = synth.make_weights(False)

    def model():
        return RAFT((H_IMG, W_IMG, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(params)

    # 2N + 1 resident frames: a pan over one larger synthetic image
    big, _ = synth.make_batch(1, H_IMG + 4 * (2 * N + 1), W_IMG + 4 * (2 * N + 1), seed0=4000)
    frames = torch.from_numpy(np.stack([big[0, 2 * k:2 * k + H_IMG, 3 * k:3 * k + W_IMG] for k in range(2 * N + 1)])).to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)  # > 50 MB L2 (H100)
    e_f1, e_f8, e_s1, e_s8, e_w1 = (model().engine() for _ in range(5))

    def fwd1():
        return [e_f1.forward(frames[k:k + 1], frames[k + 1:k + 2]).clone() for k in range(N)]

    def fwd8():
        return e_f8.forward(frames[:N], frames[1:N + 1])

    def seq1():  # one fresh call, then carries: the flows of pairs 0 .. N-1 (the first call is also timed)
        out = [e_s1.forward_sequence(frames[:2]).clone()]
        return out + [e_s1.forward_sequence(frames[k + 1:k + 2], carry=True).clone() for k in range(1, N)]

    def seq8_setup():
        e_s8.forward_sequence(frames[:N + 1])

    def seq8():  # carry: pairs N .. 2N-1
        return e_s8.forward_sequence(frames[N + 1:2 * N + 1], carry=True)

    def warm1():
        low, flow = e_w1.forward_sequence(frames[:2], return_low=True)
        for k in range(1, N):
            low, flow = e_w1.forward_sequence(frames[k + 1:k + 2], carry=True, flow_init=forward_interpolate(low),
                                              return_low=True)
        return flow

    def span(fn, setup=None):
        if setup is not None:
            setup()
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    arms = {"forward_b1": (fwd1, None), "sequence_t1": (seq1, None), "forward_b8": (fwd8, None),
            "sequence_t8_carry": (seq8, seq8_setup), "warm_t1": (warm1, None)}
    for _ in range(args.warmup):
        for fn, setup in arms.values():
            span(fn, setup)
    # the flows of the arms, bit for bit
    f1, s1 = torch.cat(fwd1()), torch.cat(seq1())
    seq8_setup()
    ref8 = e_f8.forward(frames[N:2 * N], frames[N + 1:2 * N + 1]).clone()
    identical = bool(torch.equal(f1, s1) and torch.equal(fwd8(), f1) and torch.equal(seq8(), ref8))

    times = {k: [] for k in arms}
    order = list(arms)
    for i in range(args.steps):
        for k in (order if i % 2 == 0 else order[::-1]):
            times[k].append(span(*arms[k]))
    rate = {k: N / statistics.median(v) for k, v in times.items()}

    # colour coding: the kernel (L2-warm, back to back) against the host function plus the device-to-host copy
    flows8 = s1.contiguous()
    color = {}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for B in (1, N):
        f = flows8[:B]
        for _ in range(10):
            flow_to_color(f, convert_to_bgr=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(args.color_reps):
            flow_to_color(f, convert_to_bgr=True)
        b.record()
        torch.cuda.synchronize()
        gpu_us = a.elapsed_time(b) * 1e3 / args.color_reps
        host = []
        for _ in range(args.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h = f.cpu().numpy()
            for x in h:
                flow_utils.flow_to_color(x, convert_to_bgr=True)
            host.append(time.perf_counter() - t0)
        color[f"B{B}"] = {"kernel_us": gpu_us, "host_with_copy_us": statistics.median(host) * 1e6,
                          "speedup": statistics.median(host) * 1e6 / gpu_us}

    # video() end to end on PNG frames (decode, upload, flow, colour, PNG encode and write)
    import cv2
    tmp = tempfile.mkdtemp(prefix="bench_video_")
    e2e = {}
    try:
        n = args.frames
        big, _ = synth.make_batch(1, H_IMG + 2 * n, W_IMG + 3 * n, seed0=4100)
        img = np.clip(np.rint(big[0] * 255), 0, 255).astype(np.uint8)
        src = os.path.join(tmp, "frames")
        os.makedirs(src)
        for k in range(n):
            cv2.imwrite(os.path.join(src, f"{k:05d}.png"), img[2 * k:2 * k + H_IMG, 3 * k:3 * k + W_IMG])
        for batch in (1, N):
            m = model()
            video(m, src, os.path.join(tmp, "warm"), batch=batch)  # graphs captured, files cached by the OS
            t = []
            for _ in range(2):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                video(m, src, os.path.join(tmp, f"out{batch}"), batch=batch)
                t.append(time.perf_counter() - t0)
            e2e[f"batch{batch}"] = {"s": min(t), "pairs_per_s": (n - 1) / min(t)}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)

    line = {
        "benchmark": "video",
        "workload": f"raft-things {H_IMG}x{W_IMG} (padded to 440x1024), {ITERS} iterations, {N} pairs per step, resident "
                    "frames, L2 flushed before each span, seeded random weights",
        "steps_per_arm": args.steps,
        "ms_per_step": {k: _ms(v) for k, v in times.items()},
        "pairs_per_s": rate,
        "sequence_t1_vs_forward_b1": rate["sequence_t1"] / rate["forward_b1"],
        "sequence_t8_vs_forward_b8": rate["sequence_t8_carry"] / rate["forward_b8"],
        "flows_bit_identical": identical,
        "flow_to_color": color,
        "video_e2e": {"frames": args.frames, **e2e},
        "gpu": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(dev.index or 0),
    }
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
