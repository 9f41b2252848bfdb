#!/usr/bin/env python
"""Frame interpolation over a frame sequence, three measurements, one JSON line:

1. sequence: RAFT.interpolate_sequence on T + 1 = 9 consecutive frames (8 pairs, each frame encoded once per direction set)
   against RAFT.interpolate on the same 8 pairs as one B = 8 batch, per output frame, for ts = [0.5] and ts = [1/8 .. 7/8].
2. per_t: the per-t work of one pass through the new entries (one rb_flow_reverse_multi per direction, one
   rb_frame_synthesize_pairs) against the per-t loop of the single-step entries (per t: two rb_flow_reverse, one
   rb_frame_synthesize), on the flows of the same pass, at T in {1, 8} and n_t in {1, 7}; both results are compared.
3. video: raft_b200.video.video_interpolate on 64 synthetic 436x1024 PNG frames (ts = [0.5], batch 8, 4 workers).

raft-things, 436x1024, 20 iterations, seeded random weights, frames resident on the GPU for 1 and 2, L2 flushed before
every timed span (outside it), arms alternating (ABBA); every span ends in a device synchronise.

    python tools/bench_video_interp.py [--steps 10] [--warmup 3] [--reps 50] [--video-frames 64]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

H_IMG, W_IMG, ITERS, T = 436, 1024, 20, 8


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed spans per arm (at least 6)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50, help="launch sequences per per-t timing (at least 20)")
    ap.add_argument("--video-frames", type=int, default=64)
    args = ap.parse_args(argv)
    if args.steps < 6 or args.reps < 20 or args.video_frames < 2:
        ap.error("--steps >= 6, --reps >= 20, --video-frames >= 2")

    import numpy as np
    import torch
    from types import SimpleNamespace
    from raft_b200 import capi, synth
    from raft_b200.engine import _floats
    from networks.RAFT import RAFT

    if not torch.cuda.is_available():
        raise SystemExit("bench_video_interp needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = RAFT((H_IMG, W_IMG, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    eng = model.engine()
    base, _ = synth.make_batch(1, H_IMG + 4 * T, W_IMG + 8 * T)
    frames_np = np.stack([base[0, 3 * k:3 * k + H_IMG, 7 * k:7 * k + W_IMG] for k in range(T + 1)])  # a camera pan
    frames = torch.from_numpy(frames_np).to(dev)
    left, right = frames[:T].contiguous(), frames[1:].contiguous()
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)  # > 50 MB L2 (H100)

    def span(fn):
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def abba(fa, fb):
        for _ in range(args.warmup):
            span(fa)
            span(fb)
        ta, tb = [], []
        for i in range(args.steps):
            for f, acc in (((fa, ta), (fb, tb)) if i % 2 == 0 else ((fb, tb), (fa, ta))):
                acc.append(span(f))
        return ta, tb

    def ms(ts_):
        return {"median": statistics.median(ts_) * 1e3, "min": min(ts_) * 1e3, "max": max(ts_) * 1e3}

    # 1. sequence against pairs
    seq_res = {}
    for label, ts in (("ts_0.5", [0.5]), ("ts_1/8..7/8", [i / 8 for i in range(1, 8)])):
        a = model.interpolate_sequence(frames, ts)
        b = model.interpolate(left, right, ts)
        assert torch.equal(a, b), label
        t_seq, t_pair = abba(lambda: model.interpolate_sequence(frames, ts), lambda: model.interpolate(left, right, ts))
        n_out = T * len(ts)
        seq_res[label] = {"sequence_ms": ms(t_seq), "pairs_ms": ms(t_pair),
                          "sequence_ms_per_frame": statistics.median(t_seq) * 1e3 / n_out,
                          "pairs_ms_per_frame": statistics.median(t_pair) * 1e3 / n_out,
                          "speedup": statistics.median(t_pair) / statistics.median(t_seq)}

    # 2. per-t work on the flows of one pass: new entries against the single-step loop
    lib, ptr = capi.lib, capi.ptr
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def events(fn, reps):
        torch.cuda.synchronize()
        a_ev.record()
        for _ in range(reps):
            fn()
        b_ev.record()
        torch.cuda.synchronize()
        return a_ev.elapsed_time(b_ev) / 1e3 / reps

    per_t = {}
    for Tn in (1, T):
        fr = frames[:Tn + 1]
        model.forward_sequence_bidirectional(fr, check=False)
        fw, bw = eng.flow_up[:Tn], eng.flow_bw
        f0, f1 = eng.images[:Tn], eng.images[1:Tn + 1]
        i0 = torch.cat([f0, f1]).contiguous()  # rb_frame_synthesize's [I0 | I1]
        one_bytes = capi.size_query(lib.rb_flow_reverse_workspace_bytes, Tn, H_IMG, W_IMG)
        one_ws = torch.empty(one_bytes, dtype=torch.uint8, device=dev)
        for n_t in (1, 7):
            ts = [0.5] if n_t == 1 else [i / 8 for i in range(1, 8)]
            out_new = torch.empty(n_t, Tn, H_IMG, W_IMG, 3, device=dev)
            out_old = torch.empty_like(out_new)
            ft = torch.empty(2, Tn, H_IMG, W_IMG, 2, device=dev)
            em = torch.empty(2, 2, Tn, H_IMG, W_IMG, dtype=torch.uint8, device=dev)
            st = capi.stream()

            def new():
                eng._reverse_and_blend(fw, bw, f0, f1, ts, out_new)

            def old():
                for i, t in enumerate(ts):
                    for k, (flow, step) in enumerate(((fw, t), (bw, 1.0 - t))):
                        capi.check(lib.rb_flow_reverse(ptr(flow), None, None, 0, 0, step, ptr(ft[k]), ptr(em[0, k]),
                                                       ptr(em[1, k]), None, None, Tn, H_IMG, W_IMG, ptr(one_ws), one_bytes,
                                                       st))
                    capi.check(lib.rb_frame_synthesize(ptr(i0), eng.Hp, eng.Wp, eng.pad[0], eng.pad[2], ptr(ft[0]),
                                                       ptr(ft[1]), ptr(em[0, 0]), ptr(em[0, 1]), t, ptr(out_old[i]), Tn,
                                                       H_IMG, W_IMG, st))

            for _ in range(5):
                new()
                old()
            assert torch.equal(out_new, out_old), (Tn, n_t)
            t_new, t_old = [], []
            for i in range(4):  # alternating blocks of launches
                for f, acc in (((new, t_new), (old, t_old)) if i % 2 == 0 else ((old, t_old), (new, t_new))):
                    acc.append(events(f, args.reps))
            per_t[f"T{Tn}_nt{n_t}"] = {"multi_us": statistics.median(t_new) * 1e6,
                                        "loop_us": statistics.median(t_old) * 1e6,
                                        "speedup": statistics.median(t_old) / statistics.median(t_new)}

    # 3. video_interpolate on synthetic PNGs
    import cv2
    from raft_b200.video import video_interpolate
    vmodel = RAFT(None, SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    with tempfile.TemporaryDirectory() as tmp:
        src, out = os.path.join(tmp, "in"), os.path.join(tmp, "out")
        os.makedirs(src)
        big, _ = synth.make_batch(1, H_IMG + args.video_frames, W_IMG + 2 * args.video_frames, seed0=77)
        for k in range(args.video_frames):
            img = np.clip(np.rint(big[0, k:k + H_IMG, 2 * k:2 * k + W_IMG] * 255), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(src, f"frame_{k:04d}.png"), img)
        video_interpolate(vmodel, src, out, [0.5], batch=T, workers=4)  # warm-up: graphs, allocations
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        files = video_interpolate(vmodel, src, out, [0.5], batch=T, workers=4)
        torch.cuda.synchronize()
        t_video = time.perf_counter() - t0

    line = {
        "benchmark": "video_interp",
        "workload": f"raft-things {H_IMG}x{W_IMG} (padded to 440x1024), {ITERS} iterations, T={T} pairs per pass, "
                    "resident frames, L2 flushed before each span, seeded random weights",
        "steps_per_arm": args.steps,
        "sequence_vs_pairs": seq_res,
        "per_t": per_t,
        "per_t_reps": args.reps,
        "video_interpolate": {"input_frames": args.video_frames, "files": len(files), "seconds": t_video,
                              "input_frames_per_s": (args.video_frames - 1) / t_video},
        "gpu": torch.cuda.get_device_name(dev),
        "power_limit_w": power_limit_w(dev.index or 0),
    }
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
