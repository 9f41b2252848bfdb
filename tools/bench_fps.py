#!/usr/bin/env python
"""Frame-rate conversion (raft_b200.video.fps_schedule + RaftEngine.interpolate_sequence_at), one JSON line per conversion:

1. stage: the per-item work of each pass -- rb_flow_reverse_items per direction and rb_frame_synthesize_items on the
   pass's items alone -- against union-and-discard through interpolate_sequence's per-t path (every pair of the pass at
   the union of the pass's times, then only the needed frames kept), on the flows of the same pass, uint8 output; both
   results are compared bit for bit before timing.  CUDA events around `--reps` launches per arm, arms alternating,
   median over the passes of the per-pass time.
2. end_to_end: interpolate_sequence_at over every pass of the clip (the bidirectional flow pass plus the item work), per
   output frame (copies included, which cost nothing) and per interpolated frame; a host clock around the whole clip,
   ending in a device synchronise, median of `--steps`.

raft-things, 436x1024, 20 iterations, seeded random weights, a seeded synthetic 49-frame clip (a camera pan) resident on
the GPU as uint8, T = 8 pairs per pass (6 passes).  Conversions 24 -> 60, 25 -> 60, 24 -> 25 and 24000/1001 -> 60.

    python tools/bench_fps.py [--steps 5] [--warmup 1] [--reps 10]
"""
import argparse
import json
import os
import statistics
import sys
import time
from fractions import Fraction

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

H_IMG, W_IMG, ITERS, T, N_FRAMES = 436, 1024, 20, 8, 49
CONVERSIONS = ((24, 60), (25, 60), (24, 25), ("24000/1001", 60))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed whole-clip runs (at least 3)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=10, help="launch sequences per stage timing (at least 5)")
    args = ap.parse_args(argv)
    if args.steps < 3 or args.reps < 5:
        ap.error("--steps >= 3, --reps >= 5")

    import numpy as np
    import torch
    from types import SimpleNamespace
    from raft_b200 import synth
    from raft_b200.video import fps_schedule
    from networks.RAFT import RAFT

    if not torch.cuda.is_available():
        raise SystemExit("bench_fps needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = RAFT((H_IMG, W_IMG, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    eng = model.engine()
    base, _ = synth.make_batch(1, H_IMG + 2 * N_FRAMES, W_IMG + 3 * N_FRAMES, seed0=1234)
    clip = np.stack([base[0, 2 * k:2 * k + H_IMG, 3 * k:3 * k + W_IMG] for k in range(N_FRAMES)])  # a camera pan
    clip = torch.from_numpy(np.clip(np.rint(clip * 255), 0, 255).astype(np.uint8)).to(dev)
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def events(fn, reps):
        torch.cuda.synchronize()
        a_ev.record()
        for _ in range(reps):
            fn()
        b_ev.record()
        torch.cuda.synchronize()
        return a_ev.elapsed_time(b_ev) / 1e3 / reps

    gpu, watts = torch.cuda.get_device_name(dev), power_limit_w(dev.index or 0)
    for fin, fout in CONVERSIONS:
        passes = fps_schedule(N_FRAMES, fin, fout, T)
        calls = [(clip[p.frames], [(k - p.frames[0], t) for _, k, t in p.items]) for p in passes]
        n_items = [len(it) for _, it in calls]
        n_union = [len({t for _, t in it}) for _, it in calls]

        # 1. the per-item stage against union-and-discard, on the flows of each pass
        t_items, t_union = [], []
        for frames, items in calls:
            eng.forward_sequence_bidirectional(frames, check=False)
            ks = [k for k, _ in items]
            its = [t for _, t in items]
            union = sorted(set(its))
            flows = (eng.flow_up[:T], eng.flow_bw, eng.images[:T], eng.images[1:])

            def item_stage():
                return eng._synthesize(*flows, its, True, False, ks)

            def union_stage():
                full = eng._synthesize(*flows, union, True, False)
                return full[[union.index(t) for t in its], ks]  # the needed frames; the rest is discarded

            assert torch.equal(item_stage(), union_stage())
            for i in range(4):  # alternating blocks of launches
                for f, acc in (((item_stage, t_items), (union_stage, t_union)) if i % 2 == 0
                               else ((union_stage, t_union), (item_stage, t_items))):
                    acc.append(events(f, args.reps))

        # 2. the whole clip through interpolate_sequence_at
        def clip_run():
            for frames, items in calls:
                model.interpolate_sequence_at(frames, items, uint8=True)

        for _ in range(args.warmup):
            clip_run()
        spans = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            clip_run()
            torch.cuda.synchronize()
            spans.append(time.perf_counter() - t0)
        n_out = sum(len(p.items) + len(p.copies) for p in passes)
        e2e = statistics.median(spans)
        line = {
            "benchmark": "fps",
            "conversion": f"{Fraction(fin)} -> {Fraction(fout)}",
            "workload": f"raft-things {H_IMG}x{W_IMG} (padded to 440x1024), {ITERS} iterations, {N_FRAMES}-frame seeded "
                        f"synthetic clip resident on the GPU (uint8), T={T} pairs per pass, uint8 output, seeded random "
                        "weights",
            "passes": len(passes),
            "items_per_pass": n_items,
            "union_times_per_pass": n_union,
            "stage_items_ms_per_pass": statistics.median(t_items) * 1e3,
            "stage_union_ms_per_pass": statistics.median(t_union) * 1e3,
            "stage_speedup": statistics.median(t_union) / statistics.median(t_items),
            "stage_reps": args.reps,
            "output_frames": n_out,
            "end_to_end_s": e2e,
            "end_to_end_ms_per_output_frame": e2e * 1e3 / n_out,
            "end_to_end_ms_per_interpolated_frame": e2e * 1e3 / sum(n_items),
            "end_to_end_steps": args.steps,
            "gpu": gpu,
            "power_limit_w": watts,
        }
        print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
