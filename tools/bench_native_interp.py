#!/usr/bin/env python
"""Interpolated frames at the input's own size (rb_frame_synthesize_items_resized, RaftEngine native=True), one JSON line
per measurement:

1. kernel: rb_frame_synthesize_items_resized alone, uint8 frames in and uint8 out, n_items = 1 and 8 (item i on frame
   pair i), output 1080x1920 and 2160x3840 from flows at 432x1024 and 544x960.  CUDA events around `--reps` launches
   after a warm-up of every shape.  Achieved bytes/s use the byte model of fused_bytes(): per item, both frames read once
   (6 B per output pixel), the output written once (3 B), and the two flows (8 B) and masks (1 B) at the network size.
2. composition: the same items through the existing entries, as the spec defines the result -- rb_frames_prepare on both
   frames, rb_flow_resize of both flows, a torch gather of both masks, rb_frame_synthesize_items -- timed the same way,
   with the outputs compared bit for bit first.  composition_bytes() is its byte model (the fp32 intermediates written
   and read back).
3. end_to_end: interpolate_sequence_at for 24 -> 60 fps on a seeded synthetic 1080x1920 clip (uint8, resident on the
   GPU), per output frame: native=True with flow sizes 432x1024 and 544x960 (T = 8 pairs per pass), and the whole network
   at 1080x1920 (what --keep-size runs) at T = 2 pairs per pass, whose correlation pyramids (4 pairs of 5.6 GB) fit the
   card.  A host clock around the whole clip, ending in a device synchronise, median of `--steps`.

raft-things, 20 iterations, seeded random weights.

    python tools/bench_native_interp.py [--reps 50] [--steps 3]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

OUT_SIZES = ((1080, 1920), (2160, 3840))
FLOW_SIZES = ((432, 1024), (544, 960))
N_ITEMS = (1, 8)
ITERS, N_FRAMES = 20, 9


def fused_bytes(n, Hs, Ws, H, W):
    """Least traffic of the fused kernel: per item both uint8 frames once, the uint8 output, two fp32 flows and two
    uint8 masks at the network size."""
    return n * (Hs * Ws * (2 * 3 + 3) + H * W * (2 * 8 + 2 * 1))


def composition_bytes(n, Hs, Ws, H, W):
    """Traffic of the composition: prepare (uint8 in, fp32 out) for both frames of every item, resize_flow (flows in,
    Hs x Ws fp32 flows out) and the two-step mask gather for both directions, then the blend reading fp32 frames, the
    resized flows and masks and writing uint8."""
    px = Hs * Ws
    prepare = 2 * px * (3 + 12)
    flows = 2 * (H * W * 8 + px * 8)
    masks = 2 * (H * W + 2 * Hs * W + 2 * px)
    blend = px * (2 * 12 + 2 * 8 + 2 * 1 + 3)
    return n * (prepare + flows + masks + blend)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50, help="launches per kernel timing (at least 10)")
    ap.add_argument("--steps", type=int, default=3, help="timed whole-clip runs (at least 3)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--skip-end-to-end", action="store_true")
    args = ap.parse_args(argv)
    if args.reps < 10 or args.steps < 3:
        ap.error("--reps >= 10, --steps >= 3")

    import numpy as np
    import torch
    from types import SimpleNamespace
    from raft_b200 import capi, synth
    from raft_b200.engine import _floats, _ints
    from raft_b200.video import fps_schedule
    from networks.RAFT import RAFT
    from networks.utils import resize_flow

    if not torch.cuda.is_available():
        raise SystemExit("bench_native_interp needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    lib, P = capi.lib, capi.ptr
    gpu, watts = torch.cuda.get_device_name(dev), power_limit_w(dev.index or 0)
    print(json.dumps({"gpu": gpu, "power_limit_w": watts}), flush=True)
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def events(fn, reps):
        fn()  # warm every shape
        torch.cuda.synchronize()
        a_ev.record()
        for _ in range(reps):
            fn()
        b_ev.record()
        torch.cuda.synchronize()
        return a_ev.elapsed_time(b_ev) / 1e3 / reps

    g = torch.Generator(device=dev).manual_seed(7)
    for Hs, Ws in OUT_SIZES:
        for H, W in FLOW_SIZES:
            for n in N_ITEMS:
                i0, i1 = (torch.randint(0, 256, (n, Hs, Ws, 3), generator=g, device=dev, dtype=torch.uint8)
                          for _ in range(2))
                f0, f1 = (torch.randn(n, H, W, 2, generator=g, device=dev) * 4 for _ in range(2))
                e0, e1 = ((torch.rand(n, H, W, generator=g, device=dev) < 0.05).to(torch.uint8) for _ in range(2))
                samples, ts = list(range(n)), [(i + 0.5) / n for i in range(n)]
                out = torch.empty(n, Hs, Ws, 3, dtype=torch.uint8, device=dev)
                ref = torch.empty_like(out)
                p0, p1 = (torch.empty(n, Hs, Ws, 3, device=dev) for _ in range(2))
                ys = ((2 * torch.arange(Hs, device=dev) + 1) * H) // (2 * Hs)
                xs = ((2 * torch.arange(Ws, device=dev) + 1) * W) // (2 * Ws)

                def fused():
                    capi.check(lib.rb_frame_synthesize_items_resized(
                        P(i0), P(i1), 1, Hs, Ws, P(f0), P(f1), P(e0), P(e1), H, W, _ints(samples), _floats(ts), n,
                        P(out), 1, 0, n, capi.stream()))

                def composition():
                    st = capi.stream()
                    capi.check(lib.rb_frames_prepare(P(i0), 1, P(p0), n, Hs, Ws, 0, 0, 0, 0, st))
                    capi.check(lib.rb_frames_prepare(P(i1), 1, P(p1), n, Hs, Ws, 0, 0, 0, 0, st))
                    r0, r1 = resize_flow(f0, (Hs, Ws)), resize_flow(f1, (Hs, Ws))
                    m0, m1 = (e[:, ys][:, :, xs].contiguous() for e in (e0, e1))
                    capi.check(lib.rb_frame_synthesize_items(
                        P(p0), P(p1), Hs, Ws, 0, 0, P(r0), P(r1), P(m0), P(m1), _ints(samples), _floats(ts), n, P(ref),
                        1, 0, n, Hs, Ws, st))

                fused()
                composition()
                torch.cuda.synchronize()
                same = bool(torch.equal(out, ref))
                t_f, t_c = [], []
                for i in range(4):  # alternating blocks
                    for fn, acc in (((fused, t_f), (composition, t_c)) if i % 2 == 0 else
                                    ((composition, t_c), (fused, t_f))):
                        acc.append(events(fn, args.reps))
                tf, tc = statistics.median(t_f), statistics.median(t_c)
                print(json.dumps({
                    "benchmark": "native_interp_kernel", "output": f"{Hs}x{Ws}", "flow": f"{H}x{W}", "n_items": n,
                    "frames": "uint8", "out": "uint8", "bit_identical_to_composition": same,
                    "fused_us": tf * 1e6, "composition_us": tc * 1e6, "speedup": tc / tf,
                    "fused_model_bytes": fused_bytes(n, Hs, Ws, H, W),
                    "fused_GBps": fused_bytes(n, Hs, Ws, H, W) / tf / 1e9,
                    "composition_model_bytes": composition_bytes(n, Hs, Ws, H, W),
                    "composition_GBps": composition_bytes(n, Hs, Ws, H, W) / tc / 1e9,
                    "reps": args.reps, "gpu": gpu, "power_limit_w": watts}), flush=True)
                del i0, i1, f0, f1, e0, e1, out, ref, p0, p1
                torch.cuda.empty_cache()

    if args.skip_end_to_end:
        return 0
    Hs, Ws = 1080, 1920
    base, _ = synth.make_batch(1, Hs + 2 * N_FRAMES, Ws + 3 * N_FRAMES, seed0=1234)
    clip = np.stack([base[0, 2 * k:2 * k + Hs, 3 * k:3 * k + Ws] for k in range(N_FRAMES)])  # a camera pan
    clip = torch.from_numpy(np.clip(np.rint(clip * 255), 0, 255).astype(np.uint8)).to(dev)
    weights = synth.make_weights(False)
    for name, size, T in (("native 432x1024", (432, 1024), 8), ("native 544x960", (544, 960), 8),
                          ("full network at 1080x1920 (--keep-size)", None, 2)):
        model = RAFT(None, SimpleNamespace(small=False), iters=ITERS, device=dev, input_size=size).load(weights)
        passes = fps_schedule(N_FRAMES, 24, 60, T)
        calls = [(clip[p.frames], [(k - p.frames[0], t) for _, k, t in p.items]) for p in passes]

        def clip_run():
            for frames, items in calls:
                out = model.interpolate_sequence_at(frames, items, uint8=True, native=size is not None)
            return out

        for _ in range(args.warmup):
            shape = tuple(clip_run().shape)
        spans = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            clip_run()
            torch.cuda.synchronize()
            spans.append(time.perf_counter() - t0)
        n_out = sum(len(p.items) + len(p.copies) for p in passes)
        n_items = sum(len(p.items) for p in passes)
        e2e = statistics.median(spans)
        print(json.dumps({
            "benchmark": "native_interp_end_to_end", "mode": name, "conversion": "24 -> 60",
            "workload": f"raft-things, {ITERS} iterations, seeded random weights, {N_FRAMES}-frame seeded synthetic "
                        f"{Hs}x{Ws} clip resident on the GPU (uint8), T={T} pairs per pass, uint8 output",
            "output_shape": shape, "output_frames": n_out, "interpolated_frames": n_items,
            "end_to_end_s": e2e, "ms_per_output_frame": e2e * 1e3 / n_out,
            "ms_per_interpolated_frame": e2e * 1e3 / n_items, "steps": args.steps,
            "peak_memory_GB": torch.cuda.max_memory_allocated(dev) / 1e9, "gpu": gpu, "power_limit_w": watts}),
            flush=True)
        del model
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
    return 0


if __name__ == "__main__":
    sys.exit(main())
