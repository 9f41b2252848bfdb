"""Measure frame-rate conversion with a shutter (F32) on the GPU, with seeded weights and frames:

1. rb_frame_expose_items (432x1024) and rb_frame_expose_items_resized (1080x1920 from 432x1024 flows) per output row
   for m = 8 / 16 / 32 samples, one launch of 64 // m rows, against the composition of existing entries: the m item
   frames in fp32 (rb_frame_synthesize_items / _resized) then a mean in torch.  Bytes model per output pixel: both read
   the same flows, masks and frame taps per sample; the composition also writes and reads back m fp32 frames
   (24 m bytes) where the expose kernel keeps the sum in registers and writes 3 bytes.
2. rb_flow_reverse_items per sample at 432x1024 (64 items per call, both directions count as two samples).
3. End to end: RAFT.motion_blur of a seeded 21-frame 1080x1920 clip, 60 -> 24 at 180 degrees, density 16 (m = 20), flow
   at 432x1024 and native frames, against its forward_sequence_bidirectional pass alone; time per output frame.

    python tools/bench_shutter.py [--reps 20]

Prints one line per number and a JSON line with the card's name and power limit.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-tf_b200")]


def _time(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def bench_expose(reps):
    from raft_b200 import capi
    from raft_b200.engine import _floats, _ints
    lib, P, st = capi.lib, capi.ptr, capi.stream()
    d = "cuda:0"
    g = torch.Generator(device=d).manual_seed(0)
    H, W, n = 432, 1024, 64
    flow = torch.randn(2, n, H, W, 2, device=d, generator=g) * 3
    empty = torch.zeros(2, n, H, W, dtype=torch.uint8, device=d)
    res = {}
    for hs, ws in ((H, W), (1080, 1920)):
        native = (hs, ws) != (H, W)
        frames = (torch.rand(2, hs, ws, 3, device=d, generator=g) * 255).to(torch.uint8) if native else \
            torch.rand(2, H, W, 3, device=d, generator=g)
        for m in (8, 16, 32):
            rows = n // m
            ent = (capi.ExposeEntry * n)(*[capi.ExposeEntry(i, 0, (i % m + 0.5) / m) for i in range(n)])
            row = (capi.ExposeRow * rows)(*[capi.ExposeRow(r * m, m, m, 0, r, 3) for r in range(rows)])
            out = torch.empty(rows, hs, ws, 3, dtype=torch.uint8, device=d)
            acc = torch.empty(2, hs, ws, 3, device=d)
            fl = (P(flow[0]), P(flow[1]), P(empty[0]), P(empty[1]))
            tab = (n, ent, n, row, rows, P(acc), 2, P(out), rows, 0, 1)
            items = torch.empty(n, hs, ws, 3, device=d)
            ts = _floats([(i % m + 0.5) / m for i in range(n)])
            smp = _ints([0] * n)
            if native:
                def expose():
                    capi.check(lib.rb_frame_expose_items_resized(P(frames), 1, hs, ws, *fl, H, W, *tab, st))

                def compose():
                    capi.check(lib.rb_frame_synthesize_items_resized(P(frames[0]), P(frames[1]), 1, hs, ws, *fl, H, W,
                                                                     smp, ts, n, P(items), 0, 0, 1, st))
                    items.view(rows, m, hs, ws, 3).mean(1)
            else:
                def expose():
                    capi.check(lib.rb_frame_expose_items(P(frames), H, W, 0, 0, *fl, *tab, H, W, st))

                def compose():
                    capi.check(lib.rb_frame_synthesize_items(P(frames[0]), P(frames[1]), H, W, 0, 0, *fl, smp, ts, n,
                                                             P(items), 0, 0, 1, H, W, st))
                    items.view(rows, m, hs, ws, 3).mean(1)
            te, tc = _time(expose, reps) / rows, _time(compose, reps) / rows
            key = f"{hs}x{ws} m={m}"
            res[key] = {"expose_ms_per_row": te, "composition_ms_per_row": tc,
                        "composition_extra_bytes_per_row": 24 * m * hs * ws}
            print(f"expose {key}: {te:.3f} ms per output row; composition {tc:.3f} ms "
                  f"(+{24 * m * hs * ws / 1e6:.0f} MB of fp32 frames written and read back)")
    return res


def bench_reverse(reps):
    from raft_b200 import capi
    from raft_b200.engine import _floats, _ints
    lib, P, st = capi.lib, capi.ptr, capi.stream()
    d = "cuda:0"
    H, W, n = 432, 1024, 64
    g = torch.Generator(device=d).manual_seed(1)
    flow = torch.randn(8, H, W, 2, device=d, generator=g) * 4
    nb = capi.size_query(lib.rb_flow_reverse_multi_workspace_bytes, n, 1, H, W)
    ws = torch.empty(nb, dtype=torch.uint8, device=d)
    ft = torch.empty(n, H, W, 2, device=d)
    em = torch.empty(2, n, H, W, dtype=torch.uint8, device=d)
    steps, smp = _floats([(i + 0.5) / n for i in range(n)]), _ints([i % 8 for i in range(n)])

    def rev():
        capi.check(lib.rb_flow_reverse_items(P(flow), 8, smp, steps, n, P(ft), P(em[0]), P(em[1]), H, W, P(ws), nb, st))
    t = _time(rev, reps) / n
    print(f"rb_flow_reverse_items at {H}x{W}: {t:.3f} ms per sample (a blended sample needs two)")
    return {"reverse_ms_per_sample": t}


def bench_end_to_end(reps):
    from networks.RAFT import RAFT
    from raft_b200 import synth
    m = RAFT(None, SimpleNamespace(small=False), iters=20, device="cuda:0", input_size=(432, 1024)).load(
        synth.make_weights(False))
    rng = np.random.default_rng(2)
    base = (rng.random((1080 + 80, 1920 + 80, 3)) * 255).astype(np.uint8)
    frames = torch.from_numpy(np.stack([base[2 * k:2 * k + 1080, 3 * k:3 * k + 1920] for k in range(21)]))
    n_out = 20 * 24 // 60 + 1
    flow = _time(lambda: m.forward_sequence_bidirectional(frames, check=False), max(2, reps // 5))
    blur = _time(lambda: m.motion_blur(frames, 180, fps=(60, 24), density=16, native=True), max(2, reps // 5))
    print(f"60 -> 24 at 180 deg, density 16, 21 frames of 1080x1920, flow at 432x1024: {blur / n_out:.1f} ms per output "
          f"frame; the flow pass alone {flow / n_out:.1f} ms per output frame")
    return {"e2e_ms_per_output_frame": blur / n_out, "flow_ms_per_output_frame": flow / n_out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_shutter: needs a CUDA device")
    with torch.no_grad():
        res = {"card": _card(), **bench_expose(args.reps), **bench_reverse(args.reps), **bench_end_to_end(args.reps)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
