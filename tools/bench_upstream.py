"""Cost of RB_SEMANTICS_UPSTREAM: raft-things at 436x1024, 32 iterations, forward pairs/s in both modes at B = 1 and B = 8
(alternating, one engine per mode and batch), and the lookup kernel alone in both modes by CUDA events.  Prints one JSON line
with the card name and power limit read in the same run.

    python tools/bench_upstream.py [--reps 5] [--steps 10]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-tf_b200")]

import torch  # noqa: E402

from raft_b200 import capi, synth  # noqa: E402
from raft_b200.engine import RaftEngine  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def _pairs_per_s(eng, l, r, steps):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        eng.forward(l, r)
    torch.cuda.synchronize()
    return steps * l.shape[0] / (time.perf_counter() - t)


def _lookup_ms(up, B, h, w, reps=50):
    lib, r, K = capi.lib, 4, 81
    g = torch.Generator(device="cuda").manual_seed(0)
    pyr = torch.randn(capi.size_query(lib.rb_corr_pyramid_bytes, B, h, w) // 4, device="cuda", generator=g)
    ys, xs = torch.meshgrid(torch.arange(h, device="cuda"), torch.arange(w, device="cuda"), indexing="ij")
    coords = (torch.stack([xs, ys], -1).float()[None].repeat(B, 1, 1, 1) + torch.randn(B, h, w, 2, device="cuda", generator=g) * 4)
    ws = torch.zeros(capi.size_query(lib.rb_update_workspace_bytes, 0, B, h, w), dtype=torch.uint8, device="cuda")
    capi.check(lib.rb_set_semantics(capi.RB_SEMANTICS_UPSTREAM if up else capi.RB_SEMANTICS_REFERENCE))
    try:
        call = lambda: capi.check(lib.rb_update_lookup(0, capi.ptr(ws), capi.ptr(pyr), capi.ptr(coords.contiguous()), B, h, w,  # noqa: E731
                                                       capi.stream()))
        for _ in range(5):
            call()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            call()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps
    finally:
        lib.rb_set_semantics(capi.RB_SEMANTICS_REFERENCE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="alternating rounds of each (mode, batch)")
    ap.add_argument("--steps", type=int, default=10, help="forward calls per round")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    params = synth.make_weights(False)
    res = {"card": _card(), "model": "raft-things", "size": [436, 1024], "iters": 32, "pairs_per_s": {}, "lookup_ms": {}}
    for B in (1, 8):
        g = torch.Generator().manual_seed(B)
        l, r = torch.rand(B, 436, 1024, 3, generator=g).pin_memory(), torch.rand(B, 436, 1024, 3, generator=g).pin_memory()
        engs = {m: RaftEngine(params, iters=32, upstream=(m == "upstream")) for m in ("reference", "upstream")}
        for e in engs.values():
            e.forward(l, r)
        runs = {m: [] for m in engs}
        for _ in range(a.reps):
            for m, e in engs.items():
                runs[m].append(round(_pairs_per_s(e, l, r, a.steps), 2))
        res["pairs_per_s"][f"B{B}"] = runs
        del engs
        torch.cuda.empty_cache()
        h, w = 55, 128
        res["lookup_ms"][f"B{B}"] = {m: [round(_lookup_ms(m == "upstream", B, h, w), 4) for _ in range(3)]
                                     for m in ("reference", "upstream")}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
