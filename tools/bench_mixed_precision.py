"""What RB_MATH_TC_FP16 (RaftEngine(mixed_precision=True)) buys against the default RB_MATH_TC.

Configurations: raft-things at 436x1024, 32 iterations, B = 1 and B = 8; raft-small at 768x1024, 20 iterations, B = 8 (the
per-GPU share of BASELINE config 5).  Per configuration:
  * pairs/s of RAFT.forward's engine (RaftEngine.forward, CUDA graph) from pinned host frames, one engine per mode, in
    alternating rounds;
  * one rb_update_step and one rb_encoder_forward (the feature encoder on both frames) in each mode, by CUDA events over
    many launches on the engine's own buffers;
  * max-abs and mean EPE between the two modes' flows on the seeded frames.
Prints one JSON line with the card name and power limit read in the same run.

    python tools/bench_mixed_precision.py [--reps 3] [--steps 10]
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

MODES = {"default": capi.RB_MATH_TC, "mixed": capi.RB_MATH_TC_FP16}
CONFIGS = [("raft-things", False, 436, 1024, 32, 1), ("raft-things", False, 436, 1024, 32, 8),
           ("raft-small", True, 768, 1024, 20, 8)]


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


def _events_ms(call, reps):
    for _ in range(3):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        call()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _kernels_ms(eng, mode, reps):
    """rb_update_step (without mask) and the feature encoder on both frames, on the engine's buffers after a forward."""
    lib, P = capi.lib, capi.ptr
    B = eng.pairs
    capi.check(lib.rb_set_math_mode(mode))
    try:
        coords = eng.coords1.clone()  # rb_update_step advances coords1; time it on a scratch copy
        step = lambda: capi.check(lib.rb_update_step(int(eng.small), P(eng.blob), P(eng.ws), P(coords), None, None, B,  # noqa: E731
                                                     eng.h, eng.w, capi.stream()))
        fout = torch.empty_like(eng.fmaps[:2 * B])
        enc = lambda: eng.fnet(eng.images, out=fout)  # noqa: E731
        return round(_events_ms(step, reps), 4), round(_events_ms(enc, max(reps // 4, 5)), 4)
    finally:
        lib.rb_set_math_mode(capi.RB_MATH_TC)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="alternating rounds of each mode")
    ap.add_argument("--steps", type=int, default=10, help="forward calls per round")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"card": _card(), "configs": []}
    for name, small, H, W, iters, B in CONFIGS:
        params = synth.make_weights(small)
        l, r = (torch.from_numpy(x).pin_memory() for x in synth.make_batch(B, H, W))
        engs = {m: RaftEngine(params, small=small, iters=iters, mixed_precision=(m == "mixed")) for m in MODES}
        flows = {m: e.forward(l, r).clone() for m, e in engs.items()}
        d = (flows["mixed"] - flows["default"]).double()
        row = {"model": name, "B": B, "size": [H, W], "iters": iters,
               "flow_diff": {"max_abs": float(d.abs().max()), "mean_epe": float(d.norm(dim=-1).mean()),
                             "max_abs_flow": float(flows["default"].abs().max())},
               "pairs_per_s": {m: [] for m in MODES}}
        for _ in range(a.reps):
            for m, e in engs.items():
                row["pairs_per_s"][m].append(round(_pairs_per_s(e, l, r, a.steps), 2))
        row["update_step_ms"], row["fnet_encoder_ms"] = {}, {}
        for m, e in engs.items():
            row["update_step_ms"][m], row["fnet_encoder_ms"][m] = _kernels_ms(e, MODES[m], 100)
        res["configs"].append(row)
        del engs, flows
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
