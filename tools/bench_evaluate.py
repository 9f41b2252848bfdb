"""Throughput of raft_b200.evaluate's pipeline (upstream's Sintel validation protocol) and of rb_flow_metrics.

Writes a synthetic Sintel-layout dataset (raft_b200.synth.write_sintel_tree: 8-bit PNG frames and .flo ground truth,
436x1024, 8 scenes x 9 frames = 64 pairs, 'clean' only) to a temporary directory, then reports in one JSON line:
  * the evaluator's pipeline in pairs/s (decoding threads, pinned staging, RaftEngine.forward, rb_flow_metrics; seeded
    raft-things weights, 32 iterations, 4 threads) at batch 1 and 8 on a warmed engine, against RaftEngine.forward
    alone on resident uint8 frames at the same batch -- the gap is what host decoding and staging cost -- and one
    whole evaluate() call (engine construction and graph capture included);
  * rb_flow_metrics per launch at B = 1 and 8 (CUDA events over 200 launches) with its algorithmic bytes/s
    (flow + ground truth read once: 16 B per pixel);
  * the card's name and power limit, read in the same run.

    python tools/bench_evaluate.py [--scenes 8] [--reps 2] [--workers 4]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-tf_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from raft_b200 import capi, synth  # noqa: E402

H, W, ITERS = 436, 1024, 32


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def _pipeline_rate(engine, pairs, batch, workers, reps):
    """The evaluator's pipeline (decode threads, pinned staging, forward, rb_flow_metrics) on a warmed engine: pairs/s."""
    from raft_b200.evaluate import _run
    _run(engine, pairs, False, batch, workers, False)  # warm-up: graph capture, page cache
    rates = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        _run(engine, pairs, False, batch, workers, False)
        torch.cuda.synchronize()
        rates.append(round(len(pairs) / (time.perf_counter() - t), 2))
    return rates


def _forward_rate(params, batch, steps):
    """RaftEngine.forward alone on resident uint8 frames (the evaluator's input type) at the evaluator's batch."""
    from raft_b200.engine import RaftEngine
    eng = RaftEngine(params, iters=ITERS)
    l, r = synth.make_batch(batch, H, W)
    l, r = (torch.from_numpy(np.round(255 * x).astype(np.uint8)).cuda() for x in (l, r))
    eng.forward(l, r)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        eng.forward(l, r)
    torch.cuda.synchronize()
    return round(steps * batch / (time.perf_counter() - t), 2)


def _metrics_us(B, launches=200):
    lib, P = capi.lib, capi.ptr
    g = torch.Generator(device="cuda").manual_seed(0)
    flow = torch.randn(B, H, W, 2, device="cuda", generator=g) * 10
    gt = torch.randn(B, H, W, 2, device="cuda", generator=g) * 10
    stats = torch.empty(B, 6, dtype=torch.float64, device="cuda")
    nbytes = capi.size_query(lib.rb_flow_metrics_workspace_bytes, B, H, W)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    call = lambda: capi.check(lib.rb_flow_metrics(P(flow), 1.0, P(gt), None, B, H, W, None, P(stats), P(ws), nbytes,  # noqa: E731
                                                 capi.stream()))
    for _ in range(5):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        call()
    b.record()
    torch.cuda.synchronize()
    us = 1000.0 * a.elapsed_time(b) / launches
    return {"B": B, "us": round(us, 2), "algorithmic_GBps": round(B * H * W * 16 / (us * 1e-6) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=8, help="scenes of 9 frames (8 pairs each)")
    ap.add_argument("--reps", type=int, default=2, help="timed evaluate passes per batch size")
    ap.add_argument("--workers", type=int, default=4)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from networks.RAFT import RAFT
    params = synth.make_weights(False)
    res = {"card": _card(), "size": [H, W], "iters": ITERS, "workers": a.workers}
    with tempfile.TemporaryDirectory() as root:
        t = time.perf_counter()
        res["pairs"] = synth.write_sintel_tree(root, a.scenes, 9, H, W, dstypes=("clean",))
        res["dataset_write_s"] = round(time.perf_counter() - t, 1)
        from raft_b200.engine import RaftEngine
        from raft_b200.evaluate import evaluate, sintel_pairs
        pairs = sintel_pairs(root, "clean")
        res["pipeline"] = []
        for batch in (1, 8):
            engine = RaftEngine(params, iters=ITERS)
            rates = _pipeline_rate(engine, pairs, batch, a.workers, a.reps)
            del engine
            fwd = _forward_rate(params, batch, max(16 // batch, 2) * 4)
            res["pipeline"].append({"batch": batch, "pipeline_pairs_per_s": rates, "forward_pairs_per_s": fwd,
                                    "pipeline_over_forward": round(max(rates) / fwd, 3)})
            torch.cuda.empty_cache()
        model = RAFT(None, SimpleNamespace(small=False)).load(params)
        t = time.perf_counter()
        out = evaluate(model, root, "sintel", dstypes=("clean",), batch=8, workers=a.workers)
        res["evaluate_call_s"] = round(time.perf_counter() - t, 2)
        res["epe"] = out["splits"]["clean"]["epe"]
    res["flow_metrics"] = [_metrics_us(B) for B in (1, 8)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
