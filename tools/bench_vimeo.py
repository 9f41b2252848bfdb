"""Throughput of raft_b200.evaluate's Vimeo-90K pipeline (frame interpolation scored by PSNR / SSIM) and of
rb_frame_metrics.

Writes a synthetic Vimeo-90K-layout triplet tree (raft_b200.synth.write_vimeo_tree: 8-bit PNG triplets of 256x448, the
dataset's frame size) to a temporary directory, then reports in one JSON line:
  * the evaluator's pipeline in triplets/s (decoding threads, pinned staging, RaftEngine.interpolate at t = 0.5,
    rb_frame_metrics; seeded raft-things weights, 20 iterations, 4 threads) at batch 1 and 8 on a warmed engine, against
    RaftEngine.interpolate alone on resident uint8 frames at the same batch -- the gap is what decoding, staging and
    scoring cost;
  * rb_frame_metrics per launch (CUDA events over 200 launches) at 256x448 and 436x1024, B = 1 and 8, with its
    algorithmic bytes/s (fp32 prediction and uint8 ground truth read once: 15 B per pixel);
  * the host oracle (tests/vfi_oracle.py, numpy / scipy fp64) per 256x448 triplet, for contrast;
  * the card's name and power limit, read in the same run.

    python tools/bench_vimeo.py [--triplets 64] [--reps 2] [--workers 4]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from raft_b200 import capi, synth  # noqa: E402

H, W, ITERS = 256, 448, 20


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def _pipeline_rate(engine, trips, batch, workers, reps):
    """The evaluator's pipeline (decode threads, pinned staging, interpolate, rb_frame_metrics) on a warmed engine."""
    from raft_b200.evaluate import _run_vimeo
    _run_vimeo(engine, trips, batch, workers, False)  # warm-up: graph capture, page cache
    rates = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        _run_vimeo(engine, trips, batch, workers, False)
        torch.cuda.synchronize()
        rates.append(round(len(trips) / (time.perf_counter() - t), 2))
    return rates


def _interpolate_rate(params, batch, steps):
    """RaftEngine.interpolate(left, right, [0.5]) alone on resident uint8 frames at the evaluator's batch."""
    from raft_b200.engine import RaftEngine
    eng = RaftEngine(params, iters=ITERS)
    l, r = synth.make_batch(batch, H, W)
    l, r = (torch.from_numpy(np.round(255 * x).astype(np.uint8)).cuda() for x in (l, r))
    eng.interpolate(l, r, [0.5])
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        eng.interpolate(l, r, [0.5])
    torch.cuda.synchronize()
    return round(steps * batch / (time.perf_counter() - t), 2)


def _metrics_us(B, h, w, launches=200):
    lib, P = capi.lib, capi.ptr
    g = torch.Generator(device="cuda").manual_seed(0)
    gt = torch.randint(0, 256, (B, h, w, 3), device="cuda", generator=g, dtype=torch.uint8)
    pred = (gt.float() / 255 + torch.randn(B, h, w, 3, device="cuda", generator=g) * 0.03).contiguous()
    stats = torch.empty(B, 2, dtype=torch.float64, device="cuda")
    nbytes = capi.size_query(lib.rb_frame_metrics_workspace_bytes, B, h, w)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    call = lambda: capi.check(lib.rb_frame_metrics(P(pred), 0, P(gt), B, h, w, P(stats), P(ws), nbytes,  # noqa: E731
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
    return {"B": B, "size": [h, w], "us": round(us, 2), "algorithmic_GBps": round(B * h * w * 15 / (us * 1e-6) / 1e9, 1)}


def _oracle_ms(n=4):
    import vfi_oracle
    rng = np.random.default_rng(0)
    gt = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    pred = (gt / np.float32(255) + rng.normal(0, 0.03, gt.shape)).astype(np.float32)
    t = time.perf_counter()
    vfi_oracle.frame_stats(pred, gt)
    return round(1000.0 * (time.perf_counter() - t) / n, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--triplets", type=int, default=64)
    ap.add_argument("--reps", type=int, default=2, help="timed evaluator passes per batch size")
    ap.add_argument("--workers", type=int, default=4)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    params = synth.make_weights(False)
    res = {"card": _card(), "size": [H, W], "iters": ITERS, "workers": a.workers, "triplets": a.triplets}
    with tempfile.TemporaryDirectory() as root:
        t = time.perf_counter()
        synth.write_vimeo_tree(root, [(H, W)] * a.triplets)
        res["dataset_write_s"] = round(time.perf_counter() - t, 1)
        from raft_b200.engine import RaftEngine
        from raft_b200.evaluate import vimeo_triplets
        trips = vimeo_triplets(root)
        res["pipeline"] = []
        for batch in (1, 8):
            engine = RaftEngine(params, iters=ITERS)
            rates = _pipeline_rate(engine, trips, batch, a.workers, a.reps)
            del engine
            interp = _interpolate_rate(params, batch, max(32 // batch, 4))
            res["pipeline"].append({"batch": batch, "pipeline_triplets_per_s": rates,
                                    "interpolate_triplets_per_s": interp,
                                    "pipeline_over_interpolate": round(max(rates) / interp, 3)})
            torch.cuda.empty_cache()
    res["frame_metrics"] = [_metrics_us(B, h, w) for h, w in ((H, W), (436, 1024)) for B in (1, 8)]
    res["oracle_ms_per_triplet"] = _oracle_ms()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
