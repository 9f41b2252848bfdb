"""Cost of the warm start (F10): rb_flow_forward_interpolate against upstream's host path, forward with and without
flow_init, and submit() warm against cold.  One JSON line:
  * rb_flow_forward_interpolate per launch (CUDA events over --launches launches) at grids 55x128 (436x1024 frames) and
    135x240 (1080p frames), B = 1 and 8, with L2 warm (back-to-back launches) and flushed (a 256 MB write before each
    timed launch); on flows like RAFT's, and the worst cases: one valid source per sample, every source in one cell;
  * upstream's host path per pair on the same machine: flow_low to the host, upstream's numpy + scipy griddata
    forward_interpolate per sample, the result back to the device;
  * RaftEngine.forward against forward(flow_init=..., return_low=True), raft-things at 436x1024, 32 iterations, B = 1 and
    8, the two arms alternated over --rounds rounds;
  * submit() on a synthetic Sintel test tree (436x1024, 'clean'), warm against cold, batch 1 and 8, in pairs/s;
  * the card's name and power limit, read in the same run.

    python tools/bench_warm_start.py [--launches 200] [--rounds 3] [--scenes 4]
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


def _flow(kind, B, h, w, seed=0):
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    if kind == "raft":  # smooth motion of a few pixels plus noise; some sources leave the grid
        f = [np.stack([g.uniform(-2, 2) + 1.5 * np.sin(xx / w * 6 + g.uniform(0, 6)),
                       g.uniform(-2, 2) + 1.5 * np.cos(yy / h * 6 + g.uniform(0, 6))], -1) + g.normal(0, 0.5, (h, w, 2))
             for _ in range(B)]
        f = np.stack(f)
    elif kind == "one_valid":  # every source but one leaves the grid, the one lands in a corner
        f = np.full((B, h, w, 2), 1.0e4, np.float32)
        f[:, 0, 0] = (0.5, 0.5)
    else:  # "one_cell": every source lands in cell (w/2, h/2)
        f = np.stack([w / 2 + 0.5 - xx, h / 2 + 0.5 - yy], -1)[None].repeat(B, 0)
        f = f + g.uniform(-0.49, 0.49, f.shape)
    return torch.from_numpy(np.ascontiguousarray(f, np.float32)).cuda()


def _kernel_us(kind, B, h, w, launches):
    lib, P = capi.lib, capi.ptr
    src = _flow(kind, B, h, w)
    out = torch.empty_like(src)
    n = capi.size_query(lib.rb_flow_forward_interpolate_workspace_bytes, B, h, w)
    ws = torch.empty(n, dtype=torch.uint8, device="cuda")
    call = lambda: capi.check(lib.rb_flow_forward_interpolate(P(src), P(out), B, h, w, P(ws), n, capi.stream()))  # noqa: E731
    for _ in range(5):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        call()
    b.record()
    torch.cuda.synchronize()
    warm = 1000.0 * a.elapsed_time(b) / launches
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
    for e0, e1 in ev:
        flush.fill_(1)
        e0.record()
        call()
        e1.record()
    torch.cuda.synchronize()
    cold = 1000.0 * sum(e0.elapsed_time(e1) for e0, e1 in ev) / launches
    return {"flow": kind, "B": B, "grid": [h, w], "us_l2_warm": round(warm, 2), "us_l2_flushed": round(cold, 2)}


def _host_ms(B, h, w, reps=5):
    """upstream's path per pair: .cpu(), numpy + scipy forward_interpolate per sample, back to the device."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_warm_start import upstream_forward_interpolate
    low = _flow("raft", B, h, w)
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        host = low.cpu().numpy()
        res = [upstream_forward_interpolate(np.ascontiguousarray(host[b].transpose(2, 0, 1))).transpose(1, 2, 0)
               for b in range(B)]
        torch.from_numpy(np.ascontiguousarray(np.stack(res))).cuda()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1000.0 / B)
    return {"B": B, "grid": [h, w], "ms_per_pair": round(min(times), 2), "ms_per_pair_median": round(float(np.median(times)), 2)}


def _forward_rates(params, B, rounds, steps):
    from networks.utils import forward_interpolate
    from raft_b200.engine import RaftEngine
    eng = RaftEngine(params, iters=ITERS)
    l, r = synth.make_batch(B, H, W)
    l, r = (torch.from_numpy(np.round(255 * x).astype(np.uint8)).cuda() for x in (l, r))
    low, _ = eng.forward(l, r, return_low=True)
    init = forward_interpolate(low)
    arms = {"cold": lambda: eng.forward(l, r), "warm": lambda: eng.forward(l, r, flow_init=init, return_low=True)}
    for f in arms.values():
        f()
    out = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(steps):
                f()
            torch.cuda.synchronize()
            out[k].append(round(steps * B / (time.perf_counter() - t), 2))
    return {"B": B, "cold_pairs_per_s": out["cold"], "warm_pairs_per_s": out["warm"]}


def _write_test_tree(root, scenes, frames):
    import cv2
    for i in range(scenes):
        d = os.path.join(root, "test", "clean", f"scene_{i}")
        os.makedirs(d)
        for k in range(0, frames, 2):
            for j, f in enumerate(synth.make_pair(H, W, 900 + 10 * i + k)):
                if k + j < frames:
                    cv2.imwrite(os.path.join(d, f"frame_{k + j + 1:04d}.png"), np.round(255 * f).astype(np.uint8))
    return scenes * (frames - 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scenes", type=int, default=8, help="scenes of 9 frames in the synthetic Sintel test tree")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from networks.RAFT import RAFT
    from raft_b200.evaluate import submit
    res = {"card": _card(), "launches": a.launches}
    res["forward_interpolate"] = [_kernel_us("raft", B, h, w, a.launches) for h, w in ((55, 128), (135, 240)) for B in (1, 8)]
    res["forward_interpolate"] += [_kernel_us(k, B, h, w, a.launches) for k in ("one_valid", "one_cell")
                                   for h, w in ((55, 128), (135, 240)) for B in (1, 8)]
    res["upstream_host_path"] = [_host_ms(B, h, w) for h, w in ((55, 128), (135, 240)) for B in (1, 8)]
    params = synth.make_weights(False)
    res["forward"] = {"size": [H, W], "iters": ITERS, "runs": [_forward_rates(params, B, a.rounds, max(16 // B, 2) * 2)
                                                                for B in (1, 8)]}
    torch.cuda.empty_cache()
    model = RAFT(None, SimpleNamespace(small=False)).load(params)
    with tempfile.TemporaryDirectory() as root:
        n = _write_test_tree(root, a.scenes, 9)
        res["submit"] = {"pairs": n, "runs": []}
        for batch in (1, 8):
            for warm in (False, True, False, True):
                with tempfile.TemporaryDirectory() as out:
                    t = time.perf_counter()
                    submit(model, root, "sintel", out, dstypes=("clean",), batch=batch, warm_start=warm)
                    res["submit"]["runs"].append({"batch": batch, "warm": warm,
                                                  "pairs_per_s": round(n / (time.perf_counter() - t), 2)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
