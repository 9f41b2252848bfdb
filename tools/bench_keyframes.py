#!/usr/bin/env python
"""Several-keyframe label propagation (rb_labels_propagate_keys, video_propagate with keyframes, DAVIS with a keyframe
step), one JSON line per measurement, each with the card's name and power limit:

1. kernels: one rb_labels_propagate_keys row with one voting side and with two, against one rb_labels_propagate row,
   for 436x1024 rows with labels at their own size and for 432x1024 rows with labels at 1080x1920.  The rows are a
   seeded smooth random displacement field with zero status (so both sides vote where the table gives two).  CUDA
   events around `--reps` back-to-back calls of the C entries on preallocated buffers (8 rows per call), median of 5
   windows.
2. video_propagate end to end (decode, upload, bidirectional flow, chains, labels, PNG writes) on a seeded synthetic
   24-frame 436x1024 pan as PNG files, raft-things, 20 iterations, batch 8, 4 workers: one key on frame 0, keys every 8
   frames (0, 8, 16 and the last frame 23) and every 24 frames (0 and 23); host clock, median of `--steps` runs, and
   torch.cuda.max_memory_allocated over the runs (the interval store included).
3. J&F of the DAVIS protocol on a synthetic write_davis_tree tree (3 sequences of 24 frames at 480x854, 3 objects,
   seeded weights) with one key and with a keyframe every 8 and every 4 frames: a sanity figure, not a quality claim.

Seeded random weights; everything is written to a temporary directory.

    python tools/bench_keyframes.py [--reps 100] [--steps 3]
"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_interpolate import power_limit_w  # noqa: E402

T, N_CLIP, ITERS = 8, 24, 20


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100, help="calls per kernel timing window (at least 20)")
    ap.add_argument("--steps", type=int, default=3, help="timed whole-clip runs (at least 3)")
    args = ap.parse_args(argv)
    if args.reps < 20 or args.steps < 3:
        ap.error("--reps >= 20, --steps >= 3")

    import cv2
    import numpy as np
    import torch
    from scipy.ndimage import gaussian_filter
    from types import SimpleNamespace
    from networks.RAFT import RAFT
    from raft_b200 import capi, synth
    from raft_b200.evaluate import evaluate
    from raft_b200.video import video_propagate, write_labels

    if not torch.cuda.is_available():
        raise SystemExit("bench_keyframes needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    ctx = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index or 0)}
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(call):
        for _ in range(5):
            call()
        windows = []
        for _ in range(5):
            torch.cuda.synchronize()
            a_ev.record()
            for _ in range(args.reps):
                call()
            b_ev.record()
            torch.cuda.synchronize()
            windows.append(a_ev.elapsed_time(b_ev) / 1e3 / args.reps)
        return statistics.median(windows), windows

    # 1. the kernels
    rng = np.random.default_rng(0)
    for (H, W), (Hs, Ws) in (((436, 1024), (436, 1024)), ((432, 1024), (1080, 1920))):
        acc = []
        for _ in range(2):
            f = gaussian_filter(rng.normal(0, 1, (T, H, W, 2)), sigma=(0, 24, 24, 0), mode="wrap")
            acc.append(torch.from_numpy((6.0 * f / np.abs(f).max()).astype(np.float32)).to(dev))
        st = torch.zeros(T, H, W, dtype=torch.uint8, device=dev)
        keys = torch.from_numpy(np.stack([(np.arange(Hs * Ws).reshape(Hs, Ws) // (5000 + 7 * i) % 7)
                                          for i in range(2)]).astype(np.uint8)).to(dev)
        labels = torch.empty(T, Hs, Ws, dtype=torch.uint8, device=dev)
        status = torch.empty_like(labels)
        one = torch.tensor([[0, -1, 0, 0]] * T, dtype=torch.int32, device=dev)
        two = torch.tensor([[0, 1, T - r, r + 1] for r in range(T)], dtype=torch.int32, device=dev)
        single = (capi.ptr(acc[0]), capi.ptr(st), T, H, W, capi.ptr(keys[0]), Hs, Ws, capi.ptr(labels),
                  capi.ptr(status), capi.stream())
        t_single, w_single = timed(lambda: capi.check(capi.lib.rb_labels_propagate(*single)))
        res = {}
        for name, rows in (("one_side", one), ("two_sides", two)):
            a = (capi.ptr(acc[0]), capi.ptr(st), capi.ptr(acc[1]), capi.ptr(st), capi.ptr(rows), T, H, W,
                 capi.ptr(keys), 2, Hs, Ws, capi.ptr(labels), capi.ptr(status), capi.stream())
            t, w = timed(lambda: capi.check(capi.lib.rb_labels_propagate_keys(*a)))
            res[name] = (t, w)
        print(json.dumps({"benchmark": "propagate_keys_kernel", "flow_hw": [H, W], "labels_hw": [Hs, Ws],
                          "us_per_row_labels_propagate": t_single / T * 1e6,
                          "us_per_row_keys_one_side": res["one_side"][0] / T * 1e6,
                          "us_per_row_keys_two_sides": res["two_sides"][0] / T * 1e6,
                          "two_sides_over_single": res["two_sides"][0] / t_single,
                          "windows_us": {"labels_propagate": [x * 1e6 / T for x in w_single],
                                         **{k: [x * 1e6 / T for x in v[1]] for k, v in res.items()}}, **ctx}),
              flush=True)
        del acc, st, keys, labels, status

    # 2. video_propagate with keyframes
    Hc, Wc = 436, 1024
    model = RAFT((Hc, Wc, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, Hc + 2 * N_CLIP, Wc + 3 * N_CLIP, seed0=4321)
    pan = [np.clip(np.rint(base[0, 2 * k:2 * k + Hc, 3 * k:3 * k + Wc] * 255), 0, 255).astype(np.uint8)
           for k in range(N_CLIP)]
    tmp = tempfile.mkdtemp(prefix="bench_keyframes_")
    try:
        d = os.path.join(tmp, "frames")
        os.makedirs(d)
        for k, img in enumerate(pan):
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
        key = np.zeros((Hc, Wc), np.uint8)
        key[100:300, 200:600] = 1
        key[150:400, 500:900] = 2
        names = []
        for i in range(N_CLIP):
            names.append(os.path.join(tmp, f"key{i}.png"))
            write_labels(names[-1], np.roll(key, 3 * i, 1), synth.DAVIS_PALETTE)
        every8 = list(range(0, N_CLIP, 8)) + [N_CLIP - 1]
        runs = {"one key on frame 0": (names[0], 0), "a keyframe every 8": ([names[k] for k in every8], every8),
                "a keyframe every 24": ([names[0], names[-1]], [0, N_CLIP - 1])}
        for label, (labels, frames) in runs.items():
            times, peak = [], 0
            for i in range(args.steps + 1):
                out = os.path.join(tmp, "out")
                shutil.rmtree(out, ignore_errors=True)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(dev)
                t0 = time.perf_counter()
                video_propagate(model, d, out, labels, frame=frames, batch=T, workers=4)
                torch.cuda.synchronize()
                if i:  # the first run captures the CUDA graph
                    times.append(time.perf_counter() - t0)
                    peak = max(peak, torch.cuda.max_memory_allocated(dev))
            t = statistics.median(times)
            print(json.dumps({"benchmark": "video_propagate_keyframes", "keys": label, "key_frames": frames,
                              "workload": f"video_propagate, raft-things {Hc}x{Wc}, {ITERS} iterations, {N_CLIP}-frame "
                                          f"seeded synthetic pan as PNG files, batch {T}, 4 workers, seeded weights",
                              "s_per_clip": t, "ms_per_frame": t * 1e3 / N_CLIP, "runs_s": times,
                              "max_memory_allocated_MB": peak / 2 ** 20, **ctx}), flush=True)

        # 3. DAVIS with a keyframe step
        root = os.path.join(tmp, "davis")
        synth.write_davis_tree(root, [(f"seq{i}", N_CLIP) for i in range(3)], objects=3)
        dm = RAFT(None, SimpleNamespace(small=False), device=dev).load(synth.make_weights(False))
        for step in (None, 8, 4):
            t0 = time.perf_counter()
            res = evaluate(dm, root, "davis", batch=T, keyframe_step=step)
            torch.cuda.synchronize()
            r = res["splits"]["val"]
            print(json.dumps({"benchmark": "davis_keyframe_step", "keyframe_step": step,
                              "workload": f"DAVIS-2017 protocol on a synthetic 480x854 tree, 3 sequences of {N_CLIP} "
                                          "frames, 3 objects, seeded weights (a sanity figure, not a quality claim)",
                              "J&F": r["J&F-Mean"], "J": r["J-Mean"], "F": r["F-Mean"], "J_decay": r["J-Decay"],
                              "s_per_tree": time.perf_counter() - t0, **ctx}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
