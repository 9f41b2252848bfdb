#!/usr/bin/env python
"""Keyframe label propagation (rb_flow_accumulate, rb_labels_propagate, rb_label_metrics, video_propagate and DAVIS
evaluation), one JSON line per measurement:

1. kernels: one rb_flow_accumulate step and one rb_labels_propagate row, for 436x1024 flows with labels at their own size
   and for 432x1024 flows with labels at 1080x1920.  The flows are a seeded smooth random field (a few pixels of motion)
   with bw = -fw plus noise.  CUDA events around `--reps` back-to-back calls of the C entries on preallocated buffers
   (8 steps per accumulate call, 8 rows per labels call), median of 5 windows.  Bytes per step: the model's minimum
   (pull flow, prev row and status read, acc and status written: 8 + 8 + 1 + 8 + 1 B per pixel, the test flow only
   where it is sampled) next to the measured time.
2. rb_label_metrics per 480x854 frame with 1, 5 and 10 objects (bound_pix 8, DAVIS's): the same timing, 8 frames per
   call.  Bytes: two uint8 maps read (2 B per pixel) and the counts; work: per object present in a tile, three
   neighbours per pixel for each boundary and a disk search of up to 201 offsets per boundary pixel.
3. video_propagate end to end (decode, upload, bidirectional flow, accumulation, labels, PNG writes) on a seeded
   synthetic 24-frame 436x1024 pan as PNG files, raft-things, 20 iterations, batch 8, 4 workers, the keyframe on frame 0
   and on the last frame (the reverse sweep re-runs every pass but the last); host clock, median of `--steps` runs,
   against forward_sequence_bidirectional(check=False) alone on the same passes with the frames on the device.
4. DAVIS evaluation throughput on a synthetic 480x854 tree (3 sequences of 24 frames, 3 objects), batch 1 and 8.

Seeded random weights; everything is written to a temporary directory.

    python tools/bench_propagate.py [--reps 100] [--steps 3]
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
for _p in (ROOT, os.path.join(ROOT, "raft-tf_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
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
    import propagate_oracle as P
    from networks.RAFT import RAFT
    from networks.utils import accumulate_flow, label_metrics, propagate_labels
    from raft_b200 import capi, synth
    from raft_b200.evaluate import evaluate
    from raft_b200.video import interp_schedule, video_propagate, write_labels

    if not torch.cuda.is_available():
        raise SystemExit("bench_propagate needs a CUDA device")
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

    # 1. the accumulation step and the labels
    rng = np.random.default_rng(0)
    for (H, W), (Hs, Ws) in (((436, 1024), (436, 1024)), ((432, 1024), (1080, 1920))):
        f = gaussian_filter(rng.normal(0, 1, (T, H, W, 2)), sigma=(0, 24, 24, 0), mode="wrap")
        fw = (4.0 * f / np.abs(f).max()).astype(np.float32)
        bw = (-fw + rng.normal(0, 0.3, fw.shape)).astype(np.float32)
        fw_d, bw_d = torch.from_numpy(fw).to(dev), torch.from_numpy(bw).to(dev)
        acc = torch.zeros(T + 1, H, W, 2, device=dev)
        st = torch.zeros(T + 1, H, W, dtype=torch.uint8, device=dev)
        accumulate_flow(fw_d, bw_d, acc, st)
        want_a, want_s = P.accumulate(fw[:1], bw[:1], np.zeros((2, H, W, 2), np.float32), np.zeros((2, H, W), np.uint8))
        assert np.array_equal(acc[1].cpu().numpy().view(np.uint32), want_a[1].view(np.uint32))
        assert np.array_equal(st[1].cpu().numpy(), want_s[1])
        key = torch.from_numpy((np.arange(Hs * Ws).reshape(Hs, Ws) // 5000 % 7).astype(np.uint8)).to(dev)
        labels, status = propagate_labels(acc, st, key)
        acc_args = (capi.ptr(fw_d), capi.ptr(bw_d), T, H, W, T, 1.0, 0.01, 0.5, 0, capi.ptr(acc), capi.ptr(st),
                    capi.stream())
        lab_args = (capi.ptr(acc), capi.ptr(st), T, H, W, capi.ptr(key), Hs, Ws, capi.ptr(labels), capi.ptr(status),
                    capi.stream())
        t_acc, w_acc = timed(lambda: capi.check(capi.lib.rb_flow_accumulate(*acc_args)))
        t_lab, w_lab = timed(lambda: capi.check(capi.lib.rb_labels_propagate(*lab_args)))
        step, row = t_acc / T, t_lab / T
        step_bytes = H * W * (8 + 8 + 1 + 8 + 1)
        row_bytes = Hs * Ws * 2 + H * W * 9
        print(json.dumps({"benchmark": "propagate_kernels", "flow_hw": [H, W], "labels_hw": [Hs, Ws],
                          "us_per_accumulate_step": step * 1e6, "accumulate_step_min_bytes": step_bytes,
                          "accumulate_GBps": step_bytes / step / 1e9, "us_per_labels_row": row * 1e6,
                          "labels_row_min_bytes": row_bytes, "labels_GBps": row_bytes / row / 1e9,
                          "status_counts_last_row": [int((st[-1] == k).sum()) for k in range(3)],
                          "windows_accumulate_us": [w * 1e6 for w in w_acc],
                          "windows_labels_us": [w * 1e6 for w in w_lab], **ctx}), flush=True)
        del fw_d, bw_d, acc, st, labels, status

    # 2. the label metrics
    H, W, n = 480, 854, 8
    yy, xx = np.mgrid[0:H, 0:W]
    for objs in (1, 5, 10):
        pred = np.zeros((n, H, W), np.uint8)
        for i in range(n):
            for o in range(1, objs + 1):
                cy, cx = rng.uniform(0, H), rng.uniform(0, W)
                pred[i][((yy - cy) / rng.uniform(30, 120)) ** 2 + ((xx - cx) / rng.uniform(30, 200)) ** 2 <= 1] = o
        gt = np.stack([np.roll(p, (3, -4), (0, 1)) for p in pred])
        p_d, g_d = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
        counts = label_metrics(p_d, g_d, objs, 8)
        args_lm = (capi.ptr(p_d), capi.ptr(g_d), n, H, W, objs, 8, capi.ptr(counts), capi.stream())
        t, w = timed(lambda: capi.check(capi.lib.rb_label_metrics(*args_lm)))
        c = counts.cpu().numpy()
        print(json.dumps({"benchmark": "label_metrics", "hw": [H, W], "objects": objs, "bound_pix": 8,
                          "us_per_frame": t / n * 1e6, "min_bytes_per_frame": 2 * H * W + objs * 48,
                          "GBps": 2 * H * W / (t / n) / 1e9, "boundary_pixels_per_frame": float(c[..., 2:4].sum() / n),
                          "windows_us": [x * 1e6 for x in w], **ctx}), flush=True)

    # 3. video_propagate and the flow alone; 4. DAVIS
    Hc, Wc = 436, 1024
    model = RAFT((Hc, Wc, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, Hc + 2 * N_CLIP, Wc + 3 * N_CLIP, seed0=4321)
    pan = [np.clip(np.rint(base[0, 2 * k:2 * k + Hc, 3 * k:3 * k + Wc] * 255), 0, 255).astype(np.uint8)
           for k in range(N_CLIP)]
    tmp = tempfile.mkdtemp(prefix="bench_propagate_")
    try:
        d = os.path.join(tmp, "frames")
        os.makedirs(d)
        for k, img in enumerate(pan):
            cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)
        key = np.zeros((Hc, Wc), np.uint8)
        key[100:300, 200:600] = 1
        key[150:400, 500:900] = 2
        write_labels(os.path.join(tmp, "key.png"), key, synth.DAVIS_PALETTE)
        times = {0: [], N_CLIP - 1: []}
        for i in range(args.steps + 1):
            for K in times:
                out = os.path.join(tmp, "out")
                shutil.rmtree(out, ignore_errors=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                _, last = video_propagate(model, d, out, os.path.join(tmp, "key.png"), frame=K, batch=T, workers=4)
                torch.cuda.synchronize()
                if i:  # the first run captures the CUDA graph
                    times[K].append(time.perf_counter() - t0)
        engine = model.engine()
        passes = interp_schedule(N_CLIP, T)
        clips = [torch.from_numpy(np.stack([pan[i] for i in p.frames])).to(dev) for p in passes]
        for c in clips:
            engine.forward_sequence_bidirectional(c, check=False)
        runs = []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            a_ev.record()
            for c in clips:
                engine.forward_sequence_bidirectional(c, check=False)
            b_ev.record()
            torch.cuda.synchronize()
            runs.append(a_ev.elapsed_time(b_ev) / 1e3)
        flow = statistics.median(runs)
        for K, ts in times.items():
            t = statistics.median(ts)
            print(json.dumps({"benchmark": "video_propagate", "key_frame": K,
                              "workload": f"video_propagate, raft-things {Hc}x{Wc}, {ITERS} iterations, {N_CLIP}-frame "
                                          f"seeded synthetic pan as PNG files, batch {T}, 4 workers, seeded weights",
                              "s_per_clip": t, "ms_per_frame": t * 1e3 / N_CLIP, "runs_s": ts,
                              "flow_only_s_per_clip": flow, "ratio_to_flow_only": t / flow, **ctx}), flush=True)
        print(json.dumps({"benchmark": "flow_only", "workload": f"forward_sequence_bidirectional(check=False) on the "
                          f"{len(passes)} passes of batch {T} over the same clip, frames on the device",
                          "s_per_clip": flow, "runs_s": runs, **ctx}), flush=True)
        root = os.path.join(tmp, "davis")
        synth.write_davis_tree(root, [(f"seq{i}", N_CLIP) for i in range(3)], objects=3)
        dm = RAFT(None, SimpleNamespace(small=False), device=dev).load(synth.make_weights(False))
        for batch in (1, 8):
            res, ts = None, []
            for i in range(args.steps + 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = evaluate(dm, root, "davis", batch=batch)
                torch.cuda.synchronize()
                if i:
                    ts.append(time.perf_counter() - t0)
            t = statistics.median(ts)
            r = res["splits"]["val"]
            print(json.dumps({"benchmark": "davis_eval", "batch": batch, "workload": f"DAVIS-2017 protocol on a "
                              f"synthetic 480x854 tree, 3 sequences of {N_CLIP} frames, 3 objects, seeded weights",
                              "s_per_tree": t, "frames_per_s": 3 * N_CLIP / t, "runs_s": ts,
                              "J&F": r["J&F-Mean"], **ctx}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
