#!/usr/bin/env python
"""Scene-cut detection (rb_scene_cut_scores and video_interpolate(scene_cut=...)), one JSON line per measurement:

1. kernel: rb_scene_cut_scores on N = 9 frames at 436x1024 and 1080x1920, natural-looking frames (a pan over
   tests/data/frame_0016.png with a little noise) and uniform ones (every pixel in one bin: the worst case for the
   histogram's atomics).  CUDA events around `--reps` launches (memset + two kernels each), median of 5 such windows;
   bytes/s on the N H W 3 frame bytes read, against the H100 SXM data sheet's 3.35 TB/s.  The histograms are checked
   against np.bincount first.
   pass: the scene-cut steps of one pass on an idle GPU -- the T + 1 pinned frames copied to the device buffer, scored,
   and the scores copied back (a wait on the stream) -- host clock, median of 50.
2. no_cuts: video_interpolate(fps=(24, 60)) end to end (decode, upload, flow, interpolation, PNG writes) on a seeded
   synthetic 25-frame pan without cuts, with scene_cut=None and with a threshold, arms alternating; the files of both
   arms are compared byte for byte before timing.  Host clock around each call, which returns after its last write.
3. with_cuts: the same clip with frames 5..9 and 20..24 darkened to a quarter (x // 4: a shot in other colours),
   both arms again: cut pairs found, items and passes that made no engine work, time per output frame.

raft-things, 20 iterations, seeded random weights, frames at their own 436x1024 size, T = 8 pairs per pass, 4 workers.
Frames are written to a temporary directory.

    python tools/bench_scene_cut.py [--reps 200] [--steps 5]
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

HBM_TBS = 3.35
N_KERNEL, N_CLIP, H_IMG, W_IMG, ITERS, T, THR = 9, 25, 436, 1024, 20, 8, 0.5


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200, help="launches per kernel timing window (at least 200)")
    ap.add_argument("--steps", type=int, default=5, help="timed whole-clip runs per arm (at least 3)")
    args = ap.parse_args(argv)
    if args.reps < 200 or args.steps < 3:
        ap.error("--reps >= 200, --steps >= 3")

    import cv2
    import numpy as np
    import torch
    from types import SimpleNamespace
    from networks.RAFT import RAFT
    from raft_b200 import capi, synth
    from raft_b200.video import fps_schedule, video_interpolate

    if not torch.cuda.is_available():
        raise SystemExit("bench_scene_cut needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    gpu, watts = torch.cuda.get_device_name(dev), power_limit_w(dev.index or 0)
    ctx = {"gpu": gpu, "power_limit_w": watts}
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    # 1. the kernel
    src = cv2.imread(os.path.join(ROOT, "tests", "data", "frame_0016.png"))
    rng = np.random.default_rng(0)
    for H, W in ((436, 1024), (1080, 1920)):
        natural = np.stack([np.clip(cv2.resize(np.roll(src, 5 * k, axis=1), (W, H)).astype(np.int16)
                                    + rng.integers(-6, 7, (H, W, 3)), 0, 255).astype(np.uint8)
                            for k in range(N_KERNEL)])
        uniform = np.full((N_KERNEL, H, W, 3), 77, np.uint8)
        for kind, host in (("natural", natural), ("uniform", uniform)):
            frames = torch.from_numpy(host).to(dev)
            hist = torch.empty(N_KERNEL, 512, dtype=torch.int32, device=dev)
            scores = torch.empty(N_KERNEL - 1, dtype=torch.float32, device=dev)
            st = capi.stream()

            def call():
                capi.check(capi.lib.rb_scene_cut_scores(capi.ptr(frames), N_KERNEL, H, W, capi.ptr(hist),
                                                        capi.ptr(scores), st))

            call()
            q = host.astype(np.int64) >> 5
            bins = (q[..., 0] * 64 + q[..., 1] * 8 + q[..., 2]).reshape(N_KERNEL, -1)
            want = np.stack([np.bincount(b, minlength=512) for b in bins])
            assert np.array_equal(hist.cpu().numpy(), want), (kind, H, W)
            for _ in range(20):
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
            t = statistics.median(windows)
            nbytes = N_KERNEL * H * W * 3
            print(json.dumps({"benchmark": "scene_cut_kernel", "frames": kind, "N": N_KERNEL, "H": H, "W": W,
                              "us_per_call": t * 1e6, "frame_bytes": nbytes, "GB_per_s": nbytes / t / 1e9,
                              "share_of_hbm_peak": nbytes / t / (HBM_TBS * 1e12), "reps": args.reps,
                              "windows_us": [w * 1e6 for w in windows], **ctx}), flush=True)

    # the scene-cut work of one pass on an idle GPU: the pinned frames of a pass (T + 1 at 436x1024) to the device buffer,
    # the scores, and their copy back, which waits for the stream (host clock, median of 50)
    from networks.utils import scene_cut_scores
    pinned = torch.from_numpy(natural[:T + 1, :H_IMG, :W_IMG].copy()).pin_memory()
    on_dev = torch.empty(pinned.shape, dtype=torch.uint8, device=dev)
    spans = []
    for i in range(60):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        on_dev.copy_(pinned, non_blocking=True)
        scene_cut_scores(on_dev).cpu()
        if i >= 10:
            spans.append(time.perf_counter() - t0)
    print(json.dumps({"benchmark": "scene_cut_pass", "frames": T + 1, "H": H_IMG, "W": W_IMG,
                      "ms_upload_score_readback": statistics.median(spans) * 1e3,
                      "ms_min": min(spans) * 1e3, "ms_max": max(spans) * 1e3, **ctx}), flush=True)

    # 2. and 3. end to end
    model =RAFT((H_IMG, W_IMG, 3), SimpleNamespace(small=False), iters=ITERS, device=dev).load(synth.make_weights(False))
    base, _ = synth.make_batch(1, H_IMG + 2 * N_CLIP, W_IMG + 3 * N_CLIP, seed0=4321)
    pan = [np.clip(np.rint(base[0, 2 * k:2 * k + H_IMG, 3 * k:3 * k + W_IMG] * 255), 0, 255).astype(np.uint8)
           for k in range(N_CLIP)]
    shots = [(k // 5) % 3 == 1 for k in range(N_CLIP)]  # frames 5..9 and 20..24 a dark shot: cuts at pairs 4, 9, 19
    tmp = tempfile.mkdtemp(prefix="bench_scene_cut_")
    try:
        for name, imgs in (("no_cuts", pan), ("with_cuts", [f // 4 if s else f for f, s in zip(pan, shots)])):
            d = os.path.join(tmp, name)
            os.makedirs(d)
            for k, img in enumerate(imgs):
                cv2.imwrite(os.path.join(d, f"frame_{k:04d}.png"), img)

            def run(out, thr):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = video_interpolate(model, d, out, batch=T, workers=4, fps=(24, 60), scene_cut=thr)
                torch.cuda.synchronize()
                return time.perf_counter() - t0, res

            _, plain = run(os.path.join(tmp, "a"), None)
            _, (paths, cuts) = run(os.path.join(tmp, "b"), THR)
            same = [open(p, "rb").read() == open(q, "rb").read() for p, q in zip(plain, paths)]
            if name == "no_cuts":
                assert cuts == [] and all(same) and len(plain) == len(paths), "scene_cut changed a clip without cuts"
            times = {None: [], THR: []}
            for i in range(2 * args.steps):
                thr = (None, THR)[i % 2] if (i // 2) % 2 == 0 else (THR, None)[i % 2]  # ABBA
                shutil.rmtree(os.path.join(tmp, "c"), ignore_errors=True)
                times[thr].append(run(os.path.join(tmp, "c"), thr)[0])
            passes = fps_schedule(N_CLIP, 24, 60, T)
            n_items = sum(len(p.items) for p in passes)
            skipped = sum(1 for p in passes for _, k, _ in p.items if k in cuts)
            idle = sum(1 for p in passes if all(k in cuts for _, k, _ in p.items))
            n_out = len(plain)
            t_none, t_thr = statistics.median(times[None]), statistics.median(times[THR])
            print(json.dumps({
                "benchmark": f"scene_cut_{name}",
                "workload": f"video_interpolate(fps=(24, 60)), raft-things {H_IMG}x{W_IMG}, {ITERS} iterations, "
                            f"{N_CLIP}-frame seeded synthetic pan as PNG files, batch {T}, 4 workers, seeded random "
                            "weights",
                "threshold": THR, "cuts": cuts, "output_frames": n_out, "items": n_items, "items_copied": skipped,
                "passes": len(passes), "passes_without_engine_call": idle,
                "files_identical_to_plain": sum(same), "s_plain": t_none, "s_scene_cut": t_thr,
                "ms_per_output_frame_plain": t_none * 1e3 / n_out, "ms_per_output_frame_scene_cut": t_thr * 1e3 / n_out,
                "overhead": t_thr / t_none - 1.0, "runs_plain_s": times[None], "runs_scene_cut_s": times[THR],
                **ctx}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
