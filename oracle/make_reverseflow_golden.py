#!/usr/bin/env python
"""Golden vectors for the flow reversal of frame interpolation (F6): runs the UNMODIFIED reference function
flow_utils.py:reverse_flow_avg_skip_static (lines 166-274 of gonglixue/RAFT-tf; it needs only numpy, cv2 and copy) in
process and stores its inputs and 5-tuple outputs in tests/golden/reverse_flow.npz.  tests/test_reverse_flow.py holds the
numpy restatement (tests/interp_oracle.py) to them bit for bit and tests/test_gpu_interpolate.py holds rb_flow_reverse
to them.  Generated with numpy 2.3 (python-float scalars are 'weak': `flow01 * time_step` stays float32).  The reference
loops over pixels in Python, so the cases are small.  bg = im0 ^ 0x80 where no pixel is meant to be static;
time_step 0 appears only without static pixels (inf * 0 is NaN, on which the reference raises).  Test infrastructure;
the reference checkout is only read here:
    RAFT_REFERENCE=<reference checkout> python oracle/make_reverseflow_golden.py"""
import contextlib
import importlib.util
import io
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ["RAFT_REFERENCE"]


def _cases(rng):
    def u8(h, w):
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)

    def moving(im0):  # no pixel static: every channel differs by 128
        return im0 ^ np.uint8(0x80)

    out = []
    yy, xx = np.mgrid[0:24, 0:32].astype(np.float32)
    smooth = np.stack([np.sin(xx / 5) * 3 + 0.7, np.cos(yy / 4) * 2 - 0.4], -1).astype(np.float32)
    im = u8(24, 32)
    out += [("smooth_t1", smooth, moving(im), im, 1.0), ("smooth_t1_3", smooth, moving(im), im, 1.0 / 3.0)]
    noise = rng.normal(0, 4, (20, 28, 2)).astype(np.float32)
    im = u8(20, 28)
    out += [("noise_t05", noise, moving(im), im, 0.5), ("noise_t0", noise, moving(im), im, 0.0)]
    ties = rng.choice(np.array([-2.5, -1.5, -0.5, 0.5, 1.5, 2.5], np.float32), (12, 16, 2))
    im = u8(12, 16)
    out += [("ties", ties, moving(im), im, 1.0), ("ties_t05", ties * np.float32(2), moving(im), im, 0.5)]
    huge = (rng.choice(np.array([-1, 1], np.float32), (10, 14, 2)) * rng.choice(np.array([1e30, 1e6, 3e3], np.float32),
                                                                                  (10, 14, 2))).astype(np.float32)
    im = u8(10, 14)
    out.append(("huge", huge, moving(im), im, 1.0))
    yy, xx = np.mgrid[0:16, 0:20].astype(np.float32)
    mag = (10.0 ** rng.uniform(-3, 3, (16, 20, 2))).astype(np.float32)
    converge = np.stack([-(xx + mag[..., 0]), -(yy + mag[..., 1])], -1).astype(np.float32)  # all onto (0, 0)
    im = u8(16, 20)
    out.append(("converge", converge, moving(im), im, 1.0))
    inf = rng.normal(0, 3, (14, 18, 2)).astype(np.float32)
    inf.reshape(-1)[rng.choice(inf.size, 40, replace=False)] = np.float32(np.inf)
    inf.reshape(-1)[rng.choice(inf.size, 40, replace=False)] = np.float32(-np.inf)
    im = u8(14, 18)
    out.append(("inf_tm05", inf, moving(im), im, -0.5))
    # uint8 static masks on both sides of the wrap: deltas -12..12 per channel (bg = im0 - 5 wraps to 251: not static)
    im = u8(18, 22)
    delta = rng.integers(-12, 13, (18, 22, 1)) * np.ones((1, 1, 3), np.int64)
    delta[rng.random((18, 22)) < 0.3] = rng.integers(-12, 13, 3)
    bg = ((im.astype(np.int64) + delta) % 256).astype(np.uint8)
    out.append(("u8_static", rng.normal(0, 2, (18, 22, 2)).astype(np.float32), bg, im, 1.0))
    imf = rng.uniform(0, 255, (15, 19, 3)).astype(np.float32)
    bgf = (imf + rng.normal(0, 8, imf.shape)).astype(np.float32)
    out.append(("f32_images", rng.normal(0, 2, (15, 19, 2)).astype(np.float32), bgf, imf, 0.5))
    im = u8(9, 11)
    out.append(("all_static", rng.normal(0, 2, (9, 11, 2)).astype(np.float32), im.copy(), im, 1.0))
    bg = im.copy()
    bg[4, 6] ^= np.uint8(0x80)
    out.append(("one_source", rng.normal(0, 2, (9, 11, 2)).astype(np.float32), bg, im, 1.0))
    im = u8(1, 17)
    out.append(("row", rng.normal(0, 3, (1, 17, 2)).astype(np.float32), moving(im), im, 1.0))
    im = u8(13, 1)
    out.append(("column", rng.normal(0, 3, (13, 1, 2)).astype(np.float32), moving(im), im, 0.5))
    return out


def main():
    spec = importlib.util.spec_from_file_location("ref_flow_utils", os.path.join(REF, "flow_utils.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    rng = np.random.default_rng(20261015)
    out = {}
    for name, flow, bg, im0, ts in _cases(rng):
        with contextlib.redirect_stdout(io.StringIO()):  # the reference prints two progress lines per call
            res = ref.reverse_flow_avg_skip_static(flow.copy(), bg.copy(), im0.copy(), float(ts))
        out[f"{name}/flow"], out[f"{name}/bg"], out[f"{name}/im0"] = flow, bg, im0
        out[f"{name}/time_step"] = np.array(ts, np.float64)
        for k, r in enumerate(res):
            out[f"{name}/out{k}"] = np.asarray(r)
    path = os.path.join(ROOT, "tests", "golden", "reverse_flow.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; numpy", np.__version__)


if __name__ == "__main__":
    main()
