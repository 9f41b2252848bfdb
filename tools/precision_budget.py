#!/usr/bin/env python
"""Reproduces the operand-format table of DESIGN.md section 2 (why every product costs 3 fp16 MMAs).

The CPU oracle is run with the operands of every convolution and of the correlation matmul rounded the way each
tensor-core format would round them (oracle/raft_oracle.py: EMULATE), fp32 accumulation emulated by fp64 sums of the
rounded products, and the final flow is compared with the fp64 oracle.  The row fp16_conv rounds the conv operands only
and keeps the correlation matmul exact (tests/mixed_oracle.py): the boundary of upstream RAFT's --mixed_precision and of
RB_MATH_TC_FP16.  Test infrastructure: imports oracle/ and tests/mixed_oracle.py.

    python tools/precision_budget.py                 # 128x256 frames, 32 iterations (the DESIGN.md table; ~2 min)
    python tools/precision_budget.py --quick         # 64x96, 8 iterations (what tests/test_precision_budget.py runs)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "raft-tf_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

MODES = [None, "bf16", "fp16", "fp16_conv", "tf32", "bf16x3", "fp16x3"]
COST = {None: "-", "bf16": 1, "fp16": 1, "fp16_conv": 1, "tf32": 2, "bf16x3": 3, "fp16x3": 3}


def budget(H, W, iters, small, modes=MODES):
    from oracle import raft_oracle as O
    from raft_b200 import synth
    p = synth.make_weights(small)
    l, r = synth.make_batch(1, H, W)
    lt, rt = torch.from_numpy(l), torch.from_numpy(r)
    ref = O.RAFTOracle(p, small=small, iters=iters, dtype=torch.float64).forward(lt, rt)
    out = {}
    import contextlib
    import mixed_oracle
    for m in modes:
        O.EMULATE = None if m == "fp16_conv" else m
        try:
            # emulated formats: fp64 arithmetic on rounded operands == exact products, (better than) fp32 accumulation;
            # the fp32 row is the plain fp32 oracle
            dt = torch.float32 if m is None else torch.float64
            with mixed_oracle.fp16_convs() if m == "fp16_conv" else contextlib.nullcontext():
                f = O.RAFTOracle(p, small=small, iters=iters, dtype=dt).forward(lt, rt)
        finally:
            O.EMULATE = None
        out["fp32" if m is None else m] = float((f.double() - ref).abs().max())
    out["max_flow"] = float(ref.abs().max())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    H, W, iters = (64, 96, 8) if a.quick else (128, 256, 32)
    res = {"things": budget(H, W, iters, False), "small": budget(H, W, iters, True), "H": H, "W": W, "iters": iters}
    print(f"| operand format | raft-things | raft-small | cost (fp16-MMA units) |   ({H}x{W}, {iters} iterations, max-abs error of the final flow vs fp64)")
    print("|---|---|---|---|")
    for m in MODES:
        k = "fp32" if m is None else m
        print(f"| {k} | {res['things'][k]:.1e} | {res['small'][k]:.1e} | {COST[m]} |")
    print(f"max |flow|: things {res['things']['max_flow']:.2f} px, small {res['small']['max_flow']:.2f} px")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
