"""Operand traffic of the update step's tensor-core convs: for each conv_tc_kernel launch of one rb_update_step (B = 1,
440x1024 -> 55 x 128 grid), its kernel time from torch.profiler, the bytes its TMA loads move from L2 into shared memory,
and its MMA FLOPs, both over that time.

Bytes come from the launch log (rb_debug_conv_log: tile width N, pixel box, tiles, halo rows, kh, kw, channel chunks):
per 128-pixel x N-channel tile and 64-channel chunk, the weight tiles (kh kw N rows of 128 B per plane) plus the
activation boxes (kh kw boxes of 128 rows, or kw halo boxes of `halo rows`, of 128 B per plane).  Rows TMA zero-fills outside the image count too, so this is what
lands in shared memory, an upper bound of the L2 reads.  FLOPs are the MMAs issued: 2 x 128 x N x
64 per tile, chunk and tap, times the wgmma per product (3 split, 1 single pass).

    python tools/conv_traffic.py [--steps 20] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "raft-tf_b200"))


FIELDS = ("block_n", "bw_log2", "grid", "stages", "total_tiles", "halo_rows", "kh", "kw", "chunks", "passes")


def conv_bytes(rec):
    """(weight bytes, activation bytes) the TMA loads of one launch move into shared memory."""
    r = dict(zip(FIELDS, rec))
    planes = 1 if r["passes"] == 1 else 2
    per_tile_chunk = planes * r["kh"] * r["kw"] * 128  # bytes per row of a tile's operands, over the taps
    act_rows = r["halo_rows"] / r["kh"] if r["halo_rows"] else 128  # per tap: one halo box per kx feeds all kh taps
    return (r["total_tiles"] * r["chunks"] * per_tile_chunk * r["block_n"],
            int(r["total_tiles"] * r["chunks"] * per_tile_chunk * act_rows))


def conv_flops(rec):
    r = dict(zip(FIELDS, rec))
    return 2 * r["total_tiles"] * 128 * r["block_n"] * 64 * r["chunks"] * r["kh"] * r["kw"] * r["passes"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--json", help="also write the table as JSON here")
    a = ap.parse_args()
    import torch
    from raft_b200 import capi, synth
    from raft_b200.weights import pack_update_block
    assert torch.cuda.is_available(), "conv_traffic measures kernel times on the GPU"
    dev = torch.device("cuda:0")
    lib = capi.lib
    B, h, w, s = 1, 55, 128, 0
    torch.manual_seed(0)
    pyr = torch.randn(capi.size_query(lib.rb_corr_pyramid_bytes, B, h, w) // 4, device=dev)
    grid = torch.stack(torch.meshgrid(torch.arange(w), torch.arange(h), indexing="xy"), -1).float()[None]
    coords = (grid + torch.rand(B, h, w, 2) * 8 - 4).to(dev).contiguous()
    ws = torch.zeros(capi.size_query(lib.rb_update_workspace_bytes, s, B, h, w), dtype=torch.uint8, device=dev)
    blob = pack_update_block(synth.make_weights(False), False, dev)
    net = torch.tanh(torch.randn(B, h, w, 128, device=dev))
    inp = torch.relu(torch.randn(B, h, w, 128, device=dev))
    capi.check(lib.rb_update_set_state(s, capi.ptr(blob), capi.ptr(ws), capi.ptr(net), capi.ptr(inp), B, h, w, capi.stream()))
    capi.check(lib.rb_update_lookup(s, capi.ptr(ws), capi.ptr(pyr), capi.ptr(coords), B, h, w, capi.stream()))
    c1 = coords.clone()

    def step():
        capi.check(lib.rb_update_step(s, capi.ptr(blob), capi.ptr(ws), capi.ptr(c1), None, None, B, h, w, capi.stream()))

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    capi.check(lib.rb_debug_conv_override(0, 0, 0, 0))  # restarts the launch log
    step()
    torch.cuda.synchronize()
    rec = (C.c_int * len(FIELDS))()
    n = lib.rb_debug_conv_log(0, rec)
    assert n > 0, capi.lib.rb_last_error()
    recs = []
    for i in range(n):
        assert lib.rb_debug_conv_log(i, rec) == n
        recs.append(tuple(rec))
    names = ["convf1", "convf2", "convc1", "convc2", "motion", "zr1", "q1", "zr2", "q2", "fh1", "fh2"]
    assert n == len(names), (n, recs)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    kern = [e for e in ev if e.get("cat") == "kernel" and "conv_tc_kernel" in e.get("name", "")]
    kern.sort(key=lambda e: e["args"]["correlation"])  # host launch order
    assert len(kern) == n * a.steps, (len(kern), n, a.steps)
    dur = [0.0] * n
    for i, e in enumerate(kern):
        dur[i % n] += e["dur"] / a.steps  # us
    print(f"device {torch.cuda.get_device_name(0)}; B = {B}, {h} x {w} grid; mean over {a.steps} steps")
    print(f"{'conv':7s} {'N':>4s} {'box':>6s} {'halo':>5s} {'tiles':>5s} {'grid':>4s} {'ring':>4s} {'us':>7s} "
          f"{'W MB':>7s} {'A MB':>7s} {'TB/s':>6s} {'TFLOP/s':>8s}")
    rows, tw, ta, tt, tf = [], 0, 0, 0.0, 0
    for nm, r, t in zip(names, recs, dur):
        wb, ab = conv_bytes(r)
        block_n, bwl, grid_, stages, tiles, halo_rows = r[:6]
        flops = conv_flops(r)
        tw += wb; ta += ab; tt += t; tf += flops
        box = f"{128 >> bwl}x{1 << bwl}"
        print(f"{nm:7s} {block_n:4d} {box:>6s} {halo_rows:5d} {tiles:5d} {grid_:4d} {stages:4d} {t:7.1f} {wb / 1e6:7.1f} "
              f"{ab / 1e6:7.1f} {(wb + ab) / t / 1e6:6.2f} {flops / t / 1e6:8.1f}")
        rows.append(dict(conv=nm, block_n=block_n, box=box, halo_rows=halo_rows, tiles=tiles, grid=grid_, stages=stages,
                         us=t, weight_bytes=wb, act_bytes=ab, flops=flops))
    print(f"{'sum':7s} {'':4s} {'':>6s} {'':>5s} {'':>5s} {'':>4s} {'':>4s} {tt:7.1f} {tw / 1e6:7.1f} {ta / 1e6:7.1f} "
          f"{(tw + ta) / tt / 1e6:6.2f} {tf / tt / 1e6:8.1f}   (sum of kernel times; the two side-stream convs overlap)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(device=torch.cuda.get_device_name(0), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
