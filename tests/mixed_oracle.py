"""Mixed precision (RB_MATH_TC_FP16) on top of the oracle of oracle/raft_oracle.py (TEST INFRASTRUCTURE ONLY).

Upstream RAFT's --mixed_precision runs fnet, cnet and the update block under torch autocast: every conv multiplies
fp16(a) by fp16(w); the correlation is built from fmap.float() outside it.  ``fp16_convs()`` restates that boundary on the
oracle for the duration of a block: whatever conv2d the oracle runs at that point (its own, or upstream_oracle's) is
called on fp16-rounded input and weights -- in fp64 the products are then exact and the sums better than fp32 -- and
nothing else changes: the correlation matmul, the lookup, norms, gates, residuals, coords1 += delta and the upsampling
keep the oracle's own precision, as on the GPU.  Enter it inside upstream_oracle.upstream_semantics() to combine both.

``fold_batch_norm`` restates the one structural difference the GPU keeps on purpose: batch norm is folded into the conv
weights and bias at pack time (rb_encoder_weights_pack), so it is the FOLDED weight that gets rounded to fp16.
"""
from __future__ import annotations

import contextlib
from typing import Dict

import numpy as np

from oracle import raft_oracle as O


def _round16(t):
    return t.half().to(t.dtype)


@contextlib.contextmanager
def fp16_convs():
    """Conv operands rounded to fp16 (round to nearest, like autocast's cast), the correlation exact, while the block
    runs."""
    inner = O.conv2d

    def conv2d_fp16(x, W, b, stride=1, activation=None):
        return inner(_round16(x), _round16(W), b, stride, activation)

    O.conv2d = conv2d_fp16
    try:
        yield
    finally:
        O.conv2d = inner


def fold_batch_norm(params: Dict[str, np.ndarray], small: bool, name: str) -> Dict[str, np.ndarray]:
    """``params`` with every conv of encoder ``name`` that batch norm follows replaced by the folded conv the library packs
    (csrc/encoder.cu, rb_encoder_weights_pack_host): s = gamma / sqrt(var + 1e-5) in fp64, W' = fl32(W * s),
    b' = fl32(b * s + beta - mean * s).  Run the oracle's encoder with norm "none" on the result."""
    from raft_b200 import capi
    lib = capi.lib
    out = dict(params)
    for i in range(lib.rb_encoder_num_convs(int(small))):
        conv = f"{name}/{lib.rb_encoder_conv_name(int(small), i).decode()}"
        norm = lib.rb_encoder_norm_name(int(small), i).decode()
        if not norm:
            continue
        norm = f"{name}/{norm}"
        g, beta = (np.asarray(params[f"{norm}/{k}"], np.float32).astype(np.float64) for k in ("gamma", "beta"))
        mu, var = (np.asarray(params[f"{norm}/{k}/EMA"], np.float32).astype(np.float64) for k in ("mean", "variance"))
        s = g / np.sqrt(var + 1e-5)
        W = np.asarray(params[conv + "/W"], np.float32).astype(np.float64)
        b = np.asarray(params[conv + "/b"], np.float32).astype(np.float64)
        out[conv + "/W"] = (W * s).astype(np.float32)
        out[conv + "/b"] = (b * s + (beta - mu * s)).astype(np.float32)
    return out
