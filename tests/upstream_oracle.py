"""Upstream (princeton-vl RAFT, PyTorch) semantics on top of the oracle of oracle/raft_oracle.py (TEST INFRASTRUCTURE ONLY).

RB_SEMANTICS_UPSTREAM (include/raft_b200.h) changes three things against the reference's TF port, and nothing else:
  * stride-2 convs pad k // 2 before (PyTorch's symmetric padding) instead of TF 'SAME''s total / 2  (conv2d_up);
  * the correlation lookup is upstream's bilinear_sampler + F.grid_sample(align_corners=True, padding_mode="zeros")
    (sample_corr_up; in fp32 it restates the GPU sampler bit for bit, fma contraction included);
  * raft-small's upflow8 multiplies the flow by 8 (upflow8_up).
``upstream_semantics()`` swaps these into oracle.raft_oracle for the duration of a block, so the encoders, the update loop
and RAFTOracle run unchanged on top of them; ``UpstreamOracle`` is RAFTOracle under it.
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O

_conv2d_tf = O.conv2d


def conv2d_up(x, W, b, stride=1, activation=None):
    """Conv2D with PyTorch's padding = k // 2 (odd kernels: the output is ceil(n / stride) as with 'SAME')."""
    if stride == 1:  # symmetric (k - 1) / 2 either way
        return _conv2d_tf(x, W, b, 1, activation)
    kh, kw = int(W.shape[0]), int(W.shape[1])
    y = F.conv2d(x.permute(0, 3, 1, 2), W.permute(3, 2, 0, 1).contiguous(), b, stride=stride, padding=(kh // 2, kw // 2))
    y = y.permute(0, 2, 3, 1).contiguous()
    return activation(y) if activation is not None else y


def upflow8_up(flow):
    """upstream utils.upflow8: 8 * F.interpolate(flow, 8x, bilinear, align_corners=True)."""
    return 8.0 * O.resize_bilinear_align_corners(flow, 8 * flow.shape[1], 8 * flow.shape[2])


def _fma32(a, b, c):
    """fp32 fma(a, b, c) with a single rounding: a * b is exact in fp64; the fp64 sum is corrected where it lands exactly on
    an fp32 rounding midpoint (the only case in which rounding it again differs from rounding the exact value)."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)  # s + e == p + c exactly (TwoSum)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    d = s - r64
    nb = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    tie = (d != 0) & (2.0 * np.abs(d) == np.abs(nb.astype(np.float64) - r64))
    fix = tie & (e != 0) & (np.sign(e) == np.sign(d))
    return np.where(fix, nb, r)


def _unnorm(x, n, dt):
    """upstream bilinear_sampler's normalisation and PyTorch's CUDA unnormalisation, each step rounded in dtype dt."""
    nm1 = dt(n - 1)
    g = (dt(2) * x) / nm1 - dt(1)
    ix = ((g + dt(1)) * dt(0.5)) * nm1
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(ix) <= dt(16777216.0), ix, dt(-100.0)).astype(dt)


def sample_corr_up(pyramid, coords, num_levels=4, radius=4):
    """SampleCorr with upstream's CorrBlock sampler.  pyramid: levels [B*h*w, h_l, w_l, 1]; coords [b,h,w,2] -> [b,h,w,L*D*D],
    channel = level*D*D + i*D + j (window column i walks x).  fp32 input: the GPU sampler's operation order bit for bit
    (include/raft_b200.h); fp64: the same steps in fp64, summed nw + ne + sw + se."""
    dt = np.float32 if coords.dtype == torch.float32 else np.float64
    b, h, w, _ = coords.shape
    c = coords.detach().cpu().numpy().astype(dt).reshape(b * h * w, 2)
    D = 2 * radius + 1
    d = np.arange(-radius, radius + 1).astype(dt)
    out = []
    for l in range(num_levels):
        V = pyramid[l].detach().cpu().numpy().astype(dt)
        N, Hl, Wl = V.shape[:3]
        flat = V.reshape(N, Hl * Wl)
        inv = dt(1.0 / 2 ** l)
        ix = _unnorm((c[:, 0:1] * inv) + d[None], Wl, dt)  # [N, D] per window column i
        iy = _unnorm((c[:, 1:2] * inv) + d[None], Hl, dt)  # [N, D] per window row j
        x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
        wx0, wx1 = (x0 + 1).astype(dt) - ix, ix - x0.astype(dt)
        wy0, wy1 = (y0 + 1).astype(dt) - iy, iy - y0.astype(dt)

        def val(xx, yy):  # [N, D(i), D(j)], 0 outside the level
            X, Y = np.broadcast_to(xx[:, :, None], (N, D, D)), np.broadcast_to(yy[:, None, :], (N, D, D))
            ok = (X >= 0) & (X < Wl) & (Y >= 0) & (Y < Hl)
            idx = np.where(ok, Y * Wl + X, 0).reshape(N, -1)
            return np.where(ok, np.take_along_axis(flat, idx, 1).reshape(N, D, D), dt(0))
        Inw, Ine, Isw, Ise = val(x0, y0), val(x0 + 1, y0), val(x0, y0 + 1), val(x0 + 1, y0 + 1)
        nw, ne = wx0[:, :, None] * wy0[:, None, :], wx1[:, :, None] * wy0[:, None, :]
        sw, se = wx0[:, :, None] * wy1[:, None, :], wx1[:, :, None] * wy1[:, None, :]
        if dt is np.float32:
            v = _fma32(Ise, se, _fma32(Isw, sw, _fma32(Ine, ne, Inw * nw)))
        else:
            v = Inw * nw + Ine * ne + Isw * sw + Ise * se
        out.append(torch.from_numpy(np.ascontiguousarray(v.reshape(b, h, w, D * D))))
    return torch.cat(out, dim=-1)


@contextlib.contextmanager
def upstream_semantics():
    """oracle.raft_oracle with upstream's stride-2 padding, lookup and upflow8 while the block runs."""
    saved = O.conv2d, O.sample_corr, O.upflow8
    O.conv2d, O.sample_corr, O.upflow8 = conv2d_up, sample_corr_up, upflow8_up
    try:
        yield
    finally:
        O.conv2d, O.sample_corr, O.upflow8 = saved


class UpstreamOracle(O.RAFTOracle):
    """RAFTOracle under upstream_semantics(): princeton-vl RAFT's test_mode forward (frames in [0, 1], H, W multiples of 8)."""

    def forward(self, left, right, iters=None, return_lowres=False):
        with upstream_semantics():
            return super().forward(left, right, iters, return_lowres)
