"""numpy restatement of frame-rate conversion with a shutter (rb_frame_expose_items / _resized, csrc/interp.cu), built
from interp_oracle's and native_oracle's reversal and blend, for the tests.

Every sample of an output frame is the fp32 value of its item (k, t) -- the reversal of flow_fw[k] by fl32(s t) and of
flow_bw[k] by fl32(s (1 - t)), then the blend of frames k and k + 1 at fl32(t) -- or the prepared input frame itself; the
frame is the fp32 sum from +0.0 of its m values in sample order, each add rounded on its own, divided by m in fp32 and
quantised as vfi_oracle.quantise (rb_frame_metrics' rule).  Also the known-path clip of the quality test.
"""
from __future__ import annotations

import numpy as np

import interp_oracle
import native_oracle
from vfi_oracle import quantise

f32 = np.float32


def item_value(frames, flow_fw, flow_bw, k, t, flow_scale=1.0, hw=None):
    """[H,W,3] fp32 value of the item (k, t): frames [F,H,W,3] prepared fp32 (hw None), or raw [F,Hs,Ws,3] uint8 / fp32
    frames blended at their own size hw from the [F-1,H,W,2] flows (native_oracle)."""
    f0 = interp_oracle.reverse_flow(flow_fw[k:k + 1], time_step=float(f32(flow_scale * t)))
    f1 = interp_oracle.reverse_flow(flow_bw[k:k + 1], time_step=float(f32(flow_scale * (1.0 - t))))
    blend = interp_oracle.synthesize if hw is None else native_oracle.synthesize_resized
    return blend(frames[k:k + 1], frames[k + 1:k + 2], f0[0], f1[0], f0[1], f1[1], float(f32(t)))[0]


def frame_value(frames, i, hw=None):
    """[H,W,3] fp32: input frame i as the kernels read it (raw frames prepared as rb_frames_prepare does)."""
    return np.asarray(frames[i], f32) if hw is None else native_oracle.prepare(frames[i:i + 1])[0]


def expose(values, m):
    """The output frame of m sample values: the fp32 sum from +0.0 in order, / m, quantised."""
    acc = np.zeros_like(values[0], dtype=f32)
    for v in values:
        acc = (acc + np.asarray(v, f32)).astype(f32)
    return quantise((acc / f32(m)).astype(f32))


def motion_blur(frames, flow_fw, flow_bw, samples, m, flow_scale=1.0, hw=None, bgr=False):
    """The frames [N,H,W,3] uint8 of the samples (n, i, t) of raft_b200.video.shutter_schedule() on these frames, each
    value computed once per sample in order."""
    rows = {}
    for n, i, t in samples:
        v = frame_value(frames, i, hw) if t is None else item_value(frames, flow_fw, flow_bw, i, t, flow_scale, hw)
        rows.setdefault(n, []).append(v)
    out = np.stack([expose(rows[n], m) for n in sorted(rows)])
    return out[..., ::-1].copy() if bgr else out


def pan_clip(F, hw, pan=(1.5, 0.7)):
    """The known-path clip [F,Hs,Ws,3] uint8 of stabfill_oracle.render: the texture panned by `pan` pixels per frame."""
    from stabfill_oracle import render
    G = np.stack([np.array([[1.0, 0.0, pan[0] * t], [0.0, 1.0, pan[1] * t], [0.0, 0.0, 1.0]]) for t in range(F)])
    return render(G, hw)


def pan_flows(n_pairs, hw, step, pan=(1.5, 0.7)):
    """The exact flows (fw, bw) [n_pairs,Hs,Ws,2] fp32 between frames `step` apart of pan_clip: frame k's pixel p shows
    the texture at p + k pan, so it moves by -step pan."""
    fw = np.broadcast_to(np.array([-step * pan[0], -step * pan[1]], f32), (n_pairs,) + tuple(hw) + (2,)).copy()
    return fw, -fw
