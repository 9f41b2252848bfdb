"""numpy restatement of the resized frame synthesis (rb_frame_synthesize_pairs_resized / _items_resized, csrc/interp.cu),
built from resize_oracle and interp_oracle, for the tests.

Output pixel p = (x, y) of the frames' Hs x Ws, from flows and empty masks at the network's H x W:
  flow  rb_flow_resize of the reversed flow to Hs x Ws (resize_oracle.resize_flow: cv2's float bilinear resize, then
        u *= fl32(Ws / W), v *= fl32(Hs / H));
  mask  empty[ys, xs], ys = ((2y+1) H) div (2 Hs), xs = ((2x+1) W) div (2 Ws) in 64-bit integers -- the network pixel
        whose area holds p's centre.  Neither cv2's INTER_NEAREST (floor(y Hs / H) style) nor INTER_NEAREST_EXACT picks
        the same pixels at 432x1024 -> 1080x1920;
  frame uint8 values as np.float32(u) / 255 (rb_frames_prepare), fp32 values as they are;
then interp_oracle.synthesize at Hs x Ws.
"""
from __future__ import annotations

import numpy as np

import interp_oracle
import resize_oracle

f32 = np.float32


def nearest_index(src, dst):
    """[dst] int64: the source index of each of dst output positions, ((2d+1) src) div (2 dst)."""
    d = np.arange(int(dst), dtype=np.int64)
    return ((2 * d + 1) * np.int64(src)) // (2 * np.int64(dst))


def nearest(mask, Hs, Ws):
    """[B,H,W] masks -> [B,Hs,Ws] by the centre-containment rule."""
    mask = np.asarray(mask)
    H, W = mask.shape[1:3]
    return mask[:, nearest_index(H, Hs)][:, :, nearest_index(W, Ws)]


def prepare(frames):
    """[B,Hs,Ws,3] uint8 -> np.float32(u) / 255 (correctly rounded fp32 division); fp32 as it is."""
    frames = np.asarray(frames)
    return (frames.astype(f32) / f32(255)).astype(f32) if frames.dtype == np.uint8 else frames.astype(f32)


def synthesize_resized(frame0, frame1, flow_t0, flow_t1, empty0, empty1, t):
    """[B,Hs,Ws,3] frames, [B,H,W,2] flows from time t and [B,H,W] empty masks at the network size -> [B,Hs,Ws,3] fp32."""
    Hs, Ws = np.asarray(frame0).shape[1:3]
    return interp_oracle.synthesize(prepare(frame0), prepare(frame1),
                                    resize_oracle.resize_flow(np.asarray(flow_t0, f32), Hs, Ws),
                                    resize_oracle.resize_flow(np.asarray(flow_t1, f32), Hs, Ws),
                                    nearest(empty0, Hs, Ws), nearest(empty1, Hs, Ws), t)
