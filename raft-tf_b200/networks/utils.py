"""Drop-in mirror of the reference's ``networks/utils.py`` on torch CUDA tensors; every function
runs a raft_b200 CUDA kernel through the C ABI (no TF, no CPU fallback).  NHWC like the reference."""
import torch

from raft_b200 import capi


def coords_grid(batch, ht, wd, device=None):
    """utils.py:4-11 -> [b,h,w,2] with channel 0 = x, 1 = y."""
    device = torch.device(device if device is not None else "cuda")
    out = torch.empty(int(batch), int(ht), int(wd), 2, dtype=torch.float32, device=device)
    with torch.cuda.device(out.device):
        capi.check(capi.lib.rb_coords_grid(capi.ptr(out), int(batch), int(ht), int(wd), capi.stream()))
    return out


def bilinear_sampler(img, coords):
    """utils.py:101-103 (tf_grid_sample, :39-99): img [n,H,W,1], coords [n,a,b,2] (x,y pixels)
    -> [n,a,b,1].  Truncation toward zero, index clamping, weights from the clamped x1/y1."""
    n, H, W, c = img.shape
    assert c == 1, "the reference only samples the single-channel correlation volume"
    a, b = coords.shape[1], coords.shape[2]
    img, coords = img.contiguous().float(), coords.contiguous().float()
    out = torch.empty(n, a, b, 1, dtype=torch.float32, device=img.device)
    with torch.cuda.device(img.device):
        capi.check(capi.lib.rb_bilinear_sample(capi.ptr(img), capi.ptr(coords), capi.ptr(out), n, H, W, a * b,
                                               capi.stream()))
    return out


def upflow8(flow):
    """utils.py:105-111: bilinear x8 (align_corners=True) WITHOUT multiplying by 8 (reference quirk)."""
    b, h, w, _ = flow.shape
    coords1 = (flow + coords_grid(b, h, w, flow.device)).contiguous()
    out = torch.empty(b, 8 * h, 8 * w, 2, dtype=torch.float32, device=flow.device)
    with torch.cuda.device(out.device):
        capi.check(capi.lib.rb_upflow8(capi.ptr(coords1), capi.ptr(out), b, h, w, 1.0, capi.stream()))
    return out


def fb_consistency(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5, flow_scale=1.0):
    """Extension (no counterpart in the reference): forward-backward consistency of two [B,H,W,2] flows on the GPU
    (rb_flow_fb_check; Sundaram et al. 2010, UnFlow's alpha1 / alpha2 as defaults).  flow_scale multiplies both flows
    first: 8.0 for raft-small, whose upflow8 output is in 1/8-resolution units.  Returns (occ_fw, occ_bw), [B,H,W]
    uint8: 0 consistent, 1 inconsistent (occluded), 2 the flow leaves the frame."""
    assert flow_fw.shape == flow_bw.shape and flow_fw.dim() == 4 and flow_fw.shape[-1] == 2, (flow_fw.shape, flow_bw.shape)
    assert flow_fw.device == flow_bw.device, (flow_fw.device, flow_bw.device)
    b, H, W, _ = flow_fw.shape
    fw, bw = flow_fw.contiguous().float(), flow_bw.contiguous().float()
    occ_fw = torch.empty(b, H, W, dtype=torch.uint8, device=fw.device)
    occ_bw = torch.empty_like(occ_fw)
    with torch.cuda.device(fw.device):
        capi.check(capi.lib.rb_flow_fb_check(capi.ptr(fw), capi.ptr(bw), capi.ptr(occ_fw), capi.ptr(occ_bw), b, H, W,
                                             float(flow_scale), float(alpha1), float(alpha2), capi.stream()))
    return occ_fw, occ_bw
