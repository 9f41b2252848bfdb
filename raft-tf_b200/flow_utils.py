"""Flow colour coding used by the CLI (the reference's infer_raft.py:25,43 calls
flow_utils.flow_to_color(flow, convert_to_bgr=True)).  Independent numpy implementation of the
Middlebury colour wheel (Baker et al., ICCV 2007): same normalisation by the maximum radius
(+1e-5) and floor(255*col) quantisation as the reference's flow_utils.py:95-121.  reverse_flow_avg_skip_static is the
reference's flow reversal (flow_utils.py:166-274) and resize_flow (flow_utils.py:277-284) its flow resize, both computed on
the GPU; they import torch only when called."""
import numpy as np

_SEGMENTS = (("RY", 15), ("YG", 6), ("GC", 4), ("CB", 11), ("BM", 13), ("MR", 6))


def make_colorwheel():
    n = sum(k for _, k in _SEGMENTS)
    wheel = np.zeros((n, 3))
    # each segment ramps one channel up or down while another stays saturated
    plan = [(0, 1, +1), (1, 0, -1), (1, 2, +1), (2, 1, -1), (2, 0, +1), (0, 2, -1)]
    pos = 0
    for (_, k), (sat, ramp, sign) in zip(_SEGMENTS, plan):
        t = np.floor(255 * np.arange(k) / k)
        wheel[pos:pos + k, sat] = 255
        wheel[pos:pos + k, ramp] = t if sign > 0 else 255 - t
        pos += k
    return wheel


def flow_to_color(flow_uv, clip_flow=None, convert_to_bgr=False):
    """[H,W,2] flow -> [H,W,3] uint8 colour image.  Pinned bit for bit against the reference function run in-process
    (oracle/make_flowcolor_golden.py -> tests/golden/flow_to_color.npz), which fixes the floating-point TYPE of every
    step for float32 flows (flow_utils.py:58-121): direction / radius in the flow's dtype, interpolation weight and
    colours in float64, floor(255*col) quantisation."""
    flow_uv = np.asarray(flow_uv)
    assert flow_uv.ndim == 3 and flow_uv.shape[2] == 2
    if clip_flow is not None:
        flow_uv = np.clip(flow_uv, 0, clip_flow)
    u, v = flow_uv[..., 0], flow_uv[..., 1]
    ft = u.dtype if u.dtype.kind == "f" else np.dtype(np.float64)
    rad = np.sqrt(np.square(u) + np.square(v))
    den = (rad.max() + np.asarray(1e-5, dtype=ft)).astype(ft)  # rad_max + epsilon in the flow's precision
    u, v = (u / den).astype(ft), (v / den).astype(ft)
    wheel = make_colorwheel()
    n = wheel.shape[0]
    rad = np.sqrt(np.square(u) + np.square(v))
    fk = ((np.arctan2(-v, -u) / np.asarray(np.pi, dtype=ft)).astype(ft) + 1) / 2 * (n - 1) + 1
    k0 = np.minimum(np.floor(fk).astype(np.int32), n - 2)
    k1 = k0 + 1
    k1[k1 == n] = 1
    f = fk.astype(np.float64) - k0  # float64 from here on, like (float32 array - int32 array) in numpy
    inside = rad <= 1
    img = np.zeros(u.shape + (3,), np.uint8)
    for ch in range(3):
        col = (1 - f) * (wheel[k0, ch] / 255.0) + f * (wheel[k1, ch] / 255.0)
        col = np.where(inside, 1 - rad * (1 - col), col * 0.75)
        img[..., 2 - ch if convert_to_bgr else ch] = np.floor(255 * col)
    return img


def reverse_flow_avg_skip_static(flow01_origin, bg, im0, time_step=1.0):
    """The reference's flow_utils.py:166-274 on cuda:0, same name, arguments and 5-tuple: the flow 0 -> 1 projected to
    time `time_step`, giving the flow from there back to frame 0 (rb_flow_reverse, bit for bit with the reference under
    numpy >= 2).  flow01_origin: [H,W,2] float32; bg, im0: [H,W,C] uint8 or float32 (None for both: nothing static).
    Returns numpy (flow10 float32 [H,W,2], empty uint8, uint8(count > 1), static_mask int64 [H,W,1], empty eroded by
    5x5 uint8).  Differences: a NaN flow is skipped (the reference raises), and nothing is printed."""
    import torch
    from networks.utils import reverse_flow

    flow = np.asarray(flow01_origin)
    if flow.dtype != np.float32:
        raise TypeError(f"reverse_flow_avg_skip_static: flow must be float32, got {flow.dtype}")
    if flow.ndim != 3 or flow.shape[2] != 2:
        raise ValueError(f"reverse_flow_avg_skip_static: flow must be [H,W,2], got {flow.shape}")
    imgs = []
    for im in (bg, im0):
        if im is None:
            imgs.append(None)
            continue
        im = np.asarray(im)
        if im.dtype not in (np.uint8, np.float32):
            raise TypeError(f"reverse_flow_avg_skip_static: images must be uint8 or float32, got {im.dtype}")
        if im.ndim != 3 or im.shape[:2] != flow.shape[:2]:
            raise ValueError(f"reverse_flow_avg_skip_static: images must be [H,W,C] with the flow's H, W, got {im.shape}")
        imgs.append(torch.from_numpy(np.ascontiguousarray(im))[None].to("cuda:0"))
    f = torch.from_numpy(np.ascontiguousarray(flow))[None].to("cuda:0")
    out = reverse_flow(f, float(time_step), *imgs)
    flow10, empty, multi, static, eroded = (t[0].cpu().numpy() for t in out)
    return flow10, empty, multi, static.astype(np.int64)[..., None], eroded


def resize_flow(flow, dW, dH):
    """The reference's flow_utils.py:277-284 on cuda:0, same name, arguments and return value: [H,W,2] float32 numpy
    flow -> [dH,dW,2] float32, each channel resized like cv2.resize and u, v scaled by dW / W and dH / H
    (rb_flow_resize, bit for bit with the reference under numpy >= 2)."""
    import torch
    from networks.utils import resize_flow as _resize_flow

    flow = np.asarray(flow)
    if flow.dtype != np.float32:
        raise TypeError(f"resize_flow: flow must be float32, got {flow.dtype}")
    if flow.ndim != 3 or flow.shape[2] != 2:
        raise ValueError(f"resize_flow: flow must be [H,W,2], got {flow.shape}")
    f = torch.from_numpy(np.ascontiguousarray(flow))[None].to("cuda:0")
    return _resize_flow(f, (int(dH), int(dW)))[0].cpu().numpy()


def write_flo(path, flow_uv):
    """Middlebury .flo file (magic 202021.25, int32 width, int32 height, float32 [H,W,2] row-major u,v) -- the
    format of the reference's unused writer (flow_utils.py:302-318)."""
    f = np.ascontiguousarray(flow_uv, dtype=np.float32)
    assert f.ndim == 3 and f.shape[2] == 2
    with open(path, "wb") as fh:
        np.array([202021.25], np.float32).tofile(fh)
        np.array([f.shape[1], f.shape[0]], np.int32).tofile(fh)
        f.tofile(fh)


def read_kitti_flow(path):
    """KITTI's 16-bit flow PNG -> (flow [H,W,2] float32, valid [H,W] uint8), like upstream RAFT's readFlowKITTI and the
    mask of validate_kitti: in OpenCV's BGR order channel 2 is u, channel 1 is v and channel 0 the valid flag; flow =
    (x - 2**15) / 64 (exact in float32), valid = flag >= 0.5."""
    import cv2
    raw = cv2.imread(str(path), cv2.IMREAD_ANYDEPTH | cv2.IMREAD_COLOR)
    if raw is None:
        raise FileNotFoundError(f"cannot read KITTI flow {path}")
    if raw.dtype != np.uint16 or raw.ndim != 3 or raw.shape[2] != 3:
        raise ValueError(f"{path}: a KITTI flow is a 3-channel 16-bit PNG, got {raw.dtype} {raw.shape}")
    flow = (raw[..., 2:0:-1].astype(np.float32) - np.float32(2 ** 15)) / np.float32(64.0)
    return np.ascontiguousarray(flow), (raw[..., 0] >= 0.5).astype(np.uint8)


def write_kitti_flow(path, flow):
    """[H,W,2] flow -> KITTI's 16-bit flow PNG, the inverse of read_kitti_flow and the bytes of upstream RAFT's
    writeFlowKITTI: u, v as uint16(64 * flow + 2**15) in float32 (truncated), the valid flag 1 everywhere, channels in
    OpenCV's BGR order (flag, v, u)."""
    import cv2
    uv = np.asarray(flow, dtype=np.float32)
    if uv.ndim != 3 or uv.shape[2] != 2:
        raise ValueError(f"write_kitti_flow: flow must be [H,W,2], got {uv.shape}")
    uv = np.float32(64.0) * uv + np.float32(2 ** 15)
    valid = np.ones([uv.shape[0], uv.shape[1], 1])
    raw = np.concatenate([uv, valid], axis=-1).astype(np.uint16)
    if not cv2.imwrite(str(path), raw[..., ::-1]):
        raise OSError(f"cannot write {path}")


def read_flo(path):
    with open(path, "rb") as fh:
        magic = np.fromfile(fh, np.float32, 1)[0]
        assert abs(magic - 202021.25) < 1e-3, "not a .flo file"
        w, h = np.fromfile(fh, np.int32, 2)
        return np.fromfile(fh, np.float32, 2 * int(w) * int(h)).reshape(int(h), int(w), 2)
