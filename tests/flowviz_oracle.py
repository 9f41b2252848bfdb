"""Oracle of rb_flow_to_color (csrc/flowviz.cu): flow_utils.flow_to_color step by step, with the one difference the kernel
makes on purpose -- arctan2 computed in fp64 and rounded once to fp32, because numpy's float32 arctan2 is not correctly
rounded and depends on the machine's SIMD kernels.

Neither the kernel's fp64 atan2 (CUDA: within 2 ulp) nor numpy's is correctly rounded, so where the fp64 value lies within
a few double ulps of an fp32 rounding midpoint the two may round to neighbouring floats.  flow_to_color returns those
pixels as `ambiguous`; there a neighbouring direction moves the colour by at most 1 LSB."""
import numpy as np

WHEEL_ULPS = 4  # fp64 ulps around an fp32 midpoint that count as ambiguous (CUDA's 2 + numpy's 1, plus one spare)


def _wheel():
    import flow_utils
    return flow_utils.make_colorwheel()


def atan2_f32(y, x):
    """fl32(atan2((double)y, (double)x)) and whether the fp64 value lies within WHEEL_ULPS double ulps of an fp32
    rounding midpoint."""
    d = np.arctan2(np.asarray(y, np.float64), np.asarray(x, np.float64))
    r = d.astype(np.float32)
    lo = np.nextafter(r, np.float32(-np.inf)).astype(np.float64)
    hi = np.nextafter(r, np.float32(np.inf)).astype(np.float64)
    rd = r.astype(np.float64)
    near = np.minimum(np.abs(d - (rd + lo) / 2), np.abs(d - (rd + hi) / 2))
    return r, near <= WHEEL_ULPS * np.spacing(np.abs(d))


def flow_to_color(flow_uv, clip_flow=None, convert_to_bgr=False):
    """[H,W,2] float32 flow -> ([H,W,3] uint8 image, [H,W] bool ambiguous), the numerics of the kernel."""
    flow = np.asarray(flow_uv)
    assert flow.ndim == 3 and flow.shape[2] == 2 and flow.dtype == np.float32, (flow.shape, flow.dtype)
    if clip_flow is not None:
        flow = np.clip(flow, 0, np.float32(clip_flow))
    u, v = flow[..., 0], flow[..., 1]
    rad = np.sqrt(np.square(u) + np.square(v))
    den = (rad.max() + np.float32(1e-5)).astype(np.float32)
    u, v = u / den, v / den
    wheel = _wheel()
    n = wheel.shape[0]
    rad = np.sqrt(np.square(u) + np.square(v))
    at, ambiguous = atan2_f32(-v, -u)
    fk = ((at / np.float32(np.pi)) + np.float32(1)) / np.float32(2) * np.float32(n - 1) + np.float32(1)
    k0 = np.minimum(np.floor(fk).astype(np.int32), n - 2)
    k1 = k0 + 1
    k1[k1 == n] = 1
    f = fk.astype(np.float64) - k0
    inside = rad <= 1
    img = np.zeros(u.shape + (3,), np.uint8)
    for ch in range(3):
        col = (1 - f) * (wheel[k0, ch] / 255.0) + f * (wheel[k1, ch] / 255.0)
        col = np.where(inside, 1 - rad * (1 - col), col * 0.75)
        img[..., 2 - ch if convert_to_bgr else ch] = np.floor(255 * col)
    return img, ambiguous


def flow_to_color_batch(flows, clip_flow=None, convert_to_bgr=False):
    """[B,H,W,2] -> ([B,H,W,3] uint8, [B,H,W] bool): each sample on its own."""
    out = [flow_to_color(f, clip_flow, convert_to_bgr) for f in np.asarray(flows)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def assert_matches(got, flows, clip_flow=None, convert_to_bgr=False):
    """got [B,H,W,3] uint8 equals the oracle on every non-ambiguous pixel and is within 1 LSB on the ambiguous ones."""
    want, amb = flow_to_color_batch(flows, clip_flow, convert_to_bgr)
    got = np.asarray(got)
    assert got.shape == want.shape and got.dtype == np.uint8, (got.shape, got.dtype)
    diff = np.abs(got.astype(np.int16) - want.astype(np.int16)).max(-1)
    bad = (diff > 0) & ~amb
    assert not bad.any(), f"{int(bad.sum())} non-ambiguous pixels differ, first at {np.argwhere(bad)[0].tolist()}"
    assert diff.max(initial=0) <= 1, int(diff.max())
    return int(amb.sum())
