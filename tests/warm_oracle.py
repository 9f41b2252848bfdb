"""Upstream RAFT's forward_interpolate (core/utils/utils.py) as a numpy brute force in fp64, for the tests of
rb_flow_forward_interpolate: every grid point takes the (dx, dy) of the valid source with the smallest squared distance
fl64(fl64((qx - x1)^2) + fl64((qy - y1)^2)); equal distances go to the lower source index y*w + x; a sample without a
valid source gives zeros."""
import numpy as np

_CHUNK = 1 << 23  # distances per block of grid points


def _sample(f, unique):
    h, w, _ = f.shape
    y0, x0 = np.mgrid[0:h, 0:w]
    with np.errstate(invalid="ignore"):
        x1 = (x0 + f[..., 0].astype(np.float64)).ravel()
        y1 = (y0 + f[..., 1].astype(np.float64)).ravel()
        valid = (x1 > 0) & (x1 < w) & (y1 > 0) & (y1 < h)
    src = np.flatnonzero(valid)  # ascending: argmin's first minimum is the lowest index
    out = np.zeros((h * w, 2), np.float32)
    uniq = np.ones(h * w, bool)
    if src.size:
        sx, sy = x1[src], y1[src]
        qx, qy = x0.ravel().astype(np.float64), y0.ravel().astype(np.float64)
        step = max(1, _CHUNK // src.size)
        for a in range(0, h * w, step):
            tx = qx[a:a + step, None] - sx[None]
            ty = qy[a:a + step, None] - sy[None]
            d = tx * tx
            d += ty * ty
            k = np.argmin(d, axis=1)
            out[a:a + step] = f.reshape(-1, 2)[src[k]]
            if unique:
                best = d[np.arange(len(k)), k]
                uniq[a:a + step] = (d == best[:, None]).sum(axis=1) == 1
    out = out.reshape(h, w, 2)
    return (out, uniq.reshape(h, w)) if unique else out


def forward_interpolate(flow, return_unique=False):
    """flow: [h,w,2] or [B,h,w,2] float32 (numpy or CPU torch) -> the same shape float32; with return_unique also the
    [.., h, w] bool mask of grid points whose nearest valid source is unique (scipy's griddata must agree there)."""
    f = np.asarray(flow, dtype=np.float32)
    if f.ndim == 3:
        return _sample(f, return_unique)
    res = [_sample(x, return_unique) for x in f]
    if return_unique:
        return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])
    return np.stack(res)
