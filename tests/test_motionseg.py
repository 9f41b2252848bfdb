"""Motion segmentation without a GPU: the numpy restatement of rb_homography_motion, rb_motion_evidence and
rb_motion_segment on clips with a known camera and exact flows (a perspective camera rotating about its vertical axis,
with and without a moving object), a still clip, unreliable and cut pairs, the host checks and the C entries' RB_ERR_*
returns before any CUDA call."""
import ctypes

import numpy as np
import pytest

import fb_oracle as FO
import motionseg_oracle as MO
from raft_b200 import motionseg as M

HW = (96, 160)
FOCAL = 150.0  # pixels, near the frames' width
DEG = 4.0  # the camera's turn per frame about its vertical axis


def _rotation(deg, hw=HW, f=FOCAL):
    """K R_y K^-1 in the frames' own pixels: where a still scene's pixel of frame k lands in frame k + 1."""
    Hs, Ws = hw
    K = np.array([[f, 0, 0.5 * (Ws - 1)], [0, f, 0.5 * (Hs - 1)], [0, 0, 1.0]])
    a = np.deg2rad(deg)
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    return K @ R @ np.linalg.inv(K)


def _apply(Hm, x, y):
    X = Hm[0, 0] * x + Hm[0, 1] * y + Hm[0, 2]
    Y = Hm[1, 0] * x + Hm[1, 1] * y + Hm[1, 2]
    z = Hm[2, 0] * x + Hm[2, 1] * y + Hm[2, 2]
    return X / z, Y / z


SQUARE = (60.0, 30.0, 100.0, 66.0)  # the object in frame 0: x0, y0, x1, y1 in pixels
SHIFT = 3.0  # the object's own motion per frame in pixels, on top of the camera's


def _to_frame0(k, x, y, Hm, obj):
    """Where a frame-k pixel of the object (if it is one) sat in frame 0."""
    Hi = np.linalg.inv(Hm)
    for _ in range(k):
        x, y = _apply(Hi, x - (SHIFT if obj else 0.0), y)
    return x, y


def _object_distance(k, x, y, Hm):
    """Signed distance (in frame-0 pixels, > 0 inside) of frame-k pixels from the object's boundary."""
    x0, y0 = _to_frame0(k, x, y, Hm, True)
    a, b, c, d = SQUARE
    return np.minimum(np.minimum(x0 - a, c - x0), np.minimum(y0 - b, d - y0))


def _clip(F, deg=DEG, obj=False):
    """Exact flows of F frames seen by the rotating camera (an object moving SHIFT px per frame when obj) on the frames'
    own grid, and the forward-backward masks of the occlusion check."""
    Hm = _rotation(deg)
    Hi = np.linalg.inv(Hm)
    Hs, Ws = HW
    y, x = (a.astype(np.float64) for a in np.mgrid[0:Hs, 0:Ws])
    fw, bw = np.zeros((F - 1, Hs, Ws, 2), np.float32), np.zeros((F - 1, Hs, Ws, 2), np.float32)
    for k in range(F - 1):
        qx, qy = _apply(Hm, x, y)
        rx, ry = _apply(Hi, x, y)
        if obj:
            inside = _object_distance(k, x, y, Hm) >= 0
            qx = np.where(inside, qx + SHIFT, qx)
            inside1 = _object_distance(k + 1, x, y, Hm) >= 0
            ox, oy = _apply(Hi, x - SHIFT, y)
            rx, ry = np.where(inside1, ox, rx), np.where(inside1, oy, ry)
        fw[k] = np.stack([qx - x, qy - y], -1)
        bw[k] = np.stack([rx - x, ry - y], -1)
    ofw, obw = FO.fb_check(fw, bw)
    return fw, bw, ofw, obw, Hm


def _normalised(Hm, hw=HW):
    """A homography in the frames' own pixels in F34's normalised centred coordinates."""
    Hs, Ws = hw
    L = 0.5 * max(hw)
    N = np.array([[1 / L, 0, -0.5 * (Ws - 1) / L], [0, 1 / L, -0.5 * (Hs - 1) / L], [0, 0, 1]])
    P = N @ Hm @ np.linalg.inv(N)
    return P / P[2, 2]


def test_perspective_camera_recovered_and_still():
    F = 4
    fw, bw, ofw, obw, Hm = _clip(F)
    rows = M.segment_rows(F, M.DEFAULT_WINDOW)
    mask, status, H, flags, _ = MO.segment_clip(fw, bw, ofw, obw, HW, rows)
    assert (flags == 0).all()
    for k in range(F - 1):
        np.testing.assert_allclose(H[k], _normalised(Hm), rtol=0, atol=1e-9 * np.abs(_normalised(Hm)).max())
        np.testing.assert_allclose(H[F - 1 + k], _normalised(np.linalg.inv(Hm)), rtol=0, atol=1e-9)
    np.testing.assert_allclose(M.to_pixels(H[:F - 1], HW)[0], Hm / Hm[2, 2], rtol=1e-7, atol=1e-7)
    # no pixel moves on its own; only the strips the camera turns into view or out of it lack evidence (status 1)
    assert not mask.any()
    assert 0 < status.mean() < 0.1
    # the similarity alone leaves a residual above tau near the frame edges: it is what the homography is for
    sim, _, sflags, _, _ = MO.SO.global_motion(fw[:1], ofw[:1], HW)
    e, ok = MO.field_e(fw[0], ofw[0], MO.similarity_h(sim[0], 0.5 * max(HW)), HW, 1.0, M.TAU)
    assert sflags[0] == 0 and (e[ok] >= 0.5).any()


@pytest.mark.parametrize("window", [0, M.DEFAULT_WINDOW])
def test_camera_plus_object(window):
    F = 5
    fw, bw, ofw, obw, Hm = _clip(F, obj=True)
    mask, status, _, flags, _ = MO.segment_clip(fw, bw, ofw, obw, HW, M.segment_rows(F, window))
    assert (flags == 0).all()
    Hs, Ws = HW
    y, x = (a.astype(np.float64) for a in np.mgrid[0:Hs, 0:Ws])
    for t in range(F):
        d = _object_distance(t, x, y, Hm)
        inner, outer = d >= 2, d <= -2
        assert inner.sum() > 500
        assert (mask[t][inner] == 1).all(), (t, int((mask[t][inner] == 0).sum()))
        assert (mask[t][outer] == 0).all(), (t, int((mask[t][outer] == 1).sum()))


def test_still_clip():
    F = 3
    z = np.zeros((F - 1, 24, 40, 2), np.float32)
    o = np.zeros((F - 1, 24, 40), np.uint8)
    mask, status, H, flags, ev = MO.segment_clip(z, z, o, o, (48, 80), M.segment_rows(F, 2))
    assert (flags == 0).all() and not mask.any() and not status.any()
    assert (ev[..., 0] < 1e-20).all() and (ev[0, ..., 1] == 1).all() and (ev[1, ..., 1] == 2).all()
    np.testing.assert_allclose(H, np.broadcast_to(np.eye(3), H.shape), atol=1e-12)


def test_unreliable_and_cut_pairs_unused():
    F = 5
    fw, bw, ofw, obw, _ = _clip(F, obj=True)
    T = F - 1
    H, flags = MO.fit(np.concatenate([fw, bw]), np.concatenate([ofw, obw]), HW, 1.0)
    ev = MO.evidence(fw, bw, ofw, obw, H, flags, HW)
    # an unreliable field contributes nothing: frame 1 keeps only its backward field when pair 1's forward is flagged 2
    f2 = flags.copy()
    f2[1] = 2
    ev2 = MO.evidence(fw, bw, ofw, obw, H, f2, HW)
    e, ok = MO.field_e(bw[0], obw[0], H[T], HW, 1.0, M.TAU)
    np.testing.assert_array_equal(ev2[1, ..., 0], np.where(ok, e, 0).astype(np.float32))
    np.testing.assert_array_equal(ev2[[0, 3, 4]], ev[[0, 3, 4]])
    # a cut pair: every frame equals the segmentation of its shot alone, bit for bit
    c = 2
    rows = M.segment_rows(F, M.DEFAULT_WINDOW, [c])
    mask, status, _, _, ev = MO.segment_clip(fw, bw, ofw, obw, HW, rows, cuts=[c])
    for lo, hi in ((0, c), (c + 1, F - 1)):
        n = hi - lo + 1
        m1, s1, _, _, e1 = MO.segment_clip(fw[lo:hi], bw[lo:hi], ofw[lo:hi], obw[lo:hi], HW,
                                           M.segment_rows(n, M.DEFAULT_WINDOW))
        np.testing.assert_array_equal(mask[lo:hi + 1], m1)
        np.testing.assert_array_equal(status[lo:hi + 1], s1)
        np.testing.assert_array_equal(ev[lo:hi + 1], e1)


def test_segment_rows():
    np.testing.assert_array_equal(M.segment_rows(4, 0), [[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0]])
    np.testing.assert_array_equal(M.segment_rows(5, 2, [1]), [[0, 1, 0], [1, 0, 1], [2, 2, 0], [3, 1, 1], [4, 0, 2]])


@pytest.mark.parametrize("bad", [-1, 17, 1.5, True, "3", None])
def test_window_refused(bad):
    with pytest.raises(ValueError, match="window"):
        M.check_window(bad)


@pytest.mark.parametrize("bad", [0, -1.0, float("nan"), float("inf"), 1e39, "x", None, True])
def test_tau_refused(bad):
    with pytest.raises(ValueError, match="tau"):
        M.check_tau(bad)


def test_cuts_refused():
    with pytest.raises(ValueError, match="cuts"):
        M.segment_rows(4, 1, [3])


def test_c_entries_refuse_before_cuda():
    from raft_b200 import capi
    lib = capi.lib
    p = ctypes.c_void_p(16)  # never dereferenced: every call below fails its argument checks first
    n = ctypes.c_size_t(0)
    assert lib.rb_homography_motion_workspace_bytes(0, 4, 4, ctypes.byref(n)) == -1
    assert lib.rb_homography_motion_workspace_bytes(1, 4, 4, None) == -2
    args = [p, p, 1, 4, 4, 8, 8, 1.0, p, p, 8, 0.5, p, p, None, p, 1 << 20, None]
    for i, v, rc in ((0, None, -2), (3, 0, -1), (7, 0.0, -2), (7, float("nan"), -2), (10, 0, -2), (10, 33, -2),
                     (11, 0.0, -2), (16, 0, -5)):
        a = list(args)
        a[i] = v
        assert lib.rb_homography_motion(*a) == rc, (i, v)
    ev = [p, p, p, p, p, p, None, 1, 4, 4, 8, 8, 1.0, 1.0, p, None]
    for i, v, rc in ((14, None, -2), (7, 0, -1), (12, -1.0, -2), (13, 0.0, -2), (13, float("inf"), -2)):
        a = list(ev)
        a[i] = v
        assert lib.rb_motion_evidence(*a) == rc, (i, v)
    sg = [p, 2, 4, 4, p, p, 8, 8, 1.0, 0.01, 0.5, p, 2, p, p, None]
    for i, v, rc in ((0, None, -2), (4, None, -2), (12, 0, -1), (8, 0.0, -2), (9, -1.0, -2), (10, float("nan"), -2)):
        a = list(sg)
        a[i] = v
        assert lib.rb_motion_segment(*a) == rc, (i, v)


def _degenerate(Hn=12, Wn=53):
    """A field whose only usable pixels lie on one row: F22's similarity is reliable (1/12 of the pixels), but the points
    are collinear, so the homography's system is singular."""
    rng = np.random.default_rng(3)
    flow = (rng.normal(0, 0.2, (1, Hn, Wn, 2)) + np.array([1.0, -0.5])).astype(np.float32)
    occ = np.ones((1, Hn, Wn), np.uint8)
    occ[0, 5] = 0
    return flow, occ


def test_singular_field_keeps_the_similarity():
    flow, occ = _degenerate()
    hw = (24, 106)
    sim, _, sflags, _, _ = MO.SO.global_motion(flow, occ, hw)
    assert sflags[0] == 0
    H, flags, _, _, _ = MO.homography(flow, occ, hw, 1.0, sim, sflags)
    assert flags[0] == M.SINGULAR
    np.testing.assert_array_equal(H[0], MO.similarity_h(sim[0], 0.5 * max(hw)))


def _write_2016_list(root, names):
    import os
    os.makedirs(os.path.join(root, "ImageSets", "2016"), exist_ok=True)
    with open(os.path.join(root, "ImageSets", "2016", "val.txt"), "w") as f:
        f.write("\n".join(names) + "\n")


def test_davis2016_reader(tmp_path):
    import os
    from raft_b200 import synth
    from raft_b200.davis import davis_sequences
    root = str(tmp_path / "davis")
    names = synth.write_davis_tree(root, [("alpha", 3), ("beta", 4)], H=24, W=32)
    with pytest.raises(FileNotFoundError, match="2016"):
        davis_sequences(root, "val", year="2016")
    _write_2016_list(root, names[::-1])
    seqs = davis_sequences(root, "val", year="2016")
    assert [s.name for s in seqs] == names[::-1] and [len(s.frames) for s in seqs] == [4, 3]
    os.remove(seqs[0].annotations[-1])
    with pytest.raises(ValueError, match="beta has 4 frames and 3 annotations"):
        davis_sequences(root, "val", year="2016")
    _write_2016_list(root, ["alpha", "gamma"])
    with pytest.raises(FileNotFoundError, match="gamma"):
        davis_sequences(root, "val", year="2016")


@pytest.mark.parametrize("argv,msg", [
    (["--segment-motion"], "needs --path"),
    (["--segment-window", "2"], "go with --segment-motion"),
    (["--path", "x", "--segment-motion", "--segment-window", "17"], "--segment-window"),
    (["--path", "x", "--segment-motion", "--segment-tau", "0"], "--segment-tau"),
    (["--path", "x", "--segment-motion", "--denoise", "20"], "cannot be combined with --denoise"),
    (["--path", "x", "--segment-motion", "--scene-cut", "2"], "--scene-cut"),
    (["-m", "val", "--dataset", "sintel", "--segment-motion"], "needs --dataset davis"),
    (["-m", "val", "--dataset", "davis", "--segment-motion"], "needs --data"),
    (["-m", "val", "--dataset", "davis", "--data", "d", "--segment-motion", "--path", "x"], "--path"),
])
def test_cli_refusals(argv, msg, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(argv)
    assert e.value.code == 2 and msg in capsys.readouterr().err


def test_evaluate_motion_refuses_before_reading(tmp_path):
    from types import SimpleNamespace
    from raft_b200.davis import evaluate_motion
    for model, kw in ((SimpleNamespace(input_size=(64, 96)), {}), (SimpleNamespace(input_size=None), dict(window=17)),
                      (SimpleNamespace(input_size=None), dict(tau=-1))):
        with pytest.raises(ValueError):
            evaluate_motion(model, str(tmp_path / "none"), **kw)
