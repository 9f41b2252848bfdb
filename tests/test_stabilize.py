"""Video stabilization on the CPU: the host path of raft_b200.stabilize (camera path, smoothing, zoom, transforms), the
recovery of known similarities by the fp64 fit oracle (tests/stabilize_oracle.py), and the CLI's argument checks."""
import math

import numpy as np
import pytest

import stabilize_oracle as O
from raft_b200 import stabilize as S

HW = (270, 480)


def _corners(hw):
    H, W = hw
    return np.array([[0, 0, 1], [W - 1, 0, 1], [0, H - 1, 1], [W - 1, H - 1, 1]], np.float64)


def _corner_dev(A, hw):
    """The largest distance of a [F,2,3] transform's images of the frame corners from the corners themselves."""
    c = _corners(hw)
    return float(np.abs(np.einsum("fij,cj->fci", A, c) - c[None, :, :2]).max())


def test_still_camera_gives_identity():
    A, zooms, capped = S.camera_transforms(np.tile([1.0, 0, 0, 0], (9, 1)), HW, 3.0)
    assert A.shape == (10, 2, 3) and zooms == [1.0] and capped == []
    assert np.array_equal(A, np.tile(np.array([[1.0, 0, 0], [0, 1, 0]]), (10, 1, 1)))


def test_constant_pan_is_left_as_it_is():
    A, zooms, _ = S.camera_transforms(np.tile([1.0, 0, 2.5, -1.25], (30, 1)), HW, 4.0)
    assert zooms == [1.0]
    assert _corner_dev(A, HW) < 1e-9


def test_odd_reflection_at_the_shot_ends():
    p = np.stack([np.arange(7.0) ** 2, 3.0 - 2 * np.arange(7.0)], 1)
    got = S.smooth(p, 1.0)
    R = 3
    w = np.exp(-0.5 * np.arange(-R, R + 1) ** 2)
    w /= w.sum()
    ext = lambda col, i: (2 * col[0] - col[-i] if i < 0 else 2 * col[-1] - col[2 * 6 - i] if i > 6 else col[i])  # noqa
    want = np.array([[sum(w[k + R] * ext(p[:, c], t + k) for k in range(-R, R + 1)) for c in range(2)]
                     for t in range(7)])
    assert np.allclose(got, want, rtol=0, atol=1e-12)
    assert np.allclose(got[:, 1], p[:, 1], rtol=0, atol=1e-12)  # a linear run stays
    # the radius is capped at L - 1
    q = np.array([[0.0], [1.0], [5.0]])
    w2 = np.exp(-0.5 * (np.arange(-2, 3) / 5.0) ** 2)
    w2 /= w2.sum()
    ext2 = np.array([2 * 0 - 5, 2 * 0 - 1, 0, 1, 5, 2 * 5 - 1, 2 * 5 - 0], np.float64)
    assert np.allclose(S.smooth(q, 5.0)[:, 0], [np.dot(w2, ext2[i:i + 5]) for i in range(3)], atol=1e-12)


def test_theta_is_unwrapped_across_pi():
    step = 0.3
    M = np.tile([math.cos(step), math.sin(step), 0.0, 0.0], (20, 1))
    p = S.path_params(S.camera_path(M))
    assert np.allclose(p[:, 1], step * np.arange(21), atol=1e-12)  # runs past pi without a jump
    assert np.allclose(p[:, 0], 0, atol=1e-12)


def test_each_shot_restarts_the_path():
    rng = np.random.default_rng(1)
    M = np.column_stack([1 + rng.normal(0, 1e-3, 19), rng.normal(0, 1e-3, 19), rng.normal(0, 2, 19),
                         rng.normal(0, 2, 19)])
    cuts = [6, 12]
    A, zooms, _ = S.camera_transforms(M, HW, 3.0, cuts=cuts, max_zoom=2.0)
    assert len(zooms) == 3
    for (s, e), z in zip(S.shots(20, cuts), zooms):
        a, zs, _ = S.camera_transforms(M[s:e], HW, 3.0, max_zoom=2.0)
        assert np.array_equal(a, A[s:e + 1]) and zs == [z]
    C = S.camera_path(M, cuts)
    assert all(np.array_equal(C[s], np.eye(3)) for s in (0, 7, 13))


def _brute_zoom(B, hw, max_zoom):
    H, W = hw
    hx, hy = 0.5 * (W - 1), 0.5 * (H - 1)
    c = np.array([[-hx, -hy], [hx, -hy], [-hx, hy], [hx, hy]])
    for z in np.arange(1.0, max_zoom + 1e-9, 1e-5):
        p = np.einsum("nij,cj->nci", B[:, :2, :2], c / z) + B[:, None, :2, 2]
        if (np.abs(p[..., 0]) <= hx + 1e-9).all() and (np.abs(p[..., 1]) <= hy + 1e-9).all():
            return z
    return None


@pytest.mark.parametrize("seed", range(6))
def test_zoom_closed_form_against_brute_force(seed):
    rng = np.random.default_rng(seed)
    n = 5
    B = S.motion_matrix(np.column_stack([1 + rng.normal(0, 0.01, n), rng.normal(0, 0.01, n), rng.normal(0, 8, n),
                                         rng.normal(0, 5, n)]))
    z, capped = S.shot_zoom(B, HW, 1.5)
    want = _brute_zoom(B, HW, 1.5)
    if want is None:
        assert capped and z == 1.5
    else:
        assert not capped and abs(z - want) <= 1.1e-5 and z <= want + 1e-12


def test_zoom_cap():
    B = S.motion_matrix(np.array([[1.0, 0.0, 60.0, 0.0]]))
    z, capped = S.shot_zoom(B, HW, 1.1)  # needs W / (W - 120) = 1.33
    assert capped and z == 1.1
    z, capped = S.shot_zoom(B, HW, 2.0)
    assert not capped and abs(z - 239.5 / (239.5 - 60)) < 1e-10  # within the slack
    shake = np.array([[1.0, 0, 100.0, 0], [1.0, 0, -100.0, 0]] * 2)  # a zigzag the smoothing flattens
    _, zooms, capped = S.camera_transforms(shake, HW, 2.0, max_zoom=1.2)
    assert capped == [0] and zooms == [1.2]


def test_transforms_are_uncentred_maps():
    A = S.centred_to_pixels(S.motion_matrix(np.array([[1.0, 0.0, 3.0, -2.0]]))[None][0], HW)
    assert np.allclose(A, [[[1, 0, 3], [0, 1, -2]]])
    R = S.centred_to_pixels(S.motion_matrix(np.array([[0.0, 1.0, 0.0, 0.0]])), HW)  # 90 degrees about the centre
    c = np.array([0.5 * (HW[1] - 1), 0.5 * (HW[0] - 1), 1.0])
    assert np.allclose(R[0] @ c, c[:2])


@pytest.mark.parametrize("bad", [0, -1, float("nan"), float("inf"), "x", None])
def test_sigma_refusals(bad):
    with pytest.raises(ValueError, match="sigma"):
        S.camera_transforms(np.tile([1.0, 0, 0, 0], (3, 1)), HW, bad)


def test_max_zoom_refusals():
    for bad in (0.99, float("nan"), "z"):
        with pytest.raises(ValueError, match="max_zoom"):
            S.camera_transforms(np.tile([1.0, 0, 0, 0], (3, 1)), HW, 2.0, max_zoom=bad)


@pytest.mark.parametrize("cuts", [[9], [-1], [2, 12], [1.5], ["a"]])
def test_cut_refusals(cuts):
    with pytest.raises(ValueError, match="cuts"):
        S.camera_transforms(np.tile([1.0, 0, 0, 0], (9, 1)), HW, 2.0, cuts=cuts)


def test_motion_shape_refusals():
    for bad in (np.zeros((0, 4)), np.zeros((3, 3)), np.zeros(4)):
        with pytest.raises(ValueError, match="motions"):
            S.camera_transforms(bad, HW, 2.0)


# ---- recovery of known similarities by the fit oracle --------------------------------------------------------------
M_TRUE = (1.003 * math.cos(0.004), 1.003 * math.sin(0.004), 3.7, -2.2)


@pytest.mark.parametrize("net,src,scale", [((108, 256), (270, 640), 1.0), ((96, 160), (96, 160), 1.0),
                                           ((37, 53), (101, 149), 8.0)])
def test_recovers_exact_similarity(net, src, scale):
    flow = O.similarity_flow(M_TRUE, *net, *src, flow_scale=scale)[None]
    params, weight, flags, _, _ = O.global_motion(flow, np.zeros((1,) + net, np.uint8), src, flow_scale=scale)
    assert flags[0] == 0 and weight[0] == 1.0
    assert O.corner_error(params[0], M_TRUE, src) < 1e-6


@pytest.mark.parametrize("seed", range(4))
def test_recovers_similarity_despite_outliers_occlusion_and_noise(seed):
    """30% of the pixels in one block moving 10 px differently, 10% occluded, 0.1 network px of noise: within 0.05 px
    at the frame corners."""
    Hn, Wn, Hs, Ws = 108, 256, 270, 640
    rng = np.random.default_rng(seed)
    flow = O.similarity_flow(M_TRUE, Hn, Wn, Hs, Ws)[None]
    flow += rng.normal(0, 0.1, flow.shape).astype(np.float32)
    h, w = int(Hn * 0.6), Wn // 2
    y0, x0 = rng.integers(0, Hn - h + 1), rng.integers(0, Wn - w + 1)
    ang = rng.uniform(0, 2 * np.pi)
    flow[0, y0:y0 + h, x0:x0 + w, 0] += np.float32(10 * math.cos(ang) * Wn / Ws)
    flow[0, y0:y0 + h, x0:x0 + w, 1] += np.float32(10 * math.sin(ang) * Hn / Hs)
    occ = (rng.random((1, Hn, Wn)) < 0.1).astype(np.uint8)
    flow[0, 0, 0] = np.nan  # a NaN flow counts as occluded
    params, weight, flags, _, _ = O.global_motion(flow, occ, (Hs, Ws))
    assert flags[0] == 0 and 0.85 < weight[0] < 0.95
    assert O.corner_error(params[0], M_TRUE, (Hs, Ws)) < 0.05


def test_too_few_consistent_pixels_is_unreliable():
    flow = O.similarity_flow(M_TRUE, 40, 60, 40, 60)[None]
    occ = np.ones((1, 40, 60), np.uint8)
    occ[0, :5, :5] = 0  # 25 of 2400 pixels: below the floor
    params, weight, flags, _, _ = O.global_motion(flow, occ, (40, 60))
    assert flags[0] == 1 and np.array_equal(params[0], [1, 0, 0, 0]) and weight[0] == 25 / 2400


# ---- the CLI -------------------------------------------------------------------------------------------------------
def _usage_error(argv, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


def test_cli_parses_stabilize():
    import infer_raft
    a = infer_raft.parser().parse_args(["--path", "d", "--out", "o", "--stabilize", "10", "--stabilize-zoom", "1.1",
                                        "--scene-cut", "0.4", "--flow-size", "216", "384"])
    assert (a.stabilize, a.stabilize_zoom, a.scene_cut, a.flow_size) == (10.0, 1.1, 0.4, [216, 384])
    assert infer_raft.parser().parse_args(["--path", "d"]).stabilize is None


@pytest.mark.parametrize("argv,words", [
    (["--stabilize", "10"], "needs --path"),
    (["--path", "d", "--stabilize", "10", "-m", "val"], "needs --path"),
    (["--path", "d", "--stabilize", "0"], "SIGMA"),
    (["--path", "d", "--stabilize", "nan"], "SIGMA"),
    (["--path", "d", "--stabilize", "4", "--stabilize-zoom", "0.9"], "zoom >= 1"),
    (["--path", "d", "--stabilize-zoom", "1.2"], "goes with --stabilize"),
    (["--path", "d", "--stabilize", "4", "--scene-cut", "2"], "threshold"),
    (["--path", "d", "--stabilize", "4", "--keep-size", "--flow-size", "200", "300"], "--keep-size"),
    (["--path", "d", "--stabilize", "4", "--batch", "0"], "--batch"),
] + [(["--path", "d", "--stabilize", "4"] + extra, "cannot be combined with " + extra[0])
     for extra in (["--interpolate", "0.5"], ["--fps", "60", "--input-fps", "24"], ["--warm-start"], ["--track", "p"],
                   ["--track-grid", "8"], ["--propagate", "k.png"], ["--bidirectional"], ["--native-frames"],
                   ["--native-flow"], ["--flo", "f"], ["--npy", "n"])])
def test_cli_refusals(argv, words, capsys):
    assert words in _usage_error(argv, capsys)
