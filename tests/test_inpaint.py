"""Object removal without a GPU: the numpy restatement of rb_masked_fill against an fp64 sparse Laplace solve and its
invariants, the restatement of the temporal fill, the host tables and checks, the CLI's argument errors and the C
entries' RB_ERR_* returns before any CUDA call."""
import ctypes

import numpy as np
import pytest

import inpaint_oracle as O
from raft_b200 import inpaint as I

HOLES = ("square", "ring", "border", "line", "blobs")


def hole_of(kind, H=200, W=256, seed=0):
    """The hole shapes the fill is held to: a 128x128 square, a ring around a known island, holes touching the border and
    a corner, a one-pixel line and about 30 % random blobs."""
    h = np.zeros((H, W), bool)
    yy, xx = np.mgrid[0:H, 0:W]
    if kind == "square":
        h[H // 2 - 64:H // 2 + 64, W // 2 - 64:W // 2 + 64] = True
    elif kind == "ring":
        r = np.hypot(yy - H / 2, xx - W / 2)
        h = (r > 15) & (r < 60)
    elif kind == "border":
        h[:40, :50] = True
        h[H - 30:, 100:170] = True
        h[50:90, W - 25:] = True
    elif kind == "line":
        h[H // 2, 10:W - 10] = True
    else:
        from scipy.ndimage import binary_dilation
        h = binary_dilation(np.random.default_rng(seed).random((H, W)) < 0.012, iterations=3)
    return h


def field_of(kind, C, H=200, W=256, seed=0):
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    if kind == "smooth":
        chans = [np.sin(xx / 23) + np.cos(yy / 17), 0.3 * xx / W - yy / H, np.cos((xx + yy) / 31)]
        return np.stack(chans[:C], -1).astype(np.float32)
    return (np.random.default_rng(seed).random((H, W, C)) * 255).astype(np.float32)


@pytest.mark.parametrize("C", [2, 3])
@pytest.mark.parametrize("field", ["smooth", "noise"])
@pytest.mark.parametrize("kind", HOLES)
def test_fill_is_the_laplace_solution(kind, field, C):
    v, h = field_of(field, C), hole_of(kind)
    got, flag = O.masked_fill(v, h)
    ref = O.laplace_fp64(v, h)
    known = v[~h]
    span = known.max(0) - known.min(0)
    assert flag == 0
    assert np.array_equal(got[~h], v[~h])  # the known pixels keep their bits
    assert (np.abs(got - ref).max(axis=(0, 1)) <= 2e-3 * span).all(), np.abs(got - ref).max(axis=(0, 1)) / span
    assert (got[h] >= known.min(0)).all() and (got[h] <= known.max(0)).all()


def test_constant_field_stays_bit_exact():
    for c in (np.float32(0.1), np.float32(-3.7e5), np.float32(255.0)):
        v = np.full((64, 80, 3), c, np.float32)
        for kind in HOLES:
            got, _ = O.masked_fill(v, hole_of(kind, 64, 80))
            assert np.array_equal(got, v), kind


def test_affine_field_over_a_convex_hole():
    yy, xx = np.mgrid[0:120, 0:150].astype(np.float64)
    v = np.stack([0.7 * xx - 0.2 * yy + 3, -0.1 * xx + 0.4 * yy], -1).astype(np.float32)
    h = np.zeros((120, 150), bool)
    h[20:100, 30:130] = True
    got, _ = O.masked_fill(v, h)
    span = v[~h].max(0) - v[~h].min(0)
    assert (np.abs(got - v).max(axis=(0, 1)) <= 2e-3 * span).all()


def test_fully_masked_field_is_zero_and_flagged():
    got, flag = O.masked_fill(np.ones((9, 13, 2), np.float32), np.ones((9, 13), np.uint8))
    assert flag == 1 and not got.any()


def test_fill_levels_halve_with_ceil():
    assert I.fill_levels(5, 3) == [(5, 3), (3, 2), (2, 1), (1, 1)]
    assert I.fill_levels(1, 1) == [(1, 1)]


def test_masks_rule_on_the_grid():
    rng = np.random.default_rng(1)
    masks = (rng.random((2, 23, 31)) < 0.05).astype(np.uint8) * 3
    hole, net = O.inpaint_masks(masks, I.selection_table(), 1, 9, 40)  # smaller and larger than the frames
    assert hole.shape == (2, 23, 31) and net.shape == (2, 9, 40)
    for f in range(2):  # the rule restated per network pixel
        for i in range(9):
            for j in range(40):
                ys = [y for y in range(23) if ((2 * y + 1) * 9) // 46 == i] or [((2 * i + 1) * 23) // 18]
                xs = [x for x in range(31) if ((2 * x + 1) * 40) // 62 == j] or [((2 * j + 1) * 31) // 80]
                assert net[f, i, j] == hole[f][np.ix_(ys, xs)].max()
    only = O.inpaint_masks(masks, I.selection_table([5]), 0, 23, 31)[0]
    assert not only.any()  # the label 3 is not selected


def _clip(rng, F=6, H=20, W=28, hole_frac=0.1):
    frames = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    hole = (rng.random((F, H, W)) < hole_frac).astype(np.uint8)
    fw = rng.normal(0, 1.5, (F - 1, H, W, 2)).astype(np.float32)
    bw = (-fw + rng.normal(0, 0.05, fw.shape)).astype(np.float32)
    return frames, hole, fw, bw


def test_temporal_fill_copies_non_hole_pixels_and_mirrors_on_the_reversed_clip():
    rng = np.random.default_rng(2)
    frames, hole, fw, bw = _clip(rng)
    F = len(frames)
    rows = I.inpaint_rows(F, 3)
    colour, status = O.inpaint_propagate(frames, hole, fw, bw, rows)
    keep = hole == 0
    assert np.array_equal(colour[keep], frames[keep].astype(np.float32)) and (status[keep] == 0).all()
    assert set(np.unique(status[hole == 1])) <= {1, 2, 3}
    # on the reversed clip the backward side is the forward side: a table with one side each way
    fwd = np.array([[t, 3 if t + 3 < F else F - 1 - t, 0] for t in range(F)], np.int32)
    bwd = np.array([[F - 1 - t, 0, fwd[t, 1]] for t in range(F)], np.int32)
    cf, sf = O.inpaint_propagate(frames, hole, fw, bw, fwd)
    cb, sb = O.inpaint_propagate(frames[::-1].copy(), hole[::-1].copy(), bw[::-1].copy(), fw[::-1].copy(), bwd)
    assert np.array_equal(cf, cb) and np.array_equal(sf, sb)


def test_temporal_fill_stops_at_the_window_and_at_cuts():
    rng = np.random.default_rng(3)
    F, H, W = 7, 16, 20
    frames = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    zero = np.zeros((F - 1, H, W, 2), np.float32)
    hole = np.zeros((F, H, W), np.uint8)
    hole[:, 4:9, 5:12] = 1
    hole[[2, 4], ...] = 0  # only frames 2 and 4 see behind the hole of frame 3
    hole[3, 4:9, 5:12] = 1
    for window, cuts, want in ((1, (), 1), (3, (), 1), (3, (3,), 2), (3, (2, 3), 3)):
        rows = I.inpaint_rows(F, window, cuts)[3:4]
        _, st = O.inpaint_propagate(frames, hole, zero, zero, rows)
        assert (st[0][hole[3] == 1] == want).all(), (window, cuts)
    hole[[2, 4], 4:9, 5:12] = 1  # now frames 1 and 5 are the nearest that see: window 1 reaches neither
    hole[[1, 5]] = 0
    _, st = O.inpaint_propagate(frames, hole, zero, zero, I.inpaint_rows(F, 1)[3:4])
    assert (st[0][hole[3] == 1] == 3).all()
    c, st = O.inpaint_propagate(frames, hole, zero, zero, I.inpaint_rows(F, 2)[3:4])
    assert (st[0][hole[3] == 1] == 1).all()
    ys, xs = np.nonzero(hole[3])
    assert np.array_equal(c[0, ys, xs], ((frames[1, ys, xs].astype(np.float32) + frames[5, ys, xs]) / 2))


def test_rows_table():
    rows = I.inpaint_rows(8, 3, [2, 5])
    assert rows.dtype == np.int32
    assert rows.tolist() == [[0, 2, 0], [1, 1, 1], [2, 0, 2], [3, 2, 0], [4, 1, 1], [5, 0, 2], [6, 1, 0], [7, 0, 1]]
    assert I.inpaint_rows(4, 10).tolist() == [[0, 3, 0], [1, 2, 1], [2, 1, 2], [3, 0, 3]]


@pytest.mark.parametrize("bad", [0, -1, 1.5, True, "3", None])
def test_window_refusals(bad):
    with pytest.raises(ValueError):
        I.check_window(bad)


@pytest.mark.parametrize("bad", [-1, 33, 1.0, True, None])
def test_dilate_refusals(bad):
    with pytest.raises(ValueError):
        I.check_dilate(bad)


@pytest.mark.parametrize("bad", [[], [256], [-1], [1.5], "x", 3])
def test_label_refusals(bad):
    with pytest.raises(ValueError):
        I.selection_table(bad)


def test_selection_table():
    assert I.selection_table().tolist() == [0] + [1] * 255
    t = I.selection_table([1, 7])
    assert np.flatnonzero(t).tolist() == [1, 7]


def test_rows_refuse_bad_cuts():
    with pytest.raises(ValueError):
        I.inpaint_rows(5, 2, [4])


def test_mask_listing_and_reading(tmp_path):
    from raft_b200.video import list_masks, read_labels, write_labels
    for i in range(3):
        write_labels(tmp_path / f"m_{i}.png", np.full((4, 5), i, np.uint8), palette=np.zeros((8, 3), np.uint8))
    paths = list_masks(tmp_path, 3)
    assert [read_labels(p)[0][0, 0] for p in paths] == [0, 1, 2]
    with pytest.raises(ValueError):
        list_masks(tmp_path, 4)
    with pytest.raises(FileNotFoundError):
        list_masks(tmp_path / "none", 3)


def _usage_error(argv, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


@pytest.mark.parametrize("argv,words", [
    (["--inpaint", "m/"], "needs --path"),
    (["--path", "f/", "--inpaint", "m/", "--stabilize", "5"], "cannot be combined with --stabilize"),
    (["--path", "f/", "--inpaint", "m/", "--warm-start"], "cannot be combined with --warm-start"),
    (["--path", "f/", "--inpaint", "m/", "--propagate", "k.png"], "cannot be combined with --propagate"),
    (["--path", "f/", "--inpaint", "m/", "--inpaint-window", "0"], "--inpaint-window"),
    (["--path", "f/", "--inpaint", "m/", "--inpaint-dilate", "33"], "--inpaint-dilate"),
    (["--path", "f/", "--inpaint", "m/", "--inpaint-labels", "300"], "--inpaint-labels"),
    (["--path", "f/", "--inpaint", "m/", "--scene-cut", "2"], "--scene-cut"),
    (["--path", "f/", "--inpaint", "m/", "--keep-size", "--flow-size", "64", "64"], "--flow-size"),
    (["--path", "f/", "--inpaint-window", "3"], "--inpaint-window goes with --inpaint"),
    (["--path", "f/", "--inpaint-dilate", "3"], "--inpaint-dilate goes with --inpaint"),
    (["--path", "f/", "--inpaint-labels", "1"], "--inpaint-labels goes with --inpaint"),
])
def test_cli_refusals(argv, words, capsys):
    assert words in _usage_error(argv, capsys)


def test_c_entries_refuse_bad_arguments_before_any_cuda_call():
    from raft_b200 import capi
    lib, fake = capi.lib, 4096  # a non-null pointer the checks never dereference
    n = ctypes.c_size_t(0)
    assert lib.rb_masked_fill_workspace_bytes(1, 8, 8, 2, ctypes.byref(n)) == 0 and n.value > 0
    assert lib.rb_masked_fill_workspace_bytes(1, 8, 8, 4, ctypes.byref(n)) == capi.lib.rb_masked_fill_workspace_bytes(
        1, 8, 8, 1, ctypes.byref(n)) < 0
    assert lib.rb_masked_fill_workspace_bytes(0, 8, 8, 2, ctypes.byref(n)) == -1
    assert lib.rb_masked_fill(None, fake, 1, 8, 8, 2, None, fake, 1 << 20, None) == -2
    assert lib.rb_masked_fill(fake, fake, 1, 0, 8, 2, None, fake, 1 << 20, None) == -1
    assert lib.rb_masked_fill(fake, fake, 1, 8, 8, 1, None, fake, 1 << 20, None) == -2
    assert lib.rb_masked_fill(fake, fake, 70000, 8, 8, 2, None, fake, 1 << 40, None) == -1
    assert lib.rb_masked_fill(fake, fake, 1, 8, 8, 2, None, fake, 16, None) == -5
    assert lib.rb_inpaint_masks(fake, fake, 1, 8, 8, 33, 4, 4, fake + 1, fake, None) == -2
    assert lib.rb_inpaint_masks(fake, fake, 1, 8, 8, 2, 4, 4, fake, fake, None) == -2  # hole aliases masks
    assert lib.rb_inpaint_masks(fake, fake, 0, 8, 8, 2, 4, 4, fake + 1, fake, None) == -1
    assert lib.rb_inpaint_masks(None, fake, 1, 8, 8, 2, 4, 4, fake + 1, fake, None) == -2
    args = [fake, fake, 3, 8, 8, fake, fake, 4, 4, 1.0, 0.01, 0.5, fake, 1, fake, fake, None]
    for i, v, code in ((5, None, -2), (2, 0, -1), (13, 0, -1), (9, 0.0, -2), (9, float("nan"), -2), (10, -1.0, -2),
                       (11, float("inf"), -2)):
        a = list(args)
        a[i] = v
        assert lib.rb_inpaint_propagate(*a) == code, (i, v)
