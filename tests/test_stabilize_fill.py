"""Full-frame stabilization (F26) on the CPU: the canvas margin, the CLI's argument checks, the C entries' refusals before
any CUDA call, and the geometry of the border fill through the numpy oracle (tests/stabfill_oracle.py) on a clip rendered
from an analytic texture along a known jittered camera path."""
import numpy as np
import pytest

import stabfill_oracle as SF
import stabilize_oracle as SO
from raft_b200 import stabilize as S
from raft_b200.inpaint import inpaint_rows

IDENT = np.array([[1.0, 0, 0], [0, 1, 0]])


def _shift(dx, dy, F=3):
    A = np.tile(IDENT, (F, 1, 1))
    A[1, 0, 2], A[1, 1, 2] = dx, dy
    return A


def test_margin_is_zero_without_a_border():
    assert S.fill_margin(np.tile(IDENT, (4, 1, 1)), (48, 80), (24, 40)) == (0, 0)
    zoom_in = np.array([[[0.9, 0, 3.9], [0, 0.9, 2.3]]])  # every source strictly inside
    assert S.fill_margin(zoom_in, (48, 80), (24, 40)) == (0, 0)


def test_margin_per_axis():
    # frames 48 x 80 on a 24 x 40 grid: the frame's own edge pixels sit 0.25 network pixels outside the grid
    # x: sources down to -6.5 frame pixels -> network -3.5, ceil 4, + 2 taps; y: only the frame's edge, ceil 0.25 + 2
    assert S.fill_margin(_shift(-6.5, 0), (48, 80), (24, 40)) == (3, 6)
    # y: sources up to 47 + 9 -> network (56.5) / 2 - 0.5 = 27.75, 27.75 - 23 = 4.75 -> 5 + 2
    assert S.fill_margin(_shift(0, 9), (48, 80), (24, 40)) == (7, 3)
    # frames at the grid's size: no half-pixel offset, so the axis without overshoot gets the taps alone
    assert S.fill_margin(_shift(3.0, 0), (24, 40), (24, 40)) == (2, 5)


def test_margin_cap_and_non_finite_entries():
    assert S.fill_margin(_shift(-500.0, 300.0), (48, 80), (24, 40)) == (12, 20)  # half the grid per side
    A = _shift(-6.5, 0)
    A[2, 0, 2] = np.nan
    assert S.fill_margin(A, (48, 80), (24, 40)) == (3, 6)
    with pytest.raises(ValueError, match="transforms"):
        S.fill_margin(np.zeros((3, 3, 3)), (48, 80), (24, 40))


def test_fill_motions_put_the_identity_at_cuts():
    m = np.tile([1.01, 0.02, 3.0, -1.0], (5, 1))
    got = S.fill_motions(m, [1, 3])
    assert np.array_equal(got[[1, 3]], [[1, 0, 0, 0]] * 2) and np.array_equal(got[[0, 2, 4]], m[[0, 2, 4]])
    assert m[1, 0] == 1.01  # a copy


def _usage_error(argv, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


@pytest.mark.parametrize("argv,words", [
    (["--path", "f/", "--stabilize-fill"], "--stabilize-fill goes with --stabilize"),
    (["--path", "f/", "--stabilize-window", "3"], "--stabilize-window goes with --stabilize"),
    (["--path", "f/", "--stabilize", "5", "--stabilize-window", "3"], "--stabilize-window goes with --stabilize-fill"),
    (["--path", "f/", "--stabilize", "5", "--stabilize-fill", "--stabilize-window", "0"], "--stabilize-window: N"),
    (["--path", "f/", "--inpaint", "m/", "--stabilize-fill"], "cannot be combined with --stabilize-fill"),
])
def test_cli_refusals(argv, words, capsys):
    assert words in _usage_error(argv, capsys)


def test_cli_parses_fill():
    import infer_raft
    a = infer_raft.parser().parse_args(["--path", "f/", "--stabilize", "5", "--stabilize-fill", "--stabilize-window",
                                        "4"])
    assert a.stabilize_fill and a.stabilize_window == 4 and a.stabilize_zoom is None
    a = infer_raft.parser().parse_args(["--path", "f/", "--stabilize", "5"])
    assert not a.stabilize_fill and a.stabilize_window is None


def test_c_entries_refuse_bad_arguments_before_any_cuda_call():
    from raft_b200 import capi
    lib, fake = capi.lib, 4096  # a non-null pointer the checks never dereference
    for fn in (lib.rb_flow_extend_residual, lib.rb_flow_extend_finish):
        args = [fake, fake, 2, 8, 10, 16, 20, 2, 3, 1.0, fake, fake, None]
        for i, v, code in ((0, None, -2), (1, None, -2), (10, None, -2), (11, None, -2), (2, 0, -1), (3, -1, -1),
                           (6, 0, -1), (7, -1, -1), (8, -2, -1), (9, 0.0, -2), (9, float("nan"), -2),
                           (9, float("inf"), -2), (2, 70000, -1)):
            a = list(args)
            a[i] = v
            assert fn(*a) == code, (fn.__name__, i, v)
            assert fn.__name__.encode() in lib.rb_last_error()
    args = [fake, 3, 8, 8, fake, fake, 4, 4, 1, 1, 1.0, 0.01, 0.5, fake, fake, 1, fake, fake, None]
    for i, v, code in ((0, None, -2), (4, None, -2), (13, None, -2), (14, None, -2), (16, None, -2), (1, 0, -1),
                       (15, 0, -1), (8, -1, -1), (9, -1, -1), (10, 0.0, -2), (10, float("nan"), -2), (11, -1.0, -2),
                       (12, float("inf"), -2)):
        a = list(args)
        a[i] = v
        assert lib.rb_frames_warp_affine_fill(*a) == code, (i, v)
        assert b"rb_frames_warp_affine_fill" in lib.rb_last_error()


def test_global_flow_is_similarity_flow_on_the_grid():
    M = (1.003, -0.004, 2.5, -1.25)
    for net, hw, s in (((24, 40), (48, 80), 1.0), ((11, 17), (37, 53), 8.0)):
        y, x = np.meshgrid(np.arange(net[0], dtype=np.float64), np.arange(net[1], dtype=np.float64), indexing="ij")
        u, v = SF.global_flow(M, x, y, hw, net, s)
        assert np.array_equal(np.stack([u, v], -1), SO.similarity_flow(M, *net, *hw, flow_scale=s))


def test_extension_of_a_similarity_flow_is_its_global_flow():
    """A flow that is exactly its pair's similarity has a zero residual, so its extension is the global flow on the whole
    canvas; margin 0 returns the flow."""
    M = (0.998, 0.006, -3.0, 1.5)
    hw, net, margin = (48, 80), (24, 40), (3, 5)
    flow = SO.similarity_flow(M, *net, *hw)
    ext = SF.extend(flow, M, hw, margin)
    y, x = np.meshgrid(np.arange(30, dtype=np.float64) - 3, np.arange(50, dtype=np.float64) - 5, indexing="ij")
    assert np.array_equal(ext, np.stack(SF.global_flow(M, x, y, hw, net), -1))
    assert np.array_equal(SF.extend(flow, M, hw, (0, 0)), flow)


def _known_clip(seed, **path):
    F, hw, net = 12, (48, 80), (24, 40)
    G, motions = SF.jittered_path(F, seed, **path)
    frames = SF.render(G, hw)
    fw = np.stack([SO.similarity_flow(m, *net, *hw) for m in motions])
    bw = np.stack([SO.similarity_flow(SF.inverse(m), *net, *hw) for m in motions])
    A, zooms, _ = S.camera_transforms(motions, hw, 3.0, max_zoom=1.0)
    assert zooms == [1.0]
    margin = S.fill_margin(A, hw, net)
    efw, ebw = SF.extend_flows(fw, bw, motions, hw, margin)
    colour, status = SF.warp_fill(frames, efw, ebw, net, margin, A, inpaint_rows(F, 10))
    return SF.finish(colour, status), status, SO.warp(frames, A), SF.true_view(G, A, hw)


def test_border_fill_recovers_the_true_full_frame_view():
    """A pan with rotation, zoom and translation jitter, and its analytic flows, at max_zoom = 1.  Thresholds set from a
    CPU run of the oracle before the first GPU run: the filled pixels' mean error was 0.31 grey levels (the in-frame
    pixels' 0.31 is the rounding of the rendered frames), the replicated border's 5.9, the largest filled error 1.23."""
    out, status, replicated, true = _known_clip(0)
    filled = (status == 1) | (status == 2)
    assert filled.sum() > 1500 and (status == 0).mean() > 0.9
    assert np.array_equal(out[status == 0], replicated[status == 0])  # in-frame pixels: rb_frames_warp_affine's bytes
    err = np.abs(out[..., 0] - true)[filled]
    rep = np.abs(replicated[..., 0] - true)[filled]
    assert err.mean() < 0.6 and err.max() < 3.0, (err.mean(), err.max())
    assert err.mean() < 0.15 * rep.mean(), (err.mean(), rep.mean())
    assert (out[..., 0] == out[..., 1]).all() and (out[..., 0] == out[..., 2]).all()


def test_no_spatial_fill_where_the_pan_keeps_every_border_pixel_in_reach():
    """A horizontal pan of 1.5 px per frame with horizontal jitter (sigma 3 px): every uncovered pixel lies in a frame
    at most window = 10 frames away, so nothing is left to the spatial fill."""
    out, status, replicated, true = _known_clip(0, jitter=(3.0, 0.0), rot=0, zoom=0)
    assert (status == 3).sum() == 0 and ((status == 1) | (status == 2)).sum() > 800
    filled = status > 0
    assert np.abs(out[..., 0] - true)[filled].mean() < 0.15 * np.abs(replicated[..., 0] - true)[filled].mean()
