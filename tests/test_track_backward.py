"""F17 without a GPU: the numpy restatement of rb_track_points_backward (tests/track_backward_oracle.py) against the
forward tracker on the reversed clip, chunked reverse sweeps, exact trajectories and fp64; the C entry's argument
errors; and the CLI's --track-backward checks."""
import ctypes

import numpy as np
import pytest

import track_backward_oracle as B
import track_oracle as O


def _case(rng, T, H, W, N, nan=3):
    fw = (rng.uniform(-0.3, 0.3, (T, H, W, 2)) * np.array([W, H])).astype(np.float32)
    bw = (-fw + rng.normal(0, 0.6, fw.shape)).astype(np.float32)
    for f in (fw, bw):
        for _ in range(nan):
            f[rng.integers(T), rng.integers(H), rng.integers(W), rng.integers(2)] = np.nan
    qframe = rng.integers(0, T + 1, N)
    qpos = np.stack([rng.uniform(0, W - 1, N), rng.uniform(0, H - 1, N)], -1).astype(np.float32)
    centre = rng.random(N) < 0.3
    qpos[centre] = np.floor(qpos[centre])
    return fw, bw, qframe, qpos


@pytest.mark.parametrize("scale", [1.0, 8.0])
def test_reversed_clip_identity(scale):
    """Backward from frame q equals the forward tracker on the reversed clip from frame T - q, rows reversed, on the
    rows up to q -- bit for bit."""
    rng = np.random.default_rng(31 + int(scale))
    T, H, W, N = 7, 29, 41, 600
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    fw, bw = fw / np.float32(scale), bw / np.float32(scale)
    tb, sb, (pos, st) = B.track_backward(fw, bw, qframe, qpos, flow_scale=scale)
    rfw, rbw = B.reversed_clip(fw, bw)
    tf, sf, _ = O.track(rfw, rbw, T - qframe, qpos, flow_scale=scale)
    tf, sf = tf[::-1], sf[::-1]  # row j of the reversed run is frame T - j
    rows = np.arange(T + 1)[:, None] <= qframe
    assert O.same_bits(tb[rows], tf[rows]) and np.array_equal(sb[rows], sf[rows])
    assert (sb[~rows] == O.BEFORE).all() and np.isnan(tb[~rows]).all()  # rows after the query: not stored
    assert O.same_bits(pos, tb[0]) and np.array_equal(st, sb[0])
    assert all((sb[rows] == k).any() for k in (0, 1, 2)) and not (sb[rows] == O.BEFORE).any()


def test_completes_the_forward_tracks_in_place():
    rng = np.random.default_rng(4)
    T, H, W, N = 6, 23, 31, 400
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    tf, sf, _ = O.track(fw, bw, qframe, qpos)
    tb, sb, _ = B.track_backward(fw, bw, qframe, qpos, tf, sf)
    alone, alone_s, _ = B.track_backward(fw, bw, qframe, qpos)
    after = np.arange(T + 1)[:, None] >= qframe
    assert O.same_bits(tb[after], tf[after]) and np.array_equal(sb[after], sf[after])
    assert O.same_bits(tb[~after], alone[~after]) and np.array_equal(sb[~after], alone_s[~after])
    assert not (sb == O.BEFORE).any()


def test_rows_after_the_query_are_left_as_they_were():
    rng = np.random.default_rng(6)
    T, H, W, N = 5, 17, 19, 200
    fw, bw, qframe, qpos = _case(rng, T, H, W, N)
    sentinel = np.float32(-12345.5)
    tr, ss = np.full((T + 1, N, 2), sentinel, np.float32), np.full((T + 1, N), 77, np.uint8)
    tb, sb, _ = B.track_backward(fw, bw, qframe, qpos, tr, ss)
    after = np.arange(T + 1)[:, None] > qframe
    assert (tb[after] == sentinel).all() and (sb[after] == 77).all()
    assert (sb[~after] != 77).all()


@pytest.mark.parametrize("bounds", [(0, 4, 10), (0, 1, 2, 3, 10), (0, 9, 10), (0, 5, 6, 10), (0, 10)])
def test_chunked_reverse_sweep_equals_one_pass(bounds):
    rng = np.random.default_rng(21)
    T, H, W, N = 10, 19, 27, 400
    fw, bw, qframe, qpos = _case(rng, T, H, W, N, nan=0)
    fw, bw = fw / np.float32(3), bw / np.float32(3)
    whole_t, whole_s, _ = B.track_backward(fw, bw, qframe, qpos)
    t, s = B.track_backward_passes(fw, bw, qframe, qpos, bounds)
    assert O.same_bits(t, whole_t) and np.array_equal(s, whole_s)
    assert all((whole_s == k).any() for k in range(4))


def test_carried_state_is_untouched_for_earlier_queries():
    rng = np.random.default_rng(2)
    fw, bw, _, _ = _case(rng, 3, 9, 11, 1, nan=0)
    pos = np.float32([[1.5, 2.0], [3.0, 4.0]])
    st = np.uint8([1, 0])
    _, _, (p, s) = B.track_backward(fw, bw, [2, 7], np.float32([[1, 1], [2, 2]]), first_frame=3, state=(pos, st))
    assert O.same_bits(p[0], pos[0]) and s[0] == 1  # frame 2 < first_frame: nothing stored, state kept
    assert s[1] != O.BEFORE  # frame 7 > 3 + 3: the carried (3, 4) stepped back


def test_dyadic_translation_is_exact_until_it_leaves():
    T, H, W = 40, 32, 48
    fw = np.broadcast_to(np.float32([1.5, -0.75]), (T, H, W, 2)).copy()
    qframe = np.array([T, 30, T])
    qpos = np.float32([[46.0, 2.0], [30.5, 10.25], [1.0, 30.0]])
    tracks, status, _ = B.track_backward(fw, -fw, qframe, qpos)
    for i, (f0, (x0, y0)) in enumerate(zip(qframe, qpos)):
        k = f0 - np.arange(T + 1)  # steps back from the query frame
        x, y = x0 - 1.5 * k, y0 + 0.75 * k
        gone = (x < 0) | (y > H - 1)
        leave = int(np.flatnonzero(gone & (k > 0))[-1])  # the last frame (counting down) still inside is leave + 1
        live = (k >= 0) & (np.arange(T + 1) > leave)
        assert np.array_equal(tracks[live, i, 0], x[live]) and np.array_equal(tracks[live, i, 1], y[live]), i
        assert (status[live, i] == O.CONSISTENT).all() and (status[:leave + 1, i] == O.LEFT).all(), i
        assert np.isnan(tracks[:leave + 1, i]).all() and (status[k < 0, i] == O.BEFORE).all(), i
    assert status[:, 2].tolist()[::-1].index(O.LEFT) == 1  # x = 1 - 1.5 k leaves at the first step back


def test_fp32_chain_stays_near_fp64():
    from test_track import _smooth
    rng = np.random.default_rng(5)
    T, H, W, N = 8, 48, 64, 2000
    fw = _smooth(rng, T, H, W, 3.0)
    bw = -fw + _smooth(rng, T, H, W, 0.8)
    qframe = rng.integers(T - 2, T + 1, N)
    qpos = np.stack([rng.uniform(0, W - 1, N), rng.uniform(0, H - 1, N)], -1).astype(np.float32)
    t32, s32, _ = B.track_backward(fw, bw, qframe, qpos)
    t64, s64, _ = B.track_backward(fw, bw, qframe, qpos, dt=np.float64)
    both = (s32 <= 1) & (s64 <= 1) & (np.arange(T + 1)[:, None] <= qframe)
    err = np.abs(t32.astype(np.float64) - t64)[both].max()
    assert err < 2e-4, err
    assert (s32 == s64).mean() > 0.995 and (s32 == O.LEFT).any() and (s32 == O.OCCLUDED).any()


def test_track_points_backward_argument_checks():
    """rb_track_points_backward refuses bad arguments with RB_ERR_* and a message before any CUDA call (host pointers
    below: a launch would fail, not return these codes)."""
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG = -1, -2
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = ctypes.c_float

    def call(fw=p, bw=p, T=3, H=8, W=9, n=3, s=1.0, a1=0.01, a2=0.5, qf=p, qp=p, N=4, first=0, pos=p, st=p, tr=p, ss=p):
        return lib.rb_track_points_backward(fw, bw, T, H, W, n, f(s), f(a1), f(a2), qf, qp, N, first, pos, st, tr, ss,
                                            None)

    def refused(rc, code, *words):
        assert rc == code, (rc, code)
        msg = lib.rb_last_error()
        assert b"rb_track_points_backward" in msg and all(w in msg for w in words), msg

    for name in ("fw", "bw", "qf", "qp", "pos", "st", "tr", "ss"):
        refused(call(**{name: None}), BAD_ARG, b"null")
    for kw in ({"T": 0}, {"H": 0}, {"W": -1}, {"N": 0}, {"N": -5}):
        refused(call(**kw), BAD_SHAPE, b"bad shape")
    for n in (0, -1, 4):
        refused(call(n=n), BAD_SHAPE, b"n_steps")
    for s in (0.0, -1.0, float("inf"), float("nan")):
        refused(call(s=s), BAD_ARG, b"flow_scale")
    for a1, a2 in ((-0.01, 0.5), (0.01, -0.5), (float("nan"), 0.5), (0.01, float("inf"))):
        refused(call(a1=a1, a2=a2), BAD_ARG, b"alpha")


def test_cli_track_backward_needs_points(capsys):
    import infer_raft
    for argv in (["--path", "frames", "--out", "o", "--track-backward"],
                 ["--im1", "a.png", "--im2", "b.png", "--track-backward"]):
        with pytest.raises(SystemExit) as e:
            infer_raft.main(argv)
        assert e.value.code == 2
        assert "--track-backward goes with --track-grid or --track" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:  # the other --track checks still apply
        infer_raft.main(["--path", "frames", "--out", "o", "--track-grid", "4", "--track-backward", "--warm-start"])
    assert e.value.code == 2 and "--warm-start" in capsys.readouterr().err
