"""F16 without a GPU: the numpy restatement of rb_track_points (tests/track_oracle.py) against the forward-backward check
and exact trajectories, its fp32 rounding against fp64, the chunked state, RaftEngine.track's coordinate map, the query
file, the grid, the CLI's argument checks and rb_track_points' argument errors."""
import ctypes

import numpy as np
import pytest
from scipy.ndimage import gaussian_filter

import track_oracle as O
from fb_oracle import fb_check


def _flows(rng, T, H, W, amp=0.3, noise=0.6):
    fw = rng.uniform(-amp, amp, (T, H, W, 2)) * np.array([W, H])
    bw = -fw + rng.normal(0, noise, fw.shape)
    return fw.astype(np.float32), bw.astype(np.float32)


def _smooth(rng, T, H, W, amp):
    f = gaussian_filter(rng.normal(0, 1, (T, H, W, 2)), sigma=(0, 6, 6, 0), mode="wrap")
    return (amp * f / np.abs(f).max()).astype(np.float32)


@pytest.mark.parametrize("scale", [1.0, 8.0])
def test_first_step_at_pixel_centres_is_the_fb_check(scale):
    rng = np.random.default_rng(11)
    H, W = 23, 31
    fw, bw = _flows(rng, 1, H, W)
    fw, bw = fw / np.float32(scale), bw / np.float32(scale)
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    qpos = np.stack([xs.ravel(), ys.ravel()], -1).astype(np.float32)
    tracks, status, _ = O.track(fw, bw, np.zeros(H * W), qpos, flow_scale=scale)
    occ = fb_check(fw, bw, flow_scale=scale)[0][0].ravel()
    assert np.array_equal(status[0], np.zeros(H * W)) and O.same_bits(tracks[0], qpos)
    assert np.array_equal(status[1], occ)
    assert all((occ == k).any() for k in (0, 1, 2))
    inside = occ != 2
    want = qpos + np.float32(scale) * fw[0].reshape(-1, 2)
    assert O.same_bits(tracks[1][inside], want[inside])
    assert np.isnan(tracks[1][~inside]).all()


def test_dyadic_translation_is_exact_until_it_leaves():
    T, H, W = 40, 32, 48
    fw = np.broadcast_to(np.float32([1.5, -0.75]), (T, H, W, 2)).copy()
    qframe = np.array([0, 3, 0])
    qpos = np.float32([[2.0, 30.0], [0.5, 29.25], [45.0, 1.0]])
    tracks, status, _ = O.track(fw, -fw, qframe, qpos)
    for i, (f0, (x0, y0)) in enumerate(zip(qframe, qpos)):
        k = np.arange(T + 1) - f0
        x, y = x0 + 1.5 * k, y0 - 0.75 * k
        gone = (x > W - 1) | (y < 0)
        leave = int(np.flatnonzero(gone & (k > 0))[0])  # the frame where the track leaves
        live = (k >= 0) & (np.arange(T + 1) < leave)
        assert np.array_equal(tracks[live, i, 0], x[live]) and np.array_equal(tracks[live, i, 1], y[live]), i
        assert (status[live, i] == O.CONSISTENT).all() and (status[leave:, i] == O.LEFT).all(), i
        assert np.isnan(tracks[leave:, i]).all() and np.isnan(tracks[k < 0, i]).all(), i
    assert status[:, 2].tolist().index(O.LEFT) == 2  # x = 45 + 1.5 k passes W - 1 = 47 at frame 2


def test_fp32_chain_stays_near_fp64():
    rng = np.random.default_rng(5)
    T, H, W, N = 8, 48, 64, 2000
    fw = _smooth(rng, T, H, W, 3.0)
    bw = -fw + _smooth(rng, T, H, W, 0.8)
    qframe = rng.integers(0, 3, N)
    qpos = np.stack([rng.uniform(0, W - 1, N), rng.uniform(0, H - 1, N)], -1).astype(np.float32)
    t32, s32, _ = O.track(fw, bw, qframe, qpos)
    t64, s64, _ = O.track(fw, bw, qframe, qpos, dt=np.float64)
    both = (s32 <= 1) & (s64 <= 1) & (np.arange(T + 1)[:, None] >= qframe)
    err = np.abs(t32.astype(np.float64) - t64)[both].max()
    assert err < 2e-4, err  # 8 steps of |q| < 64 px: a few fp32 ulps (3.8e-6 at 32) per step
    assert (s32 == s64).mean() > 0.995 and (s32 == O.LEFT).any() and (s32 == O.OCCLUDED).any()


@pytest.mark.parametrize("bounds", [(0, 4, 10), (0, 1, 2, 3, 10), (0, 9, 10), (0, 5, 6, 10)])
def test_chained_passes_equal_one_pass(bounds):
    rng = np.random.default_rng(21)
    T, H, W, N = 10, 19, 27, 400
    fw, bw = _flows(rng, T, H, W, amp=0.1, noise=0.3)
    qframe = rng.integers(0, T + 1, N)
    qpos = np.stack([rng.uniform(0, W - 1, N), rng.uniform(0, H - 1, N)], -1).astype(np.float32)
    whole_t, whole_s, _ = O.track(fw, bw, qframe, qpos)
    t, s = O.track_passes(fw, bw, qframe, qpos, bounds)
    assert O.same_bits(t, whole_t) and np.array_equal(s, whole_s)
    assert all((whole_s == k).any() for k in range(4))


def test_before_the_query_frame():
    rng = np.random.default_rng(3)
    T, H, W = 6, 9, 13
    fw, bw = _flows(rng, T, H, W, amp=0.05)
    qframe = np.arange(T + 1)
    qpos = np.tile(np.float32([[6.0, 4.0]]), (T + 1, 1))
    tracks, status, _ = O.track(fw, bw, qframe, qpos)
    rows = np.arange(T + 1)[:, None]
    assert (status[rows < qframe] == O.BEFORE).all() and np.isnan(tracks[rows < qframe]).all()
    assert (status[rows == qframe] == O.CONSISTENT).all() and (tracks[rows == qframe] == [6.0, 4.0]).all()
    assert (status[rows > qframe] != O.BEFORE).all()


def test_a_start_outside_the_frame_leaves_at_once():
    fw = np.zeros((2, 5, 7, 2), np.float32)
    tracks, status, _ = O.track(fw, fw, [0, 0], np.float32([[7.5, 2.0], [np.nan, 1.0]]))
    assert status[:, 0].tolist() == [0, 2, 2] and np.isnan(tracks[1:]).all()


def test_coordinate_map_round_trips_and_matches_the_engine():
    import torch
    from raft_b200.engine import track_queries, tracks_to_frames
    rng = np.random.default_rng(8)
    for src, net in (((436, 1024), (432, 1024)), ((124, 150), (128, 160)), ((720, 1280), (544, 960)), ((60, 80),) * 2):
        (Hs, Ws), (Hn, Wn) = src, net
        xy = np.concatenate([np.stack([rng.uniform(0, Ws - 1, 500), rng.uniform(0, Hs - 1, 500)], -1),
                             [[0, 0], [Ws - 1, Hs - 1], [0.25, Hs - 1.25]]])
        q = np.concatenate([rng.integers(0, 5, (len(xy), 1)), xy], -1)
        qf, qp = track_queries(q, 5, src, net)
        assert qf.dtype == np.int32 and np.array_equal(qf, q[:, 0])
        want = O.to_network(xy, src, net) if src != net else xy.astype(np.float32)
        assert O.same_bits(qp, want)
        assert (qp >= 0).all() and (qp[:, 0] <= Wn - 1).all() and (qp[:, 1] <= Hn - 1).all()
        back = tracks_to_frames(torch.from_numpy(qp), src, net).numpy()
        assert O.same_bits(back, O.from_network(qp, src, net) if src != net else qp)
        half = 0.5 * max(Ws / Wn, Hs / Hn)  # the clamp moves an edge query by less than half a network pixel
        assert np.abs(back - xy).max() < max(1e-3, half if src != net else 0), np.abs(back - xy).max()
        interior = ((xy[:, 0] >= 0.5 * Ws / Wn) & (xy[:, 0] <= Ws - 1 - 0.5 * Ws / Wn)
                    & (xy[:, 1] >= 0.5 * Hs / Hn) & (xy[:, 1] <= Hs - 1 - 0.5 * Hs / Hn))
        assert np.abs(back - xy)[interior].max() < 1e-3
    nan = tracks_to_frames(torch.full((2, 2), float("nan")), (100, 100), (64, 64))
    assert torch.isnan(nan).all()


@pytest.mark.parametrize("bad,words", [([[0, 1.0]], "[N,3]"), (np.zeros((0, 3)), "[N,3]"), ([[5, 1.0, 1.0]], "frame"),
                                       ([[-1, 1.0, 1.0]], "frame"), ([[0.5, 1.0, 1.0]], "integer"),
                                       ([[0, np.nan, 1.0]], "finite"), ([[0, 1.0, np.inf]], "finite"),
                                       ([[0, 79.5, 1.0]], "[0, 79]"), ([[0, 1.0, -0.1]], "[0, 59]"), ("abc", "[N,3]")])
def test_bad_queries(bad, words):
    from raft_b200.engine import track_queries
    with pytest.raises(ValueError) as e:
        track_queries(bad, 5, (60, 80), (64, 96))
    assert words in str(e.value)


def test_query_file_and_grid(tmp_path):
    from raft_b200.video import read_queries, track_colors, track_grid
    p = tmp_path / "q.txt"
    p.write_text("# frame x y\n0 10 20.5\n\n3 1e1 0  # a comment\n")
    assert read_queries(str(p)).tolist() == [[0, 10, 20.5], [3, 10, 0]]
    for text, words in (("0 1\n", ":1:"), ("0 1 2\n1.5 1 2\n", ":2:"), ("# none\n", "no query points"),
                        ("0 a 2\n", ":1:")):
        p.write_text(text)
        with pytest.raises(ValueError, match=words):
            read_queries(str(p))
    g = track_grid(5, 7, 3, frame=2)
    assert g.tolist() == [[2, x, y] for y in (0, 3) for x in (0, 3, 6)]
    assert len(track_grid(436, 1024, 1)) == 436 * 1024 and len(track_grid(4, 4, 5)) == 1
    for step in (0, -1, 1.5):
        with pytest.raises(ValueError):
            track_grid(4, 4, step)
    c = track_colors(10)
    assert c.shape == (10, 3) and c.dtype == np.uint8 and np.array_equal(c, track_colors(10))


@pytest.mark.parametrize("extra,words", [
    (["--track", "q.txt", "--track-grid", "4"], "pass one"),
    (["--track-grid", "4", "--interpolate", "0.5"], "--interpolate"),
    (["--track", "q.txt", "--input-fps", "24", "--fps", "60"], "--fps"),
    (["--track", "q.txt", "--warm-start"], "--warm-start"),
    (["--track", "q.txt", "--scene-cut", "0.5"], "--scene-cut"),
    (["--track-grid", "0"], "step"),
    (["--track-vis", "v"], "--track-vis"),
    (["--track-frame", "2"], "--track-frame"),
])
def test_cli_track_argument_checks(extra, words, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(["--path", "frames", "--out", "o"] + extra)
    assert e.value.code == 2
    assert words in capsys.readouterr().err
    with pytest.raises(SystemExit):
        infer_raft.main(["--track", "q.txt"])  # no --path
    assert "--path" in capsys.readouterr().err


def test_cli_track_reads_the_query_file_before_the_model(tmp_path, capsys):
    import infer_raft
    bad = tmp_path / "q.txt"
    bad.write_text("0 1\n")
    with pytest.raises(SystemExit) as e:
        infer_raft.main(["--path", str(tmp_path), "--out", str(tmp_path / "o"), "--track", str(bad)])
    err = capsys.readouterr().err
    assert e.value.code == 2 and "--track" in err and "q.txt:1:" in err


def test_track_points_argument_checks():
    """rb_track_points refuses bad arguments with RB_ERR_* and a message before any CUDA call (host pointers below: a
    launch would fail, not return these codes)."""
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG = -1, -2
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = ctypes.c_float

    def call(fw=p, bw=p, T=3, H=8, W=9, n=3, s=1.0, a1=0.01, a2=0.5, qf=p, qp=p, N=4, first=0, pos=p, st=p, tr=p, ss=p):
        return lib.rb_track_points(fw, bw, T, H, W, n, f(s), f(a1), f(a2), qf, qp, N, first, pos, st, tr, ss, None)

    def refused(rc, code, *words):
        assert rc == code, (rc, code)
        msg = lib.rb_last_error()
        assert b"rb_track_points" in msg and all(w in msg for w in words), msg

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
