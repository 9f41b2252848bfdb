"""F18 / F19 without a GPU: the fp32 restatement (tests/propagate_oracle.py) against hand cases and its own identities --
exact integer translations, the vote's tie rule, the status combination, chunked passes, the reversed clip and the
occlusion check -- plus the C entries' argument checks, the label PNG round trip and the CLI's argument errors."""
import ctypes

import numpy as np
import pytest

import fb_oracle
import propagate_oracle as P

F32 = np.float32


def _flows(rng, T, H, W, amp=2.5, noise=0.3):
    fw = rng.uniform(-amp, amp, (T, H, W, 2)).astype(F32)
    bw = (-fw + rng.normal(0, noise, fw.shape)).astype(F32)
    return fw, bw


def _translation(T, H, W, dx, dy):
    fw = np.broadcast_to(np.array([dx, dy], F32), (T, H, W, 2)).copy()
    return fw, -fw


def test_integer_translation_shifts_the_labels_exactly():
    T, H, W, dx, dy = 4, 30, 41, 2, -1
    fw, bw = _translation(T, H, W, dx, dy)
    acc, st = P.keyframe_rows(T + 1, H, W, 0)
    acc, st = P.accumulate(fw, bw, acc, st)
    key = np.random.default_rng(1).integers(0, 6, (H, W)).astype(np.uint8)
    labels, status = P.propagate(acc, st, key)
    for r in range(T + 1):
        ys, xs = np.mgrid[0:H, 0:W]
        sx, sy = xs - r * dx, ys - r * dy
        ok = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H)
        assert np.array_equal(labels[r][ok], key[sy[ok], sx[ok]])
        assert (status[r][ok] == 0).all() and (status[r][~ok] == 2).all()
        assert np.array_equal(acc[r][ok], np.broadcast_to(np.array([-r * dx, -r * dy], F32), acc[r][ok].shape))
    assert np.array_equal(labels[0], key)


def test_vote_ties_go_to_the_smaller_label_and_labels_never_blend():
    key = np.array([[7, 3], [7, 3]], np.uint8)
    assert P.vote(key, np.array([0.5], F32), np.array([0.0], F32))[0] == 3
    assert P.vote(key, np.array([0.49], F32), np.array([0.3], F32))[0] == 7
    assert P.vote(key, np.array([0.51], F32), np.array([0.7], F32))[0] == 3
    key = np.array([[1, 9], [9, 1]], np.uint8)  # two taps each: 0.25 + 0.25 against 0.25 + 0.25
    assert P.vote(key, np.array([0.5], F32), np.array([0.5], F32))[0] == 1
    key = np.array([[2, 4], [6, 4]], np.uint8)
    v = P.vote(key, np.random.default_rng(2).uniform(0, 1, 500).astype(F32),
               np.random.default_rng(3).uniform(0, 1, 500).astype(F32))
    assert set(np.unique(v)) <= {2, 4, 6}


def test_status_combination_keeps_the_largest():
    H, W = 9, 12
    pull = np.zeros((H, W, 2), F32)
    test = np.zeros((H, W, 2), F32)
    test[4, 6] = (5.0, 0.0)  # pixel (6, 4) fails the forward-backward test
    pull[:, 0] = (-1.0, 0.0)  # column 0 pulls from outside the frame
    prev = np.zeros((H, W, 2), F32)
    prev_st = np.zeros((H, W), np.uint8)
    prev_st[2, 3] = 1
    prev_st[2, 5] = 2
    acc, st = P.step(pull, test, prev, prev_st)
    assert st[4, 6] == 1 and st[2, 3] == 1 and st[2, 5] == 2 and (st[:, 0] == 2).all()
    assert st.sum() == 1 + 1 + 2 + 2 * H
    assert (acc[:, 0] == 0).all()  # clamped onto column 0: d = qc - p = 0
    prev_st[4, 6] = 2
    _, st = P.step(pull, test, prev, prev_st)
    assert st[4, 6] == 2


@pytest.mark.parametrize("scale", [1.0, 8.0])
def test_first_row_is_the_occlusion_check_and_the_scaled_flow(scale):
    rng = np.random.default_rng(4)
    T, H, W = 3, 23, 31
    fw, bw = _flows(rng, T, H, W)
    fw, bw = fw / F32(scale), bw / F32(scale)
    for K in range(T):
        acc, st = P.keyframe_rows(T + 1, H, W, K)
        acc, st = P.accumulate(fw, bw, acc, st, start=K, flow_scale=scale)
        _, occ_bw = fb_oracle.fb_check(fw[K:K + 1], bw[K:K + 1], flow_scale=scale)
        assert np.array_equal(st[K + 1], occ_bw[0])
        inside = occ_bw[0] != 2
        sb = (F32(scale) * bw[K]).astype(F32)
        assert np.array_equal(acc[K + 1][inside], sb[inside])
        assert (occ_bw[0] == 2).any() and inside.any()


@pytest.mark.parametrize("bounds", [(0, 1, 5), (0, 2, 3, 5), (0, 4, 5)])
def test_chunked_passes_equal_one_pass(bounds):
    rng = np.random.default_rng(5)
    T, H, W = 5, 17, 22
    fw, bw = _flows(rng, T, H, W)
    acc, st = P.keyframe_rows(T + 1, H, W, 0)
    whole_a, whole_s = P.accumulate(fw, bw, acc, st)
    carry = (whole_a[0], whole_s[0])
    for a, b in zip(bounds, bounds[1:]):
        ca = np.zeros((b - a + 1, H, W, 2), F32)
        cs = np.zeros((b - a + 1, H, W), np.uint8)
        ca[0], cs[0] = carry
        ca, cs = P.accumulate(fw[a:b], bw[a:b], ca, cs)
        assert np.array_equal(ca.view(np.uint32), whole_a[a:b + 1].view(np.uint32))
        assert np.array_equal(cs, whole_s[a:b + 1])
        carry = (ca[-1], cs[-1])


@pytest.mark.parametrize("scale", [1.0, 8.0])
def test_backward_equals_forward_on_the_reversed_clip(scale):
    rng = np.random.default_rng(6)
    T, H, W = 4, 19, 26
    fw, bw = _flows(rng, T, H, W)
    for K in range(T + 1):
        acc, st = P.keyframe_rows(T + 1, H, W, K)
        ba, bs = P.accumulate_backward(fw, bw, acc, st, start=K, flow_scale=scale)
        rfw, rbw = P.reversed_clip(fw, bw)
        acc, st = P.keyframe_rows(T + 1, H, W, T - K)
        fa, fs = P.accumulate(rfw, rbw, acc, st, start=T - K, flow_scale=scale)
        assert np.array_equal(ba[:K + 1].view(np.uint32), fa[::-1][:K + 1].view(np.uint32))
        assert np.array_equal(bs[:K + 1], fs[::-1][:K + 1])
        assert np.isnan(ba[K + 1:]).all() and (bs[K + 1:] == 77).all()  # rows after the key are not touched


@pytest.mark.parametrize("net,src", [((24, 40), (24, 40)), ((24, 40), (45, 80)), ((37, 53), (100, 150))])
def test_the_keyframe_row_reproduces_the_key(net, src):
    key = np.random.default_rng(7).integers(0, 255, src).astype(np.uint8)
    acc, st = P.keyframe_rows(1, *net, 0)
    labels, status = P.propagate(acc, st, key)
    assert np.array_equal(labels[0], key) and (status[0] == 0).all()


def test_accumulate_argument_checks():
    """The C entries refuse bad arguments with RB_ERR_* and a message before any CUDA call (host pointers below: a launch
    would fail, not return these codes)."""
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG = -1, -2
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = ctypes.c_float
    for name in ("rb_flow_accumulate", "rb_flow_accumulate_backward"):
        fn = getattr(lib, name)

        def call(fw=p, bw=p, T=3, H=8, W=9, n=3, s=1.0, a1=0.01, a2=0.5, start=0, acc=p, st=p):
            return fn(fw, bw, T, H, W, n, f(s), f(a1), f(a2), start, acc, st, None)

        def refused(rc, code, *words):
            assert rc == code, (name, rc, code)
            msg = lib.rb_last_error()
            assert name.encode() in msg and all(w in msg for w in words), msg

        for arg in ("fw", "bw", "acc", "st"):
            refused(call(**{arg: None}), BAD_ARG, b"null")
        for kw in ({"T": 0}, {"H": 0}, {"W": -1}):
            refused(call(**kw), BAD_SHAPE, b"bad shape")
        refused(call(H=65536, W=32768), BAD_SHAPE, b"32-bit")
        for n in (0, -1, 4):
            refused(call(n=n), BAD_SHAPE, b"n_steps")
        for start in (-1, 4):
            refused(call(start=start), BAD_ARG, b"start")
        for s in (0.0, -1.0, float("inf"), float("nan")):
            refused(call(s=s), BAD_ARG, b"flow_scale")
        for a1, a2 in ((-0.01, 0.5), (0.01, -0.5), (float("nan"), 0.5), (0.01, float("inf"))):
            refused(call(a1=a1, a2=a2), BAD_ARG, b"alpha")
    fn = lib.rb_labels_propagate

    def call(acc=p, st=p, n=2, H=8, W=9, key=p, Hs=10, Ws=12, lab=p, so=p):
        return fn(acc, st, n, H, W, key, Hs, Ws, lab, so, None)

    for arg in ("acc", "st", "key", "lab", "so"):
        assert call(**{arg: None}) == BAD_ARG and b"null" in lib.rb_last_error()
    for kw in ({"n": 0}, {"H": 0}, {"W": -1}, {"Hs": 0}, {"Ws": -3}):
        assert call(**kw) == BAD_SHAPE and b"rb_labels_propagate: bad shape" in lib.rb_last_error()
    assert call(Hs=65536, Ws=65536) == BAD_SHAPE and b"32-bit" in lib.rb_last_error()


def test_label_metrics_argument_checks():
    from raft_b200 import capi
    lib = capi.lib
    BAD_SHAPE, BAD_ARG = -1, -2
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def call(pr=p, gt=p, n=2, H=8, W=9, objs=3, r=8, c=p):
        return lib.rb_label_metrics(pr, gt, n, H, W, objs, r, c, None)

    for arg in ("pr", "gt", "c"):
        assert call(**{arg: None}) == BAD_ARG and b"null" in lib.rb_last_error()
    for kw in ({"n": 0}, {"H": 0}, {"W": -1}):
        assert call(**kw) == BAD_SHAPE and b"bad shape" in lib.rb_last_error()
    assert call(n=65536) == BAD_SHAPE and b"grid" in lib.rb_last_error()
    for objs in (0, -1, 256):
        assert call(objs=objs) == BAD_ARG and b"n_objects" in lib.rb_last_error()
    for r in (0, -1, 33):
        assert call(r=r) == BAD_ARG and b"bound_pix" in lib.rb_last_error()


def test_label_png_round_trip(tmp_path):
    from PIL import Image
    from raft_b200.synth import DAVIS_PALETTE
    from raft_b200.video import read_labels, write_labels
    lab = np.random.default_rng(8).integers(0, 12, (33, 47)).astype(np.uint8)
    write_labels(tmp_path / "p.png", lab, DAVIS_PALETTE)
    got, pal = read_labels(tmp_path / "p.png")
    assert np.array_equal(got, lab) and np.array_equal(pal[:len(DAVIS_PALETTE)], DAVIS_PALETTE)
    write_labels(tmp_path / "g.png", lab)
    got, pal = read_labels(tmp_path / "g.png")
    assert np.array_equal(got, lab) and pal is None
    Image.fromarray(np.zeros((5, 6, 3), np.uint8)).save(tmp_path / "rgb.png")
    with pytest.raises(ValueError, match="mode RGB"):
        read_labels(tmp_path / "rgb.png")


@pytest.mark.parametrize("extra,words", [
    (["--track-grid", "4"], "--track-grid"), (["--interpolate", "0.5"], "--interpolate"),
    (["--fps", "60", "--input-fps", "24"], "--fps"), (["--warm-start"], "--warm-start"),
    (["--scene-cut", "0.5"], "--scene-cut"), (["--native-frames"], "--native-frames"), (["--flo", "f"], "--flo"),
    (["--npy", "n"], "--npy"), (["--track-backward"], "--track-backward"), (["--native-flow"], "--native-flow"),
    (["--track", "q.txt"], "--track"), (["--input-fps", "24"], "--input-fps")])
def test_cli_propagate_argument_checks(extra, words, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(["--path", "frames", "--out", "o", "--propagate", "k.png"] + extra)
    assert e.value.code == 2 and f"cannot be combined with {words}" in capsys.readouterr().err


def test_cli_propagate_needs_a_frame_directory(tmp_path, capsys):
    import cv2
    import infer_raft
    from raft_b200.video import write_labels
    for argv, words in ((["--propagate", "k.png"], "needs --path"),
                        (["-m", "val", "--path", "f", "--propagate", "k.png"], "needs --path"),
                        (["--path", "f", "--propagate-frame", "2"], "--propagate-frame goes with --propagate")):
        with pytest.raises(SystemExit) as e:
            infer_raft.main(argv)
        assert e.value.code == 2 and words in capsys.readouterr().err
    (tmp_path / "frames").mkdir()
    for k in range(3):
        cv2.imwrite(str(tmp_path / "frames" / f"f{k}.png"), np.zeros((20, 30, 3), np.uint8))
    write_labels(tmp_path / "key.png", np.zeros((21, 30), np.uint8))
    base = ["--path", str(tmp_path / "frames"), "--out", str(tmp_path / "o"), "--propagate"]
    for argv, words in ((base + [str(tmp_path / "key.png")], "the key labels need the frames' size"),
                        (base + [str(tmp_path / "frames" / "f0.png")], "mode"),
                        (base + [str(tmp_path / "key.png"), "--propagate-frame", "3"], "holds 3 frames")):
        with pytest.raises(SystemExit) as e:
            infer_raft.main(argv)
        assert e.value.code == 2 and words in capsys.readouterr().err
