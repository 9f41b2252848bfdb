"""F21 on the CPU: the several-keyframe vote (tests/keyframes_oracle.py) on hand cases, the table of
raft_b200.video.keyframe_rows against a literal reading of its rules, the host-side argument checks of the new entry
points and CLI flags, and DAVIS's statistics with the keyframes left out of the scored frames."""
import itertools

import numpy as np
import pytest

import davis_oracle as D
import keyframes_oracle as KO
import propagate_oracle as P

F32 = np.float32


def _rows(rng, n, H, W, nan=True):
    acc = rng.uniform(-6, 6, (n, H, W, 2)).astype(F32)
    if nan:
        acc[0, 1, 2, 0] = np.nan
    return acc, rng.integers(0, 3, (n, H, W)).astype(np.uint8)


@pytest.mark.parametrize("which", ["a", "b"])
def test_one_side_equals_single_key_propagation(which):
    rng = np.random.default_rng(1)
    acc, st = _rows(rng, 3, 9, 13)
    keys = rng.integers(0, 5, (2, 18, 20)).astype(np.uint8)
    garbage = np.full_like(acc, np.nan), np.full_like(st, 9)
    if which == "a":
        rows = np.array([[1, -1, 0, 0]] * 3)
        got = KO.propagate_keys(acc, st, *garbage, keys, rows)
    else:
        rows = np.array([[-1, 1, 0, 0]] * 3)
        got = KO.propagate_keys(*garbage, acc, st, keys, rows)
    want = P.propagate(acc, st, keys[1])
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def _two(key_a, key_b, wa, wb, st_a=0, st_b=0, shift=(0.0, 0.0)):
    H, W = key_a.shape
    acc = np.zeros((1, H, W, 2), F32)
    acc[..., 0], acc[..., 1] = shift
    sa = np.full((1, H, W), st_a, np.uint8)
    sb = np.full((1, H, W), st_b, np.uint8)
    return KO.propagate_keys(acc, sa, acc.copy(), sb, np.stack([key_a, key_b]), np.array([[0, 1, wa, wb]]))


def test_agreeing_sides_give_their_label():
    k = np.full((6, 7), 4, np.uint8)
    lab, st = _two(k, k, 3, 5, shift=(0.3, 0.6))
    assert (lab == 4).all() and (st[:, :-1, :-1] == 0).all() and (st[:, -1] == 2).all()  # the last row leaves


def test_the_nearer_key_wins_and_the_midpoint_tie_goes_to_the_smaller_label():
    a, b = np.full((5, 6), 7, np.uint8), np.full((5, 6), 2, np.uint8)
    assert (_two(a, b, 3, 1)[0] == 7).all()  # t one frame after K_i, three before K_j: side A weighs 3
    assert (_two(a, b, 1, 3)[0] == 2).all()
    assert (_two(a, b, 2, 2)[0] == 2).all() and (_two(b, a, 2, 2)[0] == 2).all()
    # a fractional origin: side A's two labels split its weight, side B's one label keeps all of it
    a2 = np.zeros((5, 6), np.uint8)
    a2[:, 3:] = 7
    lab, _ = _two(a2, b, 3, 2, shift=(0.5, 0.0))
    assert (lab[0, :, 2] == 2).all()  # A: 0 and 7 at 1.5 each, B: 2 at 2 -> 2


@pytest.mark.parametrize("sa,sb", [(0, 1), (1, 0), (1, 2), (2, 1), (0, 2), (0, 0), (1, 1), (2, 2)])
def test_status_gating(sa, sb):
    """Side A weighs 9, side B 1: A's label wins whenever A votes; B wins only when its status gates A out."""
    a, b = np.full((4, 5), 7, np.uint8), np.full((4, 5), 2, np.uint8)
    lab, st = _two(a, b, 9, 1, st_a=sa, st_b=sb)
    assert (lab == (7 if sa <= sb else 2)).all() and (st == min(sa, sb)).all()


def test_no_side_gives_label_0_and_status_3():
    k = np.full((2, 4, 5), 6, np.uint8)
    acc, st = _rows(np.random.default_rng(2), 2, 4, 5)
    lab, s = KO.propagate_keys(acc, st, acc, st, k, np.array([[-1, -1, 0, 0], [5, -7, 1, 1]]))
    assert (lab == 0).all() and (s == 3).all()


def test_keyframe_rows_equal_the_rules_for_every_small_case():
    from raft_b200.video import keyframe_rows
    n = 0
    for F in range(2, 7):
        for m in range(1, F + 1):
            for keys in itertools.combinations(range(F), m):
                for nc in range(F):
                    for cuts in itertools.combinations(range(F - 1), nc):
                        got = keyframe_rows(F, list(keys), cuts)
                        assert got.dtype == np.int32 and got.shape == (F, 4)
                        assert np.array_equal(got, KO.keyframe_rows(F, keys, cuts)), (F, keys, cuts)
                        n += 1
    assert n > 2500


def test_keyframe_rows_hand_case():
    from raft_b200.video import keyframe_rows
    rows = keyframe_rows(10, [2, 6], cuts=[7])
    assert rows.tolist() == [[-1, 0, 0, 0], [-1, 0, 0, 0], [0, -1, 0, 0], [0, 1, 3, 1], [0, 1, 2, 2], [0, 1, 1, 3],
                             [1, -1, 0, 0], [1, -1, 0, 0], [-1, -1, 0, 0], [-1, -1, 0, 0]]
    assert keyframe_rows(4, 0).tolist() == [[0, -1, 0, 0]] * 4  # one int: the single-key table


@pytest.mark.parametrize("frames,cuts,words", [([], (), "integer"), ([2, 2], (), "strictly increasing"),
                                               ([3, 1], (), "strictly increasing"), ([0, 5], (), r"\[0, 5\)"),
                                               ([-1], (), r"\[0, 5\)"), ([1.5], (), "integer"),
                                               ([0], (4,), "cuts"), ([0], (-1,), "cuts"), ([0], (1.5,), "cuts"),
                                               ([0], 3, "cuts")])
def test_keyframe_rows_refusals(frames, cuts, words):
    from raft_b200.video import keyframe_rows
    with pytest.raises(ValueError, match=words):
        keyframe_rows(5, frames, cuts)


def test_propagate_labels_keys_needs_cuda_rows():
    import torch
    from networks.utils import propagate_labels_keys
    acc = torch.zeros(1, 4, 5, 2)
    st = torch.zeros(1, 4, 5, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA"):
        propagate_labels_keys(acc, st, acc, st, torch.zeros(1, 4, 5, dtype=torch.uint8), [[0, -1, 0, 0]])


def test_video_propagate_refuses_bad_keys_before_any_work(tmp_path):
    from raft_b200.video import video_propagate
    paths = [str(tmp_path / f"f{i}.png") for i in range(4)]  # never read: the checks come first
    k = np.zeros((3, 4), np.uint8)
    for labels, frame, words in (([k], [0, 2], "1 key label maps for 2"), ([k, k], [2, 1], "strictly increasing"),
                                 ([k, k], [0, 4], r"\[0, 4\)"), ([k, np.zeros((3, 5), np.uint8)], [0, 2], "differ"),
                                 ([k, k.astype(np.int32)], [0, 2], "uint8")):
        with pytest.raises(ValueError, match=words):
            video_propagate(None, paths, str(tmp_path / "o"), labels, frame=frame)
    with pytest.raises(ValueError, match="scene_cut"):
        video_propagate(None, paths, str(tmp_path / "o"), [k, k], frame=[0, 2], scene_cut=2.0)


def _cli_error(argv, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


def test_cli_keyframe_checks(tmp_path, capsys):
    import cv2
    from raft_b200.video import write_labels
    (tmp_path / "frames").mkdir()
    for k in range(4):
        cv2.imwrite(str(tmp_path / "frames" / f"f{k}.png"), np.zeros((20, 30, 3), np.uint8))
    write_labels(tmp_path / "k.png", np.zeros((20, 30), np.uint8))
    key = str(tmp_path / "k.png")
    base = ["--path", str(tmp_path / "frames"), "--out", str(tmp_path / "o"), "--propagate"]
    for argv, words in ((base + [key, key], "counts must match"),
                        (base + [key, key, "--propagate-frame", "0"], "counts must match"),
                        (base + [key, "--propagate-frame", "0", "2"], "counts must match"),
                        (base + [key, key, "--propagate-frame", "2", "2"], "strictly increasing"),
                        (base + [key, key, "--propagate-frame", "0", "4"], "holds 4 frames"),
                        (base + [key, key, "--propagate-frame", "0", "2", "--scene-cut", "1.5"], "not a threshold"),
                        (base + [key, "--scene-cut", "0.5"], "one key map cannot be combined with --scene-cut"),
                        (["-m", "val", "--dataset", "sintel", "--data", "d", "--keyframe-step", "4"],
                         "--keyframe-step goes with -m val --dataset davis"),
                        (["--keyframe-step", "4"], "--keyframe-step goes with"),
                        (["-m", "val", "--dataset", "davis", "--data", "d", "--keyframe-step", "0"], "must be >= 1")):
        assert words in _cli_error(argv, capsys), argv


def test_evaluate_keyframe_step_checks():
    from types import SimpleNamespace
    from raft_b200.evaluate import evaluate
    m = SimpleNamespace(input_size=None, _params={})
    with pytest.raises(ValueError, match="DAVIS"):
        evaluate(m, "d", "sintel", keyframe_step=4)
    for bad in (0, -2, 1.5, True):
        with pytest.raises(ValueError, match=">= 1"):
            evaluate(m, "d", "davis", keyframe_step=bad)


def test_summary_line_names_the_step():
    from raft_b200.evaluate import summary_lines
    r = {"J&F-Mean": 0.5, "J-Mean": 0.4, "F-Mean": 0.6}
    assert summary_lines({"dataset": "davis", "keyframe_step": 8, "splits": {"val": r}})[0].startswith(
        "Validation DAVIS-2017 (val, a keyframe every 8): J&F: 0.500000")
    assert summary_lines({"dataset": "davis", "splits": {"val": r}})[0].startswith("Validation DAVIS-2017 (val): J&F")


def test_scored_frames_leave_out_the_keyframes():
    from raft_b200.davis import keyframe_frames, scored_frames
    assert keyframe_frames(10, 4) == [0, 4, 8] and keyframe_frames(3, 100) == [0]
    assert scored_frames(10, [0, 4, 8]) == [1, 2, 3, 5, 6, 7]
    assert scored_frames(10, keyframe_frames(10, 1)) == []
    assert scored_frames(10, [0]) == list(range(1, 9))


def test_statistics_over_the_scored_frames_from_counts():
    """J, F and their M / O / D over the scored frames only, from label counts, against the evaluator's formulas."""
    import torch  # noqa: F401  (raft_b200.davis imports it)
    from raft_b200.davis import db_statistics, frame_scores, keyframe_frames, scored_frames
    rng = np.random.default_rng(3)
    F, H, W = 14, 24, 30
    gt = np.zeros((F, H, W), np.uint8)
    for t in range(F):
        gt[t, 4 + t // 2:14 + t // 2, 5:15 + t] = 1
    pred = gt.copy()
    for t in range(F):
        pred[t] = np.roll(gt[t], int(rng.integers(-2, 3)), 1)
    scored = scored_frames(F, keyframe_frames(F, 4))
    counts = D.counts(pred[scored], gt[scored], 1, 2)
    J, Fm = frame_scores(counts)
    want_j = [D.db_eval_iou(gt[t] == 1, pred[t] == 1) for t in scored]
    assert np.allclose(J[0], want_j, rtol=0, atol=1e-12)
    assert db_statistics(J[0]) == pytest.approx(D.db_statistics(np.array(want_j)), abs=1e-12)
    assert len(J[0]) == len(scored) == 9
