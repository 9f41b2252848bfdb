"""DAVIS-2017 scoring without a GPU: raft_b200.davis's J / F / statistics against the evaluator's formulas
(tests/davis_oracle.py) on edge cases and short sequences, the tree reader's refusals and the CLI's argument errors."""
import os

import numpy as np
import pytest

import davis_oracle as D


def _counts(pred, gt, r):
    return D.counts(pred[None], gt[None], 1, r)[0, 0]


@pytest.mark.parametrize("case", ["empty_pred", "empty_gt", "both_empty", "equal", "shifted", "disjoint"])
def test_j_and_f_edge_cases(case):
    from raft_b200.davis import frame_scores
    H, W = 40, 60
    gt = np.zeros((H, W), np.uint8)
    gt[10:25, 15:40] = 1
    pred = {"empty_pred": np.zeros_like(gt), "empty_gt": gt, "both_empty": np.zeros_like(gt), "equal": gt,
            "shifted": np.roll(gt, (2, 3), (0, 1)), "disjoint": np.roll(gt, (0, 30), (0, 1))}[case]
    if case in ("empty_gt", "both_empty"):
        gt = np.zeros_like(gt)
    c = _counts(pred, gt, 2)
    J, F = frame_scores(c[None, None])
    assert J[0, 0] == pytest.approx(D.db_eval_iou(gt, pred), abs=0, rel=1e-15)
    assert F[0, 0] == pytest.approx(D.f_measure(pred, gt, 2), abs=0, rel=1e-15)
    want = {"empty_pred": (0.0, 0.0), "empty_gt": (0.0, 0.0), "both_empty": (1.0, 1.0), "equal": (1.0, 1.0)}
    if case in want:
        assert (J[0, 0], F[0, 0]) == want[case]


@pytest.mark.parametrize("L", [1, 2, 3, 4, 5, 7, 40, 300])
def test_statistics_equal_the_evaluator(L):
    from raft_b200.davis import db_statistics
    rng = np.random.default_rng(L)
    v = rng.uniform(0, 1, L)
    if L > 3:
        v[1] = np.nan
    got, want = db_statistics(v), D.db_statistics(v)
    for g, w in zip(got, want):
        assert (np.isnan(g) and np.isnan(w)) or g == w


def test_aggregate_means_over_objects():
    from raft_b200.davis import aggregate_davis
    objs = [{"J-Mean": a, "J-Recall": 1.0, "J-Decay": 0.0, "F-Mean": b, "F-Recall": 0.0, "F-Decay": 0.1}
            for a, b in ((0.5, 0.7), (0.9, 0.3), (0.1, 0.2))]
    res = aggregate_davis([{"name": "a", "objects": objs[:1]}, {"name": "b", "objects": objs[1:]}])
    assert res["J-Mean"] == pytest.approx(0.5) and res["F-Mean"] == pytest.approx(0.4)
    assert res["J&F-Mean"] == pytest.approx(0.45) and res["n_objects"] == 3 and res["n_sequences"] == 2


def _tree(root, names=("a", "b"), n=3):
    from raft_b200 import synth
    synth.write_davis_tree(str(root), [(s, n) for s in names], H=24, W=32)


def test_reader_accepts_a_tree_and_refuses_missing_files(tmp_path):
    from raft_b200.davis import davis_sequences
    _tree(tmp_path)
    seqs = davis_sequences(tmp_path)
    assert [s.name for s in seqs] == ["a", "b"] and all(len(s.frames) == len(s.annotations) == 3 for s in seqs)
    os.remove(tmp_path / "Annotations" / "480p" / "b" / "00001.png")
    with pytest.raises(ValueError, match="3 frames and 2 annotations"):
        davis_sequences(tmp_path)
    os.rename(tmp_path / "Annotations" / "480p" / "b" / "00002.png", tmp_path / "Annotations" / "480p" / "b" / "x.png")
    os.remove(tmp_path / "JPEGImages" / "480p" / "b" / "00002.jpg")
    with pytest.raises(ValueError, match="no annotation 00001.png"):
        davis_sequences(tmp_path)
    with open(tmp_path / "ImageSets" / "2017" / "val.txt", "a") as f:
        f.write("ghost\n")
    with pytest.raises(FileNotFoundError):
        davis_sequences(tmp_path / "nowhere")
    os.remove(tmp_path / "ImageSets" / "2017" / "val.txt")
    with pytest.raises(FileNotFoundError, match="no sequence list"):
        davis_sequences(tmp_path)


def test_reader_refuses_a_missing_sequence_directory(tmp_path):
    from raft_b200.davis import davis_sequences
    _tree(tmp_path, names=("a",))
    with open(tmp_path / "ImageSets" / "2017" / "val.txt", "a") as f:
        f.write("ghost\n")
    with pytest.raises(FileNotFoundError, match="ghost"):
        davis_sequences(tmp_path)


def test_synthetic_tree_annotations_are_palette_label_maps(tmp_path):
    from raft_b200.video import read_labels
    _tree(tmp_path, names=("a",), n=2)
    lab, pal = read_labels(tmp_path / "Annotations" / "480p" / "a" / "00000.png")
    assert lab.shape == (24, 32) and pal is not None and set(np.unique(lab)) <= {0, 1, 2} and lab.max() > 0


@pytest.mark.parametrize("extra,words", [
    (["--split", "test"], "DAVIS-2017 test-dev"), (["--warm-start"], "DAVIS propagates labels"),
    (["--query-mode", "first"], "--query-mode goes with -m val --dataset tapvid")])
def test_cli_davis_argument_checks(extra, words, capsys):
    import infer_raft
    with pytest.raises(SystemExit) as e:
        infer_raft.main(["-m", "val", "--dataset", "davis", "--data", "d"] + extra)
    assert e.value.code == 2 and words in capsys.readouterr().err


def test_evaluate_refusals():
    from types import SimpleNamespace
    from raft_b200.evaluate import evaluate, submit
    m = SimpleNamespace(input_size=(64, 64), _params={}, upstream=False)
    with pytest.raises(ValueError, match="own size"):
        evaluate(m, "d", "davis")
    m.input_size = None
    with pytest.raises(ValueError, match="warm_start"):
        evaluate(m, "d", "davis", warm_start=True)
    with pytest.raises(ValueError, match="masks_out"):
        evaluate(m, "d", "sintel", masks_out="x")
    with pytest.raises(ValueError, match="query_mode"):
        evaluate(m, "d", "davis", query_mode="first")
    with pytest.raises(ValueError, match="test-dev"):
        submit(m, "d", "davis", "o")
