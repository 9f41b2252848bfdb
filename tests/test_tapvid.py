"""F17's TAP-Vid evaluation without a GPU: the vectorised metrics against the loop restatement (tests/tapvid_oracle.py)
and hand-built cases, query sampling, the pickle reader and its errors, and the refusals of evaluate, submit and the
CLI."""
import os
import pickle
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

import tapvid_oracle as TO
from raft_b200 import tapvid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _metrics(pred, pred_occ, gt, gt_occ, qframe, mode):
    return tapvid.video_metrics(tapvid.video_counts(pred, pred_occ, gt, gt_occ, qframe, mode))


def _random_video(rng, Q, F):
    gt = rng.uniform(0, 255, (Q, F, 2))
    gt_occ = rng.random((Q, F)) < 0.3
    pred = gt + rng.normal(0, 4, gt.shape)
    pred[rng.random((Q, F)) < 0.05] = np.nan
    pred_occ = rng.random((Q, F)) < 0.3
    qframe = rng.integers(0, F, Q)
    return pred.astype(np.float32), pred_occ, gt, gt_occ, qframe


@pytest.mark.parametrize("mode", ["first", "strided"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_metrics_equal_the_loop_restatement(mode, seed):
    rng = np.random.default_rng(seed)
    args = _random_video(rng, 40, 17)
    got = _metrics(*args, mode)
    want = TO.metrics(*(a.tolist() for a in args), mode)
    assert TO.same(got, want), (got, want)
    assert 0 < got["average_jaccard"] < 1 and 0 < got["occlusion_accuracy"] < 1


@pytest.mark.parametrize("mode", ["first", "strided"])
def test_perfect_prediction_scores_one(mode):
    rng = np.random.default_rng(3)
    _, _, gt, gt_occ, qframe = _random_video(rng, 20, 9)
    m = _metrics(gt.astype(np.float32), gt_occ, gt, gt_occ, qframe, mode)
    assert m["average_jaccard"] == 1.0 and m["average_pts_within_thresh"] == 1.0 and m["occlusion_accuracy"] == 1.0


def test_everything_predicted_occluded_has_jaccard_zero():
    rng = np.random.default_rng(4)
    _, _, gt, gt_occ, qframe = _random_video(rng, 20, 9)
    m = _metrics(gt.astype(np.float32), np.ones_like(gt_occ), gt, gt_occ, qframe, "strided")
    assert m["average_jaccard"] == 0.0 and all(m[f"jaccard_{d}"] == 0.0 for d in tapvid.THRESHOLDS)
    assert m["average_pts_within_thresh"] == 1.0  # δ ignores the predicted visibility


def test_known_counts():
    """One query on frame 0 of a 5-frame track, 'first' mode: frames 1-4 are evaluated."""
    gt = np.zeros((1, 5, 2))
    gt_occ = np.array([[False, False, False, True, False]])
    pred = np.float32([[[0, 0], [0.5, 0], [3, 0], [100, 100], [np.nan, np.nan]]])
    pred_occ = np.array([[False, False, False, False, True]])
    c = tapvid.video_counts(pred, pred_occ, gt, gt_occ, [0], "first")
    # frame 1: visible, predicted visible, 0.5 px; frame 2: 3 px; frame 3: occluded, predicted visible; frame 4:
    # visible, predicted occluded, NaN
    assert c["evaluated"] == 4 and c["visible"] == 3 and c["occlusion_correct"] == 2
    assert [c[f"within_{d}"] for d in tapvid.THRESHOLDS] == [1, 1, 2, 2, 2]
    assert [c[f"true_pos_{d}"] for d in tapvid.THRESHOLDS] == [1, 1, 2, 2, 2]
    assert [c[f"false_pos_{d}"] for d in tapvid.THRESHOLDS] == [2, 2, 1, 1, 1]
    m = tapvid.video_metrics(c)
    assert m["occlusion_accuracy"] == 0.5 and m["pts_within_1"] == 1 / 3 and m["jaccard_4"] == 2 / 4
    assert m["average_jaccard"] == (1 / 5 + 1 / 5 + 2 / 4 + 2 / 4 + 2 / 4) / 5
    assert TO.same(m, TO.metrics(pred.tolist(), pred_occ.tolist(), gt.tolist(), gt_occ.tolist(), [0], "first"))


def test_zero_denominators_are_nan_and_left_out_of_the_mean():
    m_empty = tapvid.video_metrics(tapvid.video_counts(np.zeros((0, 4, 2)), np.zeros((0, 4), bool), np.zeros((0, 4, 2)),
                                                       np.zeros((0, 4), bool), np.zeros(0, int), "first"))
    assert all(np.isnan(v) for v in m_empty.values())
    # all evaluated entries occluded and predicted occluded: OA = 1, δ and J have no denominator
    occ = np.array([[False, True, True]])
    m_occ = _metrics(np.zeros((1, 3, 2), np.float32), occ, np.zeros((1, 3, 2)), occ, [0], "first")
    assert m_occ["occlusion_accuracy"] == 1.0 and np.isnan(m_occ["average_jaccard"])
    rec = [dict(name="a", n_frames=4, n_queries=0, **m_empty), dict(name="b", n_frames=3, n_queries=1, **m_occ),
           dict(name="c", n_frames=3, n_queries=1, **{k: 0.5 for k in m_occ})]
    agg = tapvid.aggregate_tapvid(rec)
    assert agg["n_videos"] == 3 and agg["occlusion_accuracy"] == 0.75 and agg["average_jaccard"] == 0.5
    assert agg["n_scored"] == {"average_jaccard": 1, "average_pts_within_thresh": 1, "occlusion_accuracy": 2}
    assert [v["name"] for v in agg["videos"]] == ["a", "b", "c"]


def test_query_sampling():
    occ = np.ones((5, 12), bool)
    occ[0, 3:] = False  # first visible at 3
    occ[1, :] = False  # always visible
    # track 2: never visible
    occ[3, 11] = False  # visible only in its last frame
    occ[4, [0, 5, 7]] = False
    track, frame = tapvid.sample_queries(occ, "first")
    assert list(zip(track.tolist(), frame.tolist())) == [(0, 3), (1, 0), (3, 11), (4, 0)] == TO.queries(occ.tolist(),
                                                                                                          "first")
    track, frame = tapvid.sample_queries(occ, "strided")
    assert list(zip(track.tolist(), frame.tolist())) == [(1, 0), (4, 0), (0, 5), (1, 5), (4, 5), (0, 10), (1, 10)]
    assert list(zip(track.tolist(), frame.tolist())) == TO.queries(occ.tolist(), "strided")
    rng = np.random.default_rng(9)
    occ = rng.random((30, 23)) < 0.6
    for mode in ("first", "strided"):
        t, f = tapvid.sample_queries(occ, mode)
        assert list(zip(t.tolist(), f.tolist())) == TO.queries(occ.tolist(), mode)
    with pytest.raises(ValueError, match="query_mode"):
        tapvid.sample_queries(occ, "all")


def test_query_inputs_use_the_pixel_centre_convention():
    points = np.array([[[0.0, 0.0], [1.0, 1.0], [0.5, 0.25], [1 / 512, 3 / 512]]])
    qf, qp = tapvid.query_inputs(points, np.zeros(4, int), np.arange(4))
    assert qf.dtype == np.int32 and qp.dtype == np.float32
    assert qp.tolist() == [[0.0, 0.0], [255.0, 255.0], [127.5, 63.5], [0.0, 1.0]]  # -0.5 and 255.5 clamped
    assert np.array_equal(tapvid.to_pixels(points)[0, 2], [127.5, 63.5])


def _entry(rng, F, N=4, H=20, W=24, encoded=False):
    import cv2
    video = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    e = {"points": rng.random((N, F, 2)).astype(np.float32), "occluded": rng.random((N, F)) < 0.3}
    if encoded:  # PNG bytes of the BGR frames, as cv2.imencode writes them
        e["video"] = [cv2.imencode(".png", cv2.cvtColor(f, cv2.COLOR_RGB2BGR))[1].tobytes() for f in video]
    else:
        e["video"] = video
    return e, video


def _dump(path, obj):
    with open(path, "wb") as f:
        pickle.dump(obj, f)


def test_reader_dict_list_shards_and_encoded_frames(tmp_path):
    rng = np.random.default_rng(1)
    (a, va), (b, vb), (c, vc), (d, vd) = (_entry(rng, F, encoded=enc) for F, enc in ((3, False), (4, True),
                                                                                     (2, False), (5, True)))
    _dump(tmp_path / "davis.pkl", {"bear": a, "car": b})
    got = list(tapvid.read_tapvid(str(tmp_path / "davis.pkl")))
    assert [v.name for v in got] == ["bear", "car"]
    assert np.array_equal(got[0].frames, va) and np.array_equal(got[1].frames, vb)  # decoded to RGB
    assert got[0].points.dtype == np.float64 and got[0].occluded.dtype == bool
    assert np.array_equal(got[1].points, b["points"].astype(np.float64))
    shards = tmp_path / "kinetics"
    shards.mkdir()
    _dump(shards / "0001.pkl", [d])
    _dump(shards / "0000.pkl", [c, a])
    (shards / "notes.txt").write_text("not a shard")
    got = list(tapvid.read_tapvid(str(shards)))
    assert [v.name for v in got] == ["0000/0", "0000/1", "0001/0"]
    assert np.array_equal(got[0].frames, vc) and np.array_equal(got[2].frames, vd)


@pytest.mark.parametrize("change,words", [
    (lambda e: e.pop("points"), "`points`"),
    (lambda e: e.update(video=e["video"][:1], points=e["points"][:, :1], occluded=e["occluded"][:, :1]), "two"),
    (lambda e: e.update(points=e["points"][..., 0]), "[N,F,2]"),
    (lambda e: e.update(occluded=e["occluded"][:, :2]), "occluded"),
    (lambda e: e.update(points=e["points"][:, :2], occluded=e["occluded"][:, :2]), "2 frames, the video has 4"),
    (lambda e: e.update(video=e["video"].astype(np.float32)), "uint8"),
    (lambda e: e.update(video=e["video"][..., :2]), "[F,H,W,3]"),
    (lambda e: e.update(video=[b"not an image", b"x"]), "decode"),
    (lambda e: e.update(video=5), "encoded"),
])
def test_reader_errors_name_the_video(tmp_path, change, words):
    e, _ = _entry(np.random.default_rng(2), 4)
    change(e)
    _dump(tmp_path / "d.pkl", {"swan": e})
    with pytest.raises(ValueError) as err:
        list(tapvid.read_tapvid(str(tmp_path / "d.pkl")))
    assert "swan" in str(err.value) and words in str(err.value), str(err.value)


def test_reader_file_errors(tmp_path):
    with pytest.raises(FileNotFoundError):
        tapvid.tapvid_files(str(tmp_path / "none.pkl"))
    with pytest.raises(FileNotFoundError, match="no \\*.pkl"):
        tapvid.tapvid_files(str(tmp_path))
    _dump(tmp_path / "x.pkl", 42)
    with pytest.raises(ValueError, match="holds a int"):
        list(tapvid.read_tapvid(str(tmp_path / "x.pkl")))
    e, _ = _entry(np.random.default_rng(3), 3)
    big, _ = _entry(np.random.default_rng(3), 3, H=30, encoded=True)
    e["video"] = [e["video"][0].tobytes()]  # raw bytes are no image
    with pytest.raises(ValueError, match="decode"):
        tapvid.check_entry("v", e)
    import cv2
    sizes = [cv2.imencode(".png", f)[1].tobytes() for f in (np.zeros((4, 4, 3), np.uint8), np.zeros((5, 4, 3), np.uint8))]
    with pytest.raises(ValueError, match="frame 1"):
        tapvid.check_entry("v", {"video": sizes, "points": np.zeros((1, 2, 2)), "occluded": np.zeros((1, 2), bool)})
    assert len(tapvid.check_entry("w", big).frames) == 3


def test_evaluate_and_submit_refusals():
    from networks.RAFT import RAFT
    from raft_b200.evaluate import evaluate, submit
    m = RAFT(None, SimpleNamespace(small=False))
    with pytest.raises(ValueError, match="cold flows"):
        evaluate(m, "/nonexistent", "tapvid", warm_start=True)
    with pytest.raises(ValueError, match="TAP-Vid has no test split"):
        submit(m, "/nonexistent", "tapvid", "/nonexistent")
    with pytest.raises(ValueError, match="256x256"):
        evaluate(RAFT(None, SimpleNamespace(small=False), input_size=(256, 256)), "/nonexistent", "tapvid")
    with pytest.raises(ValueError, match="query_mode must be one of"):
        evaluate(m, "/nonexistent", "tapvid", query_mode="all")
    with pytest.raises(ValueError, match="query_mode belongs to TAP-Vid"):
        evaluate(m, "/nonexistent", "sintel", query_mode="first")
    with pytest.raises(RuntimeError, match="load"):
        evaluate(m, "/nonexistent", "tapvid", query_mode="strided")


def test_summary_line():
    from raft_b200.evaluate import summary_lines
    res = {"dataset": "tapvid", "query_mode": "strided",
           "splits": {"tapvid": {"average_jaccard": 0.25, "average_pts_within_thresh": 0.5, "occlusion_accuracy": 0.75}}}
    assert summary_lines(res) == ["Validation TAP-Vid (strided): AJ: 0.250000, <δ_avg>: 0.500000, OA: 0.750000"]


def test_cli_refusals(tmp_path):
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    base = [sys.executable, cli, "-m", "val", "--dataset", "tapvid", "--data", str(tmp_path)]
    for argv, words in ((base + ["--split", "test"], "TAP-Vid has no hidden-ground-truth split"),
                        (base + ["--warm-start"], "TAP-Vid tracks points through cold flows"),
                        (base[:5] + ["sintel", "--data", str(tmp_path), "--query-mode", "first"], "--query-mode goes"),
                        ([sys.executable, cli, "--query-mode", "strided"], "--query-mode goes"),
                        (base + ["--query-mode", "all"], "invalid choice")):
        r = subprocess.run(argv, cwd=tmp_path, env=env, capture_output=True, text=True)
        assert r.returncode == 2 and words in r.stderr, (argv, r.stderr)
