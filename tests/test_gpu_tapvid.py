"""F17's TAP-Vid evaluation end to end on the GPU: a synthetic pickle of three videos built from shifted crops of
tests/data/frame_0016.png (7-13 frames at sizes other than 256 x 256, one stored as encoded PNG bytes), seeded weights.
The per-video predictions equal the tracker's launches on one whole-clip pass bit for bit at every batch, the metrics
equal tests/tapvid_oracle.py on those predictions, and the CLI writes the API's result."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import tapvid_oracle as TO
import track_backward_oracle as B
import track_oracle as O
from test_gpu_track import _model, _weights

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITERS = 4


@pytest.fixture(scope="module")
def tapvid_pkl(tmp_path_factory):
    import cv2
    src = cv2.cvtColor(cv2.imread(os.path.join(ROOT, "tests", "data", "frame_0016.png")), cv2.COLOR_BGR2RGB)
    rng = np.random.default_rng(2022)
    data = {}
    for name, F, H, W, encoded in (("bear", 7, 200, 300, False), ("car", 13, 180, 240, True),
                                   ("dog", 9, 260, 330, False)):
        video = np.stack([src[20 + 2 * k:20 + 2 * k + H, 40 + 3 * k:40 + 3 * k + W] for k in range(F)])
        N = 30
        start = rng.uniform(0.05, 0.95, (N, 1, 2))
        points = (start + np.arange(F)[None, :, None] * np.array([3 / W, 2 / H]) * -1).astype(np.float32)
        occluded = rng.random((N, F)) < 0.2
        occluded[0] = True  # never visible: no query
        occluded[1] = True
        occluded[1, -1] = False  # visible only in its last frame
        occluded[2, :6] = True  # first visible at frame 6
        e = {"points": points, "occluded": occluded}
        e["video"] = ([cv2.imencode(".png", cv2.cvtColor(f, cv2.COLOR_RGB2BGR))[1].tobytes() for f in video]
                      if encoded else video)
        data[name] = e
    path = tmp_path_factory.mktemp("tapvid") / "tapvid_synth.pkl"
    with open(path, "wb") as f:
        pickle.dump(data, f)
    return str(path)


def _oracle_predictions(engine, frames, qframe, qpos, backward):
    """The launches the protocol describes, restated: one whole-clip forward_sequence_bidirectional pass, then the fp32
    restatements of rb_track_points and rb_track_points_backward on its flows."""
    fw, bw, _, _ = engine.forward_sequence_bidirectional(torch.from_numpy(np.ascontiguousarray(frames)), check=False)
    fw, bw = fw.cpu().numpy(), bw.cpu().numpy()
    t, s, _ = O.track(fw, bw, qframe, qpos, flow_scale=engine.flow_scale)
    if backward:
        t, s, _ = B.track_backward(fw, bw, qframe, qpos, t, s, flow_scale=engine.flow_scale)
    return t, s


@pytest.mark.parametrize("mode", ["first", "strided"])
def test_tapvid_end_to_end(cuda, tapvid_pkl, mode):
    from raft_b200 import tapvid
    from raft_b200.evaluate import _engine, evaluate
    m = _model(iters=ITERS)
    res = {b: evaluate(m, tapvid_pkl, "tapvid", batch=b, iters=ITERS, query_mode=mode) for b in (1, 4)}
    assert json.dumps(res[1]) == json.dumps(res[4])
    r = res[1]
    assert r["dataset"] == "tapvid" and r["iters"] == ITERS and r["query_mode"] == mode
    assert r["resolution"] == [256, 256]
    split = r["splits"]["tapvid"]
    assert split["n_videos"] == 3 and [v["name"] for v in split["videos"]] == ["bear", "car", "dog"]
    engine = _engine(m, ITERS, "sintel", input_size=tapvid.SIZE)
    per_video = []
    for v, rec in zip(tapvid.read_tapvid(tapvid_pkl), split["videos"]):
        track, frame = tapvid.sample_queries(v.occluded, mode)
        assert 0 not in track.tolist() and rec["n_queries"] == len(track) and rec["n_frames"] == len(v.frames)
        if mode == "first":
            assert (1, len(v.frames) - 1) in zip(track.tolist(), frame.tolist())
        qframe, qpos = tapvid.query_inputs(v.points, track, frame)
        bgr = v.frames[..., ::-1]  # the engine's channel order for reference weights
        want_t, want_s = _oracle_predictions(engine, bgr, qframe, qpos, mode == "strided")
        for batch in (1, 3, 4):
            t, s = tapvid.predict_video(engine, bgr, qframe, qpos, batch, backward=mode == "strided")
            assert O.same_bits(t.cpu().numpy(), want_t), (v.name, batch)
            assert np.array_equal(s.cpu().numpy(), want_s), (v.name, batch)
        if mode == "strided":
            assert not (want_s == O.BEFORE).any()
        gt = tapvid.to_pixels(v.points)[track]
        want = TO.metrics(want_t.transpose(1, 0, 2).tolist(), (want_s.T != 0).tolist(), gt.tolist(),
                          v.occluded[track].tolist(), frame.tolist(), mode)
        got = {k: rec[k] for k in want}
        assert TO.same(got, want), (v.name, got, want)
        assert 0 < want["occlusion_accuracy"] <= 1 and want["average_pts_within_thresh"] > 0
        per_video.append(want)
    for k in ("average_jaccard", "average_pts_within_thresh", "occlusion_accuracy"):
        assert split[k] == float(np.mean([w[k] for w in per_video])), k
    assert split["n_scored"] == {"average_jaccard": 3, "average_pts_within_thresh": 3, "occlusion_accuracy": 3}


def test_cli_val_tapvid(cuda, tapvid_pkl, tmp_path):
    from raft_b200.evaluate import evaluate, summary_lines
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **_weights(False))
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    argv = [sys.executable, cli, "-m", "val", "--dataset", "tapvid", "--data", tapvid_pkl, "--load", npz, "--iters",
            str(ITERS), "--out", str(tmp_path / "o"), "--batch", "4", "--query-mode", "strided"]
    r = subprocess.run(argv, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = evaluate(_model(iters=ITERS), tapvid_pkl, "tapvid", batch=2, iters=ITERS, query_mode="strided")
    with open(tmp_path / "o" / "val_tapvid.json") as f:
        assert json.dumps(json.load(f)) == json.dumps(res)
    assert summary_lines(res)[0] in r.stdout and summary_lines(res)[0].startswith("Validation TAP-Vid (strided): AJ: ")
