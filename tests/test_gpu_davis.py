"""F20's DAVIS-2017 evaluation end to end on the GPU: a synth.write_davis_tree tree (moving textured ellipses), seeded
weights.  The result is the same for every batch, equals tests/davis_oracle.py (the evaluator's formulas) on the masks
it writes, ground truth scored as prediction gives J = F = 1, and the CLI writes the API's result."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import davis_oracle as D
from test_gpu_track import _model, _weights

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITERS = 4


@pytest.fixture(scope="module")
def davis_root(tmp_path_factory):
    from raft_b200 import synth
    root = tmp_path_factory.mktemp("davis")
    synth.write_davis_tree(str(root), [("ellipses", 9), ("pair", 6)], H=120, W=200, objects=3, shift=2)
    synth.write_davis_tree(str(root / "tall"), [("tall", 7)], H=160, W=96, objects=1, seed=5100)
    os.rename(root / "tall" / "JPEGImages" / "480p" / "tall", root / "JPEGImages" / "480p" / "tall")
    os.rename(root / "tall" / "Annotations" / "480p" / "tall", root / "Annotations" / "480p" / "tall")
    with open(root / "ImageSets" / "2017" / "val.txt", "a") as f:
        f.write("tall\n")
    return str(root)


def test_davis_end_to_end(cuda, davis_root, tmp_path):
    from raft_b200.davis import davis_sequences
    from raft_b200.evaluate import evaluate, summary_lines
    from raft_b200.video import read_labels
    m = _model(iters=ITERS)
    res = {b: evaluate(m, davis_root, "davis", batch=b, iters=ITERS, masks_out=str(tmp_path / f"m{b}"))
           for b in (1, 8)}
    assert json.dumps(res[1], sort_keys=True) == json.dumps(res[8], sort_keys=True)
    r = res[1]["splits"]["val"]
    assert res[1]["dataset"] == "davis" and res[1]["iters"] == ITERS
    assert r["n_sequences"] == 3 and r["n_objects"] == 3 + 3 + 1
    seqs = davis_sequences(davis_root)
    pairs = []
    for s in seqs:
        gt = np.stack([read_labels(p)[0] for p in s.annotations])
        files = [os.path.join(tmp_path / "m1", s.name, os.path.basename(p)) for p in s.annotations]
        pred = np.stack([read_labels(f)[0] for f in files])
        assert np.array_equal(pred[0], gt[0])
        assert all(read_labels(f)[1] is not None for f in files)
        files8 = [os.path.join(tmp_path / "m8", s.name, os.path.basename(p)) for p in s.annotations]
        assert all(open(f, "rb").read() == open(g, "rb").read() for f, g in zip(files, files8))
        pairs.append((gt, pred))
    want = D.evaluate_sequences(pairs)
    for k, v in want.items():
        assert r[k] == pytest.approx(v, rel=1e-12, abs=1e-12), k
    assert 0.3 < r["J-Mean"] <= 1.0
    line = summary_lines(res[1])[0]
    assert line.startswith("Validation DAVIS-2017 (val): J&F: ")
    perfect = D.evaluate_sequences([(gt, gt) for gt, _ in pairs])
    assert perfect["J-Mean"] == perfect["F-Mean"] == perfect["J&F-Mean"] == 1.0


def test_ground_truth_as_prediction_scores_one(cuda, davis_root):
    import torch
    from networks.utils import davis_bound_pix, label_metrics
    from raft_b200.davis import davis_sequences, db_statistics, frame_scores
    from raft_b200.video import read_labels
    for s in davis_sequences(davis_root):
        gt = np.stack([read_labels(p)[0] for p in s.annotations])
        t = torch.from_numpy(gt).to(cuda)
        J, F = frame_scores(label_metrics(t, t, int(gt[0].max()), davis_bound_pix(*gt.shape[1:])).cpu().numpy())
        assert (J == 1).all() and (F == 1).all()
        assert db_statistics(J[0]) == (1.0, 1.0, 0.0)


def test_cli_davis(cuda, davis_root, tmp_path):
    from raft_b200.evaluate import evaluate
    npz = tmp_path / "w.npz"
    np.savez(npz, **_weights(False))
    cli = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")
    argv = [sys.executable, cli, "-m", "val", "--dataset", "davis", "--data", davis_root, "--load", str(npz), "--iters",
            str(ITERS), "--out", str(tmp_path / "o"), "--batch", "4"]
    r = subprocess.run(argv, capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert "Validation DAVIS-2017 (val): J&F: " in r.stdout
    with open(tmp_path / "o" / "val_davis.json") as f:
        got = json.load(f)
    want = json.loads(json.dumps(evaluate(_model(iters=ITERS), davis_root, "davis", batch=2, iters=ITERS)))
    assert got == want
    assert sorted(os.listdir(tmp_path / "o" / "davis_val")) == ["ellipses", "pair", "tall"]
