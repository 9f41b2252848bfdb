"""F33 on the CPU: the GoPro tree reader, the window selection, the ground-truth rounding, the protocol's shutter putting
every sample on a true frame, and the CLI's refusals, on synth.write_highfps_tree trees."""
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "raft-tf_b200", "infer_raft.py")


def test_reader_on_a_highfps_tree(tmp_path):
    from raft_b200 import synth
    from raft_b200.gopro import sequences
    written = synth.write_highfps_tree(str(tmp_path), "test", [("GOPR0002_00", 17), ("GOPR0001_00", 9)], 16, 24)
    seqs = sequences(str(tmp_path), "test")
    assert [n for n, _ in seqs] == ["GOPR0001_00", "GOPR0002_00"]
    assert [len(p) for _, p in seqs] == [9, 17] and seqs[1][1] == sorted(seqs[1][1])
    import cv2
    assert np.array_equal(cv2.imread(seqs[1][1][5]), written["GOPR0002_00"][5])
    assert np.array_equal(written["GOPR0002_00"][1][:, :-1], written["GOPR0002_00"][0][:, 1:])  # a 1-pixel pan
    with pytest.raises(FileNotFoundError):
        sequences(str(tmp_path), "train")
    os.makedirs(tmp_path / "train" / "empty")
    with pytest.raises(ValueError, match="no \\*.png"):
        sequences(str(tmp_path), "train")


def test_scored_windows():
    from raft_b200.gopro import scored
    # 41 frames, S = 8, M = 7: inputs 0, 8, ..., 40; input 0 needs frame -3 and input 5 (frame 40) frame 43
    assert scored(41, 8, 7) == [1, 2, 3, 4]
    assert scored(44, 8, 7) == [1, 2, 3, 4, 5]
    assert scored(41, 8, 1) == [0, 1, 2, 3, 4, 5]
    assert scored(5, 8, 7) == [] and scored(11, 8, 7) == [] and scored(12, 8, 7) == [1]


@pytest.mark.parametrize("S,M", [(0, 1), (8, 8), (8, 9), (4, 5), (8, -1), (8, 0), (8.5, 7), ("x", 7)])
def test_window_refusals(S, M):
    from raft_b200.gopro import check_window
    with pytest.raises(ValueError, match="stride"):
        check_window(S, M)


def test_ground_truth_rounds_half_to_even():
    from raft_b200.gopro import ground_truth
    w = np.zeros((2, 1, 4, 3), np.uint8)
    w[1, 0] = [[1, 1, 1], [3, 3, 3], [4, 4, 4], [255, 255, 255]]
    assert ground_truth(w)[0, :, 0].tolist() == [0, 2, 2, 128]  # 0.5 -> 0, 1.5 -> 2, 2, 127.5 -> 128
    w7 = np.arange(7, dtype=np.uint8).reshape(7, 1, 1, 1).repeat(3, -1)
    assert ground_truth(w7)[0, 0].tolist() == [3, 3, 3]


@pytest.mark.parametrize("S,M", [(8, 7), (8, 5), (4, 3), (6, 1)])
def test_protocol_samples_land_on_true_frames(S, M):
    """Shutter 360 M / S at density S: the m = M samples of input frame c sit at c + (j - (M-1)/2) / S, the true frames
    S c - (M-1)/2 .. S c + (M-1)/2, for every scored c."""
    from raft_b200.gopro import protocol, scored
    from raft_b200.video import exposure, shutter_schedule
    A, D = protocol(S, M)
    assert A == Fraction(360 * M, S) and D == S and exposure(1, 1, A, D)[1] == M
    F = 6 * S + 1
    n_in = (F - 1) // S + 1
    (ps,) = shutter_schedule(n_in, 1, 1, A, D, n_in - 1)
    rows = {}
    for n, i, t in ps.samples:
        rows.setdefault(n, []).append(i + (0 if t is None else Fraction(t).limit_denominator(1 << 20)))
    for c in scored(F, S, M):
        assert [S * u for u in rows[c]] == list(range(S * c - (M - 1) // 2, S * c + (M - 1) // 2 + 1))


@pytest.mark.parametrize("argv,what", [
    (["-m", "val", "--dataset", "gopro", "--data", "x", "--blur-frames", "8"], "--blur-frames"),
    (["-m", "val", "--dataset", "gopro", "--data", "x", "--stride", "4"], "--blur-frames"),
    (["-m", "val", "--dataset", "gopro", "--data", "x", "--warm-start"], "--warm-start"),
    (["-m", "val", "--dataset", "vimeo", "--data", "x", "--stride", "4"], "--dataset gopro"),
    (["--stride", "4"], "--dataset gopro")])
def test_cli_gopro_refusals(argv, what):
    r = subprocess.run([sys.executable, CLI] + argv, capture_output=True, text=True, timeout=120)
    error = r.stderr.strip().splitlines()[-1]
    assert r.returncode == 2 and what in error, r.stderr
