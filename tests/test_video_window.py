"""The host bookkeeping the streaming video sweeps share, on the CPU: raft_b200.video._Window (which frames a windowed
sweep keeps on the GPU, when each frame is finished, and its table rows rebased to the store) driven through
interp_schedule()'s passes on CPU tensors whose rows hold their frame or pair index; _Upload's cut list; _FrameWriter;
and print_cuts's line."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch


def _due(F, T, window, segment):
    """The pass at which each frame is due, restated per frame from the sweeps' rules: frame t needs the data of frames
    up to min(t + window, F - 1); after a pass the pairs up to ran - 1 have run, ran its last frame.  The evidence of
    motion segmentation's frame ran is only complete after the next pass (all of it after the last)."""
    from raft_b200.video import interp_schedule
    rans = [ps.frames[0] + sum(k is not None for k in ps.pairs) for ps in interp_schedule(F, T)]

    def ready(t, ran):
        need = min(t + window, F - 1)
        return ran == F - 1 or need < ran if segment else need <= ran
    return [next(j for j, ran in enumerate(rans) if ready(t, ran)) for t in range(F)]


def _sweep(F, T, window, segment):
    """One windowed sweep's bookkeeping over interp_schedule(F, T), checked at every pass."""
    from raft_b200.inpaint import inpaint_rows
    from raft_b200.motionseg import segment_rows
    from raft_b200.video import _Window, interp_schedule
    due = _due(F, T, window, segment)
    table = segment_rows(F, window) if segment else inpaint_rows(F, window)
    win = _Window(F, window, T, "cpu")
    assert win.cap == min(F, 2 * window + T + 2)
    finished = []
    for j, ps in enumerate(interp_schedule(F, T)):
        n, first = sum(k is not None for k in ps.pairs), ps.frames[0]
        s = win.alloc(frames=((), torch.int64), pairs=((), torch.int64))
        new = win.admit(first + n)
        r = win.row(first)
        assert new.stop == r + n + 1 and 0 <= new.start - r <= 1
        s["frames"][new] = torch.arange(first + new.start - r, first + n + 1)
        s["pairs"][r:r + n] = torch.arange(first, first + n)
        frames, pairs = win.kept("frames").tolist(), win.kept_pairs("pairs").tolist()
        assert len(frames) <= win.cap
        assert frames == list(range(frames[0], frames[0] + len(frames))) and pairs == frames[:-1]
        ran = first + n
        t0, m, rows = win.finish((F - 1 if ran == F - 1 else ran - 1) if segment else ran, table)
        assert list(range(t0, t0 + m)) == [t for t in range(F) if due[t] == j], (j, t0, m)
        assert rows.shape == (m, 3) and np.array_equal(rows[:, 1:], table[t0:t0 + m, 1:])
        for t, (row, nf, nb) in zip(range(t0, t0 + m), rows.tolist()):
            assert 0 <= row - nb and row + nf < len(frames), (t, row, nf, nb, len(frames))
            assert frames[row - nb:row + nf + 1] == list(range(t - nb, t + nf + 1))
            assert pairs[row - nb:row + nf] == list(range(t - nb, t + nf))
        finished += range(t0, t0 + m)
    assert finished == list(range(F))


@pytest.mark.parametrize("window", range(1, 17))
@pytest.mark.parametrize("segment", [False, True])
def test_window_keeps_what_each_frame_reaches(window, segment):
    for F in range(2, 41):
        for T in range(1, 10):
            _sweep(F, T, window, segment)


def test_window_zero_segments_each_frame_alone():
    for F in range(2, 41):
        for T in range(1, 10):
            _sweep(F, T, 0, True)


def test_window_refuses_frames_that_do_not_fit():
    from raft_b200.video import _Window
    win = _Window(10, 1, 1, "cpu")
    win.alloc(frames=((), torch.int64))
    with pytest.raises(RuntimeError, match="do not fit"):
        win.admit(9)


def test_upload_scores_the_device_copy(monkeypatch):
    import networks.utils
    from raft_b200.video import _Upload, pass_cuts
    rng = np.random.default_rng(0)
    scores = np.array([0.1, 0.7, 0.5, 0.9], np.float32)
    seen = []

    def scene_cut_scores(frames):
        seen.append(frames)
        return torch.from_numpy(scores[:len(frames) - 1])
    monkeypatch.setattr(networks.utils, "scene_cut_scores", scene_cut_scores)
    up = _Upload("cpu")
    src = torch.from_numpy(rng.integers(0, 256, (5, 3, 4, 3), dtype=np.uint8))
    for pairs, thr in (([0, 1, 2, 3], 0.5), ([4, 5, None, None], 0.05), ([8, 9, 10, 11], 1.0)):
        rows, cuts = up(src, pairs, thr)
        assert torch.equal(rows, src) and seen[-1] is rows and rows.data_ptr() == up.buf.data_ptr()
        assert cuts == pass_cuts(pairs, scores, thr)
    assert len(seen) == 3
    rows, cuts = up(src[:2], [12])  # a shorter pass, not scored: the buffer's first rows
    assert cuts == [] and len(seen) == 3 and torch.equal(rows, src[:2]) and rows.data_ptr() == up.buf.data_ptr()


@pytest.mark.parametrize("rgb", [False, True])
def test_frame_writer_writes_bgr_and_tallies(tmp_path, rgb):
    import cv2
    from raft_b200.video import _FrameWriter
    rng = np.random.default_rng(1)
    frames = rng.integers(0, 256, (3, 5, 6, 3), dtype=np.uint8)
    names = [str(tmp_path / f"frame_{i:06d}.png") for i in range(6)]
    write = _FrameWriter(names, rgb, lambda slot, n: int(slot.frames[:n].numpy().sum(dtype=np.int64)))
    slot = SimpleNamespace(event=SimpleNamespace(synchronize=lambda: None), frames=torch.from_numpy(frames))
    write(slot, 2, 2)
    write(None, 4, 0)
    for i, name in enumerate(names):
        img = cv2.imread(name)
        if i in (2, 3):
            want = frames[i - 2]
            assert np.array_equal(img, want[..., ::-1] if rgb else want)
        else:
            assert img is None
    assert write.total == int(frames[:2].sum(dtype=np.int64))
    with pytest.raises(OSError, match="cannot write"):
        _FrameWriter([str(tmp_path / "missing" / "f.png")], rgb)(slot, 0, 1)


def test_print_cuts(capsys):
    from raft_b200.video import print_cuts
    print_cuts([])
    print_cuts([0, 4, 9])
    assert capsys.readouterr().out == "scene cuts: 0\nscene cuts: 3 at pairs 0 4 9\n"
