"""F32 on the GPU: rb_frame_expose_items and _resized against tests/shutter_oracle.py bit for bit (padded crops, native
sizes, integer and clamped samples, rows split across calls with the carried accumulator, bgr), RaftEngine.motion_blur
against the oracle on the engine's own flows and at m = 1 against interpolate_sequence_at, and
video_interpolate(shutter=) against RAFT.motion_blur across batch, workers and a scene cut."""
import os

import numpy as np
import pytest
import torch

import interp_oracle
import shutter_oracle as SO
from test_gpu_video import _decoded, _files, _frames, frame_dir  # noqa: F401  (frame_dir: the module fixture)
from test_gpu_video_interp import _model

pytestmark = pytest.mark.gpu


def _reversed(fw, bw, items, flow_scale=1.0):
    """The oracle reversals of items (k, t): flow_t0, flow_t1 [n,H,W,2], empty0, empty1 [n,H,W] as the engine computes
    them (steps fl32(s t), fl32(s (1 - t)))."""
    f0 = [interp_oracle.reverse_flow(fw[k:k + 1], time_step=float(np.float32(flow_scale * t))) for k, t in items]
    f1 = [interp_oracle.reverse_flow(bw[k:k + 1], time_step=float(np.float32(flow_scale * (1.0 - t)))) for k, t in items]
    return (np.concatenate([f[0] for f in f0]), np.concatenate([f[0] for f in f1]),
            np.concatenate([f[1] for f in f0]), np.concatenate([f[1] for f in f1]))


def _run(samples, m, frames, fw, bw, hw=None, split=(), bgr=False, flow_scale=1.0, pad=(0, 0, 0, 0)):
    """The samples (n, i, t) of whole output frames through the C entry, cut into calls before the sample indices in
    split (a frame cut there carries its sum through acc), with the oracle's reversals as the flows.  frames: prepared
    fp32 [F,H,W,3] (padded by pad = top, bottom, left, right on the device) or raw [F,Hs,Ws,3] at hw."""
    from raft_b200 import capi
    lib, P = capi.lib, capi.ptr
    dev = "cuda:0"
    F = len(frames)
    if hw is None:
        t, b, l, r = pad
        padded = np.pad(np.asarray(frames, np.float32), ((0, 0), (t, b), (l, r), (0, 0)), mode="edge")
        dframes = torch.from_numpy(padded).to(dev)
        size = frames.shape[1:3]
    else:
        dframes = torch.from_numpy(np.ascontiguousarray(frames)).to(dev)
        size = hw
    H, W = fw.shape[1:3]
    ns = sorted({n for n, _, _ in samples})
    first = {n: min(g for g, s in enumerate(samples) if s[0] == n) for n in ns}
    last = {n: max(g for g, s in enumerate(samples) if s[0] == n) for n in ns}
    out = torch.full((len(ns),) + tuple(size) + (3,), 7, dtype=torch.uint8, device=dev)
    acc = torch.full((2,) + tuple(size) + (3,), float("nan"), dtype=torch.float32, device=dev)
    cuts = sorted({c for c in split if 0 < c < len(samples)} | set(range(0, len(samples), 64)) | {len(samples)})
    slot = 0
    for c0, c1 in zip(cuts, cuts[1:]):
        part = samples[c0:c1]
        items = [(i, t) for _, i, t in part if t is not None]
        ent, spans, k = [], [], 0
        for e, (n, i, t) in enumerate(part):
            ent.append(capi.ExposeEntry(-1, i, 0.0) if t is None else capi.ExposeEntry(k, i, t))
            k += t is not None
            if spans and spans[-1][0] == n:
                spans[-1][2] += 1
            else:
                spans.append([n, e, 1])
        rows, carry = [], slot
        for r, (n, e, count) in enumerate(spans):
            opened, closed = first[n] == c0 + e, last[n] == c0 + e + count - 1
            a = slot
            if not closed and not (not opened and r == 0):
                a = carry = 1 - slot
            rows.append(capi.ExposeRow(e, count, m, a, ns.index(n), opened * 1 | closed * 2))
        slot = carry
        E = (capi.ExposeEntry * len(ent))(*ent)
        R = (capi.ExposeRow * len(rows))(*rows)
        if items:
            f0, f1, e0, e1 = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in _reversed(fw, bw, items,
                                                                                                  flow_scale))
            flows = (P(f0), P(f1), P(e0), P(e1))
        else:
            flows = (None,) * 4
        tail = (len(items), E, len(ent), R, len(rows), P(acc), 2, P(out), len(ns), int(bgr), F - 1)
        if hw is None:
            rc = lib.rb_frame_expose_items(P(dframes), size[0] + pad[0] + pad[1], size[1] + pad[2] + pad[3], pad[0],
                                           pad[2], *flows, *tail, H, W, capi.stream())
        else:
            rc = lib.rb_frame_expose_items_resized(P(dframes), int(frames.dtype == np.uint8), hw[0], hw[1], *flows, H,
                                                   W, *tail, capi.stream())
        capi.check(rc)
    return out.cpu().numpy()


def _clip(F, H, W, seed):
    rng = np.random.default_rng(seed)
    frames = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    fw = (rng.normal(0, 2.5, (F - 1, H, W, 2))).astype(np.float32)
    bw = (rng.normal(0, 2.5, (F - 1, H, W, 2))).astype(np.float32)
    return frames, fw, bw


@pytest.mark.parametrize("fin,fout,A,D,cuts,split,bgr,pad,scale", [
    (60, 24, 180, 4, (), (), False, (0, 0, 0, 0), 1.0),
    (60, 24, 360, 8, (), (3, 11, 12, 30), True, (3, 2, 1, 4), 1.0),
    (24, 60, 300, 16, (), (5, 9), False, (0, 3, 0, 5), 8.0),
    (30, 30, 315, 8, (2,), (4, 20), True, (1, 1, 2, 2), 1.0)])
def test_expose_items_equals_oracle(cuda, fin, fout, A, D, cuts, split, bgr, pad, scale):
    from raft_b200.video import exposure, shutter_schedule
    frames, fw, bw = _clip(6, 21, 35, 100 + D)
    if scale != 1.0:
        fw, bw = fw / np.float32(scale), bw / np.float32(scale)
    (ps,) = shutter_schedule(6, fin, fout, A, D, 5, cuts)
    m = exposure(fin, fout, A, D)[1]
    prepared = (frames.astype(np.float32) / np.float32(255)).astype(np.float32)
    got = _run(ps.samples, m, prepared, fw, bw, split=split, bgr=bgr, flow_scale=scale, pad=pad)
    want = SO.motion_blur(prepared, fw, bw, ps.samples, m, flow_scale=scale, bgr=bgr)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("HW,hw,u8,split,bgr", [((24, 40), (61, 99), True, (), False),
                                                ((24, 40), (24, 40), False, (7,), True),
                                                ((432, 1024), (1080, 1920), True, (2,), False)])
def test_expose_items_resized_equals_oracle(cuda, HW, hw, u8, split, bgr):
    """Shutter 270 at density 6 gives m = 5 samples over e = 3/4, blends and input frames mixed.  At the 1080-class size
    only output frame 1 runs (u = 0.7, 0.85, 1, 1.15, 1.3: four blends and frame 1), split inside its row."""
    from raft_b200.video import exposure, shutter_schedule
    big = HW[0] > 100
    rng = np.random.default_rng(7)
    F = 3 if big else 5
    frames = rng.integers(0, 256, (F,) + hw + (3,), dtype=np.uint8)
    if not u8:
        frames = frames.astype(np.float32)
    fw = rng.normal(0, 2.0, (F - 1,) + HW + (2,)).astype(np.float32)
    bw = rng.normal(0, 2.0, (F - 1,) + HW + (2,)).astype(np.float32)
    (ps,) = shutter_schedule(F, 30, 30, 270, 6, F - 1)
    samples = [s for s in ps.samples if s[0] == 1] if big else ps.samples
    m = exposure(30, 30, 270, 6)[1]
    assert m == 5 and sum(t is not None for _, _, t in samples) >= 4 and any(t is None for _, _, t in samples)
    assert all(samples[c - 1][0] == samples[c][0] for c in split)  # each split cuts a row: its sum is carried
    got = _run(samples, m, frames, fw, bw, hw=hw, split=split, bgr=bgr)
    want = SO.motion_blur(frames, fw, bw, samples, m, hw=hw, bgr=bgr)
    assert np.array_equal(got, want)


def test_expose_refusals_on_device_buffers(cuda):
    """The table checks run before any CUDA call with device buffers too."""
    from raft_b200 import capi
    buf = torch.zeros(1024, device="cuda:0")
    P = capi.ptr
    e = (capi.ExposeEntry * 1)(capi.ExposeEntry(0, 0, 0.5))
    r = (capi.ExposeRow * 1)(capi.ExposeRow(0, 1, 0, 0, 0, 3))
    assert capi.lib.rb_frame_expose_items(P(buf), 4, 4, 0, 0, P(buf), P(buf), P(buf), P(buf), 1, e, 1, r, 1, P(buf), 2,
                                          P(buf), 1, 0, 1, 4, 4, capi.stream()) == -2


@pytest.mark.parametrize("small", [False, True])
def test_motion_blur_equals_oracle_on_engine_flows(cuda, small):
    from raft_b200.video import exposure, shutter_schedule
    frames = _frames(5, 64, 96)
    m = _model(small)
    fw, bw, _, _ = m.forward_sequence_bidirectional(frames, check=False)
    s = m.engine().flow_scale
    got = m.motion_blur(frames, 180, fps=(60, 24), density=4).cpu().numpy()
    (ps,) = shutter_schedule(5, 60, 24, 180, 4, 4)
    prepared = (np.asarray(frames, np.float32) / np.float32(255)).astype(np.float32)
    want = SO.motion_blur(prepared, fw.cpu().numpy(), bw.cpu().numpy(), ps.samples, exposure(60, 24, 180, 4)[1],
                          flow_scale=s)
    assert got.shape == want.shape == (2, 64, 96, 3) and np.array_equal(got, want)


def test_m1_equals_interpolate_sequence_at(cuda):
    from raft_b200.video import fps_schedule
    frames = _frames(6, 64, 96)
    m = _model()
    got = m.motion_blur(frames, 90, fps=(24, 60), density=2)
    items = [it for p in fps_schedule(6, 24, 60, 5) for it in p.items]
    ref = m.interpolate_sequence_at(frames, [(k, t) for _, k, t in items], uint8=True)
    for r, (n, _, _) in enumerate(items):
        assert torch.equal(got[n], ref[r]), n
    copies = [c for p in fps_schedule(6, 24, 60, 5) for c in p.copies]
    assert copies and len(items) + len(copies) == got.shape[0] == 13
    for n, i in copies:  # an integer time is the input frame itself, as the conversion copies it
        assert np.array_equal(got[n].cpu().numpy(), frames[i]), n


def test_motion_blur_native(cuda):
    from raft_b200.video import exposure, shutter_schedule
    frames = _frames(4, 90, 130)
    m = _model(input_size=(64, 96))
    fw, bw, _, _ = m.forward_sequence_bidirectional(frames, check=False)
    got = m.motion_blur(frames, 360, density=3, native=True).cpu().numpy()
    (ps,) = shutter_schedule(4, 1, 1, 360, 3, 3)
    want = SO.motion_blur(np.asarray(frames), fw.cpu().numpy(), bw.cpu().numpy(), ps.samples,
                          exposure(1, 1, 360, 3)[1], hw=(90, 130))
    assert got.shape == (4, 90, 130, 3) and np.array_equal(got, want)


def test_video_shutter_matches_motion_blur(cuda, frame_dir, tmp_path):
    import cv2
    from raft_b200.video import video_interpolate
    m = _model()
    clip = torch.from_numpy(_decoded(frame_dir))
    want = m.motion_blur(clip, 270, fps=(30, 24), density=6).cpu().numpy()
    runs = {}
    for batch, workers in ((1, 1), (3, 4), (8, 1), (8, 4)):
        d = tmp_path / f"b{batch}w{workers}"
        paths = video_interpolate(m, frame_dir, d, batch=batch, workers=workers, fps=(30, 24), shutter=270, density=6)
        assert len(paths) == len(want) == (10 - 1) * 24 // 30 + 1
        runs[(batch, workers)] = _files(d)
    first = runs[(1, 1)]
    assert all(r == first for r in runs.values())
    for n in range(len(want)):
        assert np.array_equal(cv2.imread(str(tmp_path / "b1w1" / f"frame_{n:06d}.png")), want[n]), n


def test_video_shutter_scene_cut(cuda, frame_dir, tmp_path):
    import cv2
    from raft_b200.video import video_interpolate
    m = _model()
    clip = _decoded(frame_dir).copy()
    clip[5:] = 255 - clip[5:]  # a cut at pair 4
    src = tmp_path / "cut"
    src.mkdir()
    for i, f in enumerate(clip):
        cv2.imwrite(str(src / f"{i:04d}.png"), f)
    want = m.motion_blur(torch.from_numpy(clip), 360, fps=(30, 30), density=4, cuts=[4]).cpu().numpy()
    files = []
    for batch in (1, 3):
        d = tmp_path / f"o{batch}"
        paths, cuts = video_interpolate(m, str(src), d, batch=batch, workers=2, fps=(30, 30), shutter=360, density=4,
                                        scene_cut=0.5)
        assert cuts == [4]
        files.append(_files(d))
        for n in range(len(want)):
            assert np.array_equal(cv2.imread(paths[n]), want[n]), (batch, n)
    assert files[0] == files[1]


def test_down_conversion_frame_count(cuda, frame_dir, tmp_path):
    from raft_b200.video import video_interpolate
    paths = video_interpolate(_model(), frame_dir, tmp_path / "o", batch=4, fps=(60, 24), shutter=180)
    assert len(paths) == (10 - 1) * 24 // 60 + 1 and all(os.path.exists(p) for p in paths)
