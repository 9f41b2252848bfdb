"""F3 resize on the GPU.

rb_frames_resize and rb_flow_resize must equal the reference's cv2.resize / resize_flow (tests/golden/resize.npz) and the
numpy restatements (tests/resize_oracle.py) bit for bit, at B = 3 with NaN/+-inf flows, batched as per sample and
graph-captured as eager.  An engine with input_size must compute from native frames exactly what it computes from frames
resized on the host, in every mode, and keep doing so when modes and source sizes alternate.  The CLI must write the
same bytes as the host-resize path it replaced."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import resize_oracle as O

pytestmark = pytest.mark.gpu

CASES = O.golden_cases()


def _same(a, b):
    a, b = np.ascontiguousarray(O.canonical_nan(a)), np.ascontiguousarray(O.canonical_nan(b))
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _golden_batch(mk, kind, case, H, W):
    """B = 3: sample 0 is the golden input, the others differ from it."""
    if kind == "flow":
        f = mk.flow_f32(H, W, bool(case))
        return np.stack([f, f * np.float32(2), -f[::-1].copy()])
    if kind == "u8":
        return mk.frames_u8(3, H, W)
    return mk.frames_f32(3, H, W)


@pytest.mark.parametrize("kind,case,H,W,Ho,Wo", CASES, ids=lambda v: str(v))
def test_kernels_equal_reference_and_restatement(cuda, kind, case, H, W, Ho, Wo):
    from networks.utils import resize_flow, resize_frames
    g, mk = np.load(O.GOLDEN), O.golden_maker()
    x = _golden_batch(mk, kind, case, H, W)
    key = O.golden_key(kind, case, H, W, Ho, Wo)
    t = torch.from_numpy(x).to(cuda)
    if kind == "flow":
        got = resize_flow(t, (Ho, Wo)).cpu().numpy()
        assert O.equals_golden(g, key, got[0])
        assert _same(got, O.resize_flow(x, Ho, Wo))
    else:
        got = resize_frames(t, (Ho, Wo)).cpu().numpy()
        ref0 = O.resize_u8(x[0], Ho, Wo) if kind == "u8" else O.resize_f32(x[0], Ho, Wo)
        assert O.equals_golden(g, key, ref0)
        if kind == "u8":
            ref0 = (ref0.astype(np.float32) / np.float32(255)).astype(np.float32)
        assert _same(got[0], ref0)
        assert _same(got, O.frames_resize(x, Ho, Wo))


def test_flow_utils_mirror_equals_reference(cuda):
    import flow_utils
    g, mk = np.load(O.GOLDEN), O.golden_maker()
    for kind, case, H, W, Ho, Wo in CASES:
        if kind == "flow":
            out = flow_utils.resize_flow(mk.flow_f32(H, W, bool(case)), Wo, Ho)
            assert out.dtype == np.float32 and O.equals_golden(g, O.golden_key(kind, case, H, W, Ho, Wo), out), (H, W)
    with pytest.raises(TypeError):
        flow_utils.resize_flow(np.zeros((4, 4, 2)), 8, 8)
    with pytest.raises(ValueError):
        flow_utils.resize_flow(np.zeros((4, 4, 3), np.float32), 8, 8)


@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("H,W,Ho,Wo,pad", [(37, 53, 45, 61, (1, 2, 3, 0)), (436, 1024, 436, 1024, (0, 0, 0, 0)),
                                           (1080, 1920, 436, 1020, (0, 0, 2, 2)), (1, 7, 60, 100, (2, 2, 2, 2))])
def test_padded_output(cuda, u8, H, W, Ho, Wo, pad):
    from networks.utils import resize_frames
    rng = np.random.default_rng(H + W)
    x = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8) if u8 else rng.random((3, H, W, 3), dtype=np.float32)
    got = resize_frames(torch.from_numpy(x).to(cuda), (Ho, Wo), pad).cpu().numpy()
    assert _same(got, O.frames_resize(x, Ho, Wo, pad))


def test_random_shapes_equal_restatement(cuda):
    from networks.utils import resize_flow, resize_frames
    rng = np.random.default_rng(12)
    for _ in range(40):
        H, W, Ho, Wo = (int(v) for v in rng.integers(1, 90, 4))
        u = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
        f = rng.random((2, H, W, 3), dtype=np.float32)
        fl = rng.normal(0, 20, (2, H, W, 2)).astype(np.float32)
        for v in (np.nan, np.inf, -np.inf):
            fl.reshape(-1)[rng.integers(0, fl.size, max(1, fl.size // 20))] = v
        for x in (u, f):
            assert _same(resize_frames(torch.from_numpy(x).to(cuda), (Ho, Wo)).cpu().numpy(), O.frames_resize(x, Ho, Wo))
        assert _same(resize_flow(torch.from_numpy(fl).to(cuda), (Ho, Wo)).cpu().numpy(), O.resize_flow(fl, Ho, Wo))


def test_batched_equals_per_sample_and_graph_equals_eager(cuda):
    from networks.utils import resize_flow, resize_frames
    rng = np.random.default_rng(2)
    u = torch.from_numpy(rng.integers(0, 256, (3, 375, 1242, 3), dtype=np.uint8)).to(cuda)
    fl = torch.from_numpy(rng.normal(0, 9, (3, 432, 1024, 2)).astype(np.float32)).to(cuda)
    a, b = resize_frames(u, (432, 1024), (2, 2, 0, 0)), resize_flow(fl, (375, 1242))
    for i in range(3):
        assert torch.equal(resize_frames(u[i:i + 1], (432, 1024), (2, 2, 0, 0)), a[i:i + 1])
        assert torch.equal(resize_flow(fl[i:i + 1], (375, 1242)), b[i:i + 1])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ga, gb = resize_frames(u, (432, 1024), (2, 2, 0, 0)), resize_flow(fl, (375, 1242))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(ga, a) and torch.equal(gb, b)


# ---- the engine with input_size ---------------------------------------------------------------------------------
def _model(p, small, B, cuda, input_size=None, shape=None):
    from networks.RAFT import RAFT
    shape = shape or (input_size + (3,))
    return RAFT(shape, SimpleNamespace(small=small), iters=4, batch=B, device=cuda, input_size=input_size).load(p)


def _native(B, H, W, u8, seed0=100):
    from raft_b200 import synth
    l, r = synth.make_batch(B, H, W, seed0=seed0)
    if u8:
        l, r = (np.round(l * 255).astype(np.uint8), np.round(r * 255).astype(np.uint8))
    return l, r


def _host_resized(frames, size):
    """What the reference's dataflow (and this CLI before) did on the host: cv2.resize per frame."""
    import cv2
    return np.stack([cv2.resize(f, dsize=(size[1], size[0])) for f in frames])


SOURCES = [(436, 1024), (1080, 1920), (375, 1242), (60, 100)]


@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("size", [(432, 1024), (436, 1024)])
def test_forward_equals_host_resize(cuda, small, size):
    from raft_b200 import synth
    p = synth.make_weights(small)
    B = 2
    m = _model(p, small, B, cuda, input_size=size)
    ref = _model(p, small, B, cuda, shape=size + (3,))
    for H, W in SOURCES:
        for u8 in (True, False):
            l, r = _native(B, H, W, u8)
            got = m.forward(l, r)
            want = ref.forward(_host_resized(l, size), _host_resized(r, size))
            assert got.shape == (B,) + size + (2,) and torch.equal(got, want), (H, W, u8)


@pytest.mark.parametrize("small", [False, True])
def test_bidirectional_and_interpolate_equal_host_resize(cuda, small):
    from raft_b200 import synth
    p = synth.make_weights(small)
    B, size = 1, (432, 1024)
    m = _model(p, small, B, cuda, input_size=size)
    ref = _model(p, small, B, cuda, shape=size + (3,))
    for (H, W), u8 in (((1080, 1920), True), ((375, 1242), False), ((60, 100), True)):
        l, r = _native(B, H, W, u8, seed0=200)
        hl, hr = _host_resized(l, size), _host_resized(r, size)
        got, want = m.forward_bidirectional(l, r), ref.forward_bidirectional(hl, hr)
        for a, b in zip(got, want):
            assert a.shape[1:3] == size and torch.equal(a, b), (H, W, u8)
        got, want = m.interpolate(l, r, [0.0, 0.4, 1.0]), ref.interpolate(hl, hr, [0.0, 0.4, 1.0])
        assert got.shape == (3, B) + size + (3,) and torch.equal(got, want), (H, W, u8)


def test_alternating_modes_and_source_sizes(cuda):
    """One engine, modes and source sizes (and dtypes) alternating: every call equals a fresh model."""
    from raft_b200 import synth
    small, B, size = False, 1, (96, 136)
    p = synth.make_weights(small)
    calls = [("f", (120, 200), True), ("b", (120, 200), True), ("f", (60, 100), True), ("i", (60, 100), False),
             ("f", (120, 200), True), ("b", (96, 136), False), ("i", (20, 30), True), ("f", (20, 30), True)]

    def call(m, kind, lr):
        if kind == "f":
            return (m.forward(*lr),)
        if kind == "b":
            return m.forward_bidirectional(*lr)
        return (m.interpolate(*lr, [0.5]),)

    one = _model(p, small, B, cuda, input_size=size)
    for k, (kind, (H, W), u8) in enumerate(calls):
        lr = _native(B, H, W, u8, seed0=300 + 10 * k)
        got = call(one, kind, lr)
        want = call(_model(p, small, B, cuda, input_size=size), kind, lr)
        for g, w in zip(got, want):
            assert torch.equal(g, w), (kind, H, W)


def test_input_size_is_checked(cuda):
    from raft_b200 import synth
    from raft_b200.engine import MIN_FRAME, RaftEngine
    p = synth.make_weights(True)
    with pytest.raises(ValueError):
        RaftEngine(p, small=True, input_size=(MIN_FRAME - 1, 100))
    RaftEngine(p, small=True, input_size=(MIN_FRAME, MIN_FRAME))


def _write_pngs(tmp_path, H, W):
    import cv2
    from raft_b200 import synth
    l, r = synth.make_batch(1, H, W, seed0=500)
    for name, img in (("a.png", l[0]), ("b.png", r[0])):
        cv2.imwrite(str(tmp_path / name), (img * 255).astype(np.uint8))


@pytest.mark.parametrize("H,W", [(436, 1024), (375, 1242)])
def test_cli_writes_the_host_resize_bytes(cuda, tmp_path, monkeypatch, H, W):
    """The CLI resizes on the GPU now; every file must be the one the host-resize path wrote (computed here the way the
    CLI used to: read_pair at 432x1024, a model of that size, the same writers)."""
    import cv2
    import infer_raft
    from flow_utils import flow_to_color, resize_flow, write_flo
    from raft_b200 import synth
    _write_pngs(tmp_path, H, W)
    p = synth.make_weights(False)
    np.savez(tmp_path / "w.npz", **p)
    monkeypatch.chdir(tmp_path)
    base = ["--im1", "a.png", "--im2", "b.png", "--load", "w.npz", "--iters", "3"]
    assert infer_raft.main(base + ["--bidirectional", "--npy", "f.npy", "--flo", "f.flo", "--interpolate", "0.5"]) == 0
    names = ["raft_flow_raft-things.png", "raft_flow_raft-things_bw.png", "raft_occ_fw.png", "raft_occ_bw.png",
             "f.npy", "f_bw.npy", "f.flo", "f_bw.flo", "raft_interp_0.png"]
    got = {n: open(n, "rb").read() for n in names}
    # the host-resize path
    os.makedirs("host")
    left, right = infer_raft.read_pair("a.png", "b.png", (432, 1024))
    m = _model(p, False, 1, cuda, shape=left.shape[1:])
    m.iters = 3
    fw, bw, ofw, obw = (t.cpu().numpy() for t in m.forward_bidirectional(left, right))
    cv2.imwrite("host/raft_flow_raft-things.png", flow_to_color(fw[0], convert_to_bgr=True))
    cv2.imwrite("host/raft_flow_raft-things_bw.png", flow_to_color(bw[0], convert_to_bgr=True))
    grey = np.array([0, 128, 255], dtype=np.uint8)
    cv2.imwrite("host/raft_occ_fw.png", grey[ofw[0]])
    cv2.imwrite("host/raft_occ_bw.png", grey[obw[0]])
    np.save("host/f.npy", fw[0])
    np.save("host/f_bw.npy", bw[0])
    write_flo("host/f.flo", fw[0])
    write_flo("host/f_bw.flo", bw[0])
    frame = m.interpolate(left, right, [0.5]).cpu().numpy()[0, 0]
    cv2.imwrite("host/raft_interp_0.png", np.clip(np.rint(255.0 * frame), 0, 255).astype(np.uint8))
    for n in names:
        assert got[n] == open(os.path.join("host", n), "rb").read(), n
    # --native-flow: the flow(s) at im1's size, equal to the reference's resize_flow of the 432x1024 flow
    assert infer_raft.main(base + ["--bidirectional", "--native-flow", "--npy", "n.npy", "--flo", "n.flo"]) == 0
    for suffix, f in (("", fw[0]), ("_bw", bw[0])):
        want = resize_flow(f, W, H)
        assert want.shape == (H, W, 2)
        assert np.load(f"n{suffix}.npy").tobytes() == want.tobytes()
        write_flo(f"host/n{suffix}.flo", want)
        assert open(f"n{suffix}.flo", "rb").read() == open(f"host/n{suffix}.flo", "rb").read()
    png = cv2.imread("raft_flow_raft-things.png")
    assert png.shape == (H, W, 3) and np.array_equal(png, flow_to_color(resize_flow(fw[0], W, H), convert_to_bgr=True))
    # --keep-size ignores --native-flow
    assert infer_raft.main(base + ["--keep-size", "--native-flow", "--npy", "k.npy"]) == 0
    assert np.load("k.npy").shape == (H, W, 2)


def test_cli_frames_of_two_sizes(cuda, tmp_path, monkeypatch):
    """im1 and im2 of different sizes were both resized to 432x1024 on the host; they still are, with the same bytes."""
    import cv2
    import infer_raft
    from raft_b200 import synth
    l, _ = synth.make_batch(1, 436, 1024, seed0=600)
    _, r = synth.make_batch(1, 375, 1242, seed0=700)
    cv2.imwrite(str(tmp_path / "a.png"), (l[0] * 255).astype(np.uint8))
    cv2.imwrite(str(tmp_path / "b.png"), (r[0] * 255).astype(np.uint8))
    p = synth.make_weights(True)
    np.savez(tmp_path / "w.npz", **p)
    monkeypatch.chdir(tmp_path)
    base = ["--im1", "a.png", "--im2", "b.png", "--load", "w.npz", "--iters", "3", "--small"]
    assert infer_raft.main(base + ["--native-flow", "--npy", "n.npy"]) == 0
    left, right = infer_raft.read_pair("a.png", "b.png", (432, 1024))
    m = _model(p, True, 1, cuda, shape=left.shape[1:])
    m.iters = 3
    want = m.forward(left, right).cpu().numpy()[0]
    from flow_utils import resize_flow
    assert np.load("n.npy").tobytes() == resize_flow(want, 1024, 436).tobytes()
    assert infer_raft.main(base + ["--npy", "f.npy"]) == 0
    assert np.load("f.npy").tobytes() == want.tobytes()
