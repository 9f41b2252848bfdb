"""F33 on the GPU: the GoPro protocol on a synth.write_highfps_tree tree -- its blurred frames are RAFT.motion_blur's
on each sequence's inputs, and its scores are vfi_oracle's PSNR / SSIM of those frames and of the sharp inputs against
np.rint of the true windows' mean."""
import numpy as np
import pytest
import torch

from test_gpu_video_interp import _model
from vfi_oracle import frame_stats, psnr

pytestmark = pytest.mark.gpu


def test_gopro_protocol_on_a_synthetic_tree(cuda, tmp_path):
    from raft_b200 import synth
    from raft_b200.gopro import evaluate, ground_truth, protocol, summary_line
    S, M = 8, 7
    written = synth.write_highfps_tree(str(tmp_path), "test", [("a", 41), ("b", 35)], 64, 96, speed=(1, 1))
    m = _model()
    res = evaluate(m, str(tmp_path), "test", S, M, batch=3)
    assert [r["scored"] for r in res["sequences"]] == [4, 3] and res["frames"] == 7
    A, D = protocol(S, M)
    for rec, (name, hi) in zip(res["sequences"], sorted(written.items())):
        inputs = hi[::S]
        blurred = m.motion_blur(torch.from_numpy(inputs), A, density=D).cpu().numpy()
        for fr in rec["per_frame"]:
            c = fr["input"]
            gt = ground_truth(hi[S * c - 3:S * c + 4])
            blur, sharp = frame_stats(blurred[c][None], gt[None])[0], frame_stats(inputs[c][None], gt[None])[0]
            assert fr["psnr"] == pytest.approx(psnr(blur[0], gt.size), rel=1e-12)
            assert fr["sharp_psnr"] == pytest.approx(psnr(sharp[0], gt.size), rel=1e-12)
            assert fr["ssim"] == pytest.approx(blur[1], abs=1e-6) and fr["sharp_ssim"] == pytest.approx(sharp[1], abs=1e-6)
    assert summary_line(res).startswith("Validation GoPro motion blur (test, stride 8, 7 frames): PSNR: ")
    assert np.isfinite(res["psnr"]) and np.isfinite(res["sharp_psnr"])
