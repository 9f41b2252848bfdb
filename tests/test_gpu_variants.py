"""Environment knobs that change how kernels are launched (read once per process) must keep results correct: the conv /
update-block / encoder parity tests are re-run in a subprocess with each knob set."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _kernel_parity(env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_kernels.py"), "-q", "-x",
                        "-k", "(conv2d or update_block or encoder) and tc", "--timeout", "300", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-1000:]


@pytest.mark.parametrize("knob", ["RAFT_B200_NO_PDL"])
def test_variant_passes_conv_and_update_parity(cuda, knob):
    name, _, value = knob.partition("=")
    _kernel_parity(dict(os.environ, **{name: value or "1"}))

