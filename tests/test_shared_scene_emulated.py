"""tests/test_gpu_shared_scene.py without a GPU: the shared-scene cases run against the kernel sources compiled for the host
(tests/emu/, as tests/test_emulated_kernels.py does for the parity suite), so that what a shared scene COMPUTES — one upload and
one update per frame feeding every attached camera, private and shared arms bit-equal, attach / detach / destroy — is checked on
any machine.  The emulation runs every launch synchronously and its CUDA events are no-ops, so the stream ordering between the
scene's stream and the cameras' streams is checked only by the device run of that file."""
import os
import shutil
import subprocess
import sys

import pytest

from tests.conftest import ROOT


def test_shared_scene_suite_passes_on_emulated_kernels():
    if not shutil.which("g++") and not os.path.exists("/usr/bin/g++"):
        pytest.skip("no host C++ compiler")
    env = dict(os.environ, HK_EMULATE_KERNELS="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "tests/test_gpu_shared_scene.py"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail
