"""tests/test_gpu_wide_tlas_device.py without a GPU: the cases run against the kernel sources compiled for the host (tests/emu/, as
tests/test_shared_scene_emulated.py does for the shared-scene suite), so that what kc_build_wide_tlas COMPUTES — the 4-wide TLAS,
ranks and stack verdict of wide_build.h, record for record, and frames equal to the host path's — is checked on any machine, in both
thread orders of the emulation (a result that depended on the order of the CTA's threads would differ between the two).  The test
that measures the host's wait needs a real device and is skipped here."""
import os
import shutil
import subprocess
import sys

import pytest

from tests.conftest import ROOT


@pytest.mark.parametrize("reverse,select", [(False, None), (True, "soups or animation")])
def test_wide_tlas_suite_passes_on_emulated_kernels(reverse, select):
    if not shutil.which("g++") and not os.path.exists("/usr/bin/g++"):
        pytest.skip("no host C++ compiler")
    env = dict(os.environ, HK_EMULATE_KERNELS="1")
    if reverse:
        env["HK_EMU_REVERSE"] = "1"
    cmd = [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "tests/test_gpu_wide_tlas_device.py"]
    if select:
        cmd += ["-k", select]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail
