"""tests/test_gpu_scene_update_edges.py without a GPU: the cases run against the kernel sources compiled for the host (tests/emu/, as
tests/test_wide_tlas_device_emulated.py does for the 4-wide TLAS suite), so that what the scene kernels COMPUTE at the edges of their
input — singular, mirrored, sheared and far transforms, emissive meshes at the chunk boundaries, the deepest chains, the cache rule,
refused non-finite models — is checked on any machine, in both thread orders of the emulation.  The selection keeps the CPU suite's
cost to about 35 s: the large soups, the 2000-emissive soup, the n = 257 families and the frames of the non-singular families run
on the device only.  The emulation runs on the host's floating point, so a NaN the device would write differently from x86 (the inverse of a zero-scaled
model) is checked only by the device run of that file."""
import os
import shutil
import subprocess
import sys

import pytest

from tests.conftest import ROOT


# 35 s on 8 cores for both passes: the zero-scale, refusal, cache-rule and chain cases, and every family at n = 33
SELECT = "(families and 33) or (render_as_the_oracle and zero) or (chunk and not 2000) or chains or cache or non_finite"


@pytest.mark.parametrize("reverse,select", [(False, SELECT), (True, "(families and 33) or cache or non_finite")])
def test_scene_update_edges_pass_on_emulated_kernels(reverse, select):
    if not shutil.which("g++") and not os.path.exists("/usr/bin/g++"):
        pytest.skip("no host C++ compiler")
    env = dict(os.environ, HK_EMULATE_KERNELS="1")
    if reverse:
        env["HK_EMU_REVERSE"] = "1"
    cmd = [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "tests/test_gpu_scene_update_edges.py"]
    if select:
        cmd += ["-k", select]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and " failed" not in tail, tail
