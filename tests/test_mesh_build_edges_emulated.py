"""tests/test_gpu_mesh_build_edges.py without a GPU: the cases run against the kernel sources compiled for the host (tests/emu/, as
tests/test_mesh_build_emulated.py does for tests/test_gpu_mesh_build.py), so that the CTA-level branches of kc_build_blas_top and the
work-list loop of kc_build_blas_bottom are checked on any machine, in both thread orders of the emulation.  Each branch is reached
with the smallest mesh that gets there (4097-4168 triangles; the fibers take about 5 ms per primitive):
  A. outliers_4097_4: CTA children of one shape, put on the work list as leaves, and more work-list entries than the bottom kernel
     has CTAs, so its claim loop goes round;
  B. copies_4097: the halves at CTA level, on an odd count;
  C. no_finite_candidate_4097: a CTA split without a finite SAH candidate, whose children enter the work list with the empty box;
  D. signed_zero[32-minus_first]: the first zero of a CTA-level node's bound in warp 1, carried across warps by the reduction.
The reverse pass runs all four, the forward pass B.  Both passes take 130 s together on 8 cores, the emulator build aside.
E's 3000-mesh call and F's frames run on the device only."""
import os
import shutil
import subprocess
import sys

import pytest

from tests.conftest import ROOT


CTA_EDGES = "outliers_4097 or copies_4097 or no_finite_candidate_4097 or (signed_zero and 32 and minus)"


@pytest.mark.parametrize("reverse,select", [(False, "copies_4097"), (True, CTA_EDGES)])
def test_mesh_build_edges_pass_on_emulated_kernels(reverse, select):
    if not shutil.which("g++") and not os.path.exists("/usr/bin/g++"):
        pytest.skip("no host C++ compiler")
    env = dict(os.environ, HK_EMULATE_KERNELS="1")
    if reverse:
        env["HK_EMU_REVERSE"] = "1"
    cmd = [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "tests/test_gpu_mesh_build_edges.py", "-k", select]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and " failed" not in tail, tail
