"""tests/test_gpu_mesh_build.py without a GPU: the cases run against the kernel sources compiled for the host (tests/emu/, as
tests/test_scene_update_edges_emulated.py does for the device scene rebuild), so that what hk_scene_add_meshes COMPUTES — the vertex
and primitive records and every mesh's BLAS, top levels split by a whole CTA and subtrees finished from the work list — is checked on
any machine, in both thread orders of the emulation.  Rendering frames on the emulation is slow, so the frame comparisons and all but
one refusal run on the device only, with the million-triangle mesh and the town and house meshes.  The meshes above 4096 primitives
(soup_5000, flat_large) have just over 4096 here (tests/test_gpu_mesh_build.py LARGE_SOUP / LARGE_GRID): both passes take 3.5 min on
8 cores, against 19.5 min with the device's 5000 and 45 000 triangles."""
import os
import shutil
import subprocess
import sys

import pytest

from tests.conftest import ROOT


SELECT = "not million and not town and not house and not frames and not queued and (not malformed or short_chunk)"


@pytest.mark.parametrize("reverse,select", [(False, SELECT), (True, SELECT + " and not soup_5000 and not flat_large")])
def test_mesh_build_passes_on_emulated_kernels(reverse, select):
    if not shutil.which("g++") and not os.path.exists("/usr/bin/g++"):
        pytest.skip("no host C++ compiler")
    env = dict(os.environ, HK_EMULATE_KERNELS="1")
    if reverse:
        env["HK_EMU_REVERSE"] = "1"
    cmd = [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", "tests/test_gpu_mesh_build.py", "-k", select]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and " failed" not in tail, tail
