"""Kernel logic without a GPU.  tests/emu/ compiles the CUDA kernel sources (bevy_hikari_b200/csrc/*.cu) for the host through
a small shim of the CUDA constructs they use, behind the same C ABI, and this test runs the `-m gpu` parity tests against
that build: every plane of every frame must equal the oracle bit for bit there too.  It checks what the kernels COMPUTE
(indexing, pass wiring, scatter resolve, tiling, upscalers, instance updates); how they run on an H100 is what `-m gpu` on the
device checks.  The emulated build is test infrastructure: the package never loads it (tests/conftest.py swaps the library
path only when HK_EMULATE_KERNELS is set)."""
import os
import shutil
import subprocess
import sys

import pytest

from tests.conftest import ROOT

FILES = ["tests/test_gpu_parity.py", "tests/test_gpu_variants.py", "tests/test_gpu_upscale.py", "tests/test_gpu_dynamic.py",
         "tests/test_gpu_frame_assembly.py", "tests/test_gpu_zz_fsr.py", "tests/test_gpu_zz_examples.py", "tests/test_gpu_zz_halo.py",
         "tests/test_gpu_wide_traversal.py", "tests/test_gpu_wide_foreign_bvh.py", "tests/test_gpu_scene_update.py",
         "tests/test_gpu_wgsl_golden.py", "tests/test_gpu_zzz_wgsl_late_cases.py", "tests/test_gpu_zzz_late_regressions.py"]
# the reverse order runs single-threaded: the files whose kernels have something an order could change (scatter claims / resolve,
# cooperative tiles and pools, the level-synchronous BVH build, halo copies), not the long fixture sequences once more
REVERSE_FILES = ["tests/test_gpu_parity.py", "tests/test_gpu_upscale.py", "tests/test_gpu_dynamic.py", "tests/test_gpu_zz_halo.py",
                 "tests/test_gpu_scene_update.py"]


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_gpu_parity_suite_passes_on_emulated_kernels(order):
    """reverse: every launch runs its blocks and threads in descending order on one host thread — results must not depend
    on the order in which the threads of a launch run"""
    if not shutil.which("g++") and not os.path.exists("/usr/bin/g++"):
        pytest.skip("no host C++ compiler")
    env = dict(os.environ, HK_EMULATE_KERNELS="1")
    if order == "reverse":
        env["HK_EMU_REVERSE"] = "1"
    files = REVERSE_FILES if order == "reverse" else FILES
    extra = []
    if order == "reverse":      # one host thread per launch: spread the tests over processes instead (pytest-xdist, when installed)
        try:
            import xdist  # noqa: F401
            extra = ["-n", str(min(4, os.cpu_count() or 1))]
        except ImportError:
            pass
    r = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + extra + files, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail


@pytest.mark.parametrize("mode,first,count", [("frames", 5000, 40), ("tiles", 7000, 15), ("halo", 9000, 12), ("soup", 11000, 30)])
def test_randomised_parity_campaign_on_emulated_kernels(mode, first, count):
    """tools/fuzz_parity.py with fixed seeds: random scene, size (down to 1 x 1), settings, upscale ratio, camera motion and
    instance animation (frames); random tile partitions against the unsharded frame (tiles)."""
    if not os.path.exists("/usr/bin/g++") and not shutil.which("g++"):
        pytest.skip("no host C++ compiler")
    env = dict(os.environ, HK_EMULATE_KERNELS="1")
    if mode == "tiles":
        env["HK_FUZZ_TILES"] = "1"
    if mode == "soup":      # random triangle soups: degenerate triangles, mirrored / non-uniform instances, several lights
        env["HK_FUZZ_SOUP"] = "1"
    if mode == "halo":      # random partitions, moving camera, motion margin + hk_halo_pull after every frame
        env["HK_FUZZ_HALO"] = "1"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "fuzz_parity.py"), str(first), str(count)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
