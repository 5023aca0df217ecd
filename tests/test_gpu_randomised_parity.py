"""The randomised parity campaign of tools/fuzz_parity.py on the H100 (exact flavour), not only on the emulated kernels.

The emulator runs the kernel logic on the host; here the same random scenes, triangle soups (degenerate triangles, mirrored and
non-uniform instances), sizes down to 1 x 1, settings, upscale ratios, camera and instance motion, tile partitions and halo pulls
meet real atomics, TMA out-of-bounds fill, warp collectives and the device's arithmetic.  Each case also draws the bit-exact
implementation switches of hk_set_tuning.  The seed ranges do not overlap those of
tests/test_emulated_kernels.py::test_randomised_parity_campaign_on_emulated_kernels."""
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode,first,count", [("frames", 105000, 60), ("soup", 111000, 40), ("tiles", 107000, 20), ("halo", 109000, 20)])
def test_randomised_parity_campaign_on_the_device(monkeypatch, mode, first, count):
    from tests.conftest import needs_real_gpu
    needs_real_gpu()        # the emulated kernels run their own fixed-seed batches (tests/test_emulated_kernels.py)
    for var in ("HK_FUZZ_SOUP", "HK_FUZZ_TILES", "HK_FUZZ_HALO"):
        monkeypatch.delenv(var, raising=False)
    if mode != "frames":
        monkeypatch.setenv({"soup": "HK_FUZZ_SOUP", "tiles": "HK_FUZZ_TILES", "halo": "HK_FUZZ_HALO"}[mode], "1")
    monkeypatch.syspath_prepend(os.path.join(ROOT, "tools"))
    import fuzz_parity
    case = fuzz_parity.one_case if mode in ("frames", "soup") else fuzz_parity.tile_case
    failures = []
    for seed in range(first, first + count):
        try:
            msg = case(seed)
        except Exception as e:      # API errors are findings too
            msg = f"seed {seed}: exception {e!r}"
        if msg:
            failures.append(msg)
    assert not failures, "\n".join(failures[:10])
