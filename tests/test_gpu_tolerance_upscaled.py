"""The PRODUCT library's tolerance contract (tests/test_gpu_tolerance.py) at upscale ratios above 1.

Above ratio 1 the render pixels are fewer than the G-buffer texels, and every tolerance unit maps a render pixel to the texel it reads
through the jittered uv (csrc/hk_device.cuh): k_spatial its own texel, each neighbour's and each depth-march tap's, k_demodulation and
k_denoise their nearest texel.  An off-by-one there reads another texel's normal, depth, instance and albedo: a different input, not
a rounding error, so it would show up here as outlier pixels.  The bounds are those of ratio 1:
  * every pass of a tolerance unit from identical inputs: spatial reuse within 1 f16 ulp, the denoise chain within 4, tone mapping
    within 5, fewer than 1e-4 outlier pixels in each (1.5 on 192x108: render 128x72, both axes exactly 1.5; 2 on 160x96; city at 1.7);
  * ids, G-buffer and temporal reservoirs bit-exact over a free-running sequence of the default pipeline (ratio 2, SMAA TU4x + TAA).
With HK_EMULATE_KERNELS=1 the "product" is the exact emulation and every bound is met with zero difference."""
import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin
from tests.conftest import EMULATED, Bench
from tests.test_gpu_parity import mismatch, reservoir_mismatch
from tests.test_gpu_tolerance import EXACT_PLANES, outlier_pixels, sync_state

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scene,config,size,ratio", [("cornell", "cornell_1080p", (192, 108), 1.5), ("cornell", "cornell_1080p", (160, 96), 2.0),
                                                     ("city", "city_4k", (160, 96), 1.7)])
def test_tolerance_units_per_pass_from_identical_inputs_above_ratio_1(scene, config, size, ratio):
    W, H = size
    b = Bench(scene, W, H, config=config, emissive_spatial_reuse=1, upscale_ratio=ratio)
    dev, orc = b.device(flavor="product"), b.oracle()
    dev.set_keep_intermediates(True)
    RW, RH = (int(np.ceil(np.float32(1.0) / np.float32(ratio) * np.float32(s))) for s in (W, H))     # ceil(size / ratio) in f32
    budget = max(1, int(1e-4 * RW * RH) + 1)       # < 1e-4 of the render pixels (+1 so that tiny test frames may have a single one)
    worst = {}
    for f in range(1, 9):
        inp = b.inputs(f) if f < 5 else b.moving_inputs(f)
        # the exact units run on the device from the oracle's state of the previous frame and must reproduce it bit for bit
        dev.prepass(inp); orc.prepass(inp)
        orc.run_pass(inp, 0); dev.run_pass(inp, 0)
        for p in (1, 2):
            orc.run_pass(inp, p); dev.run_pass(inp, p)
        for k in EXACT_PLANES[:8]:
            assert mismatch(dev.readback(k), orc.readback(k)) == 0, (f, "exact unit", k)
        for k in [L.OUT_RESERVOIR_0 + i for i in (0, 1, 2, 3)]:
            assert reservoir_mismatch(dev.readback(k), orc.readback(k)) == 0, (f, "exact unit", k)
        # ---- pass 3: spatial reuse (emissive), k_spatial, from identical inputs
        sync_state(dev, orc)
        orc.run_pass(inp, 3); dev.run_pass(inp, 3)
        n, m = outlier_pixels(dev.readback(L.OUT_RENDER_EMISSIVE), orc.readback(L.OUT_RENDER_EMISSIVE))
        worst[(f, "spatial emissive render")] = (n, m)
        assert n <= budget, (ratio, f, "emissive spatial", n, m)
        sync_state(dev, orc)
        orc.run_pass(inp, 4); dev.run_pass(inp, 4)
        for k in (L.OUT_RENDER_INDIRECT, L.OUT_VARIANCE_INDIRECT):
            assert mismatch(dev.readback(k), orc.readback(k)) == 0, (f, "indirect (exact unit)", k)
        for k in (L.OUT_RESERVOIR_0 + 6, L.OUT_RESERVOIR_0 + 7):
            assert reservoir_mismatch(dev.readback(k), orc.readback(k)) == 0, (f, "indirect (exact unit)", k)
        # ---- pass 5: spatial reuse (indirect)
        sync_state(dev, orc)
        orc.run_pass(inp, 5); dev.run_pass(inp, 5)
        n, m = outlier_pixels(dev.readback(L.OUT_RENDER_INDIRECT), orc.readback(L.OUT_RENDER_INDIRECT))
        worst[(f, "spatial indirect render")] = (n, m)
        assert n <= budget, (ratio, f, "indirect spatial", n, m)
        cur = (f & 1)
        rd, ro = dev.readback(L.OUT_RESERVOIR_0 + 8 + (1 - cur)), orc.readback(L.OUT_RESERVOIR_0 + 8 + (1 - cur))
        same_sample = (rd["sample_position"] == ro["sample_position"]).all(axis=-1) if rd.dtype.names else None
        if same_sample is not None:
            assert (~same_sample).sum() <= budget, (ratio, f, "spatial reservoir picked another sample", int((~same_sample).sum()))
        # ---- pass 6 + 7: denoise chain (nearest texel at the +-0.5-texel jittered uv) and tone mapping
        sync_state(dev, orc)
        for sgl in range(3):
            orc.run_pass(inp, 6, sgl)
        dev.run_pass(inp, 6)
        for k in (L.OUT_DENOISED_DIRECT, L.OUT_DENOISED_EMISSIVE, L.OUT_DENOISED_INDIRECT):
            n, m = outlier_pixels(dev.readback(k), orc.readback(k), ulps=4)
            worst[(f, "denoised", k)] = (n, m)
            assert n <= budget, (ratio, f, "denoise chain", k, n, m)
        orc.run_pass(inp, 7); dev.run_pass(inp, 7)
        n, m = outlier_pixels(dev.readback(L.OUT_TONE_MAPPED), orc.readback(L.OUT_TONE_MAPPED), ulps=5)
        worst[(f, "tone mapped")] = (n, m)
        assert n <= budget, (ratio, f, "tone mapping", n, m)
        sync_state(dev, orc)          # next frame starts from the oracle's state on both sides
    print(scene, ratio, {str(k): v for k, v in worst.items() if v[0]})
    if EMULATED:
        assert all(v == (0, 0.0) for v in worst.values()), worst


def test_ids_and_temporal_chain_stay_bit_exact_in_the_default_upscaled_pipeline():
    """12 frames of HikariSettings::default()'s pipeline (ratio 2, SMAA TU4x + TAA), static then moving camera, the product renders
    on its own: ids, G-buffer, albedo, sun radiance and the temporal reservoirs equal the oracle bit for bit in every frame."""
    b = Bench("cornell", 160, 96, config="cornell_1080p", taa=plugin.TAA_JASMINE, upscale_kind=plugin.UPSCALE_SMAA_TU4X, upscale_ratio=2.0)
    dev, orc = b.device(flavor="product"), b.oracle()
    for f in range(1, 13):
        inp = b.inputs(f) if f < 7 else b.moving_inputs(f)
        dev.render_frame(inp); orc.render_frame(inp)
        for k in EXACT_PLANES:
            same = reservoir_mismatch if k >= L.OUT_RESERVOIR_0 else mismatch
            assert same(dev.readback(k), orc.readback(k)) == 0, (f, k)
