"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on identical inputs.

Integer / index outputs must match bit-for-bit.  Because oracle and kernels share include/hk_math.h (explicit fmaf,
contraction off, IEEE div/sqrt, own sin/cos/exp) the floating-point planes are also required to match bit-for-bit;
the tolerance written here is therefore 0 ulp, with the looser documented bound (1 f16 ulp, <1e-4 outlier pixels,
SURVEY.md 8(c)) kept only as the fallback that the assertion message reports against."""
import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from tests.conftest import Bench

pytestmark = pytest.mark.gpu

ALL_PLANES = ([L.OUT_GBUFFER_POSITION, L.OUT_GBUFFER_NORMAL, L.OUT_GBUFFER_DEPTH_GRADIENT, L.OUT_GBUFFER_INSTANCE_MATERIAL,
               L.OUT_GBUFFER_VELOCITY_UV, L.OUT_ALBEDO, L.OUT_RENDER_DIRECT, L.OUT_RENDER_EMISSIVE, L.OUT_RENDER_INDIRECT,
               L.OUT_VARIANCE_DIRECT, L.OUT_VARIANCE_EMISSIVE, L.OUT_VARIANCE_INDIRECT, L.OUT_TONE_MAPPED] +
              [L.OUT_RESERVOIR_0 + i for i in range(10)])
DENOISED = [L.OUT_DENOISED_DIRECT, L.OUT_DENOISED_EMISSIVE, L.OUT_DENOISED_INDIRECT]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(a.shape[0], a.shape[1], -1)


def mismatch(a, b):
    """number of pixels whose bytes differ"""
    return int((bits(a) != bits(b)).any(axis=2).sum())


def reservoir_mismatch(a, b):
    """number of PackedReservoir records that differ, under the image-exact traversal mode's contract (include/hikari_b200.h
    HK_TUNE_WIDE_TRAVERSAL): a record whose sample carries no radiance may differ in sample_position.xyz — the position of whichever
    occluder the shadow ray met first, which depends on the order of the walk and which no image reads"""
    diff = (bits(a) != bits(b)).any(axis=2)
    if not diff.any():
        return 0
    dark = ((a["radiance"][..., 0] == 0) & ((a["radiance"][..., 1] & 0xFFFF) == 0) &
            (b["radiance"][..., 0] == 0) & ((b["radiance"][..., 1] & 0xFFFF) == 0))
    rest_equal = np.ones(diff.shape, bool)
    for name in a.dtype.names:
        if name == "sample_position":
            rest_equal &= a[name][..., 3] == b[name][..., 3]
        else:
            rest_equal &= (a[name] == b[name]).reshape(diff.shape + (-1,)).all(axis=-1)
    return int((diff & ~(dark & rest_equal)).sum())


def compare_all(dev, orc, planes, frame, allow=0):
    bad = {}
    for k in planes:
        n = mismatch(dev.readback(k), orc.readback(k))
        if n > allow:
            bad[k] = n
    assert not bad, f"frame {frame}: planes with differing pixels {bad} (of {dev.owned_cols * dev.owned_rows})"


def random_rays(n, seed, any_hit_fraction=0.3):
    rng = np.random.default_rng(seed)
    rays = np.zeros(n, L.RAY)
    rays["origin"] = rng.uniform([-0.9, 0.1, -0.9], [0.9, 1.9, 0.9], (n, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3))
    rays["direction"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["max_distance"] = np.float32(3.402823466e38)
    any_hit = rng.random(n) < any_hit_fraction
    rays["early_distance"] = np.where(any_hit, np.float32(65535.0), np.float32(0.0))
    rays["exclude_instance"] = np.where(rng.random(n) < 0.2, rng.integers(0, 8, n), 0xFFFFFFFF).astype(np.uint32)
    return rays


def test_trace_rays_bit_exact():
    b = Bench("cornell", 32, 32, config="cornell_256")
    dev, orc = b.device(), b.oracle()
    rays = random_rays(200_000, 1)
    hd, ho = dev.trace_rays(rays), orc.trace_rays(rays)
    for f in ("instance_index", "primitive_index"):
        assert np.array_equal(hd[f], ho[f]), f
    for f in ("distance", "u", "v"):
        assert np.array_equal(hd[f].view(np.uint32), ho[f].view(np.uint32)), f
    assert (hd["instance_index"] != 0xFFFFFFFF).mean() > 0.7   # the box is open towards the camera


@pytest.mark.parametrize("config,size,frames", [("cornell_256", 128, 12), ("cornell_1080p", 96, 12)])
def test_multi_frame_bit_exact(config, size, frames):
    """Frames 1..N from zeroed temporal state: every plane of every frame, including validation frames (3, 5, 6, ...)."""
    b = Bench("cornell", size, size, config=config)
    dev, orc = b.device(), b.oracle()
    dev.set_keep_intermediates(True)
    planes = ALL_PLANES + (DENOISED if b.settings.denoise else [])
    for f in range(1, frames + 1):
        inp = b.inputs(f)
        dev.render_frame(inp)
        orc.render_frame(inp)
        compare_all(dev, orc, planes, f)


def test_city_textured_scene_bit_exact():
    """examples/city.rs: 54 instances, 19k triangles, 14 textures (bilinear, sRGB), sun + textured emissive sphere."""
    b = Bench("city", 160, 90, config="city_4k")
    dev, orc = b.device(), b.oracle()
    dev.set_keep_intermediates(True)
    rays = random_rays(50_000, 7)
    rays["origin"] = rays["origin"] * np.float32(8.0) + np.array([0, 1, 0], np.float32)
    rays["exclude_instance"] = 0xFFFFFFFF
    hd, ho = dev.trace_rays(rays), orc.trace_rays(rays)
    for f in ("instance_index", "primitive_index", "distance", "u", "v"):
        assert np.array_equal(hd[f].view(np.uint32), ho[f].view(np.uint32)), f
    for f in range(1, 7):
        inp = b.inputs(f)
        dev.render_frame(inp)
        orc.render_frame(inp)
        compare_all(dev, orc, ALL_PLANES + DENOISED, f)
    cov = dev.readback(L.OUT_GBUFFER_POSITION)[..., 3] > 0
    assert cov.mean() > 0.5


def test_foreign_bvh_with_loose_navigator_boxes_still_matches():
    """The kernels skip the re-derived leaf box test only when upload validated that navigator boxes equal the shapes'
    own boxes (true for bvh 0.7.1).  With inflated navigator boxes they must fall back to the reference's double test."""
    from bevy_hikari_b200 import plugin
    b = Bench("cornell", 64, 64, config="cornell_1080p")
    bufs = b.world.buffers()
    for name in ("asset_nodes", "instance_nodes"):
        nodes = bufs[name]
        nav = nodes["entry_index"] < 0x80000000
        nodes["min"][nav] -= np.float32(0.05)
        nodes["max"][nav] += np.float32(0.05)
    desc = plugin.scene_desc_from_buffers(bufs)
    dev = plugin.HikariPlugin(64, 64)
    dev.upload_scene_desc(desc)
    from oracle import oracle
    orc = oracle.Oracle(64, 64, plugin.load_noise())
    orc.upload_scene_desc(desc)
    rays = random_rays(100_000, 11)
    hd, ho = dev.trace_rays(rays), orc.trace_rays(rays)
    for f in ("instance_index", "primitive_index", "distance", "u", "v"):
        assert np.array_equal(hd[f].view(np.uint32), ho[f].view(np.uint32)), f
    for f in range(1, 5):
        inp = b.inputs(f)
        dev.render_frame(inp)
        orc.render_frame(inp)
        compare_all(dev, orc, ALL_PLANES, f)


@pytest.mark.parametrize("scene,config,size", [("cornell", "cornell_1080p", (112, 80)), ("city", "city_4k", (128, 72))])
def test_moving_camera_bit_exact(scene, config, size):
    """Non-zero velocity: reprojection to other pixels, depth/normal/instance rejection, and the scatter writes to
    store_previous_spatial_reservoir(previous_coords) — racy in the reference, resolved in raster order by the oracle and
    by the claim/resolve kernels."""
    b = Bench(scene, size[0], size[1], config=config)
    dev, orc = b.device(), b.oracle()
    dev.set_keep_intermediates(True)
    moved = 0
    for f in range(1, 11):
        inp = b.moving_inputs(f)
        dev.render_frame(inp)
        orc.render_frame(inp)
        compare_all(dev, orc, ALL_PLANES + DENOISED, f)
        vel = dev.readback(L.OUT_GBUFFER_VELOCITY_UV)[..., :2]
        moved += int((np.abs(vel) > 0).any(axis=2).sum())
    assert moved > 1000


def test_scatter_at_previous_uv_one_lands_in_the_next_row():
    """light.wgsl stores a reprojected write at coords.x + size.x * coords.y, and the scatter's test admits a previous uv of exactly
    1.0: in x that is column 0 of the next row (seen on city 3840x2160 under a moving camera).  Right-edge pixels get the velocity
    that puts their previous uv at 1.0, column-0 pixels one that takes theirs out of the frame, so the wrapped write is their only one.
    The last row's write indexes past the buffer and is discarded on both sides."""
    W, H = 24, 16
    b = Bench("city", W, H, config="city_4k")              # the ground reaches both side edges
    dev, orc = b.device(), b.oracle()
    edge_uv = (np.float32(W - 1) + np.float32(0.5)) / np.float32(W)        # coords_to_uv of the last column
    for f in (1, 2):
        inp = b.inputs(f)
        dev.prepass(inp); orc.prepass(inp)
        vel = orc.readback(L.OUT_GBUFFER_VELOCITY_UV).copy()
        vel[:, W - 1, 0] = edge_uv - np.float32(1.0)           # uv.x - velocity.x == 1.0 exactly
        vel[:, 0, 0] = np.float32(0.5)                         # previous uv.x < 0: no write of its own
        dev.upload_state(L.OUT_GBUFFER_VELOCITY_UV, vel); orc.upload_state(L.OUT_GBUFFER_VELOCITY_UV, vel)
        for p in (0, 1, 2, 4):
            orc.run_pass(inp, p); dev.run_pass(inp, p)
        for k in [L.OUT_RESERVOIR_0 + i for i in range(10)]:
            assert mismatch(dev.readback(k), orc.readback(k)) == 0, (f, k)
    assert (orc.readback(L.OUT_GBUFFER_POSITION)[:H - 1, W - 1, 3] > 0).sum() >= 8      # surfaces at the right edge write


def test_nodes_one_by_one_equal_render_frame():
    """hk_prepass_run + hk_light_run + hk_post_process_run (unfused tone mapping) == hk_render_frame."""
    b = Bench("cornell", 80, 48, config="cornell_1080p")
    a, c = b.device(), b.device()
    a.set_keep_intermediates(True)
    for f in range(1, 5):
        inp = b.inputs(f)
        a.render_frame(inp)
        c.prepass(inp); c.light(inp); c.post_process(inp)
        for k in ALL_PLANES + DENOISED:
            assert mismatch(a.readback(k), c.readback(k)) == 0, (f, k)


def test_row_bands_equal_unsharded():
    """Two contexts owning half the rows each (plus ghost rows) reproduce the unsharded frame bit-for-bit."""
    b = Bench("cornell", 96, 160, config="cornell_1080p")
    full, top, bot = b.device(), b.device(0, 80), b.device(80, 160)
    for f in range(1, 8):
        inp = b.inputs(f)
        for d in (full, top, bot):
            d.render_frame(inp)
        for k in (L.OUT_TONE_MAPPED, L.OUT_RENDER_INDIRECT, L.OUT_RENDER_EMISSIVE, L.OUT_RESERVOIR_0 + 8, L.OUT_RESERVOIR_0 + 9):
            whole = full.readback(k)
            parts = np.concatenate([top.readback(k), bot.readback(k)], axis=0)
            assert mismatch(whole, parts) == 0, (f, k)


def test_2d_tiles_equal_unsharded():
    """Four contexts owning a 2x2 grid of tiles (plus ghost rows AND ghost columns) reproduce the unsharded frame."""
    b = Bench("cornell", 176, 144, config="cornell_1080p")
    full = b.device()
    tiles = [b.device(0, 72, 0, 88), b.device(0, 72, 88, 176), b.device(72, 144, 0, 88), b.device(72, 144, 88, 176)]
    for d in tiles + [full]:
        d.set_profiling(True, False)
    for f in range(1, 7):
        inp = b.inputs(f)
        for d in tiles + [full]:
            d.render_frame(inp)
        for k in (L.OUT_TONE_MAPPED, L.OUT_RENDER_INDIRECT, L.OUT_RESERVOIR_0 + 4, L.OUT_RESERVOIR_0 + 8, L.OUT_GBUFFER_POSITION):
            whole = full.readback(k)
            t = [d.readback(k) for d in tiles]
            parts = np.concatenate([np.concatenate(t[:2], axis=1), np.concatenate(t[2:], axis=1)], axis=0)
            assert mismatch(whole, parts) == 0, (f, k)
        sw = full.stats()
        st = [d.stats() for d in tiles]
        assert sum(s.tlas_rays for s in st) == sw.tlas_rays and sum(s.blas_rays for s in st) == sw.blas_rays   # ghosts not counted


def test_ray_counts_match_oracle():
    b = Bench("cornell", 64, 64, config="cornell_1080p")
    dev, orc = b.device(), b.oracle()
    dev.set_profiling(True, False)
    for f in range(1, 7):
        inp = b.inputs(f)
        dev.render_frame(inp)
        orc.render_frame(inp)
        sd, so = dev.stats(), orc.stats()
        assert (sd.primary_rays, sd.tlas_rays, sd.blas_rays) == (so.primary_rays, so.tlas_rays, so.blas_rays), f


def test_errors_are_reported_not_fatal():
    from bevy_hikari_b200 import _ffi, plugin
    p = plugin.HikariPlugin(32, 32)
    b = Bench("cornell", 32, 32, config="cornell_256")
    with pytest.raises(_ffi.HikariError, match="not uploaded"):
        p.render_frame(b.inputs(1))          # scene missing -> HK_ERR_NOT_READY (reference: node silently skips)
    p.upload_scene(b.world)
    bad = b.inputs(1)
    bad.frame.upscale_ratio = 0.5            # Upscale::ratio() clamps to [1, 2] (lib.rs:501-505); raw inputs outside are refused
    with pytest.raises(_ffi.HikariError, match="upscale_ratio"):
        p.render_frame(bad)
    p.run_frame(b.settings, b.view, b.previous_view, b.lights)
    assert p.frame_counter == 1              # frame_counter_system increments before extraction (view.rs:89-103)


def test_large_mesh_bit_exact():
    """100 352-triangle BLAS (302 k records — the size class of the reference's scene.gltf): host builder, upload and deep
    traversal, static then moving camera."""
    b = Bench("terrain", 128, 80, config="city_4k")
    assert b.world.scene_desc().primitive_count > 100000
    dev, orc = b.device(), b.oracle()
    dev.set_keep_intermediates(True)
    for f in range(1, 7):
        inp = b.inputs(f) if f < 4 else b.moving_inputs(f)
        dev.render_frame(inp)
        orc.render_frame(inp)
        compare_all(dev, orc, ALL_PLANES + DENOISED, f)
    rays = random_rays(4096, 5)
    rays["origin"] = rays["origin"] * np.float32(3.0) + np.array([0, 1.0, 0], np.float32)
    hd, ho = dev.trace_rays(rays), orc.trace_rays(rays)
    assert hd.tobytes() == ho.tobytes()
    assert (hd["instance_index"] != 0xFFFFFFFF).mean() > 0.15


@pytest.mark.parametrize("scene,size,config", [("cornell", (96, 80), "cornell_1080p"), ("city", (112, 64), "city_8k"), ("simple", (80, 64), "cornell_1080p")])
def test_pooled_indirect_kernel_bit_exact(scene, size, config):
    """kc_indirect (shared-memory ray pool with dynamic fetch, TMA-staged scene records; hk_set_tuning) writes the same bytes as the
    oracle — and therefore as the default per-pixel kernel: static and moving camera, 2 and 4 bounces, tiny and deep BLASes."""
    from bevy_hikari_b200 import plugin
    b = Bench(scene, size[0], size[1], config=config)
    dev, orc = b.device(), b.oracle()
    dev.set_tuning(plugin.TUNE_POOLED_INDIRECT, 1)
    dev.set_profiling(True, False)
    for f in range(1, 7):
        inp = b.inputs(f) if f < 4 else b.moving_inputs(f)
        dev.render_frame(inp)
        orc.render_frame(inp)
        compare_all(dev, orc, ALL_PLANES, f)
        sd, so = dev.stats(), orc.stats()
        assert (sd.tlas_rays, sd.blas_rays) == (so.tlas_rays, so.blas_rays), f


@pytest.mark.parametrize("scene,size,config", [("cornell", (96, 80), "cornell_1080p"), ("city", (131, 67), "city_8k")])
def test_spatial_reuse_tiled_and_gather_forms_bit_exact(scene, size, config):
    """kc_spatial (neighbourhood tiles staged by TMA, the default at upscale ratio 1) and k_spatial (gathers from global memory) against
    the oracle: full frame and a 2 x 2 tiling (tile origins off the 16-pixel grid, boxes hanging over the allocation), moving camera."""
    from bevy_hikari_b200 import plugin
    b = Bench(scene, size[0], size[1], config=config, emissive_spatial_reuse=1)
    orc = b.oracle()
    tiled, gather = b.device(), b.device()
    gather.set_tuning(plugin.TUNE_TILED_SPATIAL, 0)
    hx, hy = size[0] // 2 + 3, size[1] // 2 - 5
    tiles = [b.device(0, hy, 0, hx), b.device(0, hy, hx, size[0]), b.device(hy, size[1], 0, hx), b.device(hy, size[1], hx, size[0])]
    planes = [L.OUT_RENDER_EMISSIVE, L.OUT_RENDER_INDIRECT, L.OUT_VARIANCE_EMISSIVE, L.OUT_VARIANCE_INDIRECT, L.OUT_RESERVOIR_0 + 4,
              L.OUT_RESERVOIR_0 + 5, L.OUT_RESERVOIR_0 + 8, L.OUT_RESERVOIR_0 + 9, L.OUT_TONE_MAPPED]
    for f in range(1, 7):
        inp = b.inputs(f) if f < 4 else b.moving_inputs(f)
        orc.render_frame(inp)
        for d in [tiled, gather] + tiles:
            d.render_frame(inp)
        for d in (tiled, gather):
            compare_all(d, orc, planes, f)
        if f < 4:          # tiles are exact while the camera is static (the halo exchange is tested elsewhere)
            for k in planes:
                whole = orc.readback(k)
                t = [d.readback(k) for d in tiles]
                parts = np.concatenate([np.concatenate(t[:2], axis=1), np.concatenate(t[2:], axis=1)], axis=0)
                assert mismatch(whole, parts) == 0, (f, k)
