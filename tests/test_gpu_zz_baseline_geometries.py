"""Every BASELINE workload that bench.py times, held to the CPU oracle at its own resolution: `scene_1080p` (town, 120 k triangles,
3 bounces, 1920x1080), `city_4k` (3840x2160, 2 bounces, the bench's 4-tile plan) and `city_8k` (7680x4320, 4 bounces, the bench's
8-tile plan), plus the reference's default pipeline at window sizes.  Scene, size and settings come from bench.make_bench, tile
rectangles from bench.plan_tiles over the bench's quarter-resolution coverage probe, so what is checked is what the bench renders.

  * exact flavour, whole frame: frames 1-3 (frame 3 is a validation frame of the sun pass) of scene_1080p and city_4k on one
    full-frame context, every plane bit for bit; city_4k also under a moving camera (reprojection at 4K);
  * exact flavour, the bench's tile plans: each tile context alone (opened, rendered, compared, closed before the next), its owned
    rectangle of the tone-mapped frame, the three radiance planes, both spatial reservoirs and the ids against the oracle's frame;
    city_8k renders frames 2 and 3 only (cut for time; frame 3 validates the history frame 2 left, so its scatter writes run);
  * product flavour: ids, G-buffer, albedo, sun radiance and the temporal reservoirs (under the 4-wide walk's contract) equal the
    oracle over frames 1-3, but for one named pixel of city_4k (WIDE_WALK_TIE_4K); the per-pass tolerance bounds of
    test_gpu_tolerance.py at city_4k frame 2 from identical inputs, with the 4-wide walk off; the
    product's 4- and 8-tile plans of city_4k equal its own full frame bit for bit on the owned rectangles;
  * the default pipeline: HikariSettings::default() (ratio 2, SMAA TU4x + TAA) on cornell 1920x1080 and FSR 1.0 at ratio 1.5 (+ TAA)
    on city 3840x2160, 3 moving frames, every plane and every upscaler output bit for bit, extents against scaled() / upscaled().

The product's 8-tile plan is checked on the 4K frame: its reference, a full-frame product context at 8K, would need 29 GB of device
memory, and no full-frame 8K context is opened here.

Cost of the oracle per frame on 8 host threads (a 4K frame took ~33 s on the H100 host's 8 threads), and peak resident memory:
    scene_1080p  town 1920x1080, 3 bounces      ~11 s     2.3 GB
    city_4k      city 3840x2160, 2 bounces      ~24 s     8.4 GB
    city_8k      city 7680x4320, 4 bounces     ~114 s    33 GB  (+ 49 s to allocate and upload)
The file takes about 15 minutes on an H100 80GB HBM3 (700 W) whose host has 8 threads, almost all of it in the oracle.
The 8K oracle fits the 48 GB of host memory this file allows itself, so city_8k is compared with the oracle, not device against device.
Oracle planes are not kept between fixtures and tests: a 4K frame's compared planes take 5 GB, an 8K frame's 20 GB.  What a later
comparison needs is kept as one BLAKE2b digest per row of each compared rectangle, and a failure names the frame, plane, rectangle
and the rows that differ.

Device memory, at ~876 B per render pixel (bench.py): 1.8 GB for a 1080p context, 7.3 GB for 4K, about 2.1 GB for a 4K tile and
3.9 GB for an 8K strip with its ghost columns; one context at a time, plus the planes set_keep_intermediates holds.

With HK_EMULATE_KERNELS=1 (no GPU) every geometry is divided by 8 (4K, 8K) or 4 (1080p) and the tile plans are re-planned at the
scaled size: the scaled 8K frame, 960x540, has 518 k render pixels, above 2^18."""
import hashlib
from types import SimpleNamespace

import numpy as np
import pytest

import bench
from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin
from tests.conftest import EMULATED, Bench
from tests.test_gpu_parity import ALL_PLANES, DENOISED, compare_all, mismatch, reservoir_mismatch
from tests.test_gpu_tolerance import EXACT_PLANES, outlier_pixels, sync_state
from tests.test_gpu_upscale import scaled, upscaled

pytestmark = pytest.mark.gpu

FRAMES = (1, 2, 3)
# The product's 4-wide walk (primary rays) on city_4k: at one pixel the primary ray's two nearest triangles tie within the rounding of
# a box test, which csrc/hk_wide.cuh names as what that walk may change, and it keeps another triangle of the same instance than the
# reference's walk (same position and ids, another uv).  These planes differ there in every frame; with the walk off they do not.  The
# product's whole-frame check masks that pixel in these planes only; every other pixel of every compared plane must equal the oracle.
WIDE_WALK_TIE_4K = ((1309, 1233), (L.OUT_GBUFFER_VELOCITY_UV, L.OUT_ALBEDO, L.OUT_RENDER_DIRECT, L.OUT_RESERVOIR_0 + 6,
                                   L.OUT_RESERVOIR_0 + 7))
FRAMES_8K = (2, 3)   # the oracle at 8K takes 2-2.5 min per frame on 8 host threads; 3 is a validation frame of the sun pass
TILE_PLANES = (L.OUT_TONE_MAPPED, L.OUT_RENDER_DIRECT, L.OUT_RENDER_EMISSIVE, L.OUT_RENDER_INDIRECT, L.OUT_RESERVOIR_0 + 8,
               L.OUT_RESERVOIR_0 + 9, L.OUT_GBUFFER_INSTANCE_MATERIAL)


def shrink(height):
    return (4 if height <= 1080 else 8) if EMULATED else 1


def workload(config, **extra):
    """bench.make_bench(config) as a Bench (scaled down under the emulator)"""
    cfg, scene, _, W, H, view, _, _, settings = bench.make_bench(config)
    s = shrink(H)
    b = Bench(cfg["scene"], W // s, H // s, config=config, **extra)
    if not extra:
        assert bytes(b.settings) == bytes(settings)
    if s == 1:
        assert bytes(b.view) == bytes(view)
    return b


def bench_tiles(b, n):
    """bench.py's plan for n GPUs: quarter-resolution coverage probe -> cost-balanced tiles"""
    cw, ch = max(b.width // 4, 1), max(b.height // 4, 1)
    probe = plugin.HikariPlugin(cw, ch)
    probe.upload_scene(b.world)
    pv, ppv, pl = b.scene.view_inputs(cw, ch)
    probe.prepass(plugin.make_frame_inputs(b.settings, 1, pv, ppv, pl))
    coverage = probe.readback(L.OUT_GBUFFER_INSTANCE_MATERIAL)[..., 0] > 0
    probe.close()
    tiles = bench.plan_tiles(b.width, b.height, n, coverage)
    owners = np.zeros((b.height, b.width), np.int32)
    for x0, x1, r0, r1 in tiles:
        owners[r0:r1, x0:x1] += 1
    assert len(tiles) == n and (owners == 1).all(), tiles       # a partition of the frame
    return tiles


def canonical(k, a):
    """reservoir records as test_gpu_parity.reservoir_mismatch compares them under the product's 4-wide walk: a record whose sample
    carries no radiance keeps no sample position (the occluder the walk met first); byte-equal canonical records == a match there"""
    if k < L.OUT_RESERVOIR_0:
        return a
    a = a.copy()
    dark = (a["radiance"][..., 0] == 0) & ((a["radiance"][..., 1] & 0xFFFF) == 0)
    a["sample_position"][dark, :3] = 0.0
    return a


def row_digests(a):
    rows = np.ascontiguousarray(a).view(np.uint8).reshape(a.shape[0], -1)
    return [hashlib.blake2b(r.data, digest_size=16).digest() for r in rows]


def tie_mask(b):
    """the pixel and planes of WIDE_WALK_TIE_4K, at the size where the walk runs (none on the emulated kernels: the product is exact)"""
    (y, x), planes = WIDE_WALK_TIE_4K
    return {k: (y, x) for k in planes} if (b.width, b.height) == (3840, 2160) and not EMULATED else {}


def digests(ctx, planes, rects, product_contract=False, mask=None):
    """{(plane, rect): row digests} of a full-frame context's planes cut to each (x0, x1, r0, r1) rectangle; `mask` {plane: (y, x)}
    zeroes one pixel of a plane first"""
    out = {}
    for k in planes:
        whole = ctx.readback(k)
        if product_contract:
            whole = canonical(k, whole)
        if mask and k in mask:
            whole = np.ascontiguousarray(whole).copy()
            whole.view(np.uint8).reshape(whole.shape[0], whole.shape[1], -1)[mask[k]] = 0
        for x0, x1, r0, r1 in rects:
            out[(k, (x0, x1, r0, r1))] = row_digests(whole[r0:r1, x0:x1])
    return out


def differing_rows(got, want):
    """{(plane, rect): (number of differing rows, first one)} over the keys of `want`"""
    bad = {}
    for key, rows in want.items():
        d = [i for i, (a, b) in enumerate(zip(got[key], rows)) if a != b]
        if d or len(got[key]) != len(rows):
            bad[key] = (len(d), d[:1])
    return bad


def full(b):
    return (0, b.width, 0, b.height)


def reference_frames(b, tiles=(), exact_context=True, frames=FRAMES):
    """`frames` on the oracle, and (exact_context) on one full-frame exact context in lockstep, compared through compare_all on
    every plane.  Returns the comparison failures, the share of covered pixels, and per frame the digests later tests compare with:
    TILE_PLANES over the `tiles` (exact bytes), EXACT_PLANES over the whole frame (under the product's contract)."""
    orc = b.oracle()
    dev = b.device() if exact_context else None
    if dev:
        dev.set_keep_intermediates(True)
    failures, ref = [], {}
    for f in frames:
        inp = b.inputs(f)
        orc.render_frame(inp)
        if dev:
            dev.render_frame(inp)
            try:
                compare_all(dev, orc, ALL_PLANES + DENOISED, f)
            except AssertionError as e:
                failures.append(str(e))
        ref[f] = digests(orc, TILE_PLANES, tiles)
        if exact_context:
            ref[f].update(digests(orc, EXACT_PLANES, [full(b)], product_contract=True, mask=tie_mask(b)))
    covered = float((orc.readback(L.OUT_GBUFFER_INSTANCE_MATERIAL)[..., 0] > 0).mean())
    if dev:
        dev.close()
    orc.close()
    return SimpleNamespace(b=b, tiles=tiles, failures=failures, covered=covered, ref=ref, frames=frames)


@pytest.fixture(scope="module")
def scene_1080p():
    return reference_frames(workload("scene_1080p"))


@pytest.fixture(scope="module")
def city_4k():
    """the oracle's frames against the bench's 4-tile plan; its 8-tile plan at 4K for the product's own comparison"""
    b = workload("city_4k")
    ref = reference_frames(b, bench_tiles(b, 4))
    ref.plans = {4: ref.tiles, 8: bench_tiles(b, 8)}
    return ref


@pytest.fixture(scope="module")
def city_8k():
    """oracle only: the bench's 8-tile plan is compared with it, and no full-frame 8K context is opened"""
    b = workload("city_8k")
    return reference_frames(b, bench_tiles(b, 8), exact_context=False, frames=FRAMES_8K)


@pytest.mark.parametrize("config", ["scene_1080p", "city_4k"])
def test_exact_whole_frame_bit_exact(config, request):
    r = request.getfixturevalue(config)
    assert any(f % r.b.inputs(f).frame.direct_validate_interval == 0 for f in FRAMES), "no validation frame of the sun pass"
    assert not r.failures, r.failures
    assert r.covered > 0.2, r.covered


def test_exact_city_4k_moving_camera_bit_exact():
    b = workload("city_4k")
    dev, orc = b.device(), b.oracle()
    dev.set_keep_intermediates(True)
    for f in FRAMES:
        inp = b.moving_inputs(f)
        orc.render_frame(inp)
        dev.render_frame(inp)
        compare_all(dev, orc, ALL_PLANES + DENOISED, f)
    dev.close()
    orc.close()


def render_tiles(b, tiles, flavor=None, frames=FRAMES):
    """each tile on its own context, one at a time: {frame: {(plane, rect): row digests}} of its owned rectangle"""
    got = {f: {} for f in frames}
    for x0, x1, r0, r1 in tiles:
        d = b.device(r0, r1, x0, x1, flavor=flavor)
        for f in frames:
            d.render_frame(b.inputs(f))
            for k in TILE_PLANES:
                got[f][(k, (x0, x1, r0, r1))] = row_digests(d.readback(k))
        d.close()
    return got


@pytest.mark.parametrize("config,n", [("city_4k", 4), ("city_8k", 8)])
def test_exact_tile_plan_equals_the_oracle(config, n, request):
    r = request.getfixturevalue(config)
    assert len(r.tiles) == n and r.covered > 0.2, (r.tiles, r.covered)
    got = render_tiles(r.b, r.tiles, frames=r.frames)
    for f in r.frames:
        want = {key: v for key, v in r.ref[f].items() if key[0] in TILE_PLANES and key[1] in r.tiles}
        assert len(want) == n * len(TILE_PLANES)
        bad = differing_rows(got[f], want)
        assert not bad, (f, bad)


@pytest.fixture(scope="module")
def product_city_4k(city_4k):
    """frames 1-3 of city_4k on one full-frame product context: the digests its own tiles and the oracle are compared with"""
    b = city_4k.b
    dev = b.device(flavor="product")
    own = {}
    for f in FRAMES:
        dev.render_frame(b.inputs(f))
        own[f] = digests(dev, TILE_PLANES, city_4k.plans[4] + city_4k.plans[8])
        own[f].update(digests(dev, EXACT_PLANES, [full(b)], product_contract=True, mask=tie_mask(b)))
    dev.close()
    return own


@pytest.mark.parametrize("config", ["scene_1080p", "city_4k"])
def test_product_exact_planes_equal_the_oracle(config, request):
    """ids, G-buffer, albedo, sun radiance and the temporal reservoirs of the product equal the oracle (reservoirs under the 4-wide
    walk's contract) over frames 1-3, but for the one pixel of WIDE_WALK_TIE_4K on city_4k"""
    r = request.getfixturevalue(config)
    b = r.b
    if config == "scene_1080p":
        dev = b.device(flavor="product")
        own = {}
        for f in FRAMES:
            dev.render_frame(b.inputs(f))
            own[f] = digests(dev, EXACT_PLANES, [full(b)], product_contract=True)
        dev.close()
    else:
        own = request.getfixturevalue("product_city_4k")
    for f in FRAMES:
        want = {key: r.ref[f][key] for key in ((k, full(b)) for k in EXACT_PLANES)}
        bad = differing_rows(own[f], want)
        assert not bad, (f, bad)


def test_product_tolerance_units_per_pass_at_city_4k_frame_2():
    """test_gpu_tolerance.py's per-pass bounds from identical inputs at 3840x2160: frame 1 rendered by both sides and the product
    re-synchronised to the oracle's state, then frame 2 pass by pass.  The bench's city_4k runs without emissive spatial reuse; it is on
    here, as in test_gpu_tolerance.py, so that pass 3's bound measures a pass that reuses.  This checks the tolerance units, not the
    walk: the 4-wide walk is off, so that the exact units' checks do not stop at the pixel of WIDE_WALK_TIE_4K"""
    b = workload("city_4k", emissive_spatial_reuse=1)
    W, H = b.width, b.height
    dev, orc = b.device(flavor="product"), b.oracle()
    dev.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 0)
    dev.set_keep_intermediates(True)
    inp = b.inputs(1)
    orc.render_frame(inp); dev.render_frame(inp)
    sync_state(dev, orc)
    npix = W * H
    budget = max(1, int(1e-4 * npix) + 1)
    worst = {}
    f = 2
    # the loop body of test_gpu_tolerance.test_tolerance_units_per_pass_from_identical_inputs, for frame 2
    inp = b.inputs(f)
    dev.prepass(inp); orc.prepass(inp)
    orc.run_pass(inp, 0); dev.run_pass(inp, 0)
    for p in (1, 2):
        orc.run_pass(inp, p); dev.run_pass(inp, p)
    for k in EXACT_PLANES[:8]:
        assert mismatch(dev.readback(k), orc.readback(k)) == 0, (f, "exact unit", k)
    for k in [L.OUT_RESERVOIR_0 + i for i in (0, 1, 2, 3)]:
        assert reservoir_mismatch(dev.readback(k), orc.readback(k)) == 0, (f, "exact unit", k)
    # ---- pass 3: spatial reuse (emissive), from identical inputs
    sync_state(dev, orc)
    orc.run_pass(inp, 3); dev.run_pass(inp, 3)
    n, m = outlier_pixels(dev.readback(L.OUT_RENDER_EMISSIVE), orc.readback(L.OUT_RENDER_EMISSIVE))
    worst[(f, "spatial emissive render")] = (n, m)
    assert n <= budget, (f, "emissive spatial", n, m)
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
    assert n <= budget, (f, "indirect spatial", n, m)
    # the spatial reservoir it wrote: same sample chosen (bit-identical record) on all but the outlier pixels
    cur = (f & 1)
    rd, ro = dev.readback(L.OUT_RESERVOIR_0 + 8 + (1 - cur)), orc.readback(L.OUT_RESERVOIR_0 + 8 + (1 - cur))
    same_sample = (rd["sample_position"] == ro["sample_position"]).all(axis=-1) if rd.dtype.names else None
    if same_sample is not None:
        assert (~same_sample).sum() <= budget, (f, "spatial reservoir picked another sample", int((~same_sample).sum()))
    # ---- pass 6 + 7: denoise chain and tone mapping
    sync_state(dev, orc)
    for sgl in range(3):
        orc.run_pass(inp, 6, sgl)
    dev.run_pass(inp, 6)
    for k in (L.OUT_DENOISED_DIRECT, L.OUT_DENOISED_EMISSIVE, L.OUT_DENOISED_INDIRECT):
        n, m = outlier_pixels(dev.readback(k), orc.readback(k), ulps=4)       # four a-trous levels: 1 f16 ulp each
        worst[(f, "denoised", k)] = (n, m)
        assert n <= budget, (f, "denoise chain", k, n, m)
    orc.run_pass(inp, 7); dev.run_pass(inp, 7)
    n, m = outlier_pixels(dev.readback(L.OUT_TONE_MAPPED), orc.readback(L.OUT_TONE_MAPPED), ulps=5)
    assert n <= budget, (f, "tone mapping", n, m)
    print({str(k): v for k, v in worst.items() if v[0]})
    dev.close()
    orc.close()


@pytest.mark.parametrize("n", [4, 8])
def test_product_tile_plan_equals_its_own_full_frame(n, city_4k, product_city_4k):
    """fast math is deterministic per pixel: the product's tiles equal its full frame bit for bit on the owned rectangles"""
    tiles = city_4k.plans[n]
    got = render_tiles(city_4k.b, tiles, flavor="product")
    for f in FRAMES:
        want = {key: v for key, v in product_city_4k[f].items() if key[1] in tiles and key[0] in TILE_PLANES}
        assert len(want) == n * len(TILE_PLANES)
        bad = differing_rows(got[f], want)
        assert not bad, (f, bad)


DEFAULT_PIPELINES = [
    # scene, window size, settings over HikariSettings::default(), upscaler outputs
    ("cornell", (1920, 1080), None, dict(), [L.OUT_UPSCALED, L.OUT_TAA]),
    ("city", (3840, 2160), "city_4k", dict(taa=plugin.TAA_JASMINE, upscale_kind=plugin.UPSCALE_FSR1, upscale_ratio=1.5),
     [L.OUT_UPSCALED, L.OUT_FSR_SHARPENED, L.OUT_TAA]),
]


@pytest.mark.parametrize("scene,size,config,settings,outputs", DEFAULT_PIPELINES, ids=["cornell_1080p_default", "city_4k_fsr1"])
def test_default_pipeline_at_a_window_size(scene, size, config, settings, outputs):
    """three moving frames with the temporal upscalers on, every plane and every upscaler output bit for bit"""
    s = shrink(size[1])
    W, H = size[0] // s, size[1] // s
    b = Bench(scene, W, H, config=config, **settings)
    if config is None:
        b.settings = plugin.HikariSettings()          # HikariSettings::default(): Upscale::SmaaTu4x{ratio 2} + Taa::Jasmine
        assert (b.settings.upscale_kind, b.settings.upscale_ratio, b.settings.taa) == (plugin.UPSCALE_SMAA_TU4X, 2.0, plugin.TAA_JASMINE)
    ratio = b.settings.upscale_ratio
    dev, orc = b.device(), b.oracle()
    dev.set_keep_intermediates(True)
    for f in FRAMES:
        inp = b.moving_inputs(f)
        inp.temporal_upscalers = 1
        dev.render_frame(inp)
        orc.render_frame(inp)
        compare_all(dev, orc, ALL_PLANES + DENOISED + outputs, f)
    rw, rh = scaled(W, ratio), scaled(H, ratio)
    assert dev.readback(L.OUT_TONE_MAPPED).shape[:2] == (rh, rw)
    assert dev.readback(L.OUT_GBUFFER_POSITION).shape[:2] == (H, W)
    if b.settings.upscale_kind == plugin.UPSCALE_SMAA_TU4X:
        assert dev.readback(L.OUT_UPSCALED).shape[:2] == dev.readback(L.OUT_TAA).shape[:2] == (upscaled(H, ratio), upscaled(W, ratio))
    else:
        assert dev.readback(L.OUT_UPSCALED).shape[:2] == dev.readback(L.OUT_FSR_SHARPENED).shape[:2] == (H, W)
        assert dev.readback(L.OUT_TAA).shape[:2] == (rh, rw)
    dev.close()
    orc.close()
