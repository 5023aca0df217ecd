"""The light node runs its indirect pipeline on a stream of its own, beside the sun and emissive pipelines; per-kernel pass timing
(hk_set_profiling time_passes, with no single kernel selected) keeps the serial order on one stream.  The three pipelines write
disjoint planes, so both orders must give the same bytes: every case renders the same frames through a serial and a concurrent
context side by side and requires every plane — G-buffer, render / variance of each signal, all ten reservoir buffers, the denoised
signals and the tone-mapped frame — and the ray counts to be equal on every frame.  Frames 1-15 include the validation frames of
both direct passes (every 3rd / 5th) and their scatter writes."""
import numpy as np
import pytest

from bevy_hikari_b200 import plugin
from tests.conftest import Bench, cornell_animation
from tests.test_gpu_parity import ALL_PLANES, DENOISED
from tests.test_gpu_shared_scene import animate

pytestmark = pytest.mark.gpu

FRAMES = range(1, 16)


def planes_of(bench):
    if not bench.settings.denoise:
        return ALL_PLANES
    return ALL_PLANES + (DENOISED[:2] if bench.settings.indirect_bounces == 0 else DENOISED)


def make_pair(make_dev, count_rays, tuning):
    """a serial and a concurrent context over the same scene and settings"""
    devs = []
    for serial in (True, False):
        d = make_dev()
        d.set_keep_intermediates(True)
        for k, v in tuning.items():
            d.set_tuning(k, v)
        d.set_profiling(count_rays, serial)
        devs.append(d)
    return devs


def assert_same_frame(serial, concurrent, planes, frame, count_rays, label=""):
    for k in planes:
        a, b = serial.readback(k), concurrent.readback(k)
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"{label}frame {frame}: plane {k} differs"
    if count_rays:
        s, c = serial.stats(), concurrent.stats()
        assert (s.primary_rays, s.tlas_rays, s.blas_rays) == (c.primary_rays, c.tlas_rays, c.blas_rays), f"{label}frame {frame}: ray counts"
        assert s.tlas_rays > 0
    assert serial.stats().kernel_launches == concurrent.stats().kernel_launches


def run_case(bench, moving=False, count_rays=False, tuning=None, tile=None, flavor=None):
    make_dev = lambda: bench.device(*(tile or (0, None, 0, None)), flavor=flavor)
    serial, concurrent = make_pair(make_dev, count_rays, tuning or {})
    planes = planes_of(bench)
    for f in FRAMES:
        inp = bench.moving_inputs(f) if moving else bench.inputs(f)
        serial.render_frame(inp)
        concurrent.render_frame(inp)
        assert_same_frame(serial, concurrent, planes, f, count_rays)
    serial.close()
    concurrent.close()


@pytest.mark.parametrize("settings", [
    dict(),                                                                      # the benchmark's settings at a small size
    dict(indirect_bounces=0),
    dict(indirect_bounces=1, indirect_spatial_reuse=0),
    dict(indirect_bounces=2, emissive_spatial_reuse=0, indirect_spatial_reuse=0, denoise=0),
    dict(indirect_bounces=2, direct_validate_interval=1, emissive_validate_interval=2),   # scatter writes of validation every frame
])
def test_cornell_settings(settings):
    run_case(Bench("cornell", 72, 56, config="cornell_1080p", **settings))


def test_cornell_moving_camera_with_ray_counts():
    run_case(Bench("cornell", 96, 64, config="cornell_1080p"), moving=True, count_rays=True)


@pytest.mark.parametrize("scene,config", [("city", "city_4k"), ("town", "scene_1080p")])
def test_city_and_scene_rs(scene, config):
    run_case(Bench(scene, 96, 54, config=config), moving=True, count_rays=True)


@pytest.mark.parametrize("tuning", [{plugin.TUNE_POOLED_INDIRECT: 1}, {plugin.TUNE_WIDE_TRAVERSAL: 3},
                                    {plugin.TUNE_TILED_SPATIAL: 0}])
def test_run_time_choices(tuning):
    run_case(Bench("city", 96, 54, config="city_4k"), moving=True, count_rays=True, tuning=tuning)


def test_tile_context():
    run_case(Bench("cornell", 96, 64, config="cornell_1080p"), moving=True, tile=(16, 48, 24, 80))


def test_cornell_1080p():
    """the benchmark's frame with the product library, counting rays off as in its timed region"""
    run_case(Bench("cornell", 1920, 1080, config="cornell_1080p"), flavor="product")


def test_two_cameras_on_one_animated_shared_scene():
    """two cameras, each as a serial and a concurrent context, on one scene updated once per frame on the scene's own stream"""
    a = Bench("cornell", 64, 64, config="cornell_1080p")
    b = Bench("cornell", 48, 40, config="cornell_1080p", indirect_spatial_reuse=0)
    b.world = a.world
    scene = plugin.SharedScene()
    scene.upload(a.world)
    pairs = []
    for bench in (a, b):
        pair = make_pair(lambda: plugin.HikariPlugin(bench.width, bench.height, 0), True, {})
        for d in pair:
            d.attach_scene(scene)
        pairs.append(pair)
    step, state = animate(cornell_animation, 4, 3), {}
    for f in range(1, 9):
        step(f, a, scene, [d for p in pairs for d in p], state)
        for bench, pair in zip((a, b), pairs):
            for d in pair:
                d.render_frame(bench.inputs(f))
        for cam, (bench, (serial, concurrent)) in enumerate(zip((a, b), pairs)):
            assert_same_frame(serial, concurrent, planes_of(bench), f, True, f"camera {cam}, ")
    for p in pairs:
        for d in p:
            d.close()
    scene.close()
