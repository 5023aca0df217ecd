"""Shared scenes (hk_shared_scene): several cameras render ONE scene that is uploaded and animated once per frame, as the reference's
single MeshMaterialBindGroup is bound by every camera.  Each case renders the same cameras twice — every camera with a private upload
of the scene, then every camera attached to one SharedScene — and requires every plane of every frame to be bit-equal: both arms run
the same kernels on the same scene buffers.  The library creates a stream per context and per shared scene, so the shared arm also
runs the scene's uploads and updates on another stream than each camera's frames."""
import ctypes as C

import numpy as np
import pytest

from bevy_hikari_b200 import _ffi
from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin
from tests.conftest import Bench, city_animation, cornell_animation, needs_real_gpu, orthographic_inputs
from tests.test_gpu_parity import ALL_PLANES, DENOISED

pytestmark = pytest.mark.gpu


class Camera:
    """one view of the scene: size, view and settings (a Bench), and per-camera switches"""

    def __init__(self, bench, inputs=None, upscalers=False, wide=None):
        self.bench, self.inputs, self.upscalers, self.wide = bench, inputs or bench.inputs, upscalers, wide

    def device(self, world, flavor=None, upload=True):
        b = self.bench
        p = plugin.HikariPlugin(b.width, b.height, 0, flavor=flavor)
        p.set_keep_intermediates(True)
        if self.wide is not None:
            p.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, self.wide)
        if upload:
            p.upload_scene(world)
        return p

    def frame_inputs(self, f):
        inp = self.inputs(f)
        inp.temporal_upscalers = 1 if self.upscalers else 0
        return inp

    def planes(self):
        return ALL_PLANES + DENOISED + ([L.OUT_UPSCALED, L.OUT_TAA] if self.upscalers else [])


def snapshot(dev, planes):
    return {k: dev.readback(k).tobytes() for k in planes}


def two_cameras(scene, config, wide=(None, None), upscalers=False):
    """camera 0: 64 x 64 perspective, the config's settings; camera 1: 48 x 40 orthographic, 2 bounces, denoise, spatial reuse"""
    a = Bench(scene, 64, 64, config=config)
    kw = dict(taa=plugin.TAA_JASMINE) if upscalers else {}
    b = Bench(scene, 48, 40, config=config, indirect_bounces=2, denoise=1, indirect_spatial_reuse=1, emissive_spatial_reuse=1, **kw)
    cams = [Camera(a, wide=wide[0]), Camera(b, inputs=lambda f: orthographic_inputs(b, f, shift=(0.01, 0.0, 0.0)), upscalers=upscalers,
                                            wide=wide[1])]
    return a, cams


def animate(make_animation, hide_at, hide_entity):
    """per frame: the tracks move their instances; at frame `hide_at` an instance is hidden, which changes the kept set and forces
    the host path (prepare_instances + update_instances).  Shared arm: ONE update_transforms on the scene; private arm: the same
    arrays (or the host path) into every camera's own scene."""
    def step(f, bench, scene, devs, state):
        if "anim" not in state:
            state["anim"] = make_animation(bench)
        an, w = state["anim"], bench.world
        for i, track in an.tracks.items():
            w.set_instance_transform(i, an.compose(track(f), an.base[i]))
        if f == hide_at:
            w.set_instance_visible(hide_entity, False)
        w.previous_transform_system()
        if scene is not None:
            assert scene.update_transforms(w) == (f != hide_at), f
            return
        arrays = w.prepare_instance_transforms()
        assert (arrays is None) == (f == hide_at), f
        if arrays is None:
            w.prepare_instances()
            for d in devs:
                d.update_instances(w)
        else:
            models, previous, aabbs = arrays
            for d in devs:
                d.update_transforms_arrays(models, aabbs, previous)
    return step


def render_arms(make, frames, update=None, flavor=None, every_frame=True):
    """renders the cameras of make() for `frames` frames with a private scene per camera, then with one SharedScene; returns the
    read-backs of both arms (of every frame, or of the last frame only: then nothing synchronises the host before the end)"""
    arms = []
    for shared in (False, True):
        bench, cams = make()
        devs = [c.device(bench.world, flavor, upload=not shared) for c in cams]
        scene = None
        if shared:
            scene = plugin.SharedScene(0, None, flavor=flavor)
            scene.upload(bench.world)
            for d in devs:
                d.attach_scene(scene)
        state, snaps = {}, []
        for f in range(1, frames + 1):
            if update:
                update(f, bench, scene, devs, state)
            for d, c in zip(devs, cams):
                d.render_frame(c.frame_inputs(f))
            if every_frame or f == frames:
                snaps.append([snapshot(d, c.planes()) for d, c in zip(devs, cams)])
        arms.append(snaps)
        for d in devs:
            d.close()
        if scene is not None:
            scene.close()
    return arms


def assert_arms_equal(arms):
    private, shared = arms
    assert len(private) == len(shared)
    for f, (pf, sf) in enumerate(zip(private, shared)):
        for cam, (p, s) in enumerate(zip(pf, sf)):
            bad = [k for k in p if p[k] != s[k]]
            assert not bad, f"frame {f + 1}, camera {cam}: planes that differ {bad}"


def test_two_cameras_static_scene():
    assert_arms_equal(render_arms(lambda: two_cameras("cornell", "cornell_256"), 6))


def test_two_cameras_with_upscalers():
    """the second camera runs the reference's default tail (SMAA TU4x + TAA) on the shared scene"""
    assert_arms_equal(render_arms(lambda: two_cameras("cornell", "cornell_256", upscalers=True), 4))


@pytest.mark.parametrize("scene,config,animation,hide", [("cornell", "cornell_1080p", cornell_animation, 3),
                                                          ("city", "city_4k", city_animation, 5)])
def test_animated_scene_one_update_per_frame(scene, config, animation, hide):
    assert_arms_equal(render_arms(lambda: two_cameras(scene, config), 8, animate(animation, 4, hide)))


@pytest.mark.parametrize("scene,config,animation,hide", [("cornell", "cornell_1080p", cornell_animation, 3),
                                                          ("city", "city_4k", city_animation, 5)])
def test_animated_scene_wide_and_flat_cameras(scene, config, animation, hide):
    """one camera walks the 4-wide trees (HK_TUNE_WIDE_TRAVERSAL 3), the other the reference's arrays: the shared update re-derives
    the 4-wide TLAS for the first and the flat walk stays exact for the second"""
    arms = render_arms(lambda: two_cameras(scene, config, wide=(3, 0)), 8, animate(animation, 4, hide))
    assert_arms_equal(arms)


def test_back_to_back_frames_and_updates_on_separate_streams():
    """the scene and both cameras each on a stream of their own; frames and scene updates are issued back to back and nothing
    synchronises the host before the final read-backs: only the events between the streams order the updates and the frames"""
    arms = render_arms(lambda: two_cameras("city", "city_4k"), 8, animate(city_animation, 4, 5), every_frame=False)
    assert_arms_equal(arms)


def test_tiles_share_one_scene_and_one_frame_target():
    W, H = 160, 96
    tiles = [(0, 88, 0, 96), (88, 160, 0, 96)]
    b = Bench("cornell", W, H, config="cornell_1080p")
    full = b.device()
    frames = [full.frame_alloc()[0], full.frame_alloc()[0]]
    scene = plugin.SharedScene()
    scene.upload(b.world)
    devs = []
    for c0, c1, r0, r1 in tiles:
        d = plugin.HikariPlugin(W, H, 0, r0, r1, None, c0, c1)
        d.attach_scene(scene)
        devs.append(d)
    for f in range(1, 6):
        inp = b.inputs(f)
        full.render_frame(inp)
        for d in devs:
            d.set_frame_target(frames[f & 1], W)
            d.render_frame(inp)
        for d in devs:
            d.sync()
        assert full.frame_read(frames[f & 1]).tobytes() == full.readback(L.OUT_TONE_MAPPED).tobytes(), f


def test_life_cycle():
    b = Bench("cornell", 48, 40, config="cornell_256")
    ref = b.device()
    ref.set_keep_intermediates(True)
    scene = plugin.SharedScene()
    scene.upload(b.world)
    cams = []
    for _ in range(2):
        p = plugin.HikariPlugin(48, 40)
        p.set_keep_intermediates(True)
        p.attach_scene(scene)
        cams.append(p)
    scene.close()                       # the handle is gone: the attached cameras keep rendering the scene
    planes = ALL_PLANES + DENOISED
    for f in range(1, 4):
        inp = b.inputs(f)
        for d in [ref] + cams:
            d.render_frame(inp)
        want = snapshot(ref, planes)
        for d in cams:
            assert snapshot(d, planes) == want, f
    # updates through a context of a shared scene are refused and leave the scene (hence the frames) as they were
    models, previous, aabbs = b.world.prepare_instance_transforms()
    for attempt in (lambda: cams[0].upload_scene(b.world), lambda: cams[0].update_instances(b.world),
                    lambda: cams[0].update_transforms_arrays(models + np.float32(0.5), aabbs, previous)):
        with pytest.raises(_ffi.HikariError, match="shared scene"):
            attempt()
    with pytest.raises(_ffi.HikariError, match="shared scene"):
        cams[0].update_transforms(b.world)
    inp = b.inputs(4)
    for d in [ref] + cams:
        d.render_frame(inp)
    want = snapshot(ref, planes)
    for d in cams:
        assert snapshot(d, planes) == want
    # detaching: the frame calls answer NOT_READY, as on a context that never had a scene; the last detach frees the scene
    for d in cams:
        d.attach_scene(None)
        assert d._lib.hk_render_frame(d.ctx, C.byref(b.inputs(5))) == _ffi.HK_ERR_NOT_READY
        assert d._lib.hk_prepass_run(d.ctx, C.byref(b.inputs(5))) == _ffi.HK_ERR_NOT_READY
    # a detached camera is back to a private scene of its own
    cams[0].upload_scene(b.world)
    cams[0].render_frame(b.inputs(5))
    # attach after a resize: a new scene, the second camera re-sized to 64 x 48, against a private 64 x 48 camera
    b2 = Bench("cornell", 64, 48, config="cornell_256")
    ref2 = b2.device()
    scene2 = plugin.SharedScene()
    scene2.upload(b2.world)
    cam = cams[1]
    assert cam._lib.hk_context_resize(cam.ctx, 64, 48, 0, 48) == _ffi.HK_OK
    cam.attach_scene(scene2)
    for f in range(1, 4):
        ref2.render_frame(b2.inputs(f))
        cam.render_frame(b2.inputs(f))
    assert snapshot(cam, ALL_PLANES) == snapshot(ref2, ALL_PLANES)
    scene2.close()


def test_attach_keeps_the_reservoirs():
    """attaching a scene does not reset temporal state: a camera that switches from its private upload to a shared copy of the same
    scene mid-sequence renders exactly what a camera that never switched renders"""
    b = Bench("cornell", 48, 40, config="cornell_256")
    ref, dev = b.device(), b.device()
    scene = plugin.SharedScene()
    scene.upload(b.world)
    for f in range(1, 7):
        if f == 4:
            dev.attach_scene(scene)
        ref.render_frame(b.inputs(f))
        dev.render_frame(b.inputs(f))
    assert snapshot(dev, ALL_PLANES) == snapshot(ref, ALL_PLANES)


def test_scene_of_another_device_is_refused():
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    b = Bench("cornell", 32, 24, config="cornell_256")
    scene = plugin.SharedScene(1)
    scene.upload(b.world)
    dev = b.device()
    with pytest.raises(_ffi.HikariError, match="another device"):
        dev.attach_scene(scene)
    dev.render_frame(b.inputs(1))        # the context keeps its own scene


def test_second_camera_allocates_its_planes_and_nothing_of_the_scene():
    """textured city (14 textures): a private camera pays its planes + the whole scene, an attached one only its planes"""
    needs_real_gpu()
    import torch
    torch.cuda.init()

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info(0)[0]
    b = Bench("city", 320, 180, config="city_4k")
    first = b.device()                                   # a camera with the scene, so that CUDA and the library are initialised
    f0 = free()
    scene = plugin.SharedScene()
    scene.upload(b.world)
    f1 = free()
    scene_bytes = f0 - f1
    assert scene_bytes > 1 << 20, scene_bytes
    private = b.device()
    f2 = free()
    private_bytes = f1 - f2
    attached = plugin.HikariPlugin(320, 180)
    attached.attach_scene(scene)
    f3 = free()
    attached_bytes = f2 - f3
    assert private_bytes - attached_bytes >= 0.9 * scene_bytes, (scene_bytes, private_bytes, attached_bytes)
    attached.render_frame(b.inputs(1))
    scene.close()
    attached.close()                                     # the last detach frees the scene
    f4 = free()
    assert f4 - f3 >= 0.9 * (scene_bytes + attached_bytes), (f3, f4, scene_bytes, attached_bytes)
    first.close(); private.close()


def test_product_flavour_shared_equals_private():
    """the product library (tolerance build): shared and private scenes still run the same kernels on the same buffers"""
    assert_arms_equal(render_arms(lambda: two_cameras("cornell", "cornell_256"), 5, flavor="product"))
