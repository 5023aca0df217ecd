"""The 4-wide TLAS of the image-exact traversal mode derived ON THE DEVICE by hk_scene_update_transforms (kc_build_wide_tlas,
csrc/kernels_scene.cu), so that a transform update never waits for the GPU while cameras walk the 4-wide trees.

  * record for record: after every device update, the nodes, instance ranks, root and stack need equal what wide_build.h's
    build_wide derives on the host from the flat TLAS the device built (tests/cuda/wide_build_ref.cpp), on the example scenes under
    animation and on random instance soups (1 to 600 instances, coincident centres, flat boxes);
  * images: frames after device updates equal frames after hk_scene_update_instances with host-built records, every plane, under
    HK_TUNE_WIDE_TRAVERSAL 1 and 3, for one camera and for a shared scene with two cameras on streams of their own;
  * a TLAS too deep for the walk's stack: the device says so (hk_get_stats) and every ray takes the reference's walk;
  * no host wait: the update returns while the stream is still busy with queued 4K frames, in about the time it takes on an idle
    device."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
import time

import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin
from tests.conftest import ROOT, Animation, Bench, city_animation, cornell_animation, needs_real_gpu, rotation_y_about
from tests.test_gpu_parity import ALL_PLANES, DENOISED
from tests.test_gpu_scene_update import material, soup_world, unit_cube

pytestmark = pytest.mark.gpu

WIDE_LEAF = 0x80000000
WIDE_STACK = 64        # HK_WIDE_STACK of the default build


def town_animation(bench):
    """scene.rs's emissive sphere at (2, 2, 0) spins and bobs (scene.rs:85-107), as every animated frame of that example"""
    em = int(bench.world.buffers()["emissives"]["instance"][0])
    return Animation(bench, {em: lambda f: rotation_y_about(0.1 * f, (2.0, 2.0, 0.0), (0.0, 0.05 * np.sin(0.5 * f), 0.0))})


ANIMATIONS = {"cornell": ("cornell_1080p", cornell_animation), "city": ("city_4k", city_animation), "town": ("scene_1080p", town_animation)}

_REF = None


def wide_ref():
    """tests/cuda/wide_build_ref.cpp compiled for the host (cached by source and header contents in the temporary directory)"""
    global _REF
    if _REF is None:
        src = os.path.join(ROOT, "tests", "cuda", "wide_build_ref.cpp")
        csrc = os.path.join(ROOT, "bevy_hikari_b200", "csrc")
        deps = [src] + [os.path.join(csrc, f) for f in ("wide_build.h", "hk_wide.cuh", "hk_device.cuh")] + \
               [os.path.join(ROOT, "include", f) for f in ("hk_layout.h", "hk_math.h")]
        h = hashlib.sha1(b"".join(open(p, "rb").read() for p in deps)).hexdigest()[:16]
        lib = os.path.join(tempfile.gettempdir(), f"hk_wide_build_ref_{os.getuid()}_{h}.so")
        if not os.path.exists(lib):
            tmp = lib + f".{os.getpid()}.tmp"
            subprocess.run([os.environ.get("HK_CXX", "g++"), "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-ffp-contract=off",
                            "-I", os.path.join(ROOT, "tests", "emu", "include"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                            src, "-o", tmp], check=True)
            os.replace(tmp, lib)
        _REF = C.CDLL(lib)
        _REF.wide_build_ref.restype = C.c_int
        _REF.wide_build_ref.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return _REF


def host_wide(flat, n):
    """build_wide(flat, len(flat), n, nullptr) as upload_wide_tlas keeps it: (nodes, ranks, root, stack need, ok)"""
    flat = np.ascontiguousarray(flat)
    nodes = np.zeros(max(n - 1, 1), L.WIDE_NODE)
    rank = np.zeros(n, np.uint32)
    count, root, need = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    ok = wide_ref().wide_build_ref(flat.ctypes.data, len(flat), n, nodes.ctypes.data, C.byref(count), rank.ctypes.data, C.byref(root),
                                   C.byref(need))
    return nodes[:count.value], rank, root.value, need.value, bool(ok)


class WideProbe:
    """what a camera reports about the scene's 4-wide TLAS, and the share of the stack need that is not the TLAS's (the BLAS marker,
    the meshes' trees and the slack): known from the upload, whose 4-wide TLAS the host derived"""

    def __init__(self, dev, n):
        self.dev, self.n = dev, n
        _, _, _, need, ok = host_wide(dev.scene_readback(L.SCENE_INSTANCE_NODES), n)
        assert ok
        self.base = dev.stats().wide_stack_need - need

    def check(self, what, mode=3):
        """the device's 4-wide TLAS equals the host derivation from the device's flat TLAS; returns the host's stack need"""
        dev, n = self.dev, self.n
        flat = dev.scene_readback(L.SCENE_INSTANCE_NODES)
        want_nodes, want_rank, root, need, ok = host_wide(flat, n)
        got_nodes = dev.scene_readback(L.SCENE_WIDE_TLAS)
        got_rank = dev.scene_readback(L.SCENE_WIDE_INSTANCE_RANK)
        assert len(got_nodes) == len(want_nodes), (what, len(got_nodes), len(want_nodes))
        if got_nodes.tobytes() != want_nodes.tobytes():
            g, h = got_nodes.view(np.uint32).reshape(len(got_nodes), -1), want_nodes.view(np.uint32).reshape(len(want_nodes), -1)
            bad = np.nonzero((g != h).any(axis=1))[0]
            raise AssertionError(f"{what}: {len(bad)} of {len(got_nodes)} wide nodes differ, first {bad[0]}:\n device {got_nodes[bad[0]]}\n host   {want_nodes[bad[0]]}")
        assert np.array_equal(got_rank, want_rank), (what, np.nonzero(got_rank != want_rank)[0][:8])
        assert ok and root == (0 if n > 1 else WIDE_LEAF), (what, ok, hex(root))    # the root the update hands the walk
        st = dev.stats()
        assert st.wide_stack_need == need + self.base, (what, st.wide_stack_need, need, self.base)
        assert st.wide_traversal == (mode if need + self.base <= WIDE_STACK else 0), (what, st.wide_traversal, need + self.base)
        return need


def wide_device(bench, mode=3, stream=None):
    p = plugin.HikariPlugin(bench.width, bench.height, 0, 0, None, stream)
    p.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, mode)
    p.upload_scene(bench.world)
    return p


def move(anim, f):
    w = anim.bench.world
    for i, track in anim.tracks.items():
        w.set_instance_transform(i, anim.compose(track(f), anim.base[i]))
    w.previous_transform_system()
    return w


@pytest.mark.parametrize("scene", ["cornell", "city", "town"])
def test_device_wide_tlas_equals_the_host_derivation_under_animation(scene):
    config, animation = ANIMATIONS[scene]
    b = Bench(scene, 32, 24, config=config)
    dev = wide_device(b)
    n = len(b.world.buffers()["instances"])
    probe = WideProbe(dev, n)
    anim = animation(b)
    for f in range(1, 7):
        assert dev.update_transforms(move(anim, f)), f
        probe.check(f"{scene} frame {f}")
    dev.close()


@pytest.mark.parametrize("n,kind,seed", [(1, "random", 11), (2, "random", 12), (3, "coincident", 13), (4, "random", 14), (5, "flat", 15),
                                         (5, "coincident", 16), (17, "random", 17), (17, "flat", 18), (600, "random", 19)])
def test_random_instance_soups(n, kind, seed):
    rng = np.random.default_rng(seed)
    w = soup_world(rng, n, kind)
    dev = plugin.HikariPlugin(32, 24, 0, 0, None, None, 0, None)
    dev.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 3)
    dev.upload_scene(w)
    probe = WideProbe(dev, n)
    for step in range(3):
        for i in range(n):
            if rng.random() < 0.6:
                cur = w.buffers()["instances"]["model"][i].reshape(4, 4).T.astype(np.float64)
                ang = rng.uniform(-0.3, 0.3)
                c, s = np.cos(ang), np.sin(ang)
                cur = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]) @ cur
                if kind != "coincident":
                    cur[:3, 3] += rng.uniform(-1.0, 1.0, 3)
                w.set_instance_transform(i, cur.T.astype(np.float32).reshape(16).copy())
        w.previous_transform_system()
        assert dev.update_transforms(w), (n, kind, step)
        probe.check(f"{kind} n={n} step {step}")
    dev.close()


def snapshot(dev, planes):
    return {k: dev.readback(k).tobytes() for k in planes}


def assert_same(a, b, what):
    bad = [k for k in a if a[k] != b[k]]
    assert not bad, f"{what}: planes that differ {bad}"


@pytest.mark.parametrize("mode", [1, 3])
@pytest.mark.parametrize("scene", ["city", "town"])
def test_frames_after_device_updates_equal_frames_after_host_updates(scene, mode):
    config, animation = ANIMATIONS[scene]
    b = Bench(scene, 64, 48, config=config)
    on_device, on_host = wide_device(b, mode), wide_device(b, mode)
    for d in (on_device, on_host):
        d.set_keep_intermediates(True)
    anim = animation(b)
    for f in range(1, 7):
        w = move(anim, f)
        assert on_device.update_transforms(w)
        w.prepare_instances()
        on_host.update_instances(w)
        inp = b.inputs(f)
        on_device.render_frame(inp); on_host.render_frame(inp)
        assert on_device.stats().wide_traversal == on_host.stats().wide_traversal != 0
        assert_same(snapshot(on_device, ALL_PLANES + DENOISED), snapshot(on_host, ALL_PLANES + DENOISED), f"{scene} mode {mode} frame {f}")
    on_device.close(); on_host.close()


def test_shared_scene_two_cameras_on_their_own_streams():
    """one SharedScene (own stream) updated on the device, two cameras (one walking the 4-wide trees for every ray, one for primary
    rays) on streams of their own, against the same cameras with private scenes updated through the host path"""
    config, animation = ANIMATIONS["city"]
    benches = [Bench("city", 64, 48, config=config), Bench("city", 48, 40, config=config, indirect_bounces=2, denoise=1)]
    modes = (3, 1)
    scene = plugin.SharedScene()
    scene.upload(benches[0].world)
    shared = []
    for b, m in zip(benches, modes):
        p = plugin.HikariPlugin(b.width, b.height)
        p.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, m)
        p.set_keep_intermediates(True)
        p.attach_scene(scene)
        shared.append(p)
    private = []
    for b, m in zip(benches, modes):
        p = wide_device(b, m)
        p.set_keep_intermediates(True)
        private.append(p)
    anims = [animation(b) for b in benches]
    for f in range(1, 7):
        w0 = move(anims[0], f)
        assert scene.update_transforms(w0)
        w0.prepare_instances()
        w1 = move(anims[1], f)
        w1.prepare_instances()
        for p, b in zip(private, benches):
            p.update_instances(b.world)
        for s, p, b in zip(shared, private, benches):
            s.render_frame(b.inputs(f)); p.render_frame(b.inputs(f))
        for cam, (s, p) in enumerate(zip(shared, private)):
            assert s.stats().wide_traversal == p.stats().wide_traversal != 0
            assert_same(snapshot(s, ALL_PLANES + DENOISED), snapshot(p, ALL_PLANES + DENOISED), f"frame {f} camera {cam}")
    for p in shared + private:
        p.close()
    scene.close()


def chain_models(n, ratio, first):
    """n boxes along +x whose centres grow by `ratio` from one to the next, from ratio ** -first on: bvh 0.7.1's SAH build splits off
    the farthest box at almost every level, so the TLAS is a chain and its 4-wide tree needs about one stack entry per instance"""
    models = []
    for i in range(n):
        t = np.eye(4, dtype=np.float64)
        x = ratio ** (i - first)
        t[0, 0] = 0.05 * x                  # the box grows with its distance: its centre stays apart from its neighbours'
        t[:3, 3] = (x, 0.0, 0.0)
        models.append(t.T.astype(np.float32).reshape(16).copy())
    return models


def test_tlas_deeper_than_the_stack_takes_the_reference_walk():
    """a soup whose TLAS fits the walk at upload, then moves into a chain whose 4-wide TLAS needs more than HK_WIDE_STACK entries:
    the device derives the tree, finds it too deep and every launch walks the flat arrays — frames and rays equal those of a camera
    that never walks the 4-wide trees; back to a shallow TLAS, the 4-wide walk resumes"""
    rng = np.random.default_rng(21)
    n, ratio, first = 84, 6.5, 39
    w = plugin.World()                  # no emissive instance: a rescaled light would take the host path (its alias table)
    mesh, plain = w.add_mesh(*unit_cube()), w.add_material(material())
    for i in range(n):
        t = np.eye(4, dtype=np.float32)
        t[:3, 3] = rng.uniform(-20, 20, 3)
        w.add_instance(mesh, plain, t.T.reshape(16).copy())
    w.prepare()
    base = [w.buffers()["instances"]["model"][i].copy() for i in range(n)]
    b = Bench("cornell", 48, 40, config="cornell_256")
    wide, flat = (plugin.HikariPlugin(48, 40) for _ in range(2))
    wide.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 3)
    flat.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 0)
    for d in (wide, flat):
        d.set_keep_intermediates(True)
        d.upload_scene(w)
    probe = WideProbe(wide, n)
    assert wide.stats().wide_traversal == 3
    rays = np.zeros(4000, L.RAY)                   # towards the boxes of the chain around x = 1
    x = ratio ** rng.integers(-1, 3, 4000).astype(np.float64)
    rays["origin"] = np.stack([x * (1.0 + rng.uniform(-0.02, 0.02, 4000)), rng.uniform(-0.6, 0.6, 4000), np.full(4000, 6.0)], 1).astype(np.float32)
    d = np.stack([rng.uniform(-1e-3, 1e-3, 4000), rng.uniform(-0.05, 0.05, 4000), -np.ones(4000)], 1)
    rays["direction"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["max_distance"] = np.float32(3.402823466e38)
    rays["exclude_instance"] = 0xFFFFFFFF
    for f, models in enumerate([chain_models(n, ratio, first), base], 1):
        for i, m in enumerate(models):
            w.set_instance_transform(i, m)
        w.previous_transform_system()
        arrays = w.prepare_instance_transforms()
        assert arrays is not None, f
        models_, previous, aabbs = arrays
        for d in (wide, flat):
            d.update_transforms_arrays(models_, aabbs, previous)
        need = probe.check(f"step {f}")
        deep = need + probe.base > WIDE_STACK
        assert deep == (f == 1), (f, need, probe.base)
        st = wide.stats()
        assert st.wide_traversal == (0 if deep else 3) and (st.wide_stack_need > WIDE_STACK) == deep
        hw, hf = wide.trace_rays(rays), flat.trace_rays(rays)
        if deep:
            assert (hf["instance_index"] != 0xFFFFFFFF).sum() > 1000
            assert hw.tobytes() == hf.tobytes()
        inp = b.inputs(f)
        wide.render_frame(inp); flat.render_frame(inp)
        if deep:
            assert_same(snapshot(wide, ALL_PLANES + DENOISED), snapshot(flat, ALL_PLANES + DENOISED), f"deep step {f}")
    wide.close(); flat.close()


def test_update_returns_while_4k_frames_are_in_flight():
    """queue 4K city frames, then update: the call must not wait for them (the stream is still busy when it returns) and its host
    time must be about what it is on an idle device.  The same for a shared scene whose cameras run on other streams."""
    needs_real_gpu()
    import torch
    torch.cuda.init()
    b = Bench("city", 3840, 2160, config="city_4k")
    anim = city_animation(b)
    s_cam, s_cam2, s_scene = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()

    def update_host_ms(update, f, streams, queue):
        w = move(anim, f)
        models, previous, aabbs = w.prepare_instance_transforms()
        queue()
        t0 = time.perf_counter()
        update(models, aabbs, previous)
        ms = 1e3 * (time.perf_counter() - t0)
        busy = [not s.query() for s in streams]
        return ms, busy

    def measure(update, render, streams):
        """median host ms of an update on an idle device, and with three frames queued behind a synchronisation (so that the pinned
        staging slot of two calls before has landed: what is left to wait for are the frames in flight)"""
        f = 1
        for _ in range(3):                           # warm-up: staging slots and scratch are allocated by the first calls
            f += 1
            update_host_ms(update, f, streams, render)
        torch.cuda.synchronize()
        idle, flight = [], []
        for _ in range(5):
            f += 1
            torch.cuda.synchronize()
            idle.append(update_host_ms(update, f, streams, lambda: None)[0])
            render()
            f += 1
            torch.cuda.synchronize()
            ms, busy = update_host_ms(update, f, streams, lambda: [render() for _ in range(3)])
            assert all(busy), busy
            flight.append(ms)
        torch.cuda.synchronize()
        return float(np.median(idle)), float(np.median(flight))

    dev = wide_device(b, 1, s_cam.cuda_stream)
    assert dev.stats().wide_traversal == 1
    frame = [0]

    def render_one():
        frame[0] += 1
        dev.render_frame(b.inputs(frame[0]))
    idle, flight = measure(lambda m, a, p: dev.update_transforms_arrays(m, a, p), render_one, [s_cam])
    assert flight < 3.0 * idle + 2.0, (idle, flight)
    dev.close()

    scene = plugin.SharedScene(0, s_scene.cuda_stream)
    scene.upload(b.world)
    cams = []
    for s in (s_cam, s_cam2):
        p = plugin.HikariPlugin(3840, 2160, 0, 0, None, s.cuda_stream)
        p.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 1)
        p.attach_scene(scene)
        cams.append(p)

    def render_both():
        frame[0] += 1
        for p in cams:
            p.render_frame(b.inputs(frame[0]))
    idle, flight = measure(lambda m, a, p: scene.update_transforms_arrays(m, a, p), render_both, [s_cam, s_cam2])
    assert flight < 3.0 * idle + 2.0, (idle, flight)
    assert all(p.stats().wide_traversal == 1 for p in cams)
    for p in cams:
        p.close()
    scene.close()
