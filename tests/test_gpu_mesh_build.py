"""Meshes added to a live scene and built on the device (hk_scene_add_meshes, csrc/kernels_scene.cu): GpuMesh::try_from
(mod.rs:379-467) — vertex and primitive records and bvh 0.7.1's SAH build + flatten_custom of every mesh's BLAS — for meshes that
arrive while the app runs (mesh.rs:106-166 does this on the CPU and can stall a frame).

Held against the host mirror (host/hikari.cpp, the reference's CPU path): the vertex, primitive and BLAS buffers read back after the
call equal, byte for byte, those of a world that holds the same meshes in the same order, and so do the returned hk_mesh_index
records; on every mesh of the committed scenes and on meshes made for the builder's corners (one and two primitives, coincident
centroids, flat meshes with -0 and +0 on the flat axis, strips, non-finite positions, a seeded mesh of a million triangles).  Frames of
a scene whose meshes were added on the device equal frames of the same scene uploaded by the host, for both walks."""
import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin, scenes
from tests.conftest import EMULATED, Bench

pytestmark = pytest.mark.gpu

READBACK = [(L.SCENE_VERTICES, "vertices"), (L.SCENE_PRIMITIVES, "primitives"), (L.SCENE_ASSET_NODES, "asset_nodes")]
DEFAULT_MATERIAL = np.zeros((), L.MATERIAL)
for _k in ("base_color_texture", "emissive_texture", "metallic_roughness_texture", "normal_map_texture", "occlusion_texture"):
    DEFAULT_MATERIAL[_k] = 0xFFFFFFFF


def base_world():
    """a scene of one small mesh, uploaded before the meshes under test are added"""
    w = plugin.World()
    w.add_mesh(*scenes._plane_mesh(1.0))
    w.add_material(DEFAULT_MATERIAL)
    w.add_instance(0, 0, np.eye(4, dtype=np.float32).reshape(16))
    w.prepare()
    return w


def mirror(meshes):
    """the host mirror's buffers and mesh indices for the base mesh followed by `meshes`"""
    w = plugin.World()
    w.add_mesh(*scenes._plane_mesh(1.0))
    for m in meshes:
        nv = min(len(m[0]), len(m[1]), len(m[2]))        # the world takes one vertex count: the multizip rule applied here
        w.add_mesh(m[0][:nv], m[1][:nv], m[2][:nv], m[3] if len(m) > 3 else None, m[4] if len(m) > 4 else 0)
    w.add_material(DEFAULT_MATERIAL)
    for i in range(len(meshes) + 1):
        w.add_instance(i, 0, np.eye(4, dtype=np.float32).reshape(16))
    w.prepare()
    for i in range(len(meshes) + 1):
        assert w.mesh_error(i) == 0, f"mesh {i} is refused by the host mirror"
    b = w.buffers()
    return b, b["instances"]["mesh"][1:]


def assert_bytes_equal(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    for field in got.dtype.names:       # field by field, bitwise (numpy's copies of padded records do not carry the padding bytes)
        g = np.ascontiguousarray(got[field]).view(np.uint32).reshape(len(got), -1)
        h = np.ascontiguousarray(want[field]).view(np.uint32).reshape(len(want), -1)
        bad = np.nonzero((g != h).any(axis=1))[0]
        if len(bad):
            raise AssertionError(f"{what}.{field} differs in {len(bad)} of {len(got)} records, first {bad[0]}:\n device {got[bad[0]]}\n host   {want[bad[0]]}")


def assert_added_equal_the_mirror(dev, meshes, got_index, what):
    host, want_index = mirror(meshes)
    assert_bytes_equal(got_index, want_index, f"{what}: mesh index")
    for which, name in READBACK:
        assert_bytes_equal(dev.scene_readback(which), host[name], f"{what}: {name}")


def scene_meshes(name):
    return [m for m in scenes._load_npz(name)[0]]


def quad_grid(n, z=0.0, seed=0):
    """n x n quads on the plane z (two triangles each), some vertices at -0 and some at +0 on the flat axis"""
    rng = np.random.default_rng(seed)
    xs, ys = np.meshgrid(np.arange(n + 1, dtype=np.float32), np.arange(n + 1, dtype=np.float32))
    pos = np.stack([xs.ravel() * 0.1, ys.ravel() * 0.1, np.full(xs.size, z, np.float32)], 1).astype(np.float32)
    if z == 0.0:
        pos[rng.random(len(pos)) < 0.5, 2] = -0.0
    q = (np.arange(n)[None, :] + (n + 1) * np.arange(n)[:, None]).ravel()
    idx = np.stack([q, q + 1, q + n + 2, q, q + n + 2, q + n + 1], 1).astype(np.uint32).ravel()
    nrm = np.tile(np.float32([0, 0, 1]), (len(pos), 1))
    return (pos, nrm, pos[:, :2].copy(), idx)


def soup(tris, seed, spread=10.0):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-spread, spread, (tris, 3)).astype(np.float32)
    pos = (centres[:, None, :] + rng.normal(0, 0.05, (tris, 3, 3))).astype(np.float32).reshape(-1, 3)
    nrm = rng.normal(size=pos.shape).astype(np.float32)
    uv = rng.random((len(pos), 2)).astype(np.float32)
    return (pos, nrm, uv, None)


# The two meshes above BLAS_TOP_SHAPES (4096), whose top levels a whole CTA splits: 5000 and 45 000 triangles on the device, just
# over 4096 on the emulated kernels, whose fibers take about 5 ms per primitive (tests/test_mesh_build_edges_emulated.py holds the
# CTA-level edges at those sizes)
LARGE_SOUP, LARGE_GRID = (4100, 46) if EMULATED else (5000, 150)


def edge_meshes():
    one = (np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]]), np.float32([[0, 0, 1]] * 3), np.float32([[0, 0]] * 3), np.uint32([0, 1, 2]))
    two = (np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]]), np.float32([[0, 0, 1]] * 4), np.float32([[0, 0]] * 4),
           np.uint32([0, 1, 2, 2, 1, 3]))
    same = soup(1, 1)
    coincident = (np.tile(same[0], (37, 1)), np.tile(same[1], (37, 1)), np.tile(same[2], (37, 1)), None)      # the half split
    strip_pos = np.float32([[i * 0.3, (i & 1) * 0.5, 0.01 * i * i] for i in range(40)])
    strip_even = (strip_pos, strip_pos, strip_pos[:, :2], np.arange(40, dtype=np.uint32)[::-1].copy(), L.TOPOLOGY_TRIANGLE_STRIP)
    strip_odd = (strip_pos[:39], strip_pos[:39], strip_pos[:39, :2], None, L.TOPOLOGY_TRIANGLE_STRIP)
    nonfinite = list(soup(300, 2))
    p = nonfinite[0].copy()
    p[5] = [np.inf, 0, 0]; p[17] = [np.nan, 1, 2]; p[40, 1] = -np.inf; p[41] = [np.nan] * 3
    nonfinite[0] = p
    uneven = (soup(50, 3)[0], soup(50, 3)[1][:120], soup(50, 3)[2][:100], np.arange(99, dtype=np.uint32))   # multizip: 100 vertices
    return {"one": one, "two": two, "coincident": coincident, "flat_signed_zeros": quad_grid(40), "flat_z1": quad_grid(9, z=1.0),
            "strip_even": strip_even, "strip_odd": strip_odd, "nonfinite": tuple(nonfinite), "uneven_attributes": uneven,
            "soup_5000": soup(LARGE_SOUP, 4), "flat_large": quad_grid(LARGE_GRID)}


def fresh_device(width=16, height=16):
    dev = plugin.HikariPlugin(width, height)
    dev.upload_scene(base_world())
    return dev


@pytest.mark.parametrize("scene", ["cornell", "house", "house2", "house3", "town"])
def test_scene_meshes_equal_the_host_mirror(scene):
    meshes = scene_meshes(scene)
    dev = fresh_device()
    got = dev.add_mesh_sources(meshes)
    assert_added_equal_the_mirror(dev, meshes, got, scene)
    dev.close()


@pytest.mark.parametrize("case", sorted(edge_meshes()))
def test_edge_meshes_equal_the_host_mirror(case):
    mesh = edge_meshes()[case]
    dev = fresh_device()
    got = dev.add_mesh_sources([mesh])
    assert_added_equal_the_mirror(dev, [mesh], got, case)
    dev.close()


def test_meshes_added_in_several_calls_equal_one_world():
    """each call appends: buffers grow (and are replaced) between calls"""
    e = edge_meshes()
    batches = [[e["one"], e["strip_odd"]], [e["soup_5000"]], [e["two"], e["flat_large"], e["coincident"]]]
    dev = fresh_device()
    got = np.concatenate([dev.add_mesh_sources(b) for b in batches])
    assert_added_equal_the_mirror(dev, [m for b in batches for m in b], got, "three calls")
    dev.close()


def test_a_million_triangles_equal_the_host_mirror():
    mesh = soup(1 << 20, 11, spread=100.0)
    dev = fresh_device()
    got = dev.add_mesh_sources([mesh])
    assert_added_equal_the_mirror(dev, [mesh], got, "1M soup")
    dev.close()


def test_shared_scene_with_two_cameras():
    meshes = scene_meshes("cornell") + [edge_meshes()["flat_large"]]
    scene = plugin.SharedScene()
    scene.upload(base_world())
    cams = [plugin.HikariPlugin(16, 16), plugin.HikariPlugin(24, 8)]
    for c in cams:
        c.attach_scene(scene)
    got = scene.add_mesh_sources(meshes)
    for i, c in enumerate(cams):
        assert_added_equal_the_mirror(c, meshes, got, f"shared scene, camera {i}")
    for c in cams:
        c.close()
    scene.close()


REFUSALS = {
    "missing_positions": lambda m: (m[0][:0], m[1], m[2], m[3]),
    "missing_normals": lambda m: (m[0], m[1][:0], m[2], m[3]),
    "missing_uvs": lambda m: (m[0], m[1], m[2][:0], m[3]),
    "short_chunk": lambda m: (m[0], m[1], m[2], m[3][:-1]),
    "unknown_topology": lambda m: (m[0], m[1], m[2], m[3], 7),
    "no_primitive": lambda m: (m[0], m[1], m[2], m[3][:0]),
    "strip_of_two": lambda m: (m[0], m[1], m[2], m[3][:2], L.TOPOLOGY_TRIANGLE_STRIP),
    "index_out_of_range": lambda m: (m[0], m[1], m[2], np.concatenate([m[3][:-1], [len(m[0])]]).astype(np.uint32)),
    "index_beyond_the_shortest_attribute": lambda m: (m[0], m[1], m[2][:-1], m[3]),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_malformed_meshes_are_refused_and_the_scene_renders_as_before(case):
    b = Bench("cornell", 32, 24, config="cornell_256")
    good = scene_meshes("cornell")[1]
    bad = REFUSALS[case](good)
    ref, dev = b.device(), b.device()
    before = {name: dev.scene_readback(which) for which, name in READBACK}
    with pytest.raises(RuntimeError):
        dev.add_mesh_sources([good, bad])        # the whole call is refused: not even the good mesh is added
    for which, name in READBACK:
        assert_bytes_equal(dev.scene_readback(which), before[name], f"{case}: {name} after the refusal")
    for f in range(1, 3):
        ref.render_frame(b.inputs(f)); dev.render_frame(b.inputs(f))
        for k in (L.OUT_TONE_MAPPED, L.OUT_GBUFFER_INSTANCE_MATERIAL):
            assert np.array_equal(dev.readback(k), ref.readback(k)), (case, f, k)
    got = dev.add_mesh_sources([good])       # and the next valid call works
    assert got[0]["primitive"] == len(before["primitives"])
    ref.close(); dev.close()


def split_world(bench, first_added):
    """the bench's scene as a world in which meshes [first_added, ..) are device meshes (their BVH is never built on the host) and
    their instances are hidden until those meshes are on the device"""
    sc = bench.scene
    w = plugin.World()
    for t in sc.textures:
        w.add_texture(t["rgba"], t["address_mode_u"], t["address_mode_v"], t["filter_linear"], t["srgb"])
    for i, m in enumerate(sc.meshes):
        (w.add_mesh if i < first_added else w.add_device_mesh)(*m)
    for m in sc.materials:
        w.add_material(m)
    for me, ma, xf in zip(sc.inst_mesh, sc.inst_material, sc.inst_transform):
        w.add_instance(int(me), int(ma), xf, int(me) < first_added)
    w.prepare()
    return w


def show_device_instances(world, bench, first_added):
    for i, me in enumerate(bench.scene.inst_mesh):
        if int(me) >= first_added:
            world.set_instance_visible(i, True)
    world.prepare_instances()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("scene,config", [("cornell", "cornell_256"), ("town", None)])
def test_frames_with_added_meshes_equal_frames_of_the_uploaded_scene(scene, config, mode):
    """scene A: a world whose last meshes are device meshes, uploaded without them, the meshes added on the device
    (hikari_plugin_add_meshes), their instances placed from the same world; scene B: the whole world uploaded by the host.  Every
    plane of every frame and the ray counts are equal; a device-built mesh has no 4-wide tree, so A's rays take the reference's walk"""
    from tests.test_gpu_parity import ALL_PLANES
    b = Bench(scene, 48, 32, config=config) if config else Bench(scene, 48, 32)
    first_added = len(b.scene.meshes) // 2
    wa = split_world(b, first_added)
    host_nodes = wa.buffers()["asset_nodes"]
    a_dev, b_dev = plugin.HikariPlugin(b.width, b.height), b.device()
    a_dev.upload_scene(wa)
    got = a_dev.add_meshes(wa, np.arange(first_added, len(b.scene.meshes)))
    show_device_instances(wa, b, first_added)
    assert len(wa.buffers()["asset_nodes"]) == len(host_nodes) < len(b.world.buffers()["asset_nodes"]), "the host built no device BVH"
    for inst in wa.buffers()["instances"]:        # the world gives every device mesh the index the device gave it
        if int(inst["mesh"]["node_offset"]) >= len(host_nodes):
            assert inst["mesh"].tobytes() in {g.tobytes() for g in got}
    a_dev.update_instances(wa)
    for name in ("instances", "instance_nodes", "emissives", "emissive_nodes", "alias_table"):
        assert_bytes_equal(wa.buffers()[name], b.world.buffers()[name], f"{scene}: world A's {name}")
    for which, name in READBACK:
        assert_bytes_equal(a_dev.scene_readback(which), b.world.buffers()[name], f"{scene}: {name}")
    for p in (a_dev, b_dev):
        p.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, mode)
        p.set_profiling(True, False)
    for f in range(1, 5):
        inp = b.moving_inputs(f)
        a_dev.render_frame(inp); b_dev.render_frame(inp)
        for k in ALL_PLANES:
            assert a_dev.readback(k).tobytes() == b_dev.readback(k).tobytes(), f"{scene} mode {mode} frame {f}: plane {k} differs"
        sa, sb = a_dev.stats(), b_dev.stats()
        assert (sa.primary_rays, sa.tlas_rays, sa.blas_rays) == (sb.primary_rays, sb.tlas_rays, sb.blas_rays)
        assert sa.wide_traversal == 0, "a device-built mesh is in use: the 4-wide walk is off"
    a_dev.close(); b_dev.close()


@pytest.mark.parametrize("scene,config", [("cornell", "cornell_256"), ("town", None)])
def test_adding_meshes_behind_queued_frames_of_two_cameras(scene, config):
    """a shared scene on a stream of its own, two cameras on streams of their own with two frames queued each: the meshes are added
    (every mesh buffer grows: the upload's are replaced) without a host synchronisation, their instances placed, more frames
    rendered; every frame of both cameras equals a run that synchronises before the add"""
    import torch
    from tests.test_gpu_parity import ALL_PLANES
    b = Bench(scene, 48, 32, config=config) if config else Bench(scene, 48, 32)
    first_added = len(b.scene.meshes) // 2
    sizes = [(48, 32), (40, 24)]
    runs = []
    for synchronise in (False, True):
        w = split_world(b, first_added)
        shared = plugin.SharedScene()
        shared.upload(w)
        cams = [plugin.HikariPlugin(cw, ch) for cw, ch in sizes]
        for c in cams:
            c.attach_scene(shared)
        inputs = [Bench(scene, cw, ch, config=config) if config else Bench(scene, cw, ch) for cw, ch in sizes]
        frames = []
        for f in (1, 2):
            for c, bi in zip(cams, inputs):
                c.render_frame(bi.moving_inputs(f))
        if synchronise:
            torch.cuda.synchronize()
        shared.add_meshes(w, np.arange(first_added, len(b.scene.meshes)))
        frames.append([{k: c.readback(k).tobytes() for k in ALL_PLANES} for c in cams])
        show_device_instances(w, b, first_added)
        shared.update_instances(w)
        for f in (3, 4, 5):
            for c, bi in zip(cams, inputs):
                c.render_frame(bi.moving_inputs(f))
            frames.append([{k: c.readback(k).tobytes() for k in ALL_PLANES} for c in cams])
        for c in cams:
            c.close()
        shared.close()
        runs.append(frames)
    for f, (queued, synced) in enumerate(zip(*runs)):
        for cam in range(2):
            bad = [k for k in ALL_PLANES if queued[cam][k] != synced[cam][k]]
            assert not bad, f"{scene} frame {f + 2} camera {cam}: planes that differ {bad}"
