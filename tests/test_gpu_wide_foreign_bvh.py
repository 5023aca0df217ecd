"""The 4-wide walk (HK_TUNE_WIDE_TRAVERSAL, csrc/hk_wide.cuh) over flat BVHs that bvh 0.7.1 never writes.  The trees are derived on
the host (csrc/wide_build.h) from whatever flat arrays hk_scene_upload / hk_scene_update_instances accept, so every foreign array
(tests/foreign_bvh.py, checked against a brute-force query by tests/test_foreign_bvh_oracle.py) must end in one of two states,
and each case asserts which one it expects:

  * "wide": the walk is in use (hk_frame_stats.wide_traversal 3, or 1 under the default mode on a scene of at least 256 wide nodes)
    and meets test_gpu_wide_traversal.py's contract against the oracle's flat walk over the same arrays — closest-hit fields
    bit-identical on all but < 1e-4 of the rays, every shadow verdict identical, G-buffer and albedo bit-identical, images
    differing on < 1e-4 of the pixels (one pixel at these sizes);
  * "flat": wide_traversal == 0 and everything bit-exact, for arrays a 4-wide tree cannot walk like the flat one (a run of more
    than four branches below a navigator or at the top, a shape named by two leaves, a navigator box that does not enclose the boxes
    below it, a tree whose stack could outgrow the walk's).

Before wide_build.h refused runs of more than four branches, a node kept the first four and the rest were unreachable: cornell 32 x
32, mode 3, instance 6's BLAS as one navigator over its 10 leaf branches, 1 901 of 50 000 closest-hit rays (random_rays(50_000,
11), no exclusion) differed from the oracle, 404 of them losing their hit; a navigator over 5 leaf branches left 4 of the 5
triangles reachable.  Before an empty mesh was given a node without children to enter, its WIDE_EMPTY entry point ended the whole
TLAS walk: instance 0 of cornell with node_count 0, 204 of the same 50 000 rays lost their hit (both on the emulated kernels)."""
import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin, scenes
from tests import foreign_bvh as fb
from tests.conftest import Bench
from tests.test_gpu_parity import ALL_PLANES, mismatch, random_rays
from tests.test_gpu_wide_traversal import GBUFFER, IMAGES, scene_rays

pytestmark = pytest.mark.gpu

NO_HIT = 0xFFFFFFFF


def pair(b, bufs, mode):
    """device (wide mode `mode`) and oracle over the same arrays"""
    from oracle import oracle
    desc = plugin.scene_desc_from_buffers(bufs, b.scene.textures)
    dev = plugin.HikariPlugin(b.width, b.height)
    dev.upload_scene_desc(desc)
    dev.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, mode)
    orc = oracle.Oracle(b.width, b.height, plugin.load_noise())
    orc.upload_scene_desc(desc)
    return dev, orc


def closest_rays(n, seed, scale=1.0, offset=(0.0, 0.0, 0.0)):
    rays = random_rays(n, seed, any_hit_fraction=0.0)
    rays["origin"] = rays["origin"] * np.float32(scale) + np.array(offset, np.float32)
    rays["exclude_instance"] = NO_HIT
    return rays


def check_rays(dev, orc, rays, shadow, expect):
    hw, ho = dev.trace_rays(rays), orc.trace_rays(rays)
    if expect == "flat":
        assert hw.tobytes() == ho.tobytes(), "the flat walk is not bit-exact"
        return
    hit_w, hit_o = hw["instance_index"] != NO_HIT, ho["instance_index"] != NO_HIT
    assert np.array_equal(hit_w[shadow], hit_o[shadow]), "a shadow ray's verdict differs"
    c = ~shadow
    same = np.ones(int(c.sum()), bool)
    for f in ("instance_index", "primitive_index", "distance", "u", "v"):
        same &= hw[f][c].view(np.uint32) == ho[f][c].view(np.uint32)
    bad = int((~same).sum())
    assert bad <= 1e-4 * c.sum(), f"{bad} of {int(c.sum())} closest-hit rays differ from the flat walk"


def check_frames(b, dev, orc, expect, frames=3):
    allow = 0 if expect == "flat" else max(1, int(1e-4 * b.width * b.height))
    for f in range(1, frames + 1):
        inp = b.moving_inputs(f, step=(0.01, 0.004, -0.006))
        dev.render_frame(inp); orc.render_frame(inp)
        for k in (ALL_PLANES if expect == "flat" else GBUFFER):
            assert mismatch(dev.readback(k), orc.readback(k)) == 0, (f, k)
        if expect == "wide":
            for k in IMAGES:
                n_bad = mismatch(dev.readback(k), orc.readback(k))
                assert n_bad <= allow, (f, k, n_bad)


def check(b, bufs, mode, expect, n=20_000, frames=3, rays=None):
    """At mode 1 only the prepass's primary rays walk the 4-wide trees: trace_rays then takes the flat walk on the device too, and
    the G-buffer of check_frames is what holds the wide walk there; the ray dumps count as coverage only at mode 3."""
    dev, orc = pair(b, bufs, mode)
    st = dev.stats()
    assert st.wide_traversal == ({"wide": mode, "flat": 0}[expect]), (st.wide_traversal, st.wide_stack_need)
    if rays is None:
        sr, shadow = scene_rays(b, n, 3)
        rays = [(sr, shadow), (closest_rays(n // 2, 11), np.zeros(n // 2, bool))]
    for r, shadow in rays:
        check_rays(dev, orc, r, shadow, expect)
    check_frames(b, dev, orc, expect, frames)
    return dev, orc


def cornell():
    return Bench("cornell", 48, 32, config="cornell_1080p")


def city():
    return Bench("city", 48, 32, config="city_4k")


def every_blas(bufs, **kw):
    done = set()
    for i in range(len(bufs["instances"])):
        if fb.mesh_of(bufs, i) not in done and fb.triangle_count(bufs, i) > 0:
            fb.foreign_blas(bufs, i, **kw)
            done.add(fb.mesh_of(bufs, i))


def test_bvh_0_7_1_scenes_keep_the_wide_walk():
    """the scenes the product ships with: a later refusal must not quietly turn the mode off for them"""
    for name, mode, want in (("cornell", 3, 3), ("city", 3, 3), ("town", 3, 3), ("city", 1, 1), ("town", 1, 1)):
        dev = Bench(name, 16, 16, config="cornell_1080p").device()
        dev.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, mode)
        assert dev.stats().wide_traversal == want, (name, mode)


@pytest.mark.parametrize("blas,tlas", [(dict(arity=3), dict(arity=3, top=3)), (dict(arity=[4, 3]), dict(arity=4, top=4)),
                                       (dict(arity=[1, 2, 4]), dict(arity=[1, 3], top=2))])
def test_runs_of_up_to_four_branches_walk_wide(blas, tlas):
    b = cornell()
    bufs = b.world.buffers()
    every_blas(bufs, **blas)
    fb.foreign_tlas(bufs, **tlas)
    check(b, bufs, 3, "wide")


def test_runs_of_three_and_four_under_the_default_mode():
    """mode 1 (the product's default): the primary rays of a scene of at least 256 wide nodes walk the 4-wide trees"""
    b = city()
    bufs = b.world.buffers()
    every_blas(bufs, arity=[3, 4], split="random", seed=2)
    fb.foreign_tlas(bufs, arity=4, top=3)
    check(b, bufs, 1, "wide", n=8_000)


@pytest.mark.parametrize("run", [5, 8, 10])
def test_a_blas_run_of_more_than_four_branches_keeps_the_flat_walk(run):
    """cornell's tall box (instance 6, 10 triangles) under one navigator over a run of `run` branches"""
    b = cornell()
    bufs = b.world.buffers()
    lo, hi = fb.triangle_boxes(bufs, 6)
    fb.set_blas(bufs, 6, fb.flatten(fb.tree(lo, hi, arity=[2, run, 2], top=1, split="order"), lo, hi))
    check(b, bufs, 3, "flat")


def test_a_tlas_run_of_seventeen_under_the_default_mode_keeps_the_flat_walk():
    b = city()
    bufs = b.world.buffers()
    fb.foreign_tlas(bufs, arity=17, top=2)
    check(b, bufs, 1, "flat", n=8_000)


def test_a_top_level_of_five_keeps_the_flat_walk():
    b = cornell()
    bufs = b.world.buffers()
    fb.foreign_tlas(bufs, arity=2, top=5)
    check(b, bufs, 3, "flat")


@pytest.mark.parametrize("where", ["first", "last"])
def test_an_instance_of_an_empty_mesh_does_not_end_the_walk(where):
    """instance 6 (the short box: rays through its box go on to the walls and the floor) of a mesh with no records, first or last leaf
    of the TLAS"""
    b = cornell()
    bufs = b.world.buffers()
    fb.set_blas(bufs, 6, np.zeros(0, L.NODE))
    rest = [0, 1, 2, 3, 4, 5, 7]
    order = [6] + rest if where == "first" else rest + [6]
    lo, hi = fb.instance_boxes(bufs)
    fb.set_tlas(bufs, fb.flatten(fb.tree(lo, hi, arity=2, split="order", shapes=order), lo, hi))
    check(b, bufs, 3, "wide")


def test_an_empty_mesh_under_the_default_mode():
    b = city()
    bufs = b.world.buffers()
    fb.set_blas(bufs, 0, np.zeros(0, L.NODE))
    check(b, bufs, 1, "wide", n=8_000)


def test_single_record_meshes_and_a_one_instance_tlas():
    b = cornell()
    bufs = b.world.buffers()
    for i in (0, 3, 5):                                  # the walls: one of their two triangles each
        lo, hi = fb.triangle_boxes(bufs, i)
        fb.set_blas(bufs, i, fb.flatten([1], lo, hi))
    check(b, bufs, 3, "wide")
    bufs = b.world.buffers()
    lo, hi = fb.instance_boxes(bufs)
    fb.set_tlas(bufs, fb.flatten([6], lo, hi))
    check(b, bufs, 3, "wide")


@pytest.mark.parametrize("mode", [1, 3])
def test_inflated_navigator_boxes_walk_wide(mode):
    """every navigator of every BLAS and of the TLAS grown by 0.05 (then the flat walk re-derives each leaf's box; the wide walk
    tests only the navigators' boxes).  A difference could only come from a box test rounding differently at an edge.  Measured at
    mode 3 (city 96 x 54, scene_rays(b, 40_000, 3) plus 50 000 random closest-hit rays): 0 of 24 129 + 50 000 closest-hit rays and 0
    of 15 871 shadow verdicts differed, both on the emulated kernels before the fixes of this file and on an H100 after them (cornell
    on the H100: 0 as well).  So the 4-wide walk stays in use for such arrays."""
    b = city()
    bufs = b.world.buffers()
    for name in ("asset_nodes", "instance_nodes"):
        nodes = bufs[name]
        nav = nodes["entry_index"] < fb.LEAF
        nodes["min"][nav] -= np.float32(0.05)
        nodes["max"][nav] += np.float32(0.05)
    rays = closest_rays(20_000, 7, scale=8.0, offset=(0.0, 1.0, 0.0))
    sr, shadow = scene_rays(b, 20_000, 3)
    check(b, bufs, mode, "wide", rays=[(sr, shadow), (rays, np.zeros(len(rays), bool))])


@pytest.mark.parametrize("blas,tlas", [("tight", "tight"), ("tight_leaves", "exact"), ("exact", "tight_inner"), ("tight_inner", "exact"),
                                       ("exact", "tight_leaves")])
def test_navigator_boxes_that_do_not_enclose_their_shapes_keep_the_flat_walk(blas, tlas):
    """a navigator box shrunk by a quarter of its extent on every side culls hits it does not enclose, depending on the best hit so
    far, i.e. on the order of the walk (and the 4-wide walk never tests the boxes of the levels it collapses): such an array keeps the
    flat walk.  Before wide_build.h checked the boxes, all-tight binary trees on cornell 48 x 32 at mode 3 took the 4-wide walk and
    3 853 of 50 000 closest-hit rays and 48 G-buffer pixels differed from the oracle (emulated kernels)."""
    b = cornell()
    bufs = b.world.buffers()
    every_blas(bufs, arity=2, boxes=blas)
    fb.foreign_tlas(bufs, arity=2, boxes=tlas)
    check(b, bufs, 3, "flat")


def test_tight_navigator_boxes_under_the_default_mode_keep_the_flat_walk():
    """the same on the city at mode 1, where the unchecked boxes changed 6 G-buffer pixels"""
    b = city()
    bufs = b.world.buffers()
    every_blas(bufs, arity=2, boxes="tight")
    fb.foreign_tlas(bufs, arity=2, boxes="tight")
    check(b, bufs, 1, "flat", n=8_000)


@pytest.mark.parametrize("which", ["blas", "tlas"])
def test_a_shape_named_by_two_leaves_keeps_the_flat_walk(which):
    b = cornell()
    bufs = b.world.buffers()
    if which == "blas":
        lo, hi = fb.triangle_boxes(bufs, 6)
        fb.set_blas(bufs, 6, fb.flatten(fb.tree(lo, hi, shapes=list(range(10)) + [3]), lo, hi))
    else:
        lo, hi = fb.instance_boxes(bufs)
        fb.set_tlas(bufs, fb.flatten(fb.tree(lo, hi, shapes=list(range(8)) + [6]), lo, hi))
    check(b, bufs, 3, "flat")


def stack_scene(triangles=80):
    """cornell plus a stack of `triangles` parallel triangles across the view, the later ones nearer the camera"""
    sd = scenes.cornell()
    z = 1.1 + 0.01 * np.arange(triangles, dtype=np.float32)
    pos = np.zeros((3 * triangles, 3), np.float32)
    pos[0::3] = np.stack([np.full_like(z, -0.5), np.full_like(z, 0.6), z], 1)
    pos[1::3] = np.stack([np.full_like(z, 0.5), np.full_like(z, 0.6), z], 1)
    pos[2::3] = np.stack([np.zeros_like(z), np.full_like(z, 1.5), z], 1)
    nrm = np.tile(np.array([[0.0, 0.0, 1.0]], np.float32), (3 * triangles, 1))
    uv = np.zeros((3 * triangles, 2), np.float32)
    sd.meshes = list(sd.meshes) + [(pos, nrm, uv, np.arange(3 * triangles, dtype=np.uint32))]
    sd.inst_mesh = list(sd.inst_mesh) + [len(sd.meshes) - 1]
    sd.inst_material = list(sd.inst_material) + [int(sd.inst_material[2])]
    sd.inst_transform = list(sd.inst_transform) + [np.eye(4, dtype=np.float32).reshape(16)]
    scenes.SCENE_BUILDERS["_stack"] = lambda: sd
    try:
        return Bench("_stack", 48, 32, config="cornell_1080p"), triangles
    finally:
        del scenes.SCENE_BUILDERS["_stack"]


def chain_bufs(b, total, count):
    """the stack's BLAS as a chain of 4-wide levels (three leaves and the rest) over its `count` nearest triangles, farthest first:
    every ray through the stack enters the rest before the leaves, so the walk holds the leaves of every level on its stack"""
    bufs = b.world.buffers()
    inst = len(bufs["instances"]) - 1
    lo, hi = fb.triangle_boxes(bufs, inst)
    fb.set_blas(bufs, inst, fb.flatten(fb.tree(lo, hi, arity=4, split="chain", shapes=range(total - count, total)), lo, hi))
    return bufs


@pytest.mark.parametrize("need,expect", [(63, "wide"), (64, "wide"), (65, "flat")])
def test_the_deepest_stack_the_walk_can_hold(need, expect):
    """a chain's stack need grows by one per triangle: trees whose bound is 63 and 64 of the walk's 64 entries (HK_WIDE_STACK) are
    walked and 65 is refused.  The bound includes three entries of slack (context.cu: the pushes of a node step before it enters a
    child), so at a bound of 64 the walk itself holds at most 61: these rays, whose nearest child is always the deeper subtree, take
    the walk as deep as the chain goes (the TLAS entries, the BLAS marker and every level's leaves), not to entry 64.  What the cases
    pin is the bound the build reports, the refusal above 64 and the walk at the deepest tree that is accepted."""
    b, total = stack_scene()
    probe = plugin.HikariPlugin(b.width, b.height)
    probe.upload_scene_desc(plugin.scene_desc_from_buffers(chain_bufs(b, total, 30)))
    probe.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 3)
    base = probe.stats().wide_stack_need - 30                # the TLAS's share, the BLAS marker and the slack, plus 30 - 1
    bufs = chain_bufs(b, total, need - base)
    rng = np.random.default_rng(need)
    n = 10_000
    rays = np.zeros(n, L.RAY)
    rays["origin"] = (np.array([0.0, 1.0, 4.0]) + rng.uniform(-0.1, 0.1, (n, 3))).astype(np.float32)
    target = np.stack([rng.uniform(-0.1, 0.1, n), rng.uniform(0.9, 1.1, n), np.full(n, 1.0)], 1)
    d = target - rays["origin"]
    rays["direction"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["max_distance"] = np.float32(3.402823466e38)
    rays["exclude_instance"] = NO_HIT
    shadow = rng.random(n) < 0.3
    rays["max_distance"] = np.where(shadow, np.float32(2.5), rays["max_distance"])
    rays["early_distance"] = np.where(shadow, np.float32(2.4), np.float32(0.0))
    dev, orc = check(b, bufs, 3, expect, rays=[(rays, shadow)])
    assert dev.stats().wide_stack_need == need
    hits = orc.trace_rays(rays)
    stack_mesh = len(bufs["instances"]) - 1
    assert (hits["instance_index"][~shadow] == stack_mesh).mean() > 0.95
    assert (hits["primitive_index"][~shadow] - bufs["instances"]["mesh"]["primitive"][stack_mesh] == total - 1).mean() > 0.95


def test_instance_updates_switch_the_walk_with_each_tlas():
    """hk_scene_update_instances from bvh 0.7.1's TLAS to a five-branch foreign one and back: the mode follows each upload"""
    b = cornell()
    dev, orc = pair(b, b.world.buffers(), 3)
    assert dev.stats().wide_traversal == 3
    foreign = b.world.buffers()
    fb.foreign_tlas(foreign, arity=2, top=5)
    sr, shadow = scene_rays(b, 10_000, 5)
    for bufs, expect in ((foreign, "flat"), (b.world.buffers(), "wide"), (foreign, "flat")):
        desc = plugin.scene_desc_from_buffers(bufs)
        dev.update_instances_desc(desc); orc.update_instances_desc(desc)
        assert dev.stats().wide_traversal == {"wide": 3, "flat": 0}[expect]
        check_rays(dev, orc, sr, shadow, expect)
        check_rays(dev, orc, closest_rays(10_000, 13), np.zeros(10_000, bool), expect)
        inp = b.inputs(1)
        dev.render_frame(inp); orc.render_frame(inp)
        for k in GBUFFER:
            assert mismatch(dev.readback(k), orc.readback(k)) == 0, (expect, k)
