"""The device scene rebuild (hk_scene_update_transforms, csrc/kernels_scene.cu) at the edges of its input, and held to anchors that do
not go through the host mirror.

  A. transform families — mirrored, rotations about all three axes, shear, scales from 1e-3 to 1e3 and a uniform 1e-6, translations
     of 1e5 and 1e6, an axis (or all three) scaled to zero — at n = 1, 2, 33, 257 over three updates: every record equals the host
     mirror bit for bit (a singular model's inverse holds NaNs, written as the host writes them); frames with such instances in front
     of the cornell camera equal the oracle's, under the flat walk, the 4-wide walk and the pooled indirect pass; one shared scene;
  B. float64 anchors on the device's own records: inverse * model = I within c * cond(M) * 2^-24, world AABBs against the float64
     corners (starting from zero, instance.rs:298-303), emissive area / position / radius against float64 sums, and the flat TLAS's
     structure (one leaf per instance, skip links that nest, navigator boxes that enclose their subtrees exactly in f32);
  C. scale and depth: up to 20000 instances (4097 on the emulated kernels), 2000 emissives, emissive meshes at the 32-lane chunk
     boundaries of kc_scene_emissives, and the deepest chains the SAH build makes (4-wide parse depth 32, 56, 94, 95);
  D. the alias-table cache rule at its edges, against glam's rule restated here (signum, abs_diff_eq(.., 0.01));
  E. non-finite models refused by every entry point, the scene left as it was, the next valid update accepted."""
import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin
from bevy_hikari_b200._ffi import HikariError
from tests.conftest import EMULATED, Bench
from tests.test_gpu_parity import ALL_PLANES, DENOISED, compare_all
from tests.test_gpu_scene_update import assert_scene_equals_host, material, soup_world, unit_cube
from tests.test_gpu_wide_tlas_device import assert_same, chain_models, snapshot

pytestmark = pytest.mark.gpu

LEAF = 0x80000000
U = 2.0 ** -24                       # unit roundoff of f32
EMULATED_MAX_N = 4097                # the emulated kernels stop here (CPU time)

FAMILIES = ["mirrored", "rotated", "shear", "scale_wide", "scale_1e-6", "far_1e5", "far_1e6", "zero_x", "zero_y", "zero_z", "zero_all"]
ZERO = {"zero_x": [0], "zero_y": [1], "zero_z": [2], "zero_all": [0, 1, 2]}


def skip_large(n):
    if EMULATED and n > EMULATED_MAX_N:
        pytest.skip(f"n = {n}: device only (the emulated kernels run up to {EMULATED_MAX_N} instances)")


# ------------------------------------------------------------------------------------------------ transform families
def rotation(rng):
    """a uniformly random rotation (about all three axes), float64 3 x 3"""
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def shape(family, rng, emissive=False):
    """the part of an instance's model that stays fixed while it moves (so that an emissive's alias table stays cached)"""
    if emissive and family in ("zero_y", "zero_z"):
        family = "zero_x"          # |x_axis| = 0: glam's signum(det) of a rounding-noise det cannot flip the cached scale
    s = rng.uniform(0.5, 2.0, 3)
    if family == "mirrored":
        s[rng.integers(3)] *= -1.0
    elif family == "scale_wide":
        s = 10.0 ** rng.uniform(-3.0, 3.0, 3)
    elif family == "scale_1e-6":
        s = np.full(3, 1e-6)
    elif family in ZERO:
        s[ZERO[family]] = 0.0
    b = np.diag(s)
    if family == "shear":
        b = b + np.triu(rng.uniform(-1.5, 1.5, (3, 3)), 1) + np.tril(rng.uniform(-0.5, 0.5, (3, 3)), -1)
    return b


def reach(family):
    return {"far_1e5": 1e5, "far_1e6": 1e6}.get(family, 20.0)


def place(b, rng, family, centre=None):
    """column-major f32 model: translate(random within the family's reach, or `centre`) * random rotation * b"""
    t = np.eye(4)
    t[:3, :3] = rotation(rng) @ b
    t[:3, 3] = rng.uniform(-1.0, 1.0, 3) * reach(family) if centre is None else centre
    return t.T.astype(np.float32).reshape(16).copy()


def is_emissive(i):
    return i % 7 == 3                # soup_world's glowing instances


def family_world(rng, n, family):
    w = soup_world(rng, n, "random")
    shapes = [shape(family, rng, is_emissive(i)) for i in range(n)]
    for i in range(n):
        w.set_instance_transform(i, place(shapes[i], rng, family))
    w.prepare_instances()
    return w, shapes


def step_family(w, rng, family, shapes):
    for i, b in enumerate(shapes):
        w.set_instance_transform(i, place(b, rng, family))
    w.previous_transform_system()


# ------------------------------------------------------------------------------------------------ B: float64 anchors
# Each bound was calibrated on the host mirror's records (equal to the device's by contract, A) over every family and scale case of
# this file; the worst value measured is written beside it.
INVERSE_C = 8.0          # 3x3 block / translation column of the inverse, units of inverse_anchor: worst measured 4.22 (scale_1e-6)
AABB_C = 4.0             # |box - float64 box| / (2^-24 * magnitude of the sum): worst measured 2.22 (emissive soups)
AREA_C = 2.0             # |area - float64 area| / (2^-24 * (triangles * area + sum of |edge| * |vertex|)): worst measured 0.39
SPHERE_C = 3.0           # |position / radius - float64| / (2^-24 * magnitude): worst measured 1.46 (shear)


def model_rows(rec):
    """row-major float64 4 x 4 of a column-major record field"""
    return rec.reshape(4, 4).T.astype(np.float64)


def inverse_anchor(inst):
    """worst error of the inverse over the non-singular instances, the device's inverse = its inverse_transpose_model transposed,
    i.e. the record's 16 floats read row-major: the 3x3 block A against A M3 = I in units of cond(M3) 2^-24, and the translation
    column against -M3^-1 t in units of cond(M3) 2^-24 |M3^-1| |t| (the condition of the whole 4x4 grows with |t| and would let a
    far instance's 3x3 block off lightly)"""
    worst = 0.0
    for r in inst:
        m = model_rows(r["model"])
        m3, t = m[:3, :3], m[:3, 3]
        if np.linalg.matrix_rank(m3) < 3 or not np.isfinite(r["inverse_transpose_model"]).all():
            continue
        inv = r["inverse_transpose_model"].reshape(4, 4).astype(np.float64)
        k3 = np.linalg.cond(m3)
        block = np.abs(inv[:3, :3] @ m3 - np.eye(3)).max() / (k3 * U)
        m3i = np.linalg.inv(m3)
        column = np.abs(inv[:3, 3] + m3i @ t).max() / (k3 * U * (np.abs(m3i) @ np.abs(t)).max() + 1e-300)
        worst = max(worst, block, column)
    return worst


def aabb_anchor(inst, mesh_box):
    """worst |min / max - float64| over the instances, in units of 2^-24 * (|centre| + sum of |corner offsets|)"""
    worst = 0.0
    for r in inst:
        centre, half = mesh_box[int(r["mesh"]["vertex"])]
        m = model_rows(r["model"])
        c = m[:3, :3] @ centre + m[:3, 3]
        lo, hi = np.zeros(3), np.zeros(3)                       # instance.rs:298-303 starts from zero
        for index in range(8):
            v = half * np.array([2 * (index & 1) - 1, 2 * ((index >> 1) & 1) - 1, 2 * ((index >> 2) & 1) - 1], np.float64)
            t = m[:3, :3] @ v
            lo, hi = np.minimum(lo, t), np.maximum(hi, t)
        mag = np.abs(m[:3, :3]) @ (np.abs(centre) + half) + np.abs(m[:3, 3]) + 1e-300
        worst = max(worst, (np.abs(r["min"] - (lo + c)) / (U * mag)).max(), (np.abs(r["max"] - (hi + c)) / (U * mag)).max())
    return worst


def emissive_anchor(ems, inst, prims, materials):
    """worst surface area, position and radius of the emissives against float64 (the record's own instance box for the sphere)"""
    area_w = sphere_w = 0.0
    for e in ems:
        r = inst[e["instance"]]
        m = model_rows(r["model"])
        p = prims[int(r["mesh"]["primitive"]):int(r["mesh"]["primitive"]) + int(e["alias_table_count"])]["vertices"]["position"].astype(np.float64)
        v = p @ m[:3, :3].T + m[:3, 3]                           # (triangles, 3 corners, xyz)
        a, b = v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]
        areas = 0.5 * np.linalg.norm(np.cross(a, b), axis=1)
        scale = len(areas) * areas.sum() + ((np.linalg.norm(a, axis=1) + np.linalg.norm(b, axis=1)) * np.abs(v).max(axis=(1, 2))).sum() + 1e-300
        area_w = max(area_w, abs(float(e["surface_area"]) - areas.sum()) / (U * scale))
        lo, hi = r["min"].astype(np.float64), r["max"].astype(np.float64)
        pos = 0.5 * (hi + lo)
        em = materials[int(r["material"])]["emissive"].astype(np.float64)
        intensity = 255.0 * em[3] * np.linalg.norm(em[:3])
        radius = 0.5 * np.linalg.norm(hi - lo) + np.sqrt(intensity)
        sphere_w = max(sphere_w, (np.abs(e["position"] - pos) / (U * (np.abs(pos) + np.abs(hi - lo) + 1e-300))).max(),
                       abs(float(e["radius"]) - radius) / (U * (radius + 1e-300)))
    return area_w, sphere_w


def tlas_structure(nodes, inst):
    """the flat TLAS: every instance named by exactly one leaf, skip links that nest, every navigator box encloses the boxes of the
    instances below it exactly in f32.  Returns the depth of Parser::range (wide_build.h) the tree needs."""
    n = len(inst)
    entry, exit_ = nodes["entry_index"].astype(np.int64), nodes["exit_index"].astype(np.int64)
    if n == 1:
        assert len(nodes) == 1 and entry[0] == LEAF and exit_[0] == 1
        return 0
    assert len(nodes) == 3 * n - 2
    named = np.zeros(n, np.int64)
    deepest = 0
    stack = [(0, len(nodes), 0, None)]              # (begin, end, depth, navigator record) — an explicit Parser::range
    lo, hi = np.full((len(nodes), 3), np.inf, np.float32), np.full((len(nodes), 3), -np.inf, np.float32)
    order = []
    while stack:
        i, end, depth, parent = stack.pop()
        deepest = max(deepest, depth)
        while i < end:
            assert entry[i] == i + 1 and i + 1 < exit_[i] <= end, ("skip links must nest", i, entry[i], exit_[i], end)
            if entry[i + 1] >= LEAF:
                shape = int(entry[i + 1] - LEAF)
                assert shape < n and exit_[i] == i + 2 and exit_[i + 1] == i + 2, ("leaf record", i)
                named[shape] += 1
                b_lo, b_hi = inst["min"][shape], inst["max"][shape]
                assert (nodes["min"][i] <= b_lo).all() and (b_hi <= nodes["max"][i]).all(), ("leaf box", i, shape)
                lo[i], hi[i] = b_lo, b_hi
            else:
                stack.append((i + 1, int(exit_[i]), depth + 1, i))
                order.append(i)
            i = int(exit_[i])
    assert (named == 1).all(), ("instances not named exactly once", np.nonzero(named != 1)[0][:8])
    # enclosure: children before parents (reverse pre-order of the navigators), boxes of the instances below each one
    for i in reversed(sorted(order)):
        j, end = i + 1, int(exit_[i])
        while j < end:
            lo[i], hi[i] = np.minimum(lo[i], lo[j]), np.maximum(hi[i], hi[j])
            j = int(exit_[j])
        assert (nodes["min"][i] <= lo[i]).all() and (hi[i] <= nodes["max"][i]).all(), ("navigator does not enclose its subtree", i)
    return deepest


def device_records(dev):
    return {name: dev.scene_readback(which) for which, name in [(L.SCENE_INSTANCES, "instances"), (L.SCENE_INSTANCE_NODES, "instance_nodes"),
                                                                (L.SCENE_EMISSIVES, "emissives"), (L.SCENE_EMISSIVE_NODES, "emissive_nodes")]}


def cube_box():
    return np.zeros(3), np.full(3, 0.5)


def check_anchors(rec, static, mesh_box, what, singular=False):
    """B on one set of records (the device's); `static` = the world's buffers for what the update does not touch (primitives,
    materials)"""
    inst = rec["instances"]
    if not singular:
        v = inverse_anchor(inst)
        assert v <= INVERSE_C, (what, "inverse", v)
    v = aabb_anchor(inst, mesh_box)
    assert v <= AABB_C, (what, "aabb", v)
    if len(rec["emissives"]):
        a, s = emissive_anchor(rec["emissives"], inst, static["primitives"], static["materials"])
        assert a <= AREA_C and s <= SPHERE_C, (what, "emissive", a, s)
    return tlas_structure(rec["instance_nodes"], inst)


# ------------------------------------------------------------------------------------------------ A: families, records
@pytest.mark.parametrize("n", [1, 2, 33, 257])
@pytest.mark.parametrize("family", FAMILIES)
def test_transform_families_rebuild_bit_identically(family, n):
    rng = np.random.default_rng(1000 + 17 * FAMILIES.index(family) + n)
    w, shapes = family_world(rng, n, family)
    dev = plugin.HikariPlugin(32, 24, 0, 0, None, None, 0, None)
    dev.upload_scene(w)
    static = w.buffers()
    box = {int(static["instances"]["mesh"]["vertex"][0]): cube_box()}
    for step in range(3):
        step_family(w, rng, family, shapes)
        assert dev.update_transforms(w), (family, n, step)
        rec = device_records(dev)
        check_anchors(rec, static, box, f"{family} n={n} step {step}", singular=family in ZERO)      # B, before the host has run
        w.prepare_instances()
        assert_scene_equals_host(dev, w, f"{family} n={n} step {step}")
        if family in ZERO:
            it = rec["instances"]["inverse_transpose_model"]
            assert np.isnan(it).any(), "a zero-scaled model has no inverse"
            assert (it.view(np.uint32)[np.isnan(it)] == 0xFFC00000).all(), "NaNs of the inverse are x86's default NaN"
    dev.close()


def test_one_family_through_a_shared_scene():
    rng = np.random.default_rng(77)
    w, shapes = family_world(rng, 33, "zero_y")
    scene = plugin.SharedScene()
    scene.upload(w)
    cam = plugin.HikariPlugin(32, 24)
    cam.attach_scene(scene)
    for step in range(3):
        step_family(w, rng, "zero_y", shapes)
        assert scene.update_transforms(w), step
        w.prepare_instances()
        assert_scene_equals_host(cam, w, f"shared zero_y step {step}")
    cam.close()
    scene.close()


# ------------------------------------------------------------------------------------------------ A: families, frames
FRAME_CASES = [(f, walk) for f in FAMILIES for walk in ("flat", "wide")] + [(f, "pooled") for f in ZERO]
RESERVOIRS = [k for k in ALL_PLANES if k >= L.OUT_RESERVOIR_0]


def compare_wide(dev, orc, frame):
    """the 4-wide walk's contract (include/hikari_b200.h, tests/test_gpu_wide_traversal.py): a shadow ray's verdict is the reference's,
    but WHICH occluder it reports may differ, and that position is stored only with a zero-radiance sample.  So every plane but the
    reservoirs is bit-identical, and a reservoir record differs at most in the sample position of a sample whose radiance is zero."""
    compare_all(dev, orc, [k for k in ALL_PLANES if k not in RESERVOIRS], frame)
    for k in RESERVOIRS:
        a, o = dev.readback(k).reshape(-1), orc.readback(k).reshape(-1)
        differs = a.view(np.uint8).reshape(len(a), -1) != o.view(np.uint8).reshape(len(o), -1)
        bad = np.nonzero(differs.any(axis=1))[0]
        if not len(bad):
            continue
        rgb_zero = (o["radiance"][bad, 0] == 0) & ((o["radiance"][bad, 1] & 0xFFFF) == 0)       # f16 r, g | b, w
        assert rgb_zero.all(), (frame, k, "a reservoir with radiance differs", bad[~rgb_zero][:4])
        for name in a.dtype.names:
            if name != "sample_position":
                assert np.array_equal(a[name][bad].view(np.uint8), o[name][bad].view(np.uint8)), (frame, k, name, bad[:4])


@pytest.mark.parametrize("family,walk", FRAME_CASES)
def test_family_instances_in_cornell_render_as_the_oracle(family, walk):
    """four family instances (one a light) in front of the cornell camera, moved over three frames; a zero-scaled instance must
    vanish identically for every walk"""
    rng = np.random.default_rng(500 + FAMILIES.index(family))
    b = Bench("cornell", 64, 48, config="cornell_256")
    w = b.world
    mesh = w.add_mesh(*unit_cube())
    plain, glow = w.add_material(material()), w.add_material(material(emissive=(1.0, 0.8, 0.6, 0.5)))
    shapes, ids = [], []
    for k in range(4):
        sh = shape(family, rng, emissive=k == 3) * (0.25 if not family.startswith("scale") else 1.0)
        if family == "scale_wide":
            sh = sh / np.abs(sh).max() * 0.4
        shapes.append(sh)
        ids.append(w.add_instance(mesh, glow if k == 3 else plain, place(sh, rng, family, centre=(0.5 * k - 0.75, 0.9, 0.3))))
    w.prepare()
    dev = b.device()
    host = None
    if walk == "wide":
        dev.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 3)
        host = b.device()                    # the same camera updated through the host path: its 4-wide verdict is the host's
        host.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 3)
    elif walk == "pooled":
        dev.set_tuning(plugin.TUNE_POOLED_INDIRECT, 1)
    else:
        dev.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 0)
    orc = b.oracle()
    for f in range(1, 4):
        for k, (i, sh) in enumerate(zip(ids, shapes)):
            centre = (0.5 * k - 0.75, 0.9 + 0.05 * f, 0.3)
            if family.startswith("far") and k == 0:
                centre = None                      # out of sight at the family's reach: the TLAS spans 1e5 / 1e6
            w.set_instance_transform(i, place(sh, rng, family, centre=centre))
        w.previous_transform_system()
        assert dev.update_transforms(w), f
        w.prepare_instances()
        if host is not None:
            host.update_instances(w)
            assert_wide_equal(dev, host, f"{family} frame {f}")
        orc.update_instances_desc(w.scene_desc())
        inp = b.inputs(f)
        dev.render_frame(inp); orc.render_frame(inp)
        if walk == "wide":
            assert dev.stats().wide_traversal == (0 if family == "zero_all" else 3), (family, f)
            compare_wide(dev, orc, f)
        else:
            compare_all(dev, orc, ALL_PLANES, f)
    dev.close()
    if host is not None:
        host.close()


# ------------------------------------------------------------------------------------------------ C: scale
@pytest.mark.parametrize("n", [255, 256, 257, 1024, 4097, 20000])
def test_large_soups(n):
    skip_large(n)
    rng = np.random.default_rng(n)
    w = soup_world(rng, n, "random")
    dev = plugin.HikariPlugin(32, 24, 0, 0, None, None, 0, None)
    dev.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 3)
    dev.upload_scene(w)
    host = plugin.HikariPlugin(32, 24, 0, 0, None, None, 0, None)
    host.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, 3)
    host.upload_scene(w)
    static = w.buffers()
    box = {int(static["instances"]["mesh"]["vertex"][0]): cube_box()}
    for step in range(2):
        for i in range(n):
            cur = w.buffers()["instances"]["model"][i].reshape(4, 4).T.astype(np.float64)
            r = np.eye(4)
            r[:3, :3] = rotation(rng) if not is_emissive(i) else np.eye(3)
            cur = r @ cur if not is_emissive(i) else cur
            cur[:3, 3] += rng.uniform(-1.0, 1.0, 3)
            w.set_instance_transform(i, cur.T.astype(np.float32).reshape(16).copy())
        w.previous_transform_system()
        assert dev.update_transforms(w), (n, step)
        check_anchors(device_records(dev), static, box, f"n={n} step {step}")
        w.prepare_instances()
        assert_scene_equals_host(dev, w, f"n={n} step {step}")
        host.update_instances(w)
        assert_wide_equal(dev, host, f"n={n} step {step}")
    dev.close(); host.close()


def strip_mesh(triangles, rng):
    """`triangles` random triangles in the unit cube (one alias entry each)"""
    p = rng.uniform(-0.5, 0.5, (3 * triangles, 3)).astype(np.float32)
    nrm = np.tile(np.array([[0, 1, 0]], np.float32), (3 * triangles, 1))
    uv = np.zeros((3 * triangles, 2), np.float32)
    return p, nrm, uv, np.arange(3 * triangles, dtype=np.uint32)


def emissive_world(rng, n, triangles):
    """n instances of one emissive mesh of `triangles` triangles, random scales (0.2 to 2), rotations and places"""
    w = plugin.World()
    mesh_data = strip_mesh(triangles, rng)
    mesh = w.add_mesh(*mesh_data)
    glow = w.add_material(material(emissive=(1.0, 0.8, 0.6, 0.5)))
    shapes = [np.diag(rng.uniform(0.2, 2.0, 3)) for _ in range(n)]
    for b in shapes:
        w.add_instance(mesh, glow, place(b, rng, "rotated"))
    w.prepare()
    p = mesh_data[0]
    lo, hi = p.min(axis=0), p.max(axis=0)
    box = (0.5 * (hi.astype(np.float64) + lo), 0.5 * (hi.astype(np.float64) - lo))
    return w, shapes, box


@pytest.mark.parametrize("n,triangles", [(2000, 12), (3, 1), (3, 31), (3, 32), (3, 33), (3, 64), (3, 65)])
def test_emissive_soups_and_chunk_boundaries(n, triangles):
    rng = np.random.default_rng(7 * n + triangles)
    w, shapes, box = emissive_world(rng, n, triangles)
    dev = plugin.HikariPlugin(32, 24, 0, 0, None, None, 0, None)
    dev.upload_scene(w)
    static = w.buffers()
    assert len(static["emissives"]) == n and (static["emissives"]["alias_table_count"] == triangles).all()
    mesh_box = {int(static["instances"]["mesh"]["vertex"][0]): box}
    for step in range(3):
        step_family(w, rng, "rotated", shapes)
        assert dev.update_transforms(w), step
        rec = device_records(dev)
        check_anchors(rec, static, mesh_box, f"{n} emissives x {triangles} step {step}")
        tlas_structure(rec["emissive_nodes"], np.array(list(zip(rec["emissives"]["position"] - rec["emissives"]["radius"][:, None],
                                                                  rec["emissives"]["position"] + rec["emissives"]["radius"][:, None])),
                                                         dtype=[("min", np.float32, 3), ("max", np.float32, 3)]))
        w.prepare_instances()
        assert_scene_equals_host(dev, w, f"{n} emissives x {triangles} step {step}")
    dev.close()


# ------------------------------------------------------------------------------------------------ C: depth
def assert_wide_equal(dev, host, what):
    """the device's 4-wide TLAS, ranks and walk verdict equal what the host derived at upload from its own records"""
    sd, sh = dev.stats(), host.stats()
    assert (sd.wide_traversal, sd.wide_stack_need) == (sh.wide_traversal, sh.wide_stack_need), (what, sd.wide_traversal, sd.wide_stack_need,
                                                                                                 sh.wide_traversal, sh.wide_stack_need)
    for which in (L.SCENE_WIDE_TLAS, L.SCENE_WIDE_INSTANCE_RANK):
        a, b = dev.scene_readback(which), host.scene_readback(which)
        assert a.tobytes() == b.tobytes(), (what, which, len(a), len(b))


def chain3_models(n, top=1e18, ratio=6.2, scale=0.01):
    """n cubes whose centres cycle through the x, y and z axes, each 6.2^(1/3) times nearer the origin than the next, the last at
    1e18, every cube 0.01 of its distance wide: the split axis is the one with the largest centroid extent, so the SAH build peels
    one box per level on each axis in turn"""
    out = []
    for i in range(n):
        t = np.eye(4)
        c = np.zeros(3)
        c[i % 3] = top / ratio ** ((n - 1 - i) / 3.0)
        t[:3, :3] *= scale * np.abs(c).max()
        t[:3, 3] = c
        out.append(t.T.astype(np.float32).reshape(16).copy())
    return out


# How deep the SAH build can go.  A level peels off one box only when every other centre falls into the first of the six buckets
# along the split axis, i.e. the other centres' extent on that axis is below 1/5.99 of the node's; an axis therefore carries at most
# log_6(extent / 1e-5) levels (below bvh's EPSILON the half split takes over), and the extent of a box stays below about 1e19 while
# the surface areas of all three axes are finite.  Three axes: about 3 log_6(1e19 / 1e-5) = 92 levels; measured 95 (chain3_models,
# 220 instances).  One axis alone: 56 (chain_models, 84 instances; one more box overflows to infinity).  A TLAS the device builds
# therefore never reaches the 4-wide parser's limit of 200; uploaded trees reach it in tests/test_gpu_wide_foreign_bvh.py.
CHAINS = {"x 60": (lambda: chain_models(60, 6.5, 39), 32), "x 84": (lambda: chain_models(84, 6.5, 39), 56),
          "xyz 160": (lambda: chain3_models(160), 94), "xyz 220": (lambda: chain3_models(220), 95)}


@pytest.mark.parametrize("chain", sorted(CHAINS))
def test_deepest_chains(chain):
    make, depth = CHAINS[chain]
    models = make()
    n = len(models)
    rng = np.random.default_rng(depth)
    w = plugin.World()                  # no light among the instances: their scale changes, and a light's would force the host path
    mesh, plain = w.add_mesh(*unit_cube()), w.add_material(material())
    for i in range(n):
        t = np.eye(4, dtype=np.float32)
        t[:3, 3] = rng.uniform(-20, 20, 3)
        w.add_instance(mesh, plain, t.T.reshape(16).copy())
    w.prepare()
    b = Bench("cornell", 48, 40, config="cornell_256")
    wide, flat, host = (plugin.HikariPlugin(48, 40) for _ in range(3))
    for p, mode in ((wide, 3), (flat, 0), (host, 3)):
        p.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, mode)
        p.set_keep_intermediates(True)
        p.upload_scene(w)
    for i, m in enumerate(models):
        w.set_instance_transform(i, m)
    w.previous_transform_system()
    assert wide.update_transforms(w) and flat.update_transforms(w)
    rec = device_records(wide)
    got = tlas_structure(rec["instance_nodes"], rec["instances"])
    assert got == depth, (n, got)
    w.prepare_instances()
    assert_scene_equals_host(wide, w, f"chain depth {depth}")
    host.update_instances(w)
    assert_wide_equal(wide, host, f"chain depth {depth}")
    assert (host.scene_readback(L.SCENE_WIDE_TLAS).size > 0) == (depth <= 200)       # wide_build.h refuses a deeper parse
    inp = b.inputs(1)
    wide.render_frame(inp); flat.render_frame(inp)
    assert_same(snapshot(wide, ALL_PLANES + DENOISED), snapshot(flat, ALL_PLANES + DENOISED), f"chain depth {depth}")
    for p in (wide, flat, host):
        p.close()


# ------------------------------------------------------------------------------------------------ D: the cache rule
F = np.float32


def glam_scale(m16):
    """glam Mat4::to_scale_rotation_translation().0 in f32: (|x_axis| * det.signum(), |y_axis|, |z_axis|), Rust's f32::signum
    (-1 for -0.0 and negative, +1 for +0.0 and positive, NaN for NaN), and abs_diff_eq below: what this restates of glam is the
    rule.  The arithmetic is the host's, not glam's: det is the upper 3x3's in host/hikari.cpp's order and the lengths are 3-vector
    lengths, where glam 0.22 on x86 takes the 4x4 Mat4::determinant and Vec4 lengths in SSE2 order.  For an affine model the
    values agree to rounding and a non-zero det has the same sign; the sign of a det that is exactly zero depends on the order of
    the operations, so the -0.0 case checks that the library applies signum's rule to the det it computes, not that its det has
    glam's sign bit."""
    m = np.asarray(m16, F)
    with np.errstate(all="ignore"):
        det = m[0] * (m[5] * m[10] - m[6] * m[9]) - m[4] * (m[1] * m[10] - m[2] * m[9]) + m[8] * (m[1] * m[6] - m[2] * m[5])
        signum = det if np.isnan(det) else np.copysign(F(1.0), det)
        length = [np.sqrt((m[c] * m[c] + m[c + 1] * m[c + 1]) + m[c + 2] * m[c + 2]) for c in (0, 4, 8)]
    return np.array([length[0] * signum, length[1], length[2]], F), det


def abs_diff_eq(a, b, eps=F(0.01)):
    """glam Vec3::abs_diff_eq: every |a - b| <= eps (NaN: false)"""
    with np.errstate(all="ignore"):
        return bool((np.abs(a - b) <= eps).all())


def axes_model(x, y, z):
    t = np.zeros(16, F)
    t[0:3], t[4:7], t[8:11], t[15] = x, y, z, 1.0
    t[12:15] = (0.2, 0.9, 0.1)
    return t


def zero_y_models():
    """two models scaled to zero on y with |x_axis| = |z_axis| = 1, one whose det is -0.0 and one whose det is +0.0"""
    found = {}
    for bits in range(512):                                        # the signs of the nine entries
        s = [(-1.0 if bits >> k & 1 else 1.0) for k in range(9)]
        m = axes_model((s[0], s[1] * 0.0, s[2] * 0.0), (s[3] * 0.0, s[4] * 0.0, s[5] * 0.0), (s[6] * 0.0, s[7] * 0.0, s[8]))
        det = glam_scale(m)[1]
        found.setdefault(bool(np.signbit(det)), m)
    return found[True], found[False]


def cache_case_models():
    """(name, model) steps of one emissive cube: scale deltas just under / at / just over 0.01 as f32 sees them, a mirror at
    equal magnitudes, a zero-scaled light whose det rounds to -0.0 and then +0.0"""
    b = F(0.01)                                                    # z scale b -> 2b: the f32 difference is exactly 0.01f
    under_at_over = [("z=b", axes_model((1, 0, 0), (0, 1, 0), (0, 0, b))),
                     ("z=2b-", axes_model((1, 0, 0), (0, 1, 0), (0, 0, np.nextafter(2 * b, F(0))))),
                     ("z=2b (delta 0.01f)", axes_model((1, 0, 0), (0, 1, 0), (0, 0, 2 * b))),
                     ("z=2b+", axes_model((1, 0, 0), (0, 1, 0), (0, 0, np.nextafter(2 * b, F(1)))))]
    one = F(1.0)
    hi = np.nextafter(one + F(0.01), one)                          # |y| from 1: largest delta <= 0.01f, smallest above
    while not abs_diff_eq(np.array([hi], F), np.array([one], F)):
        hi = np.nextafter(hi, one)
    over = np.nextafter(hi, F(2))
    around_one = [("unit", axes_model((1, 0, 0), (0, 1, 0), (0, 0, 1))), ("y just under", axes_model((1, 0, 0), (0, hi, 0), (0, 0, 1))),
                  ("unit again", axes_model((1, 0, 0), (0, 1, 0), (0, 0, 1))), ("y just over", axes_model((1, 0, 0), (0, over, 0), (0, 0, 1))),
                  ("mirrored x", axes_model((-1, 0, 0), (0, over, 0), (0, 0, 1))), ("mirrored y", axes_model((1, 0, 0), (0, -over, 0), (0, 0, 1)))]
    neg, pos = zero_y_models()
    zero = [("unit", axes_model((1, 0, 0), (0, 1, 0), (0, 0, 1))), ("zero y, det -0", neg), ("zero y, det -0 again", neg), ("zero y, det +0", pos)]
    return under_at_over + around_one + zero


def test_cache_rule_at_its_edges():
    steps = cache_case_models()
    assert sum(1 for _, m in steps if glam_scale(m)[1] == 0 and np.signbit(glam_scale(m)[1])) >= 1, "a det of -0.0 is among the cases"
    w = plugin.World()
    mesh = w.add_mesh(*unit_cube())
    glow, plain = w.add_material(material(emissive=(1.0, 0.8, 0.6, 0.5))), w.add_material(material())
    w.add_instance(mesh, plain, axes_model((1, 0, 0), (0, 1, 0), (0, 0, 1)))
    light = w.add_instance(mesh, glow, steps[0][1])
    w.prepare()
    dev = plugin.HikariPlugin(32, 24)
    dev.upload_scene(w)
    cached_scale, cached_model = glam_scale(steps[0][1])[0], steps[0][1]
    seen = set()
    for name, m in steps[1:]:
        w.set_instance_transform(light, m)
        w.previous_transform_system()
        scale = glam_scale(m)[0]
        hit = abs_diff_eq(cached_scale, scale)                   # instance.rs:385-397
        if not hit:
            cached_scale, cached_model = scale, m
        seen.add(hit)
        assert dev.update_transforms(w) == hit, (name, cached_scale, scale)
        w.prepare_instances()
        assert_scene_equals_host(dev, w, name)
        # the light's alias table is the one a fresh world builds for the transform the cache last took
        fresh = plugin.World()
        fm = fresh.add_mesh(*unit_cube())
        fresh.add_instance(fm, fresh.add_material(material(emissive=(1.0, 0.8, 0.6, 0.5))), cached_model)
        fresh.prepare()
        assert w.buffers()["alias_table"].tobytes() == fresh.buffers()["alias_table"].tobytes(), name
    assert seen == {True, False}
    dev.close()


# ------------------------------------------------------------------------------------------------ E: non-finite models
BAD = [np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)]


@pytest.mark.parametrize("bad", range(3))
@pytest.mark.parametrize("entry", [0, 5, 13])
def test_non_finite_models_are_refused_and_the_scene_is_kept(bad, entry):
    rng = np.random.default_rng(31 + entry)
    n = 9
    w = soup_world(rng, n, "random")
    dev = plugin.HikariPlugin(32, 24)
    dev.upload_scene(w)
    scene = plugin.SharedScene()
    scene.upload(w)
    cam = plugin.HikariPlugin(32, 24)
    cam.attach_scene(scene)
    good = [w.buffers()["instances"]["model"][i].copy() for i in range(n)]
    before = {k: v.tobytes() for k, v in device_records(dev).items()}
    victim = 3 if bad == 0 else 5                                  # an emissive instance (host path) and a plain one (device path)
    m = good[victim].copy()
    m[entry] = BAD[bad]
    w.set_instance_transform(victim, m)
    w.previous_transform_system()
    for p in (dev, scene):
        with pytest.raises(HikariError, match=f"instance {victim} "):
            p.update_transforms(w)
    arrays = w.prepare_instance_transforms()
    if arrays is not None:
        bad_models, prev, aabbs = arrays
        for p in (dev, scene):
            with pytest.raises(HikariError, match=f"instance {victim} "):
                p.update_transforms_arrays(bad_models, aabbs, prev)
    w.prepare_instances()                                          # the host mirror's build stays defined on this input
    for call in (dev.update_instances, dev.upload_scene, scene.update_instances, scene.upload):
        with pytest.raises(HikariError, match=f"instance {victim} "):
            call(w)
    for p in (dev, cam):
        assert {k: v.tobytes() for k, v in device_records(p).items()} == before, "a refused call leaves the scene as it was"
    # the next valid update is accepted, on either path
    for i in range(n):
        w.set_instance_transform(i, place(np.eye(3), rng, "rotated") if not is_emissive(i) else good[i])
    w.previous_transform_system()
    dev.update_transforms(w)
    scene.update_transforms(w)
    w.prepare_instances()
    assert_scene_equals_host(dev, w, "after a refused update")
    assert_scene_equals_host(cam, w, "after a refused update (shared)")
    inp = Bench("cornell", 32, 24, config="cornell_256").inputs(1)
    dev.render_frame(inp)
    cam.close(); dev.close(); scene.close()


def test_non_finite_mesh_aabbs_are_refused():
    """hk_scene_update_transforms refuses a non-finite mesh AABB as it refuses a non-finite model (its centre enters the SAH build)"""
    rng = np.random.default_rng(41)
    w = soup_world(rng, 9, "random")
    dev = plugin.HikariPlugin(32, 24)
    dev.upload_scene(w)
    before = {k: v.tobytes() for k, v in device_records(dev).items()}
    w.previous_transform_system()
    models, prev, aabbs = w.prepare_instance_transforms()
    for bad in BAD:
        broken = aabbs.copy()
        broken[4, 3] = bad
        with pytest.raises(HikariError, match="instance 4 has a non-finite mesh AABB"):
            dev.update_transforms_arrays(models, broken, prev)
    assert {k: v.tobytes() for k, v in device_records(dev).items()} == before
    dev.update_transforms_arrays(models, aabbs, prev)
    w.prepare_instances()
    assert_scene_equals_host(dev, w, "after a refused AABB")
    dev.close()
