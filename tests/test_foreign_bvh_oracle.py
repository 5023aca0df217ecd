"""The foreign-BVH generator (tests/foreign_bvh.py) against a BVH-free answer.  tests/test_gpu_wide_foreign_bvh.py holds the 4-wide
walk to the oracle's flat walk over generated arrays; that comparison means something only if the arrays are what they claim to be.
So here the oracle walks well-formed generated trees (every navigator box encloses its shapes) and must report, for every ray, the
nearest triangle a float64 brute-force query finds among the triangles the arrays name, and the same occluded-or-not verdict for
shadow rays.  Rays whose answer float32 rounding could flip (two hits within rounding of each other, a hit on a triangle's edge, a
determinant at the reference's cut-off) are counted and bounded instead.  A failure here means the test trees are wrong, not the
kernels."""
import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin, scenes
from tests import foreign_bvh as fb
from tests.conftest import Bench

EPS = float(np.finfo(np.float32).eps)
NO_HIT = 0xFFFFFFFF


def named(records):
    """shapes the leaf records of a flat array name"""
    e = records["entry_index"]
    return sorted(int(x) - fb.LEAF for x in e[e >= fb.LEAF])


def brute_force(bufs, rays, margin=1e-5):
    """per ray: (instance, primitive) of the nearest hit in float64, the reference's triangle test (light.wgsl:364-398) in each
    instance's object space, over the instances the TLAS names and the triangles their BLASes name; and whether float32 rounding
    could change that answer"""
    n = len(rays)
    o = rays["origin"].astype(np.float64)
    d = rays["direction"].astype(np.float64)
    tmax = rays["max_distance"].astype(np.float64)
    best = np.full(n, np.inf)
    second = np.full(n, np.inf)          # nearest hit of another triangle, loose test
    loose_best = np.full(n, np.inf)
    best_id = np.full((n, 2), NO_HIT, np.int64)
    loose_id = np.full((n, 2), NO_HIT, np.int64)
    prims = bufs["primitives"]["vertices"]["position"].astype(np.float64)
    for inst in named(bufs["instance_nodes"]):
        off, cnt, prim = fb.mesh_of(bufs, inst)
        tris = named(bufs["asset_nodes"][off:off + cnt])
        if not tris:
            continue
        M = bufs["instances"]["model"][inst].astype(np.float64).reshape(4, 4).T       # column-major
        Mi = np.linalg.inv(M)
        oo = o @ Mi[:3, :3].T + Mi[:3, 3]
        dd = d @ Mi[:3, :3].T
        for t in tris:
            p0, p1, p2 = prims[prim + t]
            ab, ac = p1 - p0, p2 - p0
            uvec = np.cross(dd, ac)
            det = uvec @ ab
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / det
                ao = oo - p0
                u = (ao * uvec).sum(1) * inv
                vvec = np.cross(ao, ab)
                v = (dd * vvec).sum(1) * inv
                dist = vvec @ ac * inv
            strict = (np.abs(det) >= 2 * EPS) & (u >= margin) & (v >= margin) & (u + v <= 1 - margin) & (dist > 2 * EPS)
            loose = (np.abs(det) >= 0.5 * EPS) & (u >= -margin) & (v >= -margin) & (u + v <= 1 + margin) & (dist > 0.5 * EPS)
            strict &= dist * (1 + margin) < tmax
            loose &= dist * (1 - margin) < tmax
            ds = np.where(strict, dist, np.inf)
            dl = np.where(loose, dist, np.inf)
            take = ds < best
            best = np.where(take, ds, best)
            best_id[take] = (inst, prim + t)
            # the second-nearest loose hit of any other triangle
            lt = dl < loose_best
            second = np.where(lt, loose_best, np.minimum(second, dl))
            loose_best = np.where(lt, dl, loose_best)
            loose_id[lt] = (inst, prim + t)
    ambiguous = (loose_id != best_id).any(axis=1) | (second <= best * (1 + margin) + margin)
    ambiguous &= ~(np.isinf(best) & np.isinf(loose_best))
    return best_id, ambiguous


def random_rays(n, seed, lo, hi, aim=None, shadow_fraction=0.4):
    """origins uniform in the box lo-hi; directions uniform, or towards points uniform in the box `aim`"""
    rng = np.random.default_rng(seed)
    rays = np.zeros(n, L.RAY)
    rays["origin"] = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    dv = rng.normal(size=(n, 3)) if aim is None else rng.uniform(*aim, (n, 3)) - rays["origin"]
    rays["direction"] = (dv / np.linalg.norm(dv, axis=1, keepdims=True)).astype(np.float32)
    shadow = rng.random(n) < shadow_fraction
    far = rng.uniform(0.2, 4.0, n).astype(np.float32)
    rays["max_distance"] = np.where(shadow, far, np.float32(3.402823466e38))
    rays["early_distance"] = np.where(shadow, far - np.float32(0.1), np.float32(0.0))
    rays["exclude_instance"] = NO_HIT
    return rays, shadow


def check(bufs, rays, shadow, max_ambiguous=2e-3):
    from oracle import oracle
    orc = oracle.Oracle(8, 8, plugin.load_noise())
    orc.upload_scene_desc(plugin.scene_desc_from_buffers(bufs))
    h = orc.trace_rays(rays)
    ids, ambiguous = brute_force(bufs, rays)
    got = np.stack([h["instance_index"], h["primitive_index"]], 1).astype(np.int64)
    sure = ~ambiguous
    c = sure & ~shadow
    wrong = c & (got != ids).any(axis=1)
    assert not wrong.any(), f"{int(wrong.sum())} closest-hit rays miss the nearest triangle, e.g. {np.nonzero(wrong)[0][:5]}"
    s = sure & shadow
    occluded = h["instance_index"] != NO_HIT
    assert np.array_equal(occluded[s], ids[s, 0] != NO_HIT), "a shadow ray's verdict differs from the brute-force query"
    assert ambiguous.mean() <= max_ambiguous, f"{int(ambiguous.sum())} of {len(rays)} rays are within rounding of another answer"
    assert (ids[c, 0] != NO_HIT).sum() >= 400            # the rays do meet the scene
    return int(ambiguous.sum())


CORNELL_BOUNDS = ([-0.95, 0.05, -0.95], [0.95, 1.95, 0.95])

# (label, BLAS generator keywords for every mesh, TLAS generator keywords): every tree well formed (exact or inflated boxes)
FAMILIES = [
    ("binary_median", dict(arity=2), dict(arity=2)),
    ("runs_of_3_and_4", dict(arity=[3, 4]), dict(arity=4, top=3)),
    ("runs_of_5_8_17", dict(arity=[5, 8, 17]), dict(arity=5, top=5)),
    ("arity_1_wrappers", dict(arity=[1, 2, 1, 3]), dict(arity=[1, 2], top=2)),
    ("random_splits", dict(arity=[2, 6, 3], split="random", seed=4), dict(arity=3, top=4, split="random", seed=5)),
    ("chains", dict(arity=2, split="chain"), dict(arity=3, split="chain")),
    ("arity_8", dict(arity=8), dict(arity=8, top=8)),
    ("inflated", dict(arity=2, boxes="inflated"), dict(arity=2, boxes="inflated", delta=0.2)),
]


def foreign_scene(bench, blas_kw, tlas_kw):
    bufs = bench.world.buffers()
    done = set()
    for i in range(len(bufs["instances"])):
        key = fb.mesh_of(bufs, i)
        if key not in done and fb.triangle_count(bufs, i) > 0:
            fb.foreign_blas(bufs, i, **blas_kw)
            done.add(fb.mesh_of(bufs, i))
    fb.foreign_tlas(bufs, **tlas_kw)
    return bufs


@pytest.mark.parametrize("label,blas_kw,tlas_kw", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_generated_trees_find_the_nearest_triangle_cornell(label, blas_kw, tlas_kw):
    bufs = foreign_scene(Bench("cornell", 8, 8), blas_kw, tlas_kw)
    rays, shadow = random_rays(20_000, 31, *CORNELL_BOUNDS)
    check(bufs, rays, shadow)


@pytest.mark.parametrize("seed", [3, 17, 29])
@pytest.mark.parametrize("label,blas_kw,tlas_kw", FAMILIES[1:6], ids=[f[0] for f in FAMILIES[1:6]])
def test_generated_trees_find_the_nearest_triangle_soup(label, blas_kw, tlas_kw, seed):
    """random triangle soups (scenes.soup): degenerate and single-triangle meshes, mirrored and non-uniform instances"""
    scenes.SCENE_BUILDERS["_soup"] = lambda: scenes.soup(seed)
    try:
        b = Bench("_soup", 8, 8)
    finally:
        del scenes.SCENE_BUILDERS["_soup"]
    bufs = foreign_scene(b, dict(blas_kw, seed=seed), dict(tlas_kw, seed=seed + 1))
    rays, shadow = random_rays(20_000, seed, [-3.0] * 3, [3.0] * 3, aim=([-1.0] * 3, [1.0] * 3))
    check(bufs, rays, shadow)


def test_empty_single_record_and_one_instance_trees():
    """a mesh with no records (its instance can never be hit), meshes whose BVH is one leaf record (only that triangle can be),
    and a TLAS over one instance (only it can be)"""
    b = Bench("cornell", 8, 8)
    rays, shadow = random_rays(20_000, 37, *CORNELL_BOUNDS)
    bufs = b.world.buffers()
    fb.set_blas(bufs, 0, np.zeros(0, L.NODE))
    lo, hi = fb.triangle_boxes(bufs, 3)
    fb.set_blas(bufs, 3, fb.flatten([1], lo, hi))
    fb.foreign_tlas(bufs, arity=3)
    check(bufs, rays, shadow)
    hits = {int(i) for i in brute_force(bufs, rays)[0][:, 0]}
    assert 0 not in hits and 2 in hits
    bufs = b.world.buffers()
    lo, hi = fb.instance_boxes(bufs)
    fb.set_tlas(bufs, fb.flatten([6], lo, hi))
    assert len(bufs["instance_nodes"]) == 1
    check(bufs, rays, shadow)
    assert {int(i) for i in brute_force(bufs, rays)[0][:, 0]} <= {6, NO_HIT}


def test_flatten_writes_skip_links():
    """navigator: entry = next record, exit = behind its subtree; leaf: exit = next record; a run of five branches under one
    navigator; a single shape is one leaf record"""
    lo = np.zeros((6, 3), np.float32) + np.arange(6, dtype=np.float32)[:, None]
    hi = lo + 1
    r = fb.flatten([[0, 1, 2, 3, 4], 5], lo, hi)
    assert len(r) == 1 + 5 * 2 + 2
    assert (r[0]["entry_index"], r[0]["exit_index"]) == (1, 11)
    assert [int(x) for x in r["entry_index"][2:11:2]] == [fb.LEAF + s for s in range(5)]
    assert [int(x) for x in r["exit_index"][1:11:2]] == list(range(3, 12, 2))
    assert np.array_equal(r[0]["min"], lo[0]) and np.array_equal(r[0]["max"], hi[4])
    assert (r[11]["entry_index"], r[11]["exit_index"], r[12]["entry_index"], r[12]["exit_index"]) == (12, 13, fb.LEAF + 5, 13)
    one = fb.flatten([2], lo, hi)
    assert len(one) == 1 and one[0]["entry_index"] == fb.LEAF + 2 and one[0]["exit_index"] == 1
    t = fb.tree(lo, hi, arity=2, split="chain")
    assert t == [0, [1, [2, [3, [4, 5]]]]]
    inflated, tight = fb.flatten(t, lo, hi, boxes="inflated"), fb.flatten(t, lo, hi, boxes="tight")
    assert (inflated[0]["min"] < lo[0]).all() and (tight[2]["min"] > lo[1]).all()
