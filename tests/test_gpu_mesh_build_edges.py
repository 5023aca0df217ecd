"""hk_scene_add_meshes (csrc/kernels_scene.cu) at the edges of its two cooperative kernels: kc_build_blas_top, one 1024-thread CTA
per mesh that splits every node of more than BLAS_TOP_SHAPES = 4096 shapes, and kc_build_blas_bottom, whose CTAs take the smaller
subtrees from a work list.  tests/test_gpu_mesh_build.py meets the CTA-level split only on random soups; here every branch it has is
reached at CTA level:

  A. the threshold: soups of 4095 / 4096 / 4097 / 8192 / 8193 triangles, a root split into exactly 4096 + 4097, a CTA child of one
     shape (a work-list root that is a leaf), and a chain of such children long enough that the bottom kernel's claim loop goes round;
  B. the halves: one triangle copied 10 000 and 4097 times (an odd count: the left half is count / 2 rounded down), 9000 triangles
     whose centres span less than bvh's epsilon while their boxes differ, 5000 copies among 3000 spread triangles (halves one level
     down);
  C. non-finite positions (the patterns of test_gpu_mesh_build's `nonfinite` mesh) at 0.1 %, 10 % and 99.9 % of 20 000 triangles,
     and meshes whose root has no finite SAH candidate, so the CTA hands children with the empty box (SEG_EMPTY_BOX) to the work list;
  D. signed zeros: the first zero of a CTA-level node's bound in warp 0, in warp 1, in the last warp, past the first 1024 shapes and
     last, each sign first;
  E. one call of about 3000 meshes (single primitives, strips, unused vertices) around three large meshes: more work-list entries
     than the bottom kernel has CTAs, several top CTAs on one counter, the primitive -> mesh search over thousands of jobs;
  F. appends in sequence on a shared scene behind queued frames of two cameras: growth, in-place appends and growth again, caller
     arrays overwritten on return, transform and instance updates between the calls, a re-upload and more adds; then device-built
     meshes (an emissive one among them) under hk_scene_update_transforms.

Every case holds the device's vertex, primitive and BLAS records and the returned hk_mesh_index records to the host mirror byte for
byte, and every BLAS to float64 anchors computed on the device's own records, which do not go through either C++ builder:
  * structure: 3 m - 2 records (1 for m = 1), skip links that parse as a pre-order, every primitive in exactly one leaf;
  * boxes: a navigator is the componentwise min / max of its subtree's primitive boxes (NaN components skipped, as a join that starts
    at +-inf skips them; the sign of zero aside), or the empty box where the mesh holds non-finite positions;
  * splits: at a node of finite boxes whose centres span at least bvh's epsilon along their largest axis, the children are separated
    by bucket along that axis, bucket = trunc((c - min) / extent * 5.99) in f32 (bvh 0.7.1), and the left count is that of the
    cheapest of the five SAH candidates, costs in float64, ties within COST_TIE; below the epsilon the left child holds count / 2;
  * rays (A, B, D, E): the oracle's flat walk over the device's records finds the nearest triangle a float64 brute-force query finds
    (tests/test_foreign_bvh_oracle.py), rays within rounding of another answer counted and bounded.
tests/test_mesh_build_edges_emulated.py runs the CTA-level cases of A-D at their smallest sizes on the emulated kernels."""
import numpy as np
import pytest

from bevy_hikari_b200 import layout as L
from bevy_hikari_b200 import plugin
from tests import foreign_bvh as fb
from tests.conftest import Bench
from tests.test_foreign_bvh_oracle import check as check_rays
from tests.test_gpu_mesh_build import (READBACK, assert_added_equal_the_mirror, assert_bytes_equal, fresh_device, mirror,
                                       quad_grid, show_device_instances, soup, split_world)

pytestmark = pytest.mark.gpu

LEAF = 0x80000000
BLAS_TOP_SHAPES = 4096               # kernels_scene.cu: nodes above this many shapes are split by a whole CTA
BOTTOM_CTAS = 1056                   # kernels_scene.cu hk_launch_build_meshes: the most CTAs kc_build_blas_bottom is launched with
EPSILON = np.float32(1e-5)           # bvh 0.7.1's EPSILON: below it the centres are taken to coincide and the node is halved
BUCKET_SCALE = np.float32(6) - np.float32(0.01)
# f32 costs round each of about a dozen operations once (every term is a product or sum of non-negative values), so two candidates
# whose float64 costs differ by less than this may come out in either order in f32
COST_TIE = 1e-5


# ------------------------------------------------------------------------------------------------ anchors
def primitive_boxes(prims):
    """per primitive: its box as GpuMesh::try_from computes it, std::min(std::min(a, b), c) in f32 (a NaN first vertex poisons the
    component, a later NaN is skipped), from the device's primitive records"""
    p = prims["vertices"]["position"].astype(np.float32)
    a, b, c = p[:, 0], p[:, 1], p[:, 2]
    smin = lambda x, y: np.where(y < x, y, x)
    smax = lambda x, y: np.where(x < y, y, x)
    return smin(smin(a, b), c), smax(smax(a, b), c)


def parse(rec, m):
    """(leaves in pre-order, navigators as (record, first leaf, end leaf), internal nodes as (first leaf, first right leaf, end leaf))"""
    assert len(rec) == (1 if m == 1 else 3 * m - 2), ("record count", len(rec), m)
    entry, exit_ = rec["entry_index"].astype(np.int64), rec["exit_index"].astype(np.int64)
    leaves, navs, nodes = [], [], []

    def node(i):                     # the records of one node start at i; returns the record behind them
        assert i < len(rec), ("skip link out of range", i)
        if entry[i] >= LEAF:
            assert exit_[i] == i + 1, ("leaf exit", i)
            leaves.append(int(entry[i] - LEAF))
            return i + 1
        a = len(leaves)
        j = branch(i)
        k = len(leaves)
        end = branch(j)
        nodes.append((a, k, len(leaves)))
        return end

    def branch(i):
        assert entry[i] == i + 1, ("navigator entry", i)
        a = len(leaves)
        end = node(i + 1)
        assert exit_[i] == end, ("navigator exit", i, int(exit_[i]), end)
        navs.append((i, a, len(leaves)))
        return end

    end = node(0)
    assert end == len(rec), ("records behind the tree", end, len(rec))
    assert m == 1 or nodes, "a root of more than one shape is a leaf"
    assert sorted(leaves) == list(range(m)), "a primitive is missing from the leaves or named twice"
    return np.array(leaves, np.int64), navs, nodes


def check_blas(rec, prims, what, allow_empty=False):
    """the float64 anchors of one BLAS (records and primitives of one mesh, as the device wrote them)"""
    m = len(prims)
    leaves, navs, nodes = parse(rec, m)
    lo32, hi32 = primitive_boxes(prims)
    lo = np.where(np.isnan(lo32), np.inf, lo32).astype(np.float64)[leaves]       # in leaf order
    hi = np.where(np.isnan(hi32), -np.inf, hi32).astype(np.float64)[leaves]
    # boxes: prefix-free range min / max over the leaf ranges (sparse tables)
    def table(v, op):
        t = [v]
        while 2 ** len(t) <= len(v):
            s = 2 ** (len(t) - 1)
            t.append(op(t[-1][:-s], t[-1][s:]))
        return t

    def query(t, op, a, b):
        k = int(np.log2(b - a))
        return op(t[k][a], t[k][b - 2 ** k])
    tlo, thi = table(lo, np.minimum), table(hi, np.maximum)
    empties = 0
    for i, a, b in navs:
        got_lo, got_hi = rec["min"][i].astype(np.float64), rec["max"][i].astype(np.float64)
        if (got_lo == np.inf).all() and (got_hi == -np.inf).all() and allow_empty:
            empties += 1
            continue
        want_lo, want_hi = query(tlo, np.minimum, a, b), query(thi, np.maximum, a, b)
        assert (got_lo == want_lo).all() and (got_hi == want_hi).all(), \
            (what, "navigator", i, got_lo, got_hi, "subtree", want_lo, want_hi)
    # splits
    c32 = (lo32 + (hi32 - lo32) / np.float32(2))[leaves]        # AABB::center in f32
    finite = np.isfinite(lo32[leaves]).all(1) & np.isfinite(hi32[leaves]).all(1)
    bad_prefix = np.concatenate([[0], np.cumsum(~finite)])
    area = lambda l, h: 2.0 * ((h[0] - l[0]) * (h[1] - l[1]) + (h[0] - l[0]) * (h[2] - l[2]) + (h[1] - l[1]) * (h[2] - l[2]))
    checked = 0
    for a, k, b in nodes:
        if bad_prefix[b] != bad_prefix[a]:
            continue
        c = c32[a:b]
        cmin, cmax = c.min(0), c.max(0)
        s = cmax - cmin
        axis = 0 if (s[0] > s[1] and s[0] > s[2]) else (1 if s[1] > s[2] else 2)
        extent = s[axis]
        if extent < EPSILON:
            assert k - a == (b - a) // 2, (what, "halves", a, k, b)
            checked += 1
            continue
        x = ((c[:, axis] - cmin[axis]) / extent) * BUCKET_SCALE
        bucket = np.where(x > 0, np.minimum(np.floor(np.where(x > 0, x, 0)), 5), 0).astype(np.int64)
        assert bucket[:k - a].max() < bucket[k - a:].min(), (what, "children not separated by bucket", a, k, b)
        nl, costs = [], []
        parent = area(lo[a:b].min(0), hi[a:b].max(0))
        for i in range(5):
            left = bucket <= i
            nl.append(int(left.sum()))
            if nl[-1] in (0, b - a):
                costs.append(np.nan)
                continue
            l_, r_ = slice(a, b), slice(a, b)
            al = area(lo[l_][left].min(0), hi[l_][left].max(0))
            ar = area(lo[r_][~left].min(0), hi[r_][~left].max(0))
            costs.append((nl[-1] * al + (b - a - nl[-1]) * ar) / parent)
        costs = np.array(costs)
        best = np.nanmin(costs)
        ok = [i for i in range(5) if nl[i] == k - a and costs[i] <= best * (1 + COST_TIE)]
        assert ok, (what, "not the cheapest SAH candidate", a, k, b, nl, costs)
        checked += 1
    return {"empty_navigators": empties, "splits_checked": checked}


def device_blases(dev, got):
    """per added mesh: (its BLAS records, its primitive records), sliced from the device's buffers by its hk_mesh_index"""
    nodes, prims = dev.scene_readback(L.SCENE_ASSET_NODES), dev.scene_readback(L.SCENE_PRIMITIVES)
    out = []
    for g in got:
        off, cnt, p = int(g["node_offset"]), int(g["node_count"]), int(g["primitive"])
        m = cnt if cnt == 1 else (cnt + 2) // 3
        out.append((nodes[off:off + cnt], prims[p:p + m]))
    return out


def aimed_rays(tris, n, seed):
    """rays towards random interior points of random finite triangles without a copy, from 0.5-5 units away; 40 % shadow rays that end before or
    after that point"""
    rng = np.random.default_rng(seed)
    _, first, count = np.unique(tris.reshape(len(tris), -1), axis=0, return_index=True, return_counts=True)
    ok = np.intersect1d(first[count == 1], np.nonzero(np.isfinite(tris).all((1, 2)))[0])     # a copied triangle makes every hit a tie
    pick = tris[rng.choice(ok, n)].astype(np.float64)
    u, v = rng.uniform(0.05, 0.45, n), rng.uniform(0.05, 0.45, n)
    target = pick[:, 0] + u[:, None] * (pick[:, 1] - pick[:, 0]) + v[:, None] * (pick[:, 2] - pick[:, 0])
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    dist = rng.uniform(0.5, 5.0, n)
    rays = np.zeros(n, L.RAY)
    rays["origin"] = (target - d * dist[:, None]).astype(np.float32)
    rays["direction"] = d.astype(np.float32)
    shadow = rng.random(n) < 0.4
    far = (dist * rng.uniform(0.5, 1.5, n)).astype(np.float32)
    rays["max_distance"] = np.where(shadow, far, np.float32(3.402823466e38))
    rays["early_distance"] = np.where(shadow, far - np.float32(0.1), np.float32(0.0))
    rays["exclude_instance"] = 0xFFFFFFFF
    return rays, shadow


def check_rays_on(dev, meshes, which, seed, n=3000):
    """the mirror world's instances (one per mesh, identity) with the device's records; the TLAS holds the instance of mesh `which`"""
    bufs, _ = mirror(meshes)
    for w, name in READBACK:
        bufs[name] = dev.scene_readback(w)
    lo, hi = fb.instance_boxes(bufs)
    fb.set_tlas(bufs, fb.flatten([which + 1], lo, hi))
    _, _, p = fb.mesh_of(bufs, which + 1)
    tris = bufs["primitives"]["vertices"]["position"][p:p + fb.triangle_count(bufs, which + 1)]
    rays, shadow = aimed_rays(tris, n, seed)
    return check_rays(bufs, rays, shadow)


def add_and_check(meshes, what, rays=(), allow_empty=False, dev=None):
    """one call that adds `meshes`; records == the host mirror, anchors on every BLAS, rays on the meshes listed in `rays`"""
    own = dev is None
    dev = dev or fresh_device()
    got = dev.add_mesh_sources(meshes)
    assert_added_equal_the_mirror(dev, meshes, got, what)
    stats = [check_blas(r, p, f"{what} mesh {i}", allow_empty) for i, (r, p) in enumerate(device_blases(dev, got))]
    for k, i in enumerate(rays):
        check_rays_on(dev, meshes, i, seed=len(meshes) + k)
    if own:
        dev.close()
    return got, stats


def triangles(pos, nrm=None):
    """a non-indexed mesh of the triangles pos (n x 3 x 3)"""
    p = np.ascontiguousarray(pos, np.float32).reshape(-1, 3)
    rng = np.random.default_rng(len(p))
    return (p, rng.normal(size=p.shape).astype(np.float32) if nrm is None else nrm, rng.random((len(p), 2)).astype(np.float32), None)


def small_triangles(centres, size=0.05, seed=0):
    rng = np.random.default_rng(seed)
    return np.asarray(centres, np.float64)[:, None, :] + rng.normal(0, size, (len(centres), 3, 3))


# ------------------------------------------------------------------------------------------------ A: the threshold
def clusters(n_left, n_right, seed):
    """two clusters far apart along x: every centre of the first in bucket 0, of the second in bucket 5, so the root splits into
    exactly n_left + n_right"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 10, (n_left, 3))
    b = rng.uniform(0, 10, (n_right, 3)) + [1e4, 0, 0]
    return triangles(small_triangles(np.concatenate([a, b]), seed=seed))


def outliers(n_cluster, n_out, seed):
    """a cluster in [0, 10]^3 and `n_out` triangles at x = 10 * 7^k: each lies past 5.99 times the extent of everything nearer, so
    every CTA-level split peels off one outlier: a child of one shape, handed to the work list as a leaf"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 10, (n_cluster, 3))
    b = np.array([[10.0 * 7.0 ** (k + 1), 5, 5] for k in range(n_out)])
    return triangles(small_triangles(np.concatenate([a, b]), seed=seed))


THRESHOLD = {
    "soup_4095": lambda: soup(4095, 40), "soup_4096": lambda: soup(4096, 41), "soup_4097": lambda: soup(4097, 42),
    "soup_8192": lambda: soup(8192, 43), "soup_8193": lambda: soup(8193, 44),
    "clusters_4096_4097": lambda: clusters(4096, 4097, 45),
    "outlier_6000": lambda: outliers(6000, 1, 46),
    "outliers_4097_4": lambda: outliers(4097, 4, 47),
}


@pytest.mark.parametrize("case", sorted(THRESHOLD))
def test_threshold(case):
    mesh = THRESHOLD[case]()
    add_and_check([mesh], case, rays=[0])
    m = len(mesh[0]) // 3
    if case.startswith("outliers"):
        # the top kernel hands out one work-list entry per outlier plus the cluster's two halves: more than it launches CTAs for
        n_out = int(case.split("_")[-1])
        launched = min(BOTTOM_CTAS, 1 + 2 * (m // BLAS_TOP_SHAPES) + 1)
        assert n_out + 2 > launched, (n_out, launched)


def test_clusters_split_exactly_at_the_threshold():
    """the root's left child holds 4096 shapes (the work list), the right 4097 (one more CTA-level split)"""
    mesh = THRESHOLD["clusters_4096_4097"]()
    dev = fresh_device()
    got = dev.add_mesh_sources([mesh])
    (rec, prims), = device_blases(dev, got)
    leaves, navs, nodes = parse(rec, len(prims))
    root = max(nodes, key=lambda n: n[2] - n[0])
    assert (root[1] - root[0], root[2] - root[1]) == (4096, 4097)
    dev.close()


# ------------------------------------------------------------------------------------------------ B: the halves
def copies(n, seed):
    one = soup(1, seed)
    return (np.tile(one[0], (n, 1)), np.tile(one[1], (n, 1)), np.tile(one[2], (n, 1)), None)


def tight_centres(n, seed):
    """triangles whose boxes are symmetric about (1, 2, 3) with random half-extents: the centres agree to f32 rounding (< 1e-5)"""
    rng = np.random.default_rng(seed)
    h = rng.uniform(0.1, 1.0, (n, 3))
    c = np.array([1.0, 2.0, 3.0])
    t = np.stack([c + h * [-1, -1, -1], c + h * [1, -1, 1], c + h * [0, 1, 0]], 1)
    return triangles(t)


def coincident_among_spread(n_same, n_spread, seed):
    rng = np.random.default_rng(seed)
    same = np.tile(small_triangles([[0.3, 0.2, 0.1]], seed=seed), (n_same, 1, 1))
    spread = small_triangles(rng.uniform(-10, 10, (n_spread, 3)), seed=seed + 1)
    t = np.concatenate([same, spread])
    return triangles(t[rng.permutation(len(t))])


HALVES = {
    "copies_10000": (lambda: copies(10000, 50), False), "copies_4097": (lambda: copies(4097, 51), False),
    "tight_centres_9000": (lambda: tight_centres(9000, 52), False),
    "coincident_5000_spread_3000": (lambda: coincident_among_spread(5000, 3000, 53), True),
}


@pytest.mark.parametrize("case", sorted(HALVES))
def test_halves(case):
    """rays only where one answer exists: copies and shared centres make every hit a tie"""
    make, rays = HALVES[case]
    _, (stats,) = add_and_check([make()], case, rays=[0] if rays else [])
    assert stats["splits_checked"] > 0


# ------------------------------------------------------------------------------------------------ C: non-finite input
def nonfinite_soup(n, density, seed):
    """soup(n) with the four patterns of test_gpu_mesh_build's `nonfinite` mesh ([inf, 0, 0], [nan, 1, 2], a -inf component, a
    whole-NaN vertex) on a `density` fraction of its vertices"""
    m = list(soup(n, seed))
    p = m[0].copy()
    rng = np.random.default_rng(seed)
    hit = np.nonzero(rng.random(len(p)) < density)[0]
    kind = rng.integers(0, 4, len(hit))
    p[hit[kind == 0]] = [np.inf, 0, 0]
    p[hit[kind == 1]] = [np.nan, 1, 2]
    p[hit[kind == 2], 1] = -np.inf
    p[hit[kind == 3]] = np.nan
    m[0] = p
    return tuple(m)


def no_finite_candidate(n, seed):
    """boxes from -inf to +inf along x and flat in z, centres spread along y: every SAH cost is inf * 0 = NaN, so no candidate is
    chosen and bvh leaves both children the empty box (the split itself is bucket 0 against the rest)"""
    rng = np.random.default_rng(seed)
    y = rng.uniform(0, 10, n)
    t = np.zeros((n, 3, 3))
    t[:, 0] = np.stack([np.full(n, -np.inf), y, np.zeros(n)], 1)
    t[:, 1] = np.stack([np.full(n, np.inf), y, np.zeros(n)], 1)
    t[:, 2] = np.stack([np.zeros(n), y, np.zeros(n)], 1)
    return triangles(t)


NONFINITE = {
    "nonfinite_0.1pct": lambda: nonfinite_soup(20000, 0.001, 60), "nonfinite_10pct": lambda: nonfinite_soup(20000, 0.1, 61),
    "nonfinite_99.9pct": lambda: nonfinite_soup(20000, 0.999, 62),
    "no_finite_candidate_4097": lambda: no_finite_candidate(4097, 63), "no_finite_candidate_9000": lambda: no_finite_candidate(9000, 64),
}


@pytest.mark.parametrize("case", sorted(NONFINITE))
def test_nonfinite(case):
    mesh = NONFINITE[case]()
    with np.errstate(invalid="ignore"):
        _, (stats,) = add_and_check([mesh], case, allow_empty=True)
    if case.startswith("no_finite"):
        host, idx = mirror([mesh])
        rec = host["asset_nodes"][int(idx[0]["node_offset"]):][:int(idx[0]["node_count"])]
        empty = (rec["min"] == np.inf).all(1) & (rec["max"] == -np.inf).all(1) & (rec["entry_index"] < LEAF)
        left, right = 0, int(rec["exit_index"][0])
        assert empty[left] and empty[right], "the root's children carry the empty box"
        assert empty.sum() == stats["empty_navigators"], "the device's records carry the empty box where the mirror's do"


# ------------------------------------------------------------------------------------------------ D: signed zeros
D_CLUSTER = 4160                     # > 4096: the root's left child is split by the CTA, which writes its navigator
D_FAR = 8


def signed_zero_mesh(at, first_negative):
    """a cluster of D_CLUSTER triangles on a 0.1 grid in z = 0, then D_FAR triangles at x = 1e4 (the root splits off the cluster
    as its left child, in primitive order).  In the cluster, triangles before `at` are lifted to z in [0.5, 1]; triangle `at` has
    z = -0 on all three vertices (+0 if not first_negative); the rest have the other zero.  So the cluster's bound in z starts at
    triangle `at`'s zero, whatever the vertex order."""
    rng = np.random.default_rng(at)
    cols = 65
    ij = np.stack([np.arange(D_CLUSTER) % cols, np.arange(D_CLUSTER) // cols], 1) * 0.1
    t = np.zeros((D_CLUSTER + D_FAR, 3, 3), np.float32)
    t[:D_CLUSTER, :, :2] = ij[:, None, :] + np.float32([[0, 0], [0.08, 0], [0, 0.08]])
    first, rest = (np.float32(-0.0), np.float32(0.0)) if first_negative else (np.float32(0.0), np.float32(-0.0))
    t[:D_CLUSTER, :, 2] = rest
    t[at, :, 2] = first
    t[:at, :, 2] = rng.uniform(0.5, 1.0, (at, 3))
    t[D_CLUSTER:] = small_triangles(rng.uniform(0, 6, (D_FAR, 3)) + [1e4, 0, 0], seed=at)
    return triangles(t)


SIGNED_AT = {"0": 0, "31": 31, "32": 32, "1023": 1023, "1024": 1024, "4096": 4096, "last": D_CLUSTER - 1}


@pytest.mark.parametrize("first", ["minus_first", "plus_first"])
@pytest.mark.parametrize("at", list(SIGNED_AT))
def test_signed_zero(at, first):
    p = SIGNED_AT[at]
    mesh = signed_zero_mesh(p, first == "minus_first")
    dev = fresh_device()
    got, _ = add_and_check([mesh], f"zero at {at} {first}", rays=[0], dev=dev)
    (rec, prims), = device_blases(dev, got)
    dev.close()
    leaves, navs, nodes = parse(rec, len(prims))
    root = max(nodes, key=lambda n: n[2] - n[0])
    assert root[1] - root[0] == D_CLUSTER, "the cluster is the root's left child"
    # bvh joins its children's boxes in order with f32::min / max, which keep the first of two equal zeros
    sign = lambda v: bool(np.signbit(np.float32(v)))
    want = first == "minus_first"
    assert sign(rec["min"][0][2]) == want, ("the cluster's min z", rec["min"][0][2])
    if p == 0:
        assert sign(rec["max"][0][2]) == want, ("the cluster's max z", rec["max"][0][2])


# ------------------------------------------------------------------------------------------------ E: large batches
def small_meshes(n, seed):
    """n meshes of 1-40 triangles: single primitives, indexed and non-indexed strips and lists, meshes with unused vertices, with
    more vertices than primitives and fewer"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        kind = i % 5
        k = int(rng.integers(1, 41)) if kind else 1
        c = rng.uniform(-5, 5, 3)
        if kind == 0 or kind == 1:           # a list, non-indexed
            out.append(triangles(small_triangles(c + rng.uniform(-1, 1, (k, 3)), seed=i)))
        elif kind == 2:                      # a strip over k + 2 vertices, indexed in reverse; or non-indexed
            v = (c + rng.uniform(-1, 1, (k + 2, 3))).astype(np.float32)
            idx = np.arange(k + 2, dtype=np.uint32)[::-1].copy() if i % 2 else None
            out.append((v, v.copy(), v[:, :2].copy(), idx, L.TOPOLOGY_TRIANGLE_STRIP))
        elif kind == 3:                      # indexed over a shared pool with unused vertices: more vertices than primitives
            v = (c + rng.uniform(-1, 1, (3 * k + 7, 3))).astype(np.float32)
            idx = rng.choice(3 * k, 3 * k).astype(np.uint32)
            out.append((v, v.copy(), v[:, :2].copy(), idx))
        else:                                # a fan over 3 vertices: many more primitives than vertices
            v = (c + rng.uniform(-1, 1, (3, 3))).astype(np.float32)
            idx = np.tile(np.uint32([0, 1, 2, 2, 0, 1]), k)[:3 * k]
            out.append((v, v.copy(), v[:, :2].copy(), idx))
    return out


def test_large_batch():
    small = small_meshes(3000, 70)
    big = [soup(5000, 71), clusters(4096, 4097, 72), soup(4500, 73)]
    meshes = [big[0]] + small[:1500] + [big[1]] + small[1500:] + [big[2]]
    positions = {0: 0, 1501: 1, len(meshes) - 1: 2}
    dev = fresh_device()
    got, stats = add_and_check(meshes, "3000 meshes", dev=dev)
    shapes = [(int(g["node_count"]) + 2) // 3 for g in got]
    entries = sum(1 for s in shapes if 1 < s <= BLAS_TOP_SHAPES) + sum(2 for s in shapes if s > BLAS_TOP_SHAPES)
    assert entries > BOTTOM_CTAS, (entries, "work-list entries: the bottom kernel's CTAs must go round")
    assert sum(1 for s in shapes if s > BLAS_TOP_SHAPES) == len(positions)
    assert len({int(g["vertex"]) for g in got}) == len(meshes)
    # the large meshes, and one small mesh of each kind with a unique nearest hit (the fans repeat one triangle)
    for k, i in enumerate(list(positions) + [1, 2, 3, 4]):
        check_rays_on(dev, meshes, i, seed=700 + k)
    dev.close()


# ------------------------------------------------------------------------------------------------ F: appends in sequence
def placed(k):
    """model of the instance of extra mesh k: the soups shrunk to a few centimetres, in a row inside the cornell box"""
    m = np.diag([0.02, 0.02, 0.02, 1.0]).astype(np.float32)
    m[:3, 3] = [-0.6 + 0.25 * k, 0.4 + 0.1 * (k % 3), -0.2]
    return m.T.reshape(16)


F_EXTRA = [lambda: soup(5000, 80), lambda: soup(120, 81), lambda: quad_grid(4), lambda: soup(3000, 82), lambda: soup(300, 83),
           lambda: soup(9000, 84)]
F_CALLS = [[0], [1], [2], [3], [4], [5]]          # extra meshes per call; the first call also takes cornell's device meshes
F_EMISSIVE = 1                                     # the extra mesh whose instance gets cornell's emissive material
F_LIGHT_MATERIAL = 4


def appended_world(b, first_added, extra, device=True):
    """the bench's scene with meshes [first_added, ..) and `extra` (one instance each) as device meshes whose instances are hidden
    until added; device=False: the same scene built and shown entirely by the host (the mirror)"""
    sc = b.scene
    w = plugin.World()
    for t in sc.textures:
        w.add_texture(t["rgba"], t["address_mode_u"], t["address_mode_v"], t["filter_linear"], t["srgb"])
    for i, m in enumerate(list(sc.meshes) + list(extra)):
        (w.add_device_mesh if device and i >= first_added else w.add_mesh)(*m)
    for m in sc.materials:
        w.add_material(m)
    for me, ma, xf in zip(sc.inst_mesh, sc.inst_material, sc.inst_transform):
        w.add_instance(int(me), int(ma), xf, not device or int(me) < first_added)
    for k in range(len(extra)):
        w.add_instance(len(sc.meshes) + k, F_LIGHT_MATERIAL if k == F_EMISSIVE else 0, placed(k), not device)
    w.prepare()
    return w


def grows(counts, upload):
    """per call: whether the primitive buffer grows, by context.cu's rule (need = 48 (have + add) + 64 bytes, grown to need * 1.5,
    the upload's buffer exactly its records)"""
    cap, have, out = 48 * upload, upload, []
    for add in counts:
        need = 48 * (have + add) + 64
        out.append(cap < need)
        if cap < need:
            cap = need + need // 2
        have += add
    return out


def test_appends_in_sequence_behind_queued_frames():
    """a shared scene and two cameras; six calls, each issued while the two frames rendered since the last read-back are still in
    flight on both cameras, and without a host synchronisation; the caller arrays overwritten as soon as each call returns, instance
    updates placing the new meshes (one emissive) and device transform updates between the calls, a re-upload and two more calls,
    each again behind unread frames.  The records equal the host mirror's, and the frames in flight at each call — read back right
    after it — and the last frames equal a run that synchronises the device before each call"""
    import torch
    from tests.test_gpu_parity import ALL_PLANES
    b = Bench("cornell", 48, 32, config="cornell_256")
    first_added = len(b.scene.meshes) // 2
    extra = [f() for f in F_EXTRA]
    sources = list(b.scene.meshes) + extra
    calls = [list(range(first_added, len(b.scene.meshes))) + [len(b.scene.meshes) + k for k in F_CALLS[0]]] + \
            [[len(b.scene.meshes) + k for k in c] for c in F_CALLS[1:]]
    prims = lambda m: (len(m[3]) if m[3] is not None else len(m[0])) // 3
    upload = sum(prims(m) for m in b.scene.meshes[:first_added])
    pattern = grows([sum(prims(sources[i]) for i in c) for c in calls], upload)
    assert pattern[0] and any(not g for g in pattern) and pattern.index(False) < len(pattern) - 1 - pattern[::-1].index(True), \
        ("the calls grow, append in place, then grow again", pattern)
    host = appended_world(b, first_added, extra, device=False).buffers()
    sizes = [(48, 32), (40, 24)]
    moving = 6                                       # cornell's short box: moved by the device transform updates
    runs = []
    for synchronise in (False, True):
        w = appended_world(b, first_added, extra)
        shared = plugin.SharedScene()
        shared.upload(w)
        cams = [plugin.HikariPlugin(cw, ch) for cw, ch in sizes]
        for c in cams:
            c.attach_scene(shared)
        inputs = [Bench("cornell", cw, ch, config="cornell_256") for cw, ch in sizes]
        frames, f = [], 1
        base = np.array(b.scene.inst_transform[moving], np.float32)

        def render():
            nonlocal f
            for c, bi in zip(cams, inputs):
                c.render_frame(bi.moving_inputs(f))
            f += 1

        def read():                      # the newest frame of each camera (waits for it)
            frames.append([{k: c.readback(k).tobytes() for k in ALL_PLANES} for c in cams])

        def add(ids):
            """the call behind the frames in flight, which are read back once it has returned"""
            if synchronise:
                torch.cuda.synchronize()
            src = [tuple(None if a is None else np.array(a) for a in sources[i][:4]) + tuple(sources[i][4:]) for i in ids]
            got = shared.add_mesh_sources(src)
            for s in src:                # the library has copied what it needs
                for a in s[:4]:
                    if a is not None:
                        a[...] = 0x7F if a.dtype == np.uint32 else np.nan
            read()
            return got

        render(); render()
        for n, ids in enumerate(calls):
            got = add(ids)
            want = {i: host["instances"]["mesh"][j] for j, i in enumerate(host_instance_mesh(b, extra)) if i in ids}
            assert_bytes_equal(got, np.array([want[i] for i in ids], L.MESH_INDEX), f"call {n}: mesh index")
            for inst, me in enumerate(host_instance_mesh(b, extra)):
                if me in ids:
                    w.set_instance_visible(inst, True)
            w.prepare_instances()
            shared.update_instances(w)
            render()
            moved = base.copy()
            moved[12:15] += np.float32(0.02 * (n + 1))
            w.set_instance_transform(moving, moved)
            w.previous_transform_system()
            assert shared.update_transforms(w), f"call {n}: the transform update took the host path"
            render()
        read()
        assert_added_world(cams[0], host, "after six calls")
        device_instances = [inst for inst, me in enumerate(host_instance_mesh(b, extra)) if me >= first_added]
        for inst in device_instances:    # the upload takes the host part again: the device meshes are added once more
            w.set_instance_visible(inst, False)
        w.prepare_instances()
        render(); render()
        shared.upload(w)
        render(); render()
        ids = [i for c in calls for i in c]
        for part in (ids[:len(ids) // 2], ids[len(ids) // 2:]):
            add(part)
            render(); render()
        for inst in device_instances:
            w.set_instance_visible(inst, True)
        w.prepare_instances()
        shared.update_instances(w)
        render(); render()
        read()
        assert_added_world(cams[1], host, "after the re-upload")
        for c in cams:
            c.close()
        shared.close()
        runs.append(frames)
    assert len(runs[0]) == len(runs[1]) == len(calls) + 4
    for n, (queued, synced) in enumerate(zip(*runs)):
        for cam in range(2):
            bad = [k for k in ALL_PLANES if queued[cam][k] != synced[cam][k]]
            assert not bad, f"read-back frame {n} camera {cam}: planes that differ {bad}"


def host_instance_mesh(b, extra):
    return [int(m) for m in b.scene.inst_mesh] + [len(b.scene.meshes) + k for k in range(len(extra))]


def assert_added_world(dev, host, what):
    for which, name in READBACK:
        assert_bytes_equal(dev.scene_readback(which), host[name], f"{what}: {name}")


@pytest.mark.parametrize("mode", [0, 1])
def test_device_meshes_under_transform_updates(mode):
    """cornell with its last meshes (the ceiling light's among them) built on the device, animated by hk_scene_update_transforms:
    instance, TLAS, emissive and emissive-BVH records equal the host mirror's after every update, and every plane of every frame
    equals a world uploaded by the host, animated the same way"""
    from tests.conftest import cornell_animation
    from tests.test_gpu_parity import ALL_PLANES
    from tests.test_gpu_scene_update import assert_scene_equals_host
    b = Bench("cornell", 48, 32, config="cornell_256")
    first_added = len(b.scene.meshes) // 2
    assert any(b.scene.materials[int(ma)]["emissive"][:3].any() for me, ma in zip(b.scene.inst_mesh, b.scene.inst_material)
               if int(me) >= first_added), "an instance of a device-built mesh is emissive"
    wa = split_world(b, first_added)
    a_dev, b_dev = plugin.HikariPlugin(b.width, b.height), b.device()
    a_dev.upload_scene(wa)
    a_dev.add_meshes(wa, np.arange(first_added, len(b.scene.meshes)))
    show_device_instances(wa, b, first_added)
    a_dev.update_instances(wa)
    for p in (a_dev, b_dev):
        p.set_tuning(plugin.TUNE_WIDE_TRAVERSAL, mode)
    anim = cornell_animation(b)
    for f in range(1, 6):
        for i, fn in anim.tracks.items():
            xf = anim.compose(fn(f), anim.base[i])
            wa.set_instance_transform(i, xf)
            b.world.set_instance_transform(i, xf)
        for w, p in ((wa, a_dev), (b.world, b_dev)):
            w.previous_transform_system()
            assert p.update_transforms(w), f"frame {f}: the host path ran"
        wa.prepare_instances()
        assert_scene_equals_host(a_dev, wa, f"mode {mode} frame {f}")
        b.world.prepare_instances()
        for name in ("instances", "instance_nodes", "emissives", "emissive_nodes"):
            assert_bytes_equal(wa.buffers()[name], b.world.buffers()[name], f"frame {f}: {name} of the two worlds")
        inp = b.moving_inputs(f)
        a_dev.render_frame(inp); b_dev.render_frame(inp)
        for k in ALL_PLANES:
            assert a_dev.readback(k).tobytes() == b_dev.readback(k).tobytes(), f"mode {mode} frame {f}: plane {k} differs"
    a_dev.close(); b_dev.close()
