"""Foreign flat BVHs: skip-link arrays in the layout the reference's walk reads (light.wgsl:400-486), but over trees that bvh 0.7.1
never writes.  A tree is nested lists over shape ids (triangles of a mesh, or instances of the scene): an int is a leaf, a list is a
node whose entries are its children.  `flatten` writes it the way the walk reads it — per child a navigator record (box, entry = the
next record, exit = the record behind the child's subtree) followed by a leaf record or by the child's own branches — and
`set_blas` / `set_tlas` swap the records into a World's buffers (plugin.World.buffers), ready for plugin.scene_desc_from_buffers.

Used by tests/test_foreign_bvh_oracle.py (the trees against a brute-force closest-hit query) and tests/test_gpu_wide_foreign_bvh.py
(the 4-wide walk against the oracle's flat walk over the same arrays)."""
import numpy as np

from bevy_hikari_b200 import layout as L

LEAF = 0x80000000
F = np.float32


def instance_boxes(bufs):
    """world-space boxes of the instances: the shapes of the TLAS"""
    inst = bufs["instances"]
    return inst["min"].astype(F), inst["max"].astype(F)


def mesh_of(bufs, instance):
    """(node_offset, node_count, primitive) of an instance's mesh"""
    m = bufs["instances"]["mesh"][instance]
    return int(m["node_offset"]), int(m["node_count"]), int(m["primitive"])


def triangle_count(bufs, instance):
    off, cnt, _ = mesh_of(bufs, instance)
    e = bufs["asset_nodes"]["entry_index"][off:off + cnt]
    e = e[e >= LEAF]
    return int(e.max() - LEAF + 1) if len(e) else 0


def triangle_boxes(bufs, instance):
    """object-space boxes of the triangles of an instance's mesh: the shapes of its BLAS"""
    _, _, prim = mesh_of(bufs, instance)
    p = bufs["primitives"]["vertices"]["position"][prim:prim + triangle_count(bufs, instance)]
    return p.min(axis=1).astype(F), p.max(axis=1).astype(F)


def _arity(arity, depth):
    if isinstance(arity, int):
        return arity
    return arity[min(depth, len(arity) - 1)]


def _split(shapes, k, split, lo, hi, rng):
    k = min(k, len(shapes))
    if split == "chain":                 # k - 1 single leaves, then the rest: one leaf per level when k = 2
        return [shapes[i:i + 1] for i in range(k - 1)] + [shapes[k - 1:]]
    if split == "order":                 # the order of `shapes`, into k groups of (nearly) equal size
        return [list(part) for part in np.array_split(np.asarray(shapes), k)]
    if split == "random":
        order = rng.permutation(len(shapes))
        cuts = np.sort(rng.choice(np.arange(1, len(shapes)), k - 1, replace=False))
        return [[shapes[i] for i in part] for part in np.split(order, cuts)]
    # median: along the longest extent of the box centres, into k groups of (nearly) equal size
    c = (lo[shapes].astype(np.float64) + hi[shapes]) * 0.5
    axis = int(np.argmax(c.max(axis=0) - c.min(axis=0)))
    order = np.argsort(c[:, axis], kind="stable")
    return [[shapes[i] for i in part] for part in np.array_split(order, k)]


def tree(lo, hi, arity=2, top=None, split="median", shapes=None, seed=0):
    """the top-level branches (a list) of a tree over `shapes` (default: all of them, in order).  `arity`: children per node, 1-8 (an
    int, or one per depth, the last repeating; a node of arity 1 wraps its shapes in one more node); `top`: branches at the top level
    (default `arity`); `split`: "median", "random", "order" (groups in the order of `shapes`) or "chain" (each level holds arity - 1
    leaves, in the order of `shapes`, plus the rest)."""
    rng = np.random.default_rng(seed)
    shapes = list(range(len(lo))) if shapes is None else list(shapes)

    def node(group, depth):
        if len(group) == 1:
            return int(group[0])
        k = _arity(arity, depth)
        if k == 1:
            return [node(group, depth + 1)]
        return [node(g, depth + 1) for g in _split(group, k, split, lo, hi, rng)]

    if len(shapes) == 1:
        return [int(shapes[0])]
    return [node(g, 1) for g in _split(shapes, top or _arity(arity, 0), split, lo, hi, rng)]


def flatten(branches, lo, hi, boxes="exact", delta=0.05):
    """skip-link records (L.NODE) of the top-level `branches` over shapes with boxes lo / hi.  `boxes`: "exact" (a navigator's box is
    the union of its shapes' boxes, as bvh 0.7.1 writes it), "inflated" (grown by `delta` on every side: still encloses its shapes)
    or "tight" (shrunk by a quarter of its extent on every side: no longer encloses them; "tight_leaves" / "tight_inner" shrink only
    the navigators of leaves / of inner nodes).  A single shape is one leaf record
    without a navigator, as bvh 0.7.1 writes it; no shape is no record."""
    if len(branches) == 1 and isinstance(branches[0], int):
        out = np.zeros(1, L.NODE)
        out[0] = ((np.inf,) * 3, LEAF + branches[0], (-np.inf,) * 3, 1)
        return out
    recs = []

    def branch(n):
        i = len(recs)
        recs.append(None)
        if isinstance(n, int):
            b_lo, b_hi = lo[n], hi[n]
            recs.append(((np.inf,) * 3, LEAF + n, (-np.inf,) * 3, i + 2))
        else:
            parts = [branch(c) for c in n]
            b_lo = np.min([p[0] for p in parts], axis=0).astype(F)
            b_hi = np.max([p[1] for p in parts], axis=0).astype(F)
        n_lo, n_hi = b_lo, b_hi
        if boxes == "inflated":
            n_lo, n_hi = b_lo - F(delta), b_hi + F(delta)
        elif boxes == "tight" or boxes == ("tight_leaves" if isinstance(n, int) else "tight_inner"):
            q = (b_hi - b_lo) * F(0.25)
            n_lo, n_hi = b_lo + q, b_hi - q
        recs[i] = (tuple(n_lo), i + 1, tuple(n_hi), len(recs))
        return b_lo, b_hi

    for b in branches:
        branch(b)
    return np.array(recs, L.NODE)


def set_blas(bufs, instance, records):
    """give the mesh of `instance` (and every instance that shares it) the flat BVH `records`, appended to the asset nodes"""
    key = mesh_of(bufs, instance)
    off = len(bufs["asset_nodes"])
    bufs["asset_nodes"] = np.concatenate([bufs["asset_nodes"], np.asarray(records, L.NODE)])
    for i in range(len(bufs["instances"])):
        if mesh_of(bufs, i) == key:
            bufs["instances"]["mesh"]["node_offset"][i] = off
            bufs["instances"]["mesh"]["node_count"][i] = len(records)


def set_tlas(bufs, records):
    bufs["instance_nodes"] = np.asarray(records, L.NODE).copy()


def foreign_blas(bufs, instance, **kw):
    """set_blas with a generated tree (keywords: those of `tree`, plus `boxes` / `delta` of `flatten`)"""
    fl = {k: kw.pop(k) for k in ("boxes", "delta") if k in kw}
    lo, hi = triangle_boxes(bufs, instance)
    set_blas(bufs, instance, flatten(tree(lo, hi, **kw), lo, hi, **fl))


def foreign_tlas(bufs, **kw):
    fl = {k: kw.pop(k) for k in ("boxes", "delta") if k in kw}
    lo, hi = instance_boxes(bufs)
    set_tlas(bufs, flatten(tree(lo, hi, **kw), lo, hi, **fl))
