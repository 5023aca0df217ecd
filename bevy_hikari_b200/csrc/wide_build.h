// wide_build.h — host side of the image-exact traversal mode (hk_wide.cuh): derives 4-wide trees from the reference's flat skip-link
// BVHs (bvh 0.7.1 flatten_custom as uploaded by the host, src/mesh_material/mod.rs:185-201, instance.rs:352-437) at scene upload.
//
// A flat array is a sequence of "branches": a navigator record (box of the child, entry = next record, exit = the record behind the
// child's subtree) followed by the child — a leaf record (entry = LEAF | shape, exit = next record) or two more branches.  The tree is
// parsed back, collapsed to at most four children per node by opening the child with the largest surface area first, and written
// pre-order.  What the walk needs besides the nodes: the position of every shape's leaf in the flat array (its rank: the reference's
// strict '<' keeps the FIRST of two equidistant hits in that order, light.wgsl:416,470) and the deepest stack the tree can ask for.
// Foreign flat arrays in the same skip-link layout are accepted as long as the derived tree walks exactly like the flat one: any
// arity from 1 up, runs of up to four branches below a navigator and at the top level, navigator boxes larger than what they hold.
// ok = false — the context then keeps the exact-order walk — for an array that is not in this layout (links that do not nest, a leaf
// named twice, a leaf that names no shape), for a node that still has more than four branches after collapsing (a 4-wide node cannot
// hold them; bvh 0.7.1 writes two) and for a navigator box that does not enclose the boxes below it (its children's navigator boxes,
// or the shape's own box at a leaf).  Such a box culls hits it does not enclose, and whether it does depends on the best hit found so
// far, i.e. on the order of the walk; the 4-wide walk also never tests the boxes of the binary levels it collapses.  An empty array
// is ok with root = EMPTY: the context gives such a mesh a node without children (empty_node) to enter.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <limits>
#include <vector>

#include "hk_layout.h"
#include "hk_wide.cuh"

namespace hkw {

struct WideTree {
    bool ok = false;
    std::vector<hkd::hk_wide_node> nodes;
    uint32_t root = hkd::WIDE_EMPTY;       // node 0, LEAF | shape for a single-shape tree, EMPTY for an empty one
    std::vector<uint32_t> rank;            // per shape: position of its leaf record among the leaves of the flat array
    uint32_t stack_need = 0;               // bound on the entries a walk of this tree alone can have on the stack
    std::vector<uint32_t> node_need;       // (internal) per wide node
};

// a node without children: the walk tests nothing in it and pops
inline hkd::hk_wide_node empty_node() {
    hkd::hk_wide_node n;
    const float inf = std::numeric_limits<float>::infinity();
    for (int c = 0; c < 4; ++c) {
        n.lo_x[c] = n.lo_y[c] = n.lo_z[c] = inf; n.hi_x[c] = n.hi_y[c] = n.hi_z[c] = -inf;
        n.child[c] = hkd::WIDE_EMPTY; n.pad[c] = 0u;
    }
    return n;
}

namespace detail {

struct BNode {
    float lo[3], hi[3];
    bool leaf;
    uint32_t shape;
    std::vector<uint32_t> kids;
};

inline bool encloses(const float* lo, const float* hi, const float* inner_lo, const float* inner_hi) {
    for (int k = 0; k < 3; ++k)
        if (!(lo[k] <= inner_lo[k] && inner_hi[k] <= hi[k])) return false;      // false for NaN too
    return true;
}

struct Parser {
    const hk_node* flat;
    uint32_t count;
    std::vector<BNode>& out;
    std::vector<uint32_t>& rank;
    const float* shape_box;        // 6 per shape (min xyz, max xyz), or null when the leaves' boxes are the shapes' by construction
    uint32_t leaves = 0;
    bool ok = true;

    // children of the record range [i, end): ids into `out`
    std::vector<uint32_t> range(uint32_t i, uint32_t end, int depth) {
        std::vector<uint32_t> kids;
        if (depth > 200) { ok = false; return kids; }
        while (ok && i < end) {
            const hk_node& nav = flat[i];
            if (nav.entry_index != i + 1 || nav.exit_index <= i + 1 || nav.exit_index > end) { ok = false; break; }
            BNode b;
            for (int k = 0; k < 3; ++k) { b.lo[k] = nav.min[k]; b.hi[k] = nav.max[k]; }
            const hk_node& first = flat[i + 1];
            if (first.entry_index >= 0x80000000u) {
                const uint32_t shape = first.entry_index - 0x80000000u;
                if (nav.exit_index != i + 2 || first.exit_index != i + 2 || shape >= rank.size() || rank[shape] != 0xFFFFFFFFu) { ok = false; break; }
                b.leaf = true; b.shape = shape;
                rank[shape] = leaves++;
                if (shape_box && !encloses(b.lo, b.hi, shape_box + 6 * (size_t)shape, shape_box + 6 * (size_t)shape + 3)) { ok = false; break; }
            } else {
                b.leaf = false; b.shape = 0;
                b.kids = range(i + 1, nav.exit_index, depth + 1);
                if (b.kids.empty()) ok = false;
                for (uint32_t kid : b.kids) ok = ok && encloses(b.lo, b.hi, out[kid].lo, out[kid].hi);
            }
            out.push_back(std::move(b));
            kids.push_back((uint32_t)out.size() - 1);
            i = nav.exit_index;
        }
        // a run of more than four branches: no child of the run can be opened to make room, so a 4-wide node would drop some
        if (kids.size() > 4) ok = false;
        return kids;
    }
};

inline float half_area(const BNode& b) {
    const float sx = std::max(b.hi[0] - b.lo[0], 0.0f), sy = std::max(b.hi[1] - b.lo[1], 0.0f), sz = std::max(b.hi[2] - b.lo[2], 0.0f);
    return sx * sy + sx * sz + sy * sz;
}

// writes the wide node whose children are `kids` (after collapsing) and returns its index
inline uint32_t emit(const std::vector<BNode>& b, std::vector<uint32_t> kids, WideTree& t) {
    while (kids.size() < 4) {
        int open = -1;
        float best = -1.0f;
        for (size_t j = 0; j < kids.size(); ++j) {
            const BNode& k = b[kids[j]];
            if (k.leaf || kids.size() - 1 + k.kids.size() > 4) continue;
            const float a = half_area(k);
            if (a > best) { best = a; open = (int)j; }
        }
        if (open < 0) break;
        const std::vector<uint32_t> sub = b[kids[open]].kids;
        kids.erase(kids.begin() + open);
        kids.insert(kids.begin() + open, sub.begin(), sub.end());
    }
    const uint32_t index = (uint32_t)t.nodes.size();
    t.nodes.emplace_back();
    t.node_need.push_back(0);
    hkd::hk_wide_node n = empty_node();
    uint32_t need = 0;
    const uint32_t k = (uint32_t)std::min<size_t>(kids.size(), 4);
    for (uint32_t c = 0; c < k; ++c) {
        const BNode& kid = b[kids[c]];
        n.lo_x[c] = kid.lo[0]; n.lo_y[c] = kid.lo[1]; n.lo_z[c] = kid.lo[2];
        n.hi_x[c] = kid.hi[0]; n.hi_y[c] = kid.hi[1]; n.hi_z[c] = kid.hi[2];
        uint32_t sub_need = 0;
        if (kid.leaf) {
            n.child[c] = hkd::WIDE_LEAF | kid.shape;
        } else {
            const uint32_t ci = emit(b, kid.kids, t);
            n.child[c] = ci;
            sub_need = t.node_need[ci];
        }
        need = std::max(need, (k - 1) + sub_need);
    }
    t.nodes[index] = n;
    t.node_need[index] = need;
    return index;
}

}  // namespace detail

// `shape_count`: number of shapes the leaves may name (triangles of the mesh / instances of the scene); `shape_box`: their boxes, 6
// floats each (min xyz, max xyz), which every leaf's navigator box must enclose — null where the caller wrote those boxes itself
inline WideTree build_wide(const hk_node* flat, uint32_t count, uint32_t shape_count, const float* shape_box) {
    WideTree t;
    t.rank.assign(shape_count, 0xFFFFFFFFu);
    if (count == 0) { t.ok = true; return t; }
    if (count == 1) {                       // a single-shape BVH is one leaf record without a navigator
        if (flat[0].entry_index < 0x80000000u || flat[0].entry_index - 0x80000000u >= shape_count) return t;
        t.root = hkd::WIDE_LEAF | (flat[0].entry_index - 0x80000000u);
        t.rank[flat[0].entry_index - 0x80000000u] = 0;
        t.ok = true;
        return t;
    }
    std::vector<detail::BNode> b;
    b.reserve(count);
    detail::Parser p{flat, count, b, t.rank, shape_box};
    std::vector<uint32_t> top = p.range(0, count, 0);
    if (!p.ok || top.empty()) return t;
    t.root = detail::emit(b, top, t);
    t.stack_need = t.node_need[t.root];
    t.ok = true;
    return t;
}

}  // namespace hkw
