// hk_wide.cuh — the image-exact traversal mode (hk_set_tuning(HK_TUNE_WIDE_TRAVERSAL)): 4-wide BVH nodes, an ordered walk with a
// short stack, the reference's arithmetic on every box and triangle.
//
// The reference walks flat skip-link arrays in a fixed order (light.wgsl:400-486): one dependent record fetch per box test, no
// front-to-back order, 43 (city) / 108 (scene.rs) dependent steps per bounce ray.  Its RESULT is "the nearest triangle, the first
// in array order among equidistant ones" for closest-hit rays and "is there a triangle nearer than max_distance" for shadow rays —
// neither depends on the order of the walk, only the any-hit occluder a shadow ray happens to report does, and that position is
// stored with a zero-radiance sample that no image reads (tests/test_bvh_topology_invariance.py).  So this mode keeps
//   * the reference's box test (hkd::slab) and triangle test (hkd::triangle) on the same object-space ray, hence the same distance,
//     u and v for every (ray, triangle) pair, and
//   * first-in-array-order among equidistant hits, through the leaf ranks wide_build.h records,
// and changes the structure that is walked: each node holds the boxes of up to four children (the reference's own boxes, two binary
// levels collapsed: 128 bytes = one L2 line, eight 16-byte loads issued together), the nearest child that passes is entered, the
// others are pushed with their entry distance and dropped on pop when a nearer hit has been found since.  Dependent steps per bounce
// ray: city 43 -> 12, scene.rs 108 -> 35 (tools/exp_wide_traversal.py).  What can differ from the exact-order walk: a hit whose
// distance ties with another within the rounding of a box test (the culling decision `t_min < hit.distance` sees a different
// hit.distance), i.e. rays through an edge shared by two surfaces — measured in tests/test_wide_traversal.py.
#pragma once
#include "hk_device.cuh"

#ifndef HK_WIDE_STACK
#define HK_WIDE_STACK 64       // entries of 8 bytes in local memory; a scene whose trees could need more keeps the exact-order walk
#endif

namespace hkd {

constexpr uint32_t WIDE_EMPTY = 0xFFFFFFFFu;      // no child / walk finished
constexpr uint32_t WIDE_SENTINEL = 0xFFFFFFFEu;   // stack marker: the entries above it belong to the BLAS entered last
constexpr uint32_t WIDE_LEAF = 0x80000000u;       // child reference = WIDE_LEAF | shape (instance in the TLAS, triangle of the mesh in a BLAS)

struct hk_wide_node {          // 128 bytes, 128-byte aligned
    float lo_x[4], lo_y[4], lo_z[4], hi_x[4], hi_y[4], hi_z[4];
    uint32_t child[4];         // node index relative to the tree's first node | WIDE_LEAF + shape | WIDE_EMPTY
    uint32_t pad[4];
};
static_assert(sizeof(hk_wide_node) == 128, "one L2 line per node");

// Does the new hit (distance equal to the best so far) come before the best hit in the reference's array order?
__device__ __forceinline__ bool wide_tie_first(const DeviceScene& sc, uint32_t new_instance, uint32_t new_primitive, const Hit& hit) {
    const uint32_t a = __ldg(&sc.wide_instance_rank[new_instance]), b = __ldg(&sc.wide_instance_rank[hit.instance_index]);
    if (a != b) return a < b;
    return __ldg(&sc.wide_primitive_rank[new_primitive]) < __ldg(&sc.wide_primitive_rank[hit.primitive_index]);
}

// BOTTOM = false: traverse_top (light.wgsl:442-486) — `ray` is the world-space ray.
// BOTTOM = true:  traverse_bottom of instance `instance` alone (light.wgsl:400-440) — `ray` is already in its object space;
//                 hit.instance_index is left to the caller like the reference does.
template <bool BOTTOM>
static __device__ __forceinline__ Hit wide_walk(const DeviceScene& sc, const Ray& ray, float max_distance, float early_distance,
                                            uint32_t exclude_instance, uint32_t instance) {
    Hit hit;
    hit.u = 0.0f; hit.v = 0.0f; hit.distance = max_distance;
    hit.instance_index = U32_MAX; hit.primitive_index = U32_MAX;
    uint2 stack[HK_WIDE_STACK];        // x = reference, y = bits of the entry distance: one 8-byte local store / load per entry
    int sp = 0;
    Ray cur = ray;
    bool in_blas = BOTTOM;
    uint32_t instance_index = instance, mesh_primitive = 0;
    const hk_wide_node* nodes = sc.wide_tlas;
    uint32_t ref = sc.wide_tlas_root;
    if (BOTTOM) {
        const uint2 w = __ldg(&sc.wide_instance[instance]);            // first node of the mesh's tree | its root reference
        nodes = sc.wide_blas + w.x; ref = w.y;
        mesh_primitive = __ldg(&sc.instances[instance].mesh.primitive);
    }
    for (;;) {
        // phase 1 — interior nodes: four box tests per step, the nearest passing child is entered, the others are pushed
        while (ref < WIDE_LEAF) {
            const float4* n = reinterpret_cast<const float4*>(nodes + ref);
            const float4 lx = ldg4(n), ly = ldg4(n + 1), lz = ldg4(n + 2), hx = ldg4(n + 3), hy = ldg4(n + 4), hz = ldg4(n + 5);
            const uint4 ch = ldg4u(n + 6);
            float t0 = slab(cur, v3(lx.x, ly.x, lz.x), v3(hx.x, hy.x, hz.x));
            float t1 = slab(cur, v3(lx.y, ly.y, lz.y), v3(hx.y, hy.y, hz.y));
            float t2 = slab(cur, v3(lx.z, ly.z, lz.z), v3(hx.z, hy.z, hz.z));
            float t3 = slab(cur, v3(lx.w, ly.w, lz.w), v3(hx.w, hy.w, hz.w));
            // the reference's culling rule, slab(...) < hit.distance (light.wgsl:421,466); F32_MAX marks "not entered"
            t0 = (ch.x != WIDE_EMPTY && t0 < hit.distance) ? t0 : F32_MAX;
            t1 = (ch.y != WIDE_EMPTY && t1 < hit.distance) ? t1 : F32_MAX;
            t2 = (ch.z != WIDE_EMPTY && t2 < hit.distance) ? t2 : F32_MAX;
            t3 = (ch.w != WIDE_EMPTY && t3 < hit.distance) ? t3 : F32_MAX;
            uint32_t r0 = ch.x, r1 = ch.y, r2 = ch.z, r3 = ch.w;
            // nearest into slot 0 (three compare-exchanges); the rest keep their places
            if (t1 < t0) { float t = t0; t0 = t1; t1 = t; uint32_t r = r0; r0 = r1; r1 = r; }
            if (t2 < t0) { float t = t0; t0 = t2; t2 = t; uint32_t r = r0; r0 = r2; r2 = r; }
            if (t3 < t0) { float t = t0; t0 = t3; t3 = t; uint32_t r = r0; r0 = r3; r3 = r; }
            if (t1 < F32_MAX) { stack[sp] = make_uint2(r1, __float_as_uint(t1)); ++sp; }
            if (t2 < F32_MAX) { stack[sp] = make_uint2(r2, __float_as_uint(t2)); ++sp; }
            if (t3 < F32_MAX) { stack[sp] = make_uint2(r3, __float_as_uint(t3)); ++sp; }
            if (t0 < F32_MAX) { ref = r0; continue; }
            // nothing entered: next entry of the stack that is still nearer than the best hit
            ref = WIDE_EMPTY;
            while (sp > 0) {
                --sp;
                const uint2 e = stack[sp];
                if (e.x == WIDE_SENTINEL || __uint_as_float(e.y) < hit.distance) { ref = e.x; break; }
            }
        }
        if (ref == WIDE_EMPTY) break;
        // phase 2 — a leaf reference (or the marker that ends a BLAS)
        bool pop = true;
        if (!BOTTOM && ref == WIDE_SENTINEL) {
            in_blas = false;
            nodes = sc.wide_tlas;
            cur = ray;
        } else if (!BOTTOM && !in_blas) {
            const uint32_t candidate = ref & 0x7FFFFFFFu;
            if (candidate != exclude_instance) {
                const hk_instance* inst = sc.instances + candidate;
                instance_ray(inst, ray, cur);                              // light.wgsl:306-316
                const uint2 w = __ldg(&sc.wide_instance[candidate]);
                mesh_primitive = __ldg(&inst->mesh.primitive);
                instance_index = candidate;
                in_blas = true;
                stack[sp] = make_uint2(WIDE_SENTINEL, 0u); ++sp;
                nodes = sc.wide_blas + w.x;
                ref = w.y;
                pop = false;
            }
        } else {
            const uint32_t primitive_index = mesh_primitive + (ref & 0x7FFFFFFFu);
            const hk_primitive* prim = sc.primitives + primitive_index;
            const float4 a = ldg4(&prim->vertices[0]), b = ldg4(&prim->vertices[1]), c = ldg4(&prim->vertices[2]);
            float u, v;
            const float distance = triangle(cur, f4xyz(a), f4xyz(b), f4xyz(c), u, v);
            bool closer = distance < hit.distance;
            if (!closer && distance == hit.distance && hit.primitive_index != U32_MAX)      // equidistant: the reference keeps the first
                closer = BOTTOM ? __ldg(&sc.wide_primitive_rank[primitive_index]) < __ldg(&sc.wide_primitive_rank[hit.primitive_index])
                                : wide_tie_first(sc, instance_index, primitive_index, hit);
            if (closer) {
                hit.u = u; hit.v = v; hit.distance = distance;
                hit.primitive_index = primitive_index;
                if (!BOTTOM) hit.instance_index = instance_index;
                if (distance < early_distance) break;                       // traverse_bottom returns, traverse_top returns
            }
        }
        if (pop) {
            ref = WIDE_EMPTY;
            while (sp > 0) {
                --sp;
                const uint2 e = stack[sp];
                if (e.x == WIDE_SENTINEL || __uint_as_float(e.y) < hit.distance) { ref = e.x; break; }
            }
        }
    }
    return hit;
}

}  // namespace hkd
