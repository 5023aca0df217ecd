// kernels_scene.cu — SURVEY 8(f) rank 2: the per-frame half of the scene rebuilt ON THE DEVICE.
//
// The reference rebuilds, on the CPU and whenever anything moves (src/mesh_material/instance.rs:352-437): every instance's world
// AABB, model and inverse-transpose matrix (:286-323), the TLAS over the instances (bvh 0.7.1 BVH::build + flatten_custom, :365-371),
// every emissive's bounding sphere and surface area (:399-418) and the BVH over the emissives (:420-427) — and then re-uploads all
// of it (:430-437); its README lists "asynchronous building of acceleration structures" as to do.  hk_scene_update_instances takes
// those arrays from a host that has done this work (host/hikari.cpp); the kernels below do the work themselves from what actually
// changed — one model matrix per instance — and leave the results where the light kernels read them, stream-ordered, without a host
// round trip:
//   k_scene_instances    per instance: world AABB, inverse transpose, previous model + "moved" flag, compact traversal record
//   kc_build_flat_bvh    one CTA: bvh 0.7.1's bucketed SAH build + flatten_custom, one WARP per tree node, level by level
//   kc_scene_emissives   one warp per emissive: bounding sphere, surface area (areas in parallel, summed in the reference's order)
// The result is the reference's, bit for bit (tests/test_gpu_scene_update.py compares every record with the host mirror's):
//   * the arithmetic is host/hikari.cpp's, statement for statement, compiled without FMA contraction;
//   * a node's split (axis, buckets, SAH costs) depends on min / max / counts over the node's shapes, which no order of evaluation
//     changes (boxes never hold -0: every bound is a sum whose exact-zero result rounds to +0), and the one thing that is
//     order-sensitive — the order of the shapes inside a child, bucket by bucket, stable — is reproduced by a ballot-ranked
//     counting sort;
//   * a node's place in the flat array follows from how many tree nodes and leaves precede it in pre-order: a subtree of m shapes
//     has 2m - 1 tree nodes and writes 3m - 1 records, so both children's places are known when the parent splits.
// When a camera walks the 4-wide trees (HK_TUNE_WIDE_TRAVERSAL), one more kernel follows the TLAS build:
//   kc_build_wide_tlas   one CTA: the image-exact traversal mode's 4-wide TLAS (hk_wide.cuh) from the flat TLAS just built, byte for
//                        byte what wide_build.h derives on the host at upload, and the verdict "fits the walk's stack"
//                        (tests/test_gpu_wide_tlas_device.py holds it to the host derivation)
// What this path does NOT rebuild: alias tables (their cache rule — rebuild when the scale moved by more than 0.01,
// instance.rs:385-397 — is the caller's to check: hikari::MeshMaterialWorld::prepare_instance_transforms) and anything that changes
// the SET of instances or materials; those go through hk_scene_update_instances / hk_scene_upload.
// Meshes added to the scene (hk_scene_add_meshes) are built here too — GpuMesh::try_from of mod.rs:379-467, see "mesh assets" below:
//   k_mesh_records       one thread per vertex and per primitive: the records, each primitive's box and centre
//   kc_build_blas_top    one CTA per mesh: the top levels of its BLAS, the whole CTA on one node
//   kc_build_blas_bottom the subtrees below, taken from a work list, one warp per node
// with the same split routine (sah_split) as kc_build_flat_bvh.  Changing or removing an existing mesh is not done.
#include "hk_device.cuh"
#include "hk_wide.cuh"
#include "hk_kernels.h"

namespace hkd {

namespace {

constexpr float SCENE_BVH_EPSILON = 0.00001f;   // bvh 0.7.1 EPSILON
constexpr int SCENE_BUCKETS = 6;                // bvh 0.7.1 NUM_BUCKETS
constexpr uint32_t SCENE_LEAF = 0x80000000u;

// std::min / std::max as the host mirror uses them (first argument wins ties)
__device__ __forceinline__ float smin(float a, float b) { return b < a ? b : a; }
__device__ __forceinline__ float smax(float a, float b) { return a < b ? b : a; }

struct SBox {
    float mn[3], mx[3];
    __device__ __forceinline__ void clear() {
        mn[0] = mn[1] = mn[2] = __uint_as_float(0x7f800000u);
        mx[0] = mx[1] = mx[2] = __uint_as_float(0xff800000u);
    }
    __device__ __forceinline__ void join(const SBox& o) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { mn[k] = smin(mn[k], o.mn[k]); mx[k] = smax(mx[k], o.mx[k]); }
    }
    __device__ __forceinline__ float surface_area() const {
        const float sx = mx[0] - mn[0], sy = mx[1] - mn[1], sz = mx[2] - mn[2];
        return 2.0f * (sx * sy + sx * sz + sy * sz);
    }
};

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = smin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = smax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ uint32_t warp_sum(uint32_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ void store_node(hk_node* out, uint32_t at, const SBox& b, uint32_t entry, uint32_t exit) {
    float4* p = reinterpret_cast<float4*>(out + at);
    p[0] = make_float4(b.mn[0], b.mn[1], b.mn[2], __uint_as_float(entry));
    p[1] = make_float4(b.mx[0], b.mx[1], b.mx[2], __uint_as_float(exit));
}

// glam Mat4::transform_point3 / transform_vector3 as restated in host/hikari.cpp (column-major, no perspective divide)
__device__ __forceinline__ void xf_point3(const float* m, const float* p, float* out) {
    float r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = m[k] * p[0];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = m[4 + k] * p[1] + r[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = m[8 + k] * p[2] + r[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] = m[12 + k] + r[k];
}
__device__ __forceinline__ void xf_vector3(const float* m, const float* p, float* out) {
    float r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = m[k] * p[0];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = m[4 + k] * p[1] + r[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] = m[8 + k] * p[2] + r[k];
}
__device__ __forceinline__ float len3(const float* a) { return sqrtf((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]); }

// glam Mat4::inverse, scalar path (host/hikari.cpp mat4_inverse)
__device__ void mat4_inverse_dev(const float* m, float* out) {
    const float m00 = m[0], m01 = m[1], m02 = m[2], m03 = m[3];
    const float m10 = m[4], m11 = m[5], m12 = m[6], m13 = m[7];
    const float m20 = m[8], m21 = m[9], m22 = m[10], m23 = m[11];
    const float m30 = m[12], m31 = m[13], m32 = m[14], m33 = m[15];
    const float coef00 = m22 * m33 - m32 * m23, coef02 = m12 * m33 - m32 * m13, coef03 = m12 * m23 - m22 * m13;
    const float coef04 = m21 * m33 - m31 * m23, coef06 = m11 * m33 - m31 * m13, coef07 = m11 * m23 - m21 * m13;
    const float coef08 = m21 * m32 - m31 * m22, coef10 = m11 * m32 - m31 * m12, coef11 = m11 * m22 - m21 * m12;
    const float coef12 = m20 * m33 - m30 * m23, coef14 = m10 * m33 - m30 * m13, coef15 = m10 * m23 - m20 * m13;
    const float coef16 = m20 * m32 - m30 * m22, coef18 = m10 * m32 - m30 * m12, coef19 = m10 * m22 - m20 * m12;
    const float coef20 = m20 * m31 - m30 * m21, coef22 = m10 * m31 - m30 * m11, coef23 = m10 * m21 - m20 * m11;
    const float fac0[4] = {coef00, coef00, coef02, coef03}, fac1[4] = {coef04, coef04, coef06, coef07};
    const float fac2[4] = {coef08, coef08, coef10, coef11}, fac3[4] = {coef12, coef12, coef14, coef15};
    const float fac4[4] = {coef16, coef16, coef18, coef19}, fac5[4] = {coef20, coef20, coef22, coef23};
    const float vec0[4] = {m10, m00, m00, m00}, vec1[4] = {m11, m01, m01, m01};
    const float vec2[4] = {m12, m02, m02, m02}, vec3_[4] = {m13, m03, m03, m03};
    const float sign_a[4] = {1.0f, -1.0f, 1.0f, -1.0f}, sign_b[4] = {-1.0f, 1.0f, -1.0f, 1.0f};
    float inv[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float inv0 = vec1[k] * fac0[k] - vec2[k] * fac1[k] + vec3_[k] * fac2[k];
        const float inv1 = vec0[k] * fac0[k] - vec2[k] * fac3[k] + vec3_[k] * fac4[k];
        const float inv2 = vec0[k] * fac1[k] - vec1[k] * fac3[k] + vec3_[k] * fac5[k];
        const float inv3 = vec0[k] * fac2[k] - vec1[k] * fac4[k] + vec2[k] * fac5[k];
        inv[0][k] = inv0 * sign_a[k]; inv[1][k] = inv1 * sign_b[k]; inv[2][k] = inv2 * sign_a[k]; inv[3][k] = inv3 * sign_b[k];
    }
    const float d0 = m00 * inv[0][0], d1 = m01 * inv[1][0], d2 = m02 * inv[2][0], d3 = m03 * inv[3][0];
    const float dot1 = ((d0 + d1) + d2) + d3;
    const float rcp_det = 1.0f / dot1;
    // A singular model (an axis scaled to zero) gives rcp_det = ±inf and 0 * inf = NaN in every zero cofactor.  The device writes
    // every NaN as 0x7FFFFFFF; x86 writes its default NaN 0xFFC00000, and with finite inputs every NaN of this expansion is that one
    // (generated, then only propagated).  The reference uploads the x86 bytes, and so does the host path: write those.
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float v = inv[c][k] * rcp_det;
            out[4 * c + k] = v != v ? __uint_as_float(0xFFC00000u) : v;
        }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ instances
// instance.rs:286-323 for instance i: the mesh's Aabb (centre, half extents) carried through the new GlobalTransform.
// `previous` = PreviousMeshUniform::transform (instance.rs:111-128); nullptr = the model the record held until now.
__global__ void __launch_bounds__(128) k_scene_instances(uint32_t n, const float4* __restrict__ models, const float4* __restrict__ previous,
                                                         const float* __restrict__ mesh_aabbs, hk_instance* instances, hk_instance_trav* trav,
                                                         float4* previous_out, uint32_t* moved_out, float4* box_lo, float4* box_hi) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float m[16], p[16];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float4 v = models[4u * i + c];
        m[4 * c] = v.x; m[4 * c + 1] = v.y; m[4 * c + 2] = v.z; m[4 * c + 3] = v.w;
    }
    const float4* old = previous ? previous + 4u * i : reinterpret_cast<const float4*>(instances[i].model);
    uint32_t moved = 0u;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float4 v = old[c];
        p[4 * c] = v.x; p[4 * c + 1] = v.y; p[4 * c + 2] = v.z; p[4 * c + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) moved |= (__float_as_uint(p[k]) != __float_as_uint(m[k])) ? 1u : 0u;   // memcmp, as the host path
    const float center[3] = {mesh_aabbs[6u * i], mesh_aabbs[6u * i + 1], mesh_aabbs[6u * i + 2]};
    const float half[3] = {mesh_aabbs[6u * i + 3], mesh_aabbs[6u * i + 4], mesh_aabbs[6u * i + 5]};
    float c[3];
    xf_point3(m, center, c);
    float lo[3] = {0.0f, 0.0f, 0.0f}, hi[3] = {0.0f, 0.0f, 0.0f};       // instance.rs:298-303 starts from ZERO
#pragma unroll
    for (int index = 0; index < 8; ++index) {
        const float vtx[3] = {half[0] * (float)(2 * (index & 1) - 1), half[1] * (float)(2 * ((index >> 1) & 1) - 1),
                              half[2] * (float)(2 * ((index >> 2) & 1) - 1)};
        float t[3];
        xf_vector3(m, vtx, t);
#pragma unroll
        for (int k = 0; k < 3; ++k) { lo[k] = smin(lo[k], t[k]); hi[k] = smax(hi[k], t[k]); }
    }
    float inv[16];
    mat4_inverse_dev(m, inv);
    hk_instance* rec = instances + i;
    float4* r4 = reinterpret_cast<float4*>(rec);
    const uint32_t material = rec->material, node_index = rec->node_index;
    const float mn[3] = {lo[0] + c[0], lo[1] + c[1], lo[2] + c[2]}, mx[3] = {hi[0] + c[0], hi[1] + c[1], hi[2] + c[2]};
    r4[0] = make_float4(mn[0], mn[1], mn[2], __uint_as_float(material));
    r4[1] = make_float4(mx[0], mx[1], mx[2], __uint_as_float(node_index));
    float4* t4 = reinterpret_cast<float4*>(trav + i);
#pragma unroll
    for (int col = 0; col < 4; ++col) {
        r4[2 + col] = make_float4(m[4 * col], m[4 * col + 1], m[4 * col + 2], m[4 * col + 3]);
        // inverse().transpose(): element (row, col) of the transpose = element (col, row) of the inverse
        const float4 it = make_float4(inv[col], inv[4 + col], inv[8 + col], inv[12 + col]);
        r4[6 + col] = it;
        t4[col] = it;
        previous_out[4u * i + col] = make_float4(p[4 * col], p[4 * col + 1], p[4 * col + 2], p[4 * col + 3]);
    }
    moved_out[i] = moved;
    box_lo[i] = make_float4(mn[0], mn[1], mn[2], 0.0f);
    box_hi[i] = make_float4(mx[0], mx[1], mx[2], 0.0f);
}

// ------------------------------------------------------------------------------------------------ SAH build + flatten
// One tree node being split.  `t` = its index among the tree nodes in pre-order (what bvh calls the node index and writes back
// through set_bh_node_index), `leaves_before` = shapes that precede it in pre-order; its navigator record sits at
// t - 1 + leaves_before (the root has none).  Each node writes its own navigator: the box bvh gives a child (l_box / r_box of
// BVH::build) is the join of the child's shapes in the order the child holds them, which is the child's own bound, except when no
// SAH candidate had a cost below infinity (NaN or infinite costs): then the parent leaves both children the empty box.
constexpr uint32_t SEG_EMPTY_BOX = 1u;     // BuildSeg::flags: the navigator gets the empty box
constexpr uint32_t SEG_IDX_B = 2u;         // the segment's shape list is in idx_b (else idx_a)
struct BuildSeg {
    uint32_t begin, count, t, leaves_before, flags, mesh;     // mesh: the BLAS job of a kc_build_blas_* segment (0 for the TLAS)
};
static_assert(sizeof(BuildSeg) == 24, "scratch sizing below");

// What one split needs: the shapes' boxes and centres (indexed by shape), the two shape lists, and where the records go.
struct BuildIn {
    const float4 *box_lo, *box_hi, *center;
    uint32_t* idx[2];
    hk_node* out;                 // the flat array of this tree
    uint32_t shape_base;          // leaf records name shape - shape_base
    uint8_t* index_base;          // per shape: its node index t is written at index_base + shape * index_stride (nullptr: none)
    uint32_t index_stride;
};

// bvh 0.7.1's bucket of a centre: Rust's saturating `f32 as usize`, clamped to the last bucket as host/hikari.cpp clamps it
__device__ __forceinline__ uint32_t sah_bucket(float rel) {
    const float x = rel * ((float)SCENE_BUCKETS - 0.01f);
    if (!(x > 0.0f)) return 0u;
    if (x >= (float)SCENE_BUCKETS) return (uint32_t)SCENE_BUCKETS - 1u;
    const uint32_t b = (uint32_t)x;
    return b < (uint32_t)SCENE_BUCKETS ? b : (uint32_t)SCENE_BUCKETS - 1u;
}
__device__ __forceinline__ float4 box_center(const float4 lo, const float4 hi) {      // AABB::center
    return make_float4(lo.x + (hi.x - lo.x) / 2.0f, lo.y + (hi.y - lo.y) / 2.0f, lo.z + (hi.z - lo.z) / 2.0f, 0.0f);
}

// The join of boxes in a given order, bit for bit.  min / max over the values do not depend on the order (a NaN never wins against
// the running bound, which starts at +-inf and so is never NaN); the one thing that does is which zero a bound of 0 keeps, -0 or +0:
// the first zero in the order.  So each bound also carries (position << 1 | sign) of the first zero it met.
struct OrderedBox {
    SBox b;
    uint32_t z[6];
    __device__ __forceinline__ void clear() {
        b.clear();
#pragma unroll
        for (int k = 0; k < 6; ++k) z[k] = 0xFFFFFFFFu;
    }
    __device__ __forceinline__ void add(uint32_t pos, const float4 lo, const float4 hi) {
        const float l[3] = {lo.x, lo.y, lo.z}, h[3] = {hi.x, hi.y, hi.z};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            b.mn[k] = smin(b.mn[k], l[k]); b.mx[k] = smax(b.mx[k], h[k]);
            if (l[k] == 0.0f && z[k] == 0xFFFFFFFFu) z[k] = pos << 1 | (__float_as_uint(l[k]) >> 31);
            if (h[k] == 0.0f && z[3 + k] == 0xFFFFFFFFu) z[3 + k] = pos << 1 | (__float_as_uint(h[k]) >> 31);
        }
    }
    __device__ __forceinline__ void settle_zeros() {       // after the reduction over the team
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (b.mn[k] == 0.0f) b.mn[k] = (z[k] & 1u) ? -0.0f : 0.0f;
            if (b.mx[k] == 0.0f) b.mx[k] = (z[3 + k] & 1u) ? -0.0f : 0.0f;
        }
    }
};

// A team of threads that splits one node together: a warp (the TLAS, and a BLAS below the top levels) or a whole CTA (the top
// levels of a large BLAS).  reduce() combines per-thread values in place (mins, maxs, unsigned mins, sums); ranks() gives each
// thread's position in a stable counting sort of one round of `size` elements by bucket (SCENE_BUCKETS = no element).
struct WarpTeam {
    uint32_t lane;
    __device__ __forceinline__ uint32_t rank() const { return lane; }
    __device__ __forceinline__ uint32_t size() const { return 32u; }
    template <int NF, int NX, int NU, int NS>
    __device__ __forceinline__ void reduce(float* mins, float* maxs, uint32_t* umins, uint32_t* sums) {
#pragma unroll
        for (int i = 0; i < NF; ++i) mins[i] = warp_min(mins[i]);
#pragma unroll
        for (int i = 0; i < NX; ++i) maxs[i] = warp_max(maxs[i]);
#pragma unroll
        for (int i = 0; i < NU; ++i)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) umins[i] = min(umins[i], __shfl_xor_sync(0xffffffffu, umins[i], o));
#pragma unroll
        for (int i = 0; i < NS; ++i) sums[i] = warp_sum(sums[i]);
    }
    __device__ __forceinline__ uint32_t ranks(uint32_t bucket, uint32_t* off) {
        const uint32_t lt = (1u << lane) - 1u;
        uint32_t pos = 0u;
#pragma unroll
        for (int b = 0; b < SCENE_BUCKETS; ++b) {
            const uint32_t mask = __ballot_sync(0xffffffffu, bucket == (uint32_t)b);
            if (bucket == (uint32_t)b) pos = off[b] + (uint32_t)__popc(mask & lt);
            off[b] += (uint32_t)__popc(mask);
        }
        return pos;
    }
};

constexpr int CTA_TEAM_SLOTS = 48;         // the most values one reduce() combines (the buckets: 18 + 18 + 6)
struct CtaTeamShared {
    uint32_t red[32][CTA_TEAM_SLOTS];
    uint32_t cnt[SCENE_BUCKETS][32];
};
struct CtaTeam {
    CtaTeamShared* sh;
    uint32_t tid, warps;
    __device__ __forceinline__ uint32_t rank() const { return tid; }
    __device__ __forceinline__ uint32_t size() const { return warps * 32u; }
    template <int NF, int NX, int NU, int NS>
    __device__ void reduce(float* mins, float* maxs, uint32_t* umins, uint32_t* sums) {
        static_assert(NF + NX + NU + NS <= CTA_TEAM_SLOTS, "CtaTeamShared::red");
        WarpTeam w{tid & 31u};
        w.reduce<NF, NX, NU, NS>(mins, maxs, umins, sums);
        const uint32_t warp = tid >> 5;
        if ((tid & 31u) == 0u) {
#pragma unroll
            for (int i = 0; i < NF; ++i) sh->red[warp][i] = __float_as_uint(mins[i]);
#pragma unroll
            for (int i = 0; i < NX; ++i) sh->red[warp][NF + i] = __float_as_uint(maxs[i]);
#pragma unroll
            for (int i = 0; i < NU; ++i) sh->red[warp][NF + NX + i] = umins[i];
#pragma unroll
            for (int i = 0; i < NS; ++i) sh->red[warp][NF + NX + NU + i] = sums[i];
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < NF; ++i) { float v = mins[i]; for (uint32_t q = 0; q < warps; ++q) v = smin(v, __uint_as_float(sh->red[q][i])); mins[i] = v; }
#pragma unroll
        for (int i = 0; i < NX; ++i) { float v = maxs[i]; for (uint32_t q = 0; q < warps; ++q) v = smax(v, __uint_as_float(sh->red[q][NF + i])); maxs[i] = v; }
#pragma unroll
        for (int i = 0; i < NU; ++i) { uint32_t v = umins[i]; for (uint32_t q = 0; q < warps; ++q) v = min(v, sh->red[q][NF + NX + i]); umins[i] = v; }
#pragma unroll
        for (int i = 0; i < NS; ++i) { uint32_t v = 0u; for (uint32_t q = 0; q < warps; ++q) v += sh->red[q][NF + NX + NU + i]; sums[i] = v; }
        __syncthreads();
    }
    __device__ uint32_t ranks(uint32_t bucket, uint32_t* off) {
        const uint32_t lane = tid & 31u, warp = tid >> 5, lt = (1u << lane) - 1u;
        uint32_t in_warp = 0u;
#pragma unroll
        for (int b = 0; b < SCENE_BUCKETS; ++b) {
            const uint32_t mask = __ballot_sync(0xffffffffu, bucket == (uint32_t)b);
            if (bucket == (uint32_t)b) in_warp = (uint32_t)__popc(mask & lt);
            if (lane == 0u) sh->cnt[b][warp] = (uint32_t)__popc(mask);
        }
        __syncthreads();
        uint32_t pos = 0u;
#pragma unroll
        for (int b = 0; b < SCENE_BUCKETS; ++b) {
            uint32_t before = 0u, total = 0u;
            for (uint32_t q = 0; q < warps; ++q) {
                const uint32_t c = sh->cnt[b][q];
                before += q < warp ? c : 0u;
                total += c;
            }
            if (bucket == (uint32_t)b) pos = off[b] + before + in_warp;
            off[b] += total;
        }
        __syncthreads();
        return pos;
    }
};

// bvh 0.7.1's BVH::build for one node of >= 2 shapes (host/hikari.cpp Builder::build) over the shapes of `sg`, by a team: the
// node's own bound (its navigator, unless the parent left it the empty box), the centre bounds and the largest axis, the six
// buckets, the SAH candidates, and the children's shape lists in idx[!parity] — bucket by bucket, each bucket in the order the
// shapes had (a stable counting sort), or the two halves in order when the centres coincide or one side would be empty.
// Every thread of the team returns the same two children.
template <class Team>
__device__ void sah_split(Team& team, const BuildSeg& sg, const BuildIn& in, BuildSeg& l, BuildSeg& r) {
    const uint32_t* idx_cur = in.idx[(sg.flags & SEG_IDX_B) ? 1 : 0];
    uint32_t* idx_nxt = in.idx[(sg.flags & SEG_IDX_B) ? 0 : 1];
    const uint32_t me = team.rank(), step = team.size();
    // bounds of the shapes' boxes (in order) and of their centres
    OrderedBox ab;
    SBox cb;
    ab.clear(); cb.clear();
    for (uint32_t j = me; j < sg.count; j += step) {
        const uint32_t shape = idx_cur[sg.begin + j];
        const float4 lo = in.box_lo[shape], hi = in.box_hi[shape], c = in.center[shape];
        ab.add(j, lo, hi);
        cb.mn[0] = smin(cb.mn[0], c.x); cb.mn[1] = smin(cb.mn[1], c.y); cb.mn[2] = smin(cb.mn[2], c.z);
        cb.mx[0] = smax(cb.mx[0], c.x); cb.mx[1] = smax(cb.mx[1], c.y); cb.mx[2] = smax(cb.mx[2], c.z);
    }
    {
        float mins[6] = {ab.b.mn[0], ab.b.mn[1], ab.b.mn[2], cb.mn[0], cb.mn[1], cb.mn[2]};
        float maxs[6] = {ab.b.mx[0], ab.b.mx[1], ab.b.mx[2], cb.mx[0], cb.mx[1], cb.mx[2]};
        team.template reduce<6, 6, 6, 0>(mins, maxs, ab.z, nullptr);
#pragma unroll
        for (int k = 0; k < 3; ++k) { ab.b.mn[k] = mins[k]; ab.b.mx[k] = maxs[k]; cb.mn[k] = mins[3 + k]; cb.mx[k] = maxs[3 + k]; }
        ab.settle_zeros();
    }
    if (sg.t != 0u && me == 0u) {
        const uint32_t at = sg.t - 1u + sg.leaves_before;
        SBox own = ab.b;
        if (sg.flags & SEG_EMPTY_BOX) own.clear();
        store_node(in.out, at, own, at + 1u, at + 3u * sg.count - 1u);
    }
    const float sx = cb.mx[0] - cb.mn[0], sy = cb.mx[1] - cb.mn[1], sz = cb.mx[2] - cb.mn[2];
    const int axis = (sx > sy && sx > sz) ? 0 : (sy > sz ? 1 : 2);       // AABB::largest_axis
    const float split_axis_size = axis == 0 ? sx : (axis == 1 ? sy : sz);
    const float axis_min = axis == 0 ? cb.mn[0] : (axis == 1 ? cb.mn[1] : cb.mn[2]);
    uint32_t nl = 0u;
    bool halves = split_axis_size < SCENE_BVH_EPSILON, boxes = true;
    if (!halves) {
        SBox bb[SCENE_BUCKETS];
        uint32_t bn[SCENE_BUCKETS];
#pragma unroll
        for (int b = 0; b < SCENE_BUCKETS; ++b) { bb[b].clear(); bn[b] = 0u; }
        for (uint32_t j = me; j < sg.count; j += step) {
            const uint32_t shape = idx_cur[sg.begin + j];
            const float4 lo = in.box_lo[shape], hi = in.box_hi[shape], c = in.center[shape];
            const float ca = axis == 0 ? c.x : (axis == 1 ? c.y : c.z);
            const uint32_t bucket = sah_bucket((ca - axis_min) / split_axis_size);
            SBox b;
            b.mn[0] = lo.x; b.mn[1] = lo.y; b.mn[2] = lo.z; b.mx[0] = hi.x; b.mx[1] = hi.y; b.mx[2] = hi.z;
#pragma unroll
            for (int q = 0; q < SCENE_BUCKETS; ++q)
                if (bucket == (uint32_t)q) { bb[q].join(b); bn[q] += 1u; }
        }
        {
            float mins[3 * SCENE_BUCKETS], maxs[3 * SCENE_BUCKETS];
#pragma unroll
            for (int b = 0; b < SCENE_BUCKETS; ++b)
#pragma unroll
                for (int k = 0; k < 3; ++k) { mins[3 * b + k] = bb[b].mn[k]; maxs[3 * b + k] = bb[b].mx[k]; }
            team.template reduce<3 * SCENE_BUCKETS, 3 * SCENE_BUCKETS, 0, SCENE_BUCKETS>(mins, maxs, nullptr, bn);
#pragma unroll
            for (int b = 0; b < SCENE_BUCKETS; ++b)
#pragma unroll
                for (int k = 0; k < 3; ++k) { bb[b].mn[k] = mins[3 * b + k]; bb[b].mx[k] = maxs[3 * b + k]; }
        }
        // the split with the least SAH cost (every thread evaluates the same five candidates)
        int min_bucket = 0;
        float min_cost = __uint_as_float(0x7f800000u);
        bool chosen = false;
        const float parent_area = ab.b.surface_area();
#pragma unroll
        for (int i = 0; i < SCENE_BUCKETS - 1; ++i) {
            SBox cl, cr;
            cl.clear(); cr.clear();
            uint32_t nlc = 0u, nrc = 0u;
#pragma unroll
            for (int b = 0; b < SCENE_BUCKETS; ++b) {
                if (b <= i) { cl.join(bb[b]); nlc += bn[b]; } else { cr.join(bb[b]); nrc += bn[b]; }
            }
            const float cost = ((float)nlc * cl.surface_area() + (float)nrc * cr.surface_area()) / parent_area;
            if (cost < min_cost) { min_bucket = i; min_cost = cost; chosen = true; }
        }
        uint32_t off[SCENE_BUCKETS];
        uint32_t acc = 0u;
#pragma unroll
        for (int b = 0; b < SCENE_BUCKETS; ++b) {
            off[b] = acc; acc += bn[b];
            if (b <= min_bucket) nl += bn[b];
        }
        if (nl == 0u || nl == sg.count) {
            halves = true;          // only non-finite boxes get here (host/hikari.cpp: the halves keep the build finite)
        } else {
            boxes = chosen;
            for (uint32_t base = 0u; base < sg.count; base += step) {
                const uint32_t j = base + me;
                uint32_t shape = 0u, bucket = (uint32_t)SCENE_BUCKETS;
                if (j < sg.count) {
                    shape = idx_cur[sg.begin + j];
                    const float4 c = in.center[shape];
                    const float ca = axis == 0 ? c.x : (axis == 1 ? c.y : c.z);
                    bucket = sah_bucket((ca - axis_min) / split_axis_size);
                }
                const uint32_t pos = team.ranks(bucket, off);
                if (j < sg.count) idx_nxt[sg.begin + pos] = shape;
            }
        }
    }
    if (halves) {
        nl = sg.count / 2u;
        for (uint32_t j = me; j < sg.count; j += step) idx_nxt[sg.begin + j] = idx_cur[sg.begin + j];
    }
    const uint32_t flags = (boxes ? 0u : SEG_EMPTY_BOX) | ((sg.flags & SEG_IDX_B) ^ SEG_IDX_B);
    l = BuildSeg{sg.begin, nl, sg.t + 1u, sg.leaves_before, flags, sg.mesh};
    r = BuildSeg{sg.begin + nl, sg.count - nl, sg.t + 2u * nl, sg.leaves_before + nl, flags, sg.mesh};
}

// a node of one shape: its navigator (the shape's box, or the empty box its parent left it) and the leaf record
__device__ void sah_leaf(const BuildSeg& sg, const BuildIn& in) {
    const uint32_t at = sg.t - 1u + sg.leaves_before;
    const uint32_t shape = in.idx[(sg.flags & SEG_IDX_B) ? 1 : 0][sg.begin];
    SBox own, e;
    own.clear(); e.clear();
    if (!(sg.flags & SEG_EMPTY_BOX)) {
        SBox b;
        const float4 lo = in.box_lo[shape], hi = in.box_hi[shape];
        b.mn[0] = lo.x; b.mn[1] = lo.y; b.mn[2] = lo.z; b.mx[0] = hi.x; b.mx[1] = hi.y; b.mx[2] = hi.z;
        own.join(b);
    }
    store_node(in.out, at, own, at + 1u, at + 2u);
    store_node(in.out, at + 1u, e, SCENE_LEAF | (shape - in.shape_base), at + 2u);
    if (in.index_base) *reinterpret_cast<uint32_t*>(in.index_base + (size_t)shape * in.index_stride) = sg.t;
}

// The subtrees whose roots are in cur[0, *s_cur), level by level, one WARP per node; cur / nxt hold as many segments as the
// subtrees have shapes.  Pre-order placement makes every node's records independent of the others'.
__device__ void sah_levels(BuildSeg* cur, BuildSeg* nxt, const BuildIn& in, uint32_t* s_cur, uint32_t* s_next) {
    const uint32_t tid = threadIdx.x, warp = tid >> 5, warps = blockDim.x >> 5;
    WarpTeam team{tid & 31u};
    for (;;) {
        const uint32_t cnt = *s_cur;
        if (cnt == 0u) break;
        for (uint32_t s = warp; s < cnt; s += warps) {
            const BuildSeg sg = cur[s];
            if (sg.count == 1u) {
                if (team.lane == 0u) sah_leaf(sg, in);
                continue;
            }
            BuildSeg l, r;
            sah_split(team, sg, in, l, r);
            if (team.lane == 0u) {
                const uint32_t slot = atomicAdd(s_next, 2u);
                nxt[slot] = l; nxt[slot + 1u] = r;
            }
        }
        __syncthreads();
        if (tid == 0u) { *s_cur = *s_next; *s_next = 0u; }
        BuildSeg* ts = cur; cur = nxt; nxt = ts;
        __syncthreads();
    }
}

// The TLAS / emissive BVH: one CTA, the whole tree.
__global__ void __launch_bounds__(256) kc_build_flat_bvh(uint32_t n, const float4* __restrict__ box_lo, const float4* __restrict__ box_hi,
                                                         float4* center, uint32_t* idx_a, uint32_t* idx_b, BuildSeg* seg_a, BuildSeg* seg_b,
                                                         hk_node* out, uint8_t* index_base, uint32_t index_stride) {
    __shared__ uint32_t s_cur_count, s_next_count;
    const uint32_t tid = threadIdx.x;
    if (n == 0u) return;
    for (uint32_t i = tid; i < n; i += blockDim.x) {
        idx_a[i] = i;
        center[i] = box_center(box_lo[i], box_hi[i]);
    }
    if (tid == 0u) {
        s_next_count = 0u;
        if (n == 1u) {      // a single shape: one leaf record without a navigator
            SBox e; e.clear();
            store_node(out, 0u, e, SCENE_LEAF | 0u, 1u);
            *reinterpret_cast<uint32_t*>(index_base) = 0u;
            s_cur_count = 0u;
        } else {
            seg_a[0] = BuildSeg{0u, n, 0u, 0u, 0u, 0u};
            s_cur_count = 1u;
        }
    }
    __syncthreads();
    const BuildIn in{box_lo, box_hi, center, {idx_a, idx_b}, out, 0u, index_base, index_stride};
    sah_levels(seg_a, seg_b, in, &s_cur_count, &s_next_count);
}

// ------------------------------------------------------------------------------------------------ mesh assets (hk_scene_add_meshes)
// GpuMesh::try_from (mod.rs:379-467) for a batch of meshes: k_mesh_records packs the vertices and primitives and each primitive's
// box and centre; then the BLAS of every mesh, bvh 0.7.1's build + flatten_custom at mesh scale, in two launches that need neither a
// grid-wide barrier nor a count read back by the host:
//   kc_build_blas_top     one 1024-thread CTA per mesh splits every node of more than BLAS_TOP_SHAPES shapes, level by level, the
//                         whole CTA on one node (sah_split with a CtaTeam); every smaller node goes to a work list
//   kc_build_blas_bottom  CTAs take work-list entries by atomic counter and finish each subtree with the TLAS builder's loop
//                         (sah_levels, one warp per node)
constexpr uint32_t BLAS_TOP_SHAPES = 4096u;
constexpr uint32_t BLAS_TOP_THREADS = 1024u, BLAS_BOTTOM_THREADS = 256u;

__device__ __forceinline__ uint32_t mesh_of(const MeshJob* jobs, uint32_t n_jobs, uint32_t i, bool by_vertex) {
    uint32_t lo = 0u, hi = n_jobs;        // the last job whose first element is <= i
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) / 2u;
        if ((by_vertex ? jobs[mid].src_vertex : jobs[mid].shape_begin) <= i) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(128) k_mesh_records(uint32_t n_jobs, const MeshJob* __restrict__ jobs, uint32_t total_vertices,
                                                      uint32_t total_primitives, const float* __restrict__ positions,
                                                      const float* __restrict__ normals, const float* __restrict__ uvs,
                                                      const uint32_t* __restrict__ indices, hk_vertex* vertices, hk_primitive* primitives,
                                                      float4* box_lo, float4* box_hi, float4* center) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total_vertices) {             // vertex i of the batch
        const MeshJob& m = jobs[mesh_of(jobs, n_jobs, i, true)];
        const uint32_t v = i - m.src_vertex;
        hk_vertex* o = vertices + m.dst_vertex + v;
        o->position[0] = positions[3u * (size_t)i]; o->position[1] = positions[3u * (size_t)i + 1u]; o->position[2] = positions[3u * (size_t)i + 2u];
        o->normal[0] = normals[3u * (size_t)i]; o->normal[1] = normals[3u * (size_t)i + 1u]; o->normal[2] = normals[3u * (size_t)i + 2u];
        o->u = uvs[2u * (size_t)i]; o->v = uvs[2u * (size_t)i + 1u];
    }
    if (i < total_primitives) {           // primitive i of the batch
        const MeshJob& m = jobs[mesh_of(jobs, n_jobs, i, false)];
        const uint32_t p = i - m.shape_begin;
        uint32_t id[3];
        if (m.strip) {                    // mod.rs:433-450: odd triangles swap their first two vertices
            const uint32_t a = p, b = p + 1u, c = p + 2u;
            const uint32_t va = m.indexed ? indices[m.src_index + a] : a, vb = m.indexed ? indices[m.src_index + b] : b;
            id[0] = (p & 1u) ? vb : va; id[1] = (p & 1u) ? va : vb;
            id[2] = m.indexed ? indices[m.src_index + c] : c;
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) id[k] = m.indexed ? indices[m.src_index + 3u * p + (uint32_t)k] : 3u * p + (uint32_t)k;
        }
        float pos[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) pos[k][c] = positions[3u * ((size_t)m.src_vertex + id[k]) + (uint32_t)c];
        float4* o = reinterpret_cast<float4*>(primitives + m.dst_primitive + p);
#pragma unroll
        for (int k = 0; k < 3; ++k) o[k] = make_float4(pos[k][0], pos[k][1], pos[k][2], __uint_as_float(id[k]));
        float lo[3], hi[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {     // std::min(std::min(a, b), c) as GpuMesh::try_from
            lo[c] = smin(smin(pos[0][c], pos[1][c]), pos[2][c]);
            hi[c] = smax(smax(pos[0][c], pos[1][c]), pos[2][c]);
        }
        const float4 l4 = make_float4(lo[0], lo[1], lo[2], 0.0f), h4 = make_float4(hi[0], hi[1], hi[2], 0.0f);
        box_lo[i] = l4; box_hi[i] = h4; center[i] = box_center(l4, h4);
    }
}

struct BlasScratch {          // hk_blas_scratch_bytes
    unsigned long long* counters;       // [0] work-list entries, [1] entries taken
    float4 *box_lo, *box_hi, *center;   // per primitive of the batch
    uint32_t *idx_a, *idx_b;
    BuildSeg *seg_a, *seg_b, *work;
};

__device__ __forceinline__ BuildIn blas_in(const MeshJob& m, const BlasScratch& s, hk_node* nodes) {
    return BuildIn{s.box_lo, s.box_hi, s.center, {s.idx_a, s.idx_b}, nodes + m.dst_node, m.shape_begin, nullptr, 0u};
}

__global__ void __launch_bounds__(BLAS_TOP_THREADS) kc_build_blas_top(const MeshJob* __restrict__ jobs, BlasScratch s, hk_node* nodes) {
    __shared__ CtaTeamShared s_team;
    __shared__ uint32_t s_cur_count, s_next_count;
    const uint32_t tid = threadIdx.x;
    const MeshJob m = jobs[blockIdx.x];
    const BuildIn in = blas_in(m, s, nodes);
    for (uint32_t i = tid; i < m.shapes; i += blockDim.x) s.idx_a[m.shape_begin + i] = m.shape_begin + i;
    const BuildSeg root{m.shape_begin, m.shapes, 0u, 0u, 0u, blockIdx.x};
    if (m.shapes <= BLAS_TOP_SHAPES) {
        if (tid == 0u) {
            if (m.shapes == 1u) {         // a single primitive: one leaf record without a navigator
                SBox e; e.clear();
                store_node(in.out, 0u, e, SCENE_LEAF | 0u, 1u);
            } else {
                s.work[atomicAdd(s.counters, 1ull)] = root;
            }
        }
        return;
    }
    BuildSeg* cur = s.seg_a + m.shape_begin;
    BuildSeg* nxt = s.seg_b + m.shape_begin;
    if (tid == 0u) { cur[0] = root; s_cur_count = 1u; s_next_count = 0u; }
    __syncthreads();
    CtaTeam team{&s_team, tid, blockDim.x >> 5};
    for (;;) {
        const uint32_t cnt = s_cur_count;
        if (cnt == 0u) break;
        for (uint32_t k = 0; k < cnt; ++k) {
            const BuildSeg sg = cur[k];
            BuildSeg ch[2];
            sah_split(team, sg, in, ch[0], ch[1]);
            if (tid == 0u)
                for (int c = 0; c < 2; ++c) {
                    if (ch[c].count > BLAS_TOP_SHAPES) nxt[s_next_count++] = ch[c];
                    else s.work[atomicAdd(s.counters, 1ull)] = ch[c];
                }
            __syncthreads();
        }
        if (tid == 0u) { s_cur_count = s_next_count; s_next_count = 0u; }
        BuildSeg* ts = cur; cur = nxt; nxt = ts;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(BLAS_BOTTOM_THREADS) kc_build_blas_bottom(const MeshJob* __restrict__ jobs, BlasScratch s, hk_node* nodes) {
    __shared__ uint32_t s_cur_count, s_next_count;
    __shared__ unsigned long long s_item;
    const uint32_t tid = threadIdx.x;
    const unsigned long long items = s.counters[0];
    for (;;) {
        if (tid == 0u) s_item = atomicAdd(s.counters + 1, 1ull);
        __syncthreads();
        const unsigned long long item = s_item;
        if (item >= items) break;
        const BuildSeg root = s.work[item];
        BuildSeg* cur = s.seg_a + root.begin;
        if (tid == 0u) { cur[0] = root; s_cur_count = 1u; s_next_count = 0u; }
        __syncthreads();
        sah_levels(cur, s.seg_b + root.begin, blas_in(jobs[root.mesh], s, nodes), &s_cur_count, &s_next_count);
    }
}

// ------------------------------------------------------------------------------------------------ emissives
// instance.rs:399-418 for emissive e (its instance, alias-table slice and material are those of the last full upload): bounding
// sphere from the instance's new AABB, surface area = sum of the transformed triangles' areas (mod.rs:318-328) in primitive order.
__global__ void __launch_bounds__(128) kc_scene_emissives(uint32_t ne, hk_emissive* emissives, const hk_instance* __restrict__ instances,
                                                          const hk_material* __restrict__ materials, const hk_primitive* __restrict__ primitives,
                                                          const hk_vertex* __restrict__ vertices, float4* box_lo, float4* box_hi) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (e >= ne) return;                                   // whole warps leave together
    hk_emissive* em = emissives + e;
    const hk_instance* inst = instances + em->instance;
    float m[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) m[k] = inst->model[k];
    const uint32_t prim0 = inst->mesh.primitive, vert0 = inst->mesh.vertex, count = em->alias_table_count;   // one alias entry per triangle
    float surface_area = 0.0f;
    for (uint32_t base = 0u; base < count; base += 32u) {
        const uint32_t i = base + lane;
        float area = 0.0f;
        if (i < count) {
            const hk_primitive* pr = primitives + prim0 + i;
            float v[3][3];
#pragma unroll
            for (int k = 0; k < 3; ++k) xf_point3(m, vertices[vert0 + pr->vertices[k].index].position, v[k]);
            const float a[3] = {v[1][0] - v[0][0], v[1][1] - v[0][1], v[1][2] - v[0][2]};
            const float b[3] = {v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2]};
            const float c[3] = {a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]};   // glam cross
            area = 0.5f * fabsf(len3(c));
        }
        const uint32_t in_chunk = count - base < 32u ? count - base : 32u;
        for (uint32_t l = 0u; l < 32u; ++l) {              // the reference's left-to-right sum, every lane the same
            const float a_l = __shfl_sync(0xffffffffu, area, (int)l);
            if (l < in_chunk) surface_area += a_l;
        }
    }
    if (lane == 0u) {
        const float* ec = materials[inst->material].emissive;
        const float e4[4] = {ec[0], ec[1], ec[2], ec[3]};
        const float intensity = 255.0f * e4[3] * len3(e4);
        float pos[3], ext[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) { pos[k] = 0.5f * (inst->max[k] + inst->min[k]); ext[k] = inst->max[k] - inst->min[k]; }
        const float radius = 0.5f * len3(ext) + sqrtf(intensity);
#pragma unroll
        for (int k = 0; k < 4; ++k) em->emissive[k] = e4[k];
#pragma unroll
        for (int k = 0; k < 3; ++k) em->position[k] = pos[k];
        em->radius = radius;
        em->surface_area = surface_area;
        box_lo[e] = make_float4(pos[0] - radius, pos[1] - radius, pos[2] - radius, 0.0f);
        box_hi[e] = make_float4(pos[0] + radius, pos[1] + radius, pos[2] + radius, 0.0f);
    }
}

// ------------------------------------------------------------------------------------------------ 4-wide TLAS
// hkw::build_wide(flat, 3n - 2, n, nullptr) (wide_build.h) restated for one CTA, so that hk_scene_update_transforms leaves the 4-wide
// TLAS on the device instead of reading the flat one back.  The same tree, node for node:
//   parse     one thread per record: a navigator's branches are the chain of exit links that starts behind it (Parser::range), checked
//             as the host checks them — links that nest, at most four branches, leaf branches of two records naming a shape < n,
//             navigator boxes that enclose their branches' boxes, no deeper than the host's recursion limit — and a leaf's rank is
//             the number of leaf records before it (block-wide scan); a shape named by two leaves fails
//   collapse  level by level, one thread per wide node: open the branch with the largest half_area while the result still fits in
//             four, the first of equal areas (detail::emit); the branches left that are not leaves are the next level's wide nodes
//   sizes     bottom-up: wide subtree sizes and stack needs, need = max((k - 1) + the child's need)
//   write     top-down: pre-order indices (a node before its children, children in order) and the 128-byte nodes, empty_node padding
// state = {ready, stack need of the whole walk, node count}: ready = blas_ok && tlas ok && need <= HK_WIDE_STACK, where
// need = the TLAS's need + base_need (the BLAS marker, the meshes' need and the slack, context.cu upload_wide_tlas).  A tree the host
// would refuse leaves node count 0 and every rank 0, as upload_wide_tlas does.
constexpr uint32_t WB_OK = 8u, WB_LEAF = 16u;      // rec_meta: branch count (0-4) | WB_OK | WB_LEAF (a leaf branch: rec_kids.x = shape)
constexpr uint32_t WB_MAX_DEPTH = 200u;            // Parser::range refuses a deeper recursion

struct WideScratch {
    uint32_t* rec_meta;      // per record, and the top-level range at index `count`
    uint4* rec_kids;         // per record: the records of its branches, or .x = the shape of a leaf branch
    uint32_t* wn_bin;        // per wide node, in level order: its record (`count` = the top-level range)
    uint32_t* wn_depth;      // depth of Parser::range at which its branches are found
    uint32_t* wn_k;          // branches after collapsing
    uint4* wn_kids;          // their records
    uint4* wn_child;         // per branch: slot of its wide node, or WIDE_EMPTY (a leaf)
    uint32_t *wn_size, *wn_need, *wn_index;
    uint32_t* level;         // level l = slots [level[l], level[l + 1])
};

__device__ __forceinline__ bool wb_encloses(const hk_node& o, const hk_node& in) {
    bool r = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) r = r && o.min[k] <= in.min[k] && in.max[k] <= o.max[k];       // false for NaN, as the host
    return r;
}

// Parser::range over [p, end): the branches' records, their count | WB_OK when every link nests and `box` (if any) encloses them
__device__ uint32_t wb_branches(const hk_node* flat, uint32_t p, uint32_t end, const hk_node* box, uint4& kids) {
    uint32_t k = 0u, at[4] = {0u, 0u, 0u, 0u};
    bool ok = p < end;
    while (ok && p < end) {
        if (k == 4u) { ok = false; break; }
        const hk_node q = flat[p];
        if (q.entry_index != p + 1u || q.exit_index <= p + 1u || q.exit_index > end) { ok = false; break; }
        if (box && !wb_encloses(*box, q)) ok = false;
        at[k++] = p;
        p = q.exit_index;
    }
    kids = make_uint4(at[0], at[1], at[2], at[3]);
    return k | (ok ? WB_OK : 0u);
}

__device__ __forceinline__ float wb_half_area(const hk_node& b) {
    const float sx = smax(b.max[0] - b.min[0], 0.0f), sy = smax(b.max[1] - b.min[1], 0.0f), sz = smax(b.max[2] - b.min[2], 0.0f);
    return sx * sy + sx * sz + sy * sz;
}

// a branch found at range depth `depth`: its own parse succeeded, and a navigator with branches stays within the recursion limit
__device__ __forceinline__ bool wb_branch_ok(uint32_t meta, uint32_t depth) {
    return (meta & WB_OK) != 0u && ((meta & WB_LEAF) != 0u || depth + 1u <= WB_MAX_DEPTH);
}

__global__ void __launch_bounds__(256) kc_build_wide_tlas(uint32_t n, const hk_node* __restrict__ flat, uint32_t blas_ok, uint32_t base_need,
                                                          WideScratch s, hk_wide_node* nodes, uint32_t* rank, uint32_t* state) {
    __shared__ uint32_t s_scan[256];
    __shared__ uint32_t s_total;
    const uint32_t tid = threadIdx.x, threads = blockDim.x;
    if (n == 0u) return;
    if (n == 1u) {          // one leaf record without a navigator: root = WIDE_LEAF | 0, no nodes
        if (tid == 0u) {
            const uint32_t e = flat[0].entry_index;
            const bool ok = e >= SCENE_LEAF && e - SCENE_LEAF < n;
            rank[0] = 0u;
            state[0] = (blas_ok && ok && base_need <= (uint32_t)HK_WIDE_STACK) ? 1u : 0u;
            state[1] = base_need; state[2] = 0u;
        }
        return;
    }
    const uint32_t count = 3u * n - 2u, cap = n - 1u;       // a binary tree over n shapes collapses into at most n - 1 wide nodes
    bool bad = false;
    // ---- parse: every record as a navigator, and the top-level range
    for (uint32_t i = tid; i <= count; i += threads) {
        uint32_t meta = 0u;
        uint4 kids = make_uint4(0u, 0u, 0u, 0u);
        if (i == count) {
            meta = wb_branches(flat, 0u, count, nullptr, kids);
        } else {
            const hk_node nav = flat[i];
            if (nav.entry_index < SCENE_LEAF && i + 1u < count) {
                const hk_node first = flat[i + 1u];
                if (first.entry_index >= SCENE_LEAF) {
                    const uint32_t shape = first.entry_index - SCENE_LEAF;
                    kids.x = shape;
                    meta = WB_LEAF | ((nav.exit_index == i + 2u && first.exit_index == i + 2u && shape < n) ? WB_OK : 0u);
                } else if (nav.exit_index <= count) {
                    meta = wb_branches(flat, i + 1u, nav.exit_index, &nav, kids);
                }
            }
        }
        s.rec_meta[i] = meta;
        s.rec_kids[i] = kids;
    }
    // ---- ranks: leaf records before each leaf record, in per-thread chunks of the array
    for (uint32_t i = tid; i < n; i += threads) rank[i] = 0xFFFFFFFFu;
    const uint32_t chunk = (count + threads - 1u) / threads, c0 = min(count, tid * chunk), c1 = min(count, c0 + chunk);
    uint32_t leaves = 0u;
    for (uint32_t i = c0; i < c1; ++i) leaves += flat[i].entry_index >= SCENE_LEAF ? 1u : 0u;
    s_scan[tid] = leaves;
    if (tid == 0u) {
        s.wn_bin[0] = count; s.wn_depth[0] = 0u; s.wn_index[0] = 0u;
        s.level[0] = 0u; s.level[1] = 1u;
        s_total = 1u;
    }
    __syncthreads();
    for (uint32_t o = 1u; o < threads; o <<= 1) {
        const uint32_t v = tid >= o ? s_scan[tid - o] : 0u;
        __syncthreads();
        s_scan[tid] += v;
        __syncthreads();
    }
    const uint32_t first_rank = s_scan[tid] - leaves;
    uint32_t r = first_rank;
    for (uint32_t i = c0; i < c1; ++i) {
        const uint32_t e = flat[i].entry_index;
        if (e < SCENE_LEAF) continue;
        if (e - SCENE_LEAF < n) rank[e - SCENE_LEAF] = r;
        ++r;
    }
    __syncthreads();
    r = first_rank;
    for (uint32_t i = c0; i < c1; ++i) {       // a shape named twice keeps only one of its ranks
        const uint32_t e = flat[i].entry_index;
        if (e < SCENE_LEAF) continue;
        if (e - SCENE_LEAF < n && rank[e - SCENE_LEAF] != r) bad = true;
        ++r;
    }
    // ---- collapse, level by level
    {
        const uint32_t m = s.rec_meta[count];
        if (!wb_branch_ok(m, 0u) || (m & WB_LEAF) != 0u) bad = true;
    }
    uint32_t lb = 0u, le = 1u, levels = 0u;
    while (lb < le) {
        for (uint32_t w = lb + tid; w < le; w += threads) {
            const uint32_t b = s.wn_bin[w], depth = s.wn_depth[w], meta = s.rec_meta[b];
            bool ok = (meta & WB_OK) != 0u && (meta & WB_LEAF) == 0u;
            uint32_t k = ok ? (meta & 7u) : 0u, id[4], dp[4];
            const uint4 bk = s.rec_kids[b];
            id[0] = bk.x; id[1] = bk.y; id[2] = bk.z; id[3] = bk.w;
            for (uint32_t j = 0u; j < 4u; ++j) dp[j] = depth;
            for (uint32_t j = 0u; j < k; ++j) ok = ok && wb_branch_ok(s.rec_meta[id[j]], dp[j]);
            while (ok && k < 4u) {
                int open = -1;
                float best = -1.0f;
                for (uint32_t j = 0u; j < k; ++j) {
                    const uint32_t mj = s.rec_meta[id[j]];
                    if ((mj & WB_LEAF) != 0u || k - 1u + (mj & 7u) > 4u) continue;
                    const float a = wb_half_area(flat[id[j]]);
                    if (a > best) { best = a; open = (int)j; }
                }
                if (open < 0) break;
                const uint32_t o = (uint32_t)open, mo = s.rec_meta[id[o]], sk = mo & 7u, sd = dp[o] + 1u;
                const uint4 sub4 = s.rec_kids[id[o]];
                const uint32_t sub[4] = {sub4.x, sub4.y, sub4.z, sub4.w};
                for (uint32_t j = k; j-- > o + 1u;) { id[j + sk - 1u] = id[j]; dp[j + sk - 1u] = dp[j]; }    // the rest moves up by sk - 1
                for (uint32_t j = 0u; j < sk; ++j) {
                    id[o + j] = sub[j]; dp[o + j] = sd;
                    ok = ok && wb_branch_ok(s.rec_meta[sub[j]], sd);
                }
                k += sk - 1u;
            }
            uint32_t child[4] = {WIDE_EMPTY, WIDE_EMPTY, WIDE_EMPTY, WIDE_EMPTY};
            if (!ok) k = 0u;
            for (uint32_t c = 0u; c < k; ++c) {
                if ((s.rec_meta[id[c]] & WB_LEAF) != 0u) continue;
                const uint32_t slot = atomicAdd(&s_total, 1u);
                if (slot >= cap) { ok = false; continue; }
                s.wn_bin[slot] = id[c]; s.wn_depth[slot] = dp[c] + 1u;
                child[c] = slot;
            }
            bad = bad || !ok;
            s.wn_k[w] = k;
            s.wn_kids[w] = make_uint4(id[0], id[1], id[2], id[3]);
            s.wn_child[w] = make_uint4(child[0], child[1], child[2], child[3]);
        }
        __syncthreads();
        lb = le;
        le = min(*(volatile uint32_t*)&s_total, cap);
        ++levels;
        if (tid == 0u) s.level[levels + 1u] = le;
        __syncthreads();
    }
    const bool ok = __syncthreads_or(bad ? 1 : 0) == 0;
    if (ok) {
        // ---- sizes and needs, bottom-up
        for (uint32_t l = levels; l-- > 0u;) {
            const uint32_t l0 = s.level[l], l1 = s.level[l + 1u];
            for (uint32_t w = l0 + tid; w < l1; w += threads) {
                const uint32_t k = s.wn_k[w];
                const uint4 c4 = s.wn_child[w];
                const uint32_t ch[4] = {c4.x, c4.y, c4.z, c4.w};
                uint32_t size = 1u, need = 0u;
                for (uint32_t c = 0u; c < k; ++c) {
                    uint32_t sub = 0u;
                    if (ch[c] != WIDE_EMPTY) { size += s.wn_size[ch[c]]; sub = s.wn_need[ch[c]]; }
                    need = max(need, (k - 1u) + sub);
                }
                s.wn_size[w] = size; s.wn_need[w] = need;
            }
            __syncthreads();
        }
        // ---- pre-order indices and nodes, top-down
        const float inf = __uint_as_float(0x7f800000u), ninf = __uint_as_float(0xff800000u);
        for (uint32_t l = 0u; l < levels; ++l) {
            const uint32_t l0 = s.level[l], l1 = s.level[l + 1u];
            for (uint32_t w = l0 + tid; w < l1; w += threads) {
                const uint32_t k = s.wn_k[w], index = s.wn_index[w];
                const uint4 k4 = s.wn_kids[w], c4 = s.wn_child[w];
                const uint32_t id[4] = {k4.x, k4.y, k4.z, k4.w}, ch[4] = {c4.x, c4.y, c4.z, c4.w};
                float v[6][4];
                uint32_t ref[4];
                uint32_t next = index + 1u;
                for (uint32_t c = 0u; c < 4u; ++c) {
                    if (c >= k) {
                        v[0][c] = v[1][c] = v[2][c] = inf; v[3][c] = v[4][c] = v[5][c] = ninf;
                        ref[c] = WIDE_EMPTY;
                        continue;
                    }
                    const hk_node b = flat[id[c]];
                    v[0][c] = b.min[0]; v[1][c] = b.min[1]; v[2][c] = b.min[2];
                    v[3][c] = b.max[0]; v[4][c] = b.max[1]; v[5][c] = b.max[2];
                    if (ch[c] != WIDE_EMPTY) {
                        s.wn_index[ch[c]] = next;
                        ref[c] = next;
                        next += s.wn_size[ch[c]];
                    } else {
                        ref[c] = WIDE_LEAF | s.rec_kids[id[c]].x;
                    }
                }
                float4* out = reinterpret_cast<float4*>(nodes + index);
                for (int q = 0; q < 6; ++q) out[q] = make_float4(v[q][0], v[q][1], v[q][2], v[q][3]);
                reinterpret_cast<uint4*>(out)[6] = make_uint4(ref[0], ref[1], ref[2], ref[3]);
                reinterpret_cast<uint4*>(out)[7] = make_uint4(0u, 0u, 0u, 0u);
            }
            __syncthreads();
        }
    } else {
        for (uint32_t i = tid; i < n; i += threads) rank[i] = 0u;
    }
    if (tid == 0u) {
        const uint32_t need = (ok ? s.wn_need[0] : 0u) + base_need;
        state[0] = (blas_ok && ok && need <= (uint32_t)HK_WIDE_STACK) ? 1u : 0u;
        state[1] = need;
        state[2] = ok ? s.wn_size[0] : 0u;
    }
}

}  // namespace hkd

// ------------------------------------------------------------------------------------------------ launchers
using namespace hkd;
void hk_launch_scene_instances(uint32_t n, const float4* models, const float4* previous, const float* mesh_aabbs, hk_instance* instances,
                               hkd::hk_instance_trav* trav, float4* previous_out, uint32_t* moved_out, float4* box_lo, float4* box_hi, cudaStream_t st) {
    if (n == 0u) return;
    k_scene_instances<<<(n + 127u) / 128u, 128, 0, st>>>(n, models, previous, mesh_aabbs, instances, trav, previous_out, moved_out, box_lo, box_hi);
}
void hk_launch_build_flat_bvh(uint32_t n, const float4* box_lo, const float4* box_hi, void* scratch, hk_node* out, void* index_base,
                              uint32_t index_stride, cudaStream_t st) {
    if (n == 0u) return;
    // scratch: centre float4[n] | idx uint32[2][n] | segments BuildSeg[2][n]   (hk_scene_bvh_scratch_bytes)
    uint8_t* p = reinterpret_cast<uint8_t*>(scratch);
    float4* center = reinterpret_cast<float4*>(p); p += sizeof(float4) * (size_t)n;
    uint32_t* idx_a = reinterpret_cast<uint32_t*>(p); p += sizeof(uint32_t) * (size_t)n;
    uint32_t* idx_b = reinterpret_cast<uint32_t*>(p); p += sizeof(uint32_t) * (size_t)n;
    p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 15u) & ~(uintptr_t)15u);
    hkd::BuildSeg* seg_a = reinterpret_cast<hkd::BuildSeg*>(p); p += sizeof(hkd::BuildSeg) * (size_t)n;
    hkd::BuildSeg* seg_b = reinterpret_cast<hkd::BuildSeg*>(p);
    kc_build_flat_bvh<<<1, 256, 0, st>>>(n, box_lo, box_hi, center, idx_a, idx_b, seg_a, seg_b, out, reinterpret_cast<uint8_t*>(index_base), index_stride);
}
size_t hk_scene_bvh_scratch_bytes(uint32_t n) {
    return sizeof(float4) * (size_t)n + 2u * sizeof(uint32_t) * (size_t)n + 16u + 2u * sizeof(hkd::BuildSeg) * (size_t)n;
}
// scratch: counters | box_lo, box_hi, centre float4[N] | idx uint32[2][N] | segments, work list BuildSeg[3][N]   (N primitives)
static hkd::BlasScratch blas_scratch(uint32_t n, void* scratch) {
    hkd::BlasScratch s;
    uint8_t* p = reinterpret_cast<uint8_t*>(scratch);
    s.counters = reinterpret_cast<unsigned long long*>(p); p += 16u;
    s.box_lo = reinterpret_cast<float4*>(p); p += sizeof(float4) * (size_t)n;
    s.box_hi = reinterpret_cast<float4*>(p); p += sizeof(float4) * (size_t)n;
    s.center = reinterpret_cast<float4*>(p); p += sizeof(float4) * (size_t)n;
    s.idx_a = reinterpret_cast<uint32_t*>(p); p += sizeof(uint32_t) * (size_t)n;
    s.idx_b = reinterpret_cast<uint32_t*>(p); p += sizeof(uint32_t) * (size_t)n;
    p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 15u) & ~(uintptr_t)15u);
    s.seg_a = reinterpret_cast<hkd::BuildSeg*>(p); p += sizeof(hkd::BuildSeg) * (size_t)n;
    s.seg_b = reinterpret_cast<hkd::BuildSeg*>(p); p += sizeof(hkd::BuildSeg) * (size_t)n;
    s.work = reinterpret_cast<hkd::BuildSeg*>(p);
    return s;
}
size_t hk_blas_scratch_bytes(uint32_t primitives) {
    return 16u + 3u * sizeof(float4) * (size_t)primitives + 2u * sizeof(uint32_t) * (size_t)primitives + 16u + 3u * sizeof(hkd::BuildSeg) * (size_t)primitives;
}
int hk_launch_build_meshes(uint32_t n_jobs, const MeshJob* jobs, uint32_t total_vertices, uint32_t total_primitives, const float* positions,
                           const float* normals, const float* uvs, const uint32_t* indices, void* scratch, hk_vertex* vertices,
                           hk_primitive* primitives, hk_node* nodes, cudaStream_t st) {
    if (n_jobs == 0u) return 0;
    const hkd::BlasScratch s = blas_scratch(total_primitives, scratch);
    cudaMemsetAsync(s.counters, 0, 16u, st);
    const uint32_t threads = total_vertices > total_primitives ? total_vertices : total_primitives;
    k_mesh_records<<<(threads + 127u) / 128u, 128, 0, st>>>(n_jobs, jobs, total_vertices, total_primitives, positions, normals, uvs, indices,
                                                            vertices, primitives, s.box_lo, s.box_hi, s.center);
    kc_build_blas_top<<<n_jobs, hkd::BLAS_TOP_THREADS, 0, st>>>(jobs, s, nodes);
    // at most 2 N / BLAS_TOP_SHAPES + n_jobs subtrees from the top levels; enough CTAs to fill the device, and no more than the work
    const uint32_t want = n_jobs + 2u * (total_primitives / hkd::BLAS_TOP_SHAPES) + 1u, bottom = want < 1056u ? want : 1056u;
    kc_build_blas_bottom<<<bottom, hkd::BLAS_BOTTOM_THREADS, 0, st>>>(jobs, s, nodes);
    return 3;
}
// scratch: rec_kids uint4[3n - 1] | wn_kids, wn_child uint4[n - 1] | rec_meta uint32[3n - 1] | six uint32[n - 1] | level uint32[n + 1]
static hkd::WideScratch wide_scratch(uint32_t n, void* scratch) {
    const size_t recs = n < 2u ? 2u : 3u * (size_t)n - 1u, cap = n < 2u ? 1u : (size_t)n - 1u;
    hkd::WideScratch s;
    uint4* q = reinterpret_cast<uint4*>(scratch);
    s.rec_kids = q; q += recs;
    s.wn_kids = q; q += cap;
    s.wn_child = q; q += cap;
    uint32_t* u = reinterpret_cast<uint32_t*>(q);
    s.rec_meta = u; u += recs;
    s.wn_bin = u; u += cap;
    s.wn_depth = u; u += cap;
    s.wn_k = u; u += cap;
    s.wn_size = u; u += cap;
    s.wn_need = u; u += cap;
    s.wn_index = u; u += cap;
    s.level = u;
    return s;
}
size_t hk_wide_tlas_scratch_bytes(uint32_t n) {
    const size_t recs = n < 2u ? 2u : 3u * (size_t)n - 1u, cap = n < 2u ? 1u : (size_t)n - 1u;
    return 16u * (recs + 2u * cap) + 4u * (recs + 6u * cap + cap + 2u);
}
void hk_launch_build_wide_tlas(uint32_t n, const hk_node* flat, bool blas_ok, uint32_t base_need, void* scratch, hkd::hk_wide_node* nodes,
                               uint32_t* rank, uint32_t* state, cudaStream_t st) {
    if (n == 0u) return;
    kc_build_wide_tlas<<<1, 256, 0, st>>>(n, flat, blas_ok ? 1u : 0u, base_need, wide_scratch(n, scratch), nodes, rank, state);
}
void hk_launch_scene_emissives(uint32_t ne, hk_emissive* emissives, const hk_instance* instances, const hk_material* materials,
                               const hk_primitive* primitives, const hk_vertex* vertices, float4* box_lo, float4* box_hi, cudaStream_t st) {
    if (ne == 0u) return;
    kc_scene_emissives<<<(ne + 3u) / 4u, 128, 0, st>>>(ne, emissives, instances, materials, primitives, vertices, box_lo, box_hi);
}
