// hikari.cpp — implementation of the host mirror declared in hikari.hpp (plain C++17, no CUDA).
// Compiled with -ffp-contract=off: the f32 arithmetic below must round exactly like the reference's Rust/glam code
// would, and is compared bit-for-bit with the independent numpy restatement in oracle/scene_build.py.
#include "hikari.hpp"

#include <math.h>
#include <string.h>

#include <algorithm>
#include <limits>

namespace hikari {

// =========================================================================================== FrameUniform
// view.rs:125-139
static const float KERNEL[3][3] = {{0.0625f, 0.125f, 0.0625f}, {0.125f, 0.25f, 0.125f}, {0.0625f, 0.125f, 0.0625f}};
static const float HALTON[8][4] = {
    {0.000000f, 0.000000f, 0.500000f, 0.333333f}, {0.250000f, 0.666667f, 0.750000f, 0.111111f},
    {0.125000f, 0.444444f, 0.625000f, 0.777778f}, {0.375000f, 0.222222f, 0.875000f, 0.555556f},
    {0.062500f, 0.888889f, 0.562500f, 0.037037f}, {0.312500f, 0.370370f, 0.812500f, 0.703704f},
    {0.187500f, 0.148148f, 0.687500f, 0.481481f}, {0.437500f, 0.814815f, 0.937500f, 0.259259f}};

FrameUniform FrameUniform::extract_component(const HikariSettings& s, const FrameCounter& counter) {  // view.rs:145-192
    FrameUniform u;
    memset(static_cast<hk_frame_uniform*>(&u), 0, sizeof(hk_frame_uniform));
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) u.kernel[c][r] = KERNEL[c][r];
    memcpy(u.halton, HALTON, sizeof(HALTON));
    for (int i = 0; i < 4; ++i) u.clear_color[i] = s.clear_color[i];
    u.number = (uint32_t)counter.value;
    u.direct_validate_interval = (uint32_t)s.direct_validate_interval;
    u.emissive_validate_interval = (uint32_t)s.emissive_validate_interval;
    u.indirect_bounces = (uint32_t)s.indirect_bounces;
    u.temporal_reuse = s.temporal_reuse ? 1u : 0u;
    u.emissive_spatial_reuse = s.emissive_spatial_reuse ? 1u : 0u;
    u.indirect_spatial_reuse = s.indirect_spatial_reuse ? 1u : 0u;
    u.max_temporal_reuse_count = (uint32_t)s.max_temporal_reuse_count;
    u.max_spatial_reuse_count = (uint32_t)s.max_spatial_reuse_count;
    u.max_reservoir_lifetime = s.max_reservoir_lifetime;
    u.solar_angle = s.solar_angle;
    u.max_indirect_luminance = s.max_indirect_luminance;
    u.upscale_ratio = s.upscale.ratio();
    return u;
}

hk_frame_inputs make_frame_inputs(const HikariSettings& settings, const FrameCounter& counter, const ViewInputs& view) {
    hk_frame_inputs in;
    memset(&in, 0, sizeof(in));
    in.frame = FrameUniform::extract_component(settings, counter);
    in.view = view.view;
    in.previous_view = view.previous_view;
    in.lights = view.lights;
    in.denoise = settings.denoise ? 1u : 0u;
    in.taa_jitter = settings.taa == Taa::Jasmine ? 1u : 0u;               // prepass.rs:193-196 TEMPORAL_ANTI_ALIASING
    in.smaa_tu4x = settings.upscale.kind == Upscale::SmaaTu4x ? 1u : 0u;  // prepass.rs:197-199 SMAA_TU4X
    in.fsr1 = settings.upscale.kind == Upscale::Fsr1 ? 1u : 0u;           // post_process.rs:1279
    in.fsr_sharpness = settings.upscale.sharpness();                      // FsrConstantsUniform::sharpness, post_process.rs:530
    return in;
}

// ================================================================================================ bvh 0.7.1
// BVH::build + flatten_custom restated from the published source of the pinned dependency (Cargo.toml:20).
namespace {

constexpr float BVH_EPSILON = 0.00001f;
constexpr int NUM_BUCKETS = 6;
const float INF = std::numeric_limits<float>::infinity();

// Rust's `f32 as usize`: saturating, NaN -> 0 (a C++ cast of NaN or of a negative value is undefined)
size_t rust_as_usize(float x) {
    if (!(x > 0.0f)) return 0;
    if (x >= 18446744073709551616.0f) return std::numeric_limits<size_t>::max();
    return (size_t)x;
}

struct Box {
    float mn[3] = {INF, INF, INF};
    float mx[3] = {-INF, -INF, -INF};
    void join(const Box& o) {
        for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], o.mn[k]); mx[k] = std::max(mx[k], o.mx[k]); }
    }
    void grow(const float p[3]) {
        for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], p[k]); mx[k] = std::max(mx[k], p[k]); }
    }
    float surface_area() const {
        float sx = mx[0] - mn[0], sy = mx[1] - mn[1], sz = mx[2] - mn[2];
        return 2.0f * (sx * sy + sx * sz + sy * sz);
    }
    int largest_axis() const {
        float sx = mx[0] - mn[0], sy = mx[1] - mn[1], sz = mx[2] - mn[2];
        if (sx > sy && sx > sz) return 0;
        if (sy > sz) return 1;
        return 2;
    }
};

struct BvhNode {
    bool leaf = false;
    uint32_t shape = 0;
    Box l_box, r_box;
    uint32_t l_index = 0, r_index = 0;
};

struct Builder {
    const std::vector<Box>& boxes;
    std::vector<std::array<float, 3>> centers;
    std::vector<BvhNode> nodes;
    std::vector<uint32_t> shape_node;

    explicit Builder(const std::vector<Box>& b) : boxes(b), centers(b.size()), shape_node(b.size(), 0) {
        for (size_t i = 0; i < b.size(); ++i)
            for (int k = 0; k < 3; ++k) centers[i][k] = b[i].mn[k] + (b[i].mx[k] - b[i].mn[k]) / 2.0f;  // AABB::center
    }
    Box joint(const std::vector<uint32_t>& idx, size_t lo, size_t hi) const {
        Box r;
        for (size_t i = lo; i < hi; ++i) r.join(boxes[idx[i]]);
        return r;
    }
    uint32_t build(const std::vector<uint32_t>& indices) {
        if (indices.size() == 1) {
            uint32_t node_index = (uint32_t)nodes.size();
            BvhNode n; n.leaf = true; n.shape = indices[0];
            nodes.push_back(n);
            shape_node[indices[0]] = node_index;
            return node_index;
        }
        Box aabb_bounds, centroid_bounds;
        for (uint32_t i : indices) { aabb_bounds.join(boxes[i]); centroid_bounds.grow(centers[i].data()); }
        uint32_t node_index = (uint32_t)nodes.size();
        nodes.emplace_back();
        int axis = centroid_bounds.largest_axis();
        float split_axis_size = centroid_bounds.mx[axis] - centroid_bounds.mn[axis];
        std::vector<uint32_t> l_idx, r_idx;
        Box l_box, r_box;
        if (split_axis_size < BVH_EPSILON) {
            size_t half = indices.size() / 2;
            l_idx.assign(indices.begin(), indices.begin() + half);
            r_idx.assign(indices.begin() + half, indices.end());
            l_box = joint(l_idx, 0, l_idx.size());
            r_box = joint(r_idx, 0, r_idx.size());
        } else {
            size_t b_size[NUM_BUCKETS] = {0};
            Box b_box[NUM_BUCKETS];
            std::vector<uint32_t> assign[NUM_BUCKETS];
            for (uint32_t i : indices) {
                float rel = (centers[i][axis] - centroid_bounds.mn[axis]) / split_axis_size;
                size_t bucket = rust_as_usize(rel * ((float)NUM_BUCKETS - 0.01f));
                if (bucket >= (size_t)NUM_BUCKETS) bucket = NUM_BUCKETS - 1;    // only for non-finite boxes (bvh 0.7.1 panics there)
                b_size[bucket] += 1;
                b_box[bucket].join(boxes[i]);
                assign[bucket].push_back(i);
            }
            int min_bucket = 0;
            float min_cost = INF;
            for (int i = 0; i < NUM_BUCKETS - 1; ++i) {
                Box cl, cr; size_t nl = 0, nr = 0;
                for (int b = 0; b <= i; ++b) { cl.join(b_box[b]); nl += b_size[b]; }
                for (int b = i + 1; b < NUM_BUCKETS; ++b) { cr.join(b_box[b]); nr += b_size[b]; }
                float cost = ((float)nl * cl.surface_area() + (float)nr * cr.surface_area()) / aabb_bounds.surface_area();
                if (cost < min_cost) { min_bucket = i; min_cost = cost; l_box = cl; r_box = cr; }
            }
            for (int b = 0; b <= min_bucket; ++b) l_idx.insert(l_idx.end(), assign[b].begin(), assign[b].end());
            for (int b = min_bucket + 1; b < NUM_BUCKETS; ++b) r_idx.insert(r_idx.end(), assign[b].begin(), assign[b].end());
            if (l_idx.empty() || r_idx.empty()) {
                // Finite boxes put the smallest centre in bucket 0 and the largest in bucket 5, so both sides hold a shape.  Only
                // non-finite boxes (NaN centres, NaN costs) get here; the halves keep the build finite.  The library refuses such
                // a scene at upload (hk_scene_upload), but this builder runs first.
                const size_t half = indices.size() / 2;
                l_idx.assign(indices.begin(), indices.begin() + half);
                r_idx.assign(indices.begin() + half, indices.end());
                l_box = joint(l_idx, 0, l_idx.size());
                r_box = joint(r_idx, 0, r_idx.size());
            }
        }
        uint32_t l = build(l_idx);
        uint32_t r = build(r_idx);
        BvhNode& n = nodes[node_index];
        n.leaf = false; n.l_box = l_box; n.r_box = r_box; n.l_index = l; n.r_index = r;
        return node_index;
    }
};

hk_node pack(const Box& aabb, uint32_t entry_index, uint32_t exit_index, uint32_t primitive_index) {  // mod.rs:185-201
    hk_node n;
    n.entry_index = (entry_index == 0xFFFFFFFFu) ? (primitive_index | 0x80000000u) : entry_index;
    n.exit_index = exit_index;
    for (int k = 0; k < 3; ++k) { n.min[k] = aabb.mn[k]; n.max[k] = aabb.mx[k]; }
    return n;
}

struct Flattener {
    const std::vector<BvhNode>& nodes;
    std::vector<hk_node>& out;
    uint32_t flat(uint32_t ni, uint32_t next_free) {
        const BvhNode& n = nodes[ni];
        if (n.leaf) {
            uint32_t next_shape = next_free + 1;
            out.push_back(pack(Box(), 0xFFFFFFFFu, next_shape, n.shape));
            return next_shape;
        }
        uint32_t after_l = branch(n.l_box, n.l_index, next_free);
        return branch(n.r_box, n.r_index, after_l);
    }
    uint32_t branch(const Box& box, uint32_t index, uint32_t next_free) {
        out.push_back(pack(Box(), 0, 0, 0));  // dummy
        uint32_t after = flat(index, next_free + 1);
        out[next_free] = pack(box, next_free + 1, after, 0xFFFFFFFFu);
        return after;
    }
};

}  // namespace

std::vector<hk_node> build_flat_bvh(const std::vector<std::array<float, 3>>& aabb_min,
                                    const std::vector<std::array<float, 3>>& aabb_max, std::vector<uint32_t>* shape_node_index) {
    std::vector<hk_node> out;
    size_t n = aabb_min.size();
    if (n == 0) { if (shape_node_index) shape_node_index->clear(); return out; }
    std::vector<Box> boxes(n);
    for (size_t i = 0; i < n; ++i)
        for (int k = 0; k < 3; ++k) { boxes[i].mn[k] = aabb_min[i][k]; boxes[i].mx[k] = aabb_max[i][k]; }
    Builder b(boxes);
    std::vector<uint32_t> all(n);
    for (size_t i = 0; i < n; ++i) all[i] = (uint32_t)i;
    b.build(all);
    out.reserve(3 * n);
    Flattener f{b.nodes, out};
    f.flat(0, 0);
    if (shape_node_index) *shape_node_index = b.shape_node;
    return out;
}

// ==================================================================================================== glam
namespace {

// Mat4::transform_point3 (no perspective divide); m is column-major
void transform_point3(const float m[16], const float p[3], float out[3]) {
    float r[4];
    for (int k = 0; k < 4; ++k) r[k] = m[k] * p[0];
    for (int k = 0; k < 4; ++k) r[k] = m[4 + k] * p[1] + r[k];
    for (int k = 0; k < 4; ++k) r[k] = m[8 + k] * p[2] + r[k];
    for (int k = 0; k < 4; ++k) r[k] = m[12 + k] + r[k];
    out[0] = r[0]; out[1] = r[1]; out[2] = r[2];
}
void transform_vector3(const float m[16], const float p[3], float out[3]) {
    float r[3];
    for (int k = 0; k < 3; ++k) r[k] = m[k] * p[0];
    for (int k = 0; k < 3; ++k) r[k] = m[4 + k] * p[1] + r[k];
    for (int k = 0; k < 3; ++k) r[k] = m[8 + k] * p[2] + r[k];
    out[0] = r[0]; out[1] = r[1]; out[2] = r[2];
}
// Mat4::inverse (cofactor expansion, glam scalar path)
void mat4_inverse(const float m[16], float out[16]) {
    float m00 = m[0], m01 = m[1], m02 = m[2], m03 = m[3];
    float m10 = m[4], m11 = m[5], m12 = m[6], m13 = m[7];
    float m20 = m[8], m21 = m[9], m22 = m[10], m23 = m[11];
    float m30 = m[12], m31 = m[13], m32 = m[14], m33 = m[15];
    float coef00 = m22 * m33 - m32 * m23, coef02 = m12 * m33 - m32 * m13, coef03 = m12 * m23 - m22 * m13;
    float coef04 = m21 * m33 - m31 * m23, coef06 = m11 * m33 - m31 * m13, coef07 = m11 * m23 - m21 * m13;
    float coef08 = m21 * m32 - m31 * m22, coef10 = m11 * m32 - m31 * m12, coef11 = m11 * m22 - m21 * m12;
    float coef12 = m20 * m33 - m30 * m23, coef14 = m10 * m33 - m30 * m13, coef15 = m10 * m23 - m20 * m13;
    float coef16 = m20 * m32 - m30 * m22, coef18 = m10 * m32 - m30 * m12, coef19 = m10 * m22 - m20 * m12;
    float coef20 = m20 * m31 - m30 * m21, coef22 = m10 * m31 - m30 * m11, coef23 = m10 * m21 - m20 * m11;
    float fac0[4] = {coef00, coef00, coef02, coef03}, fac1[4] = {coef04, coef04, coef06, coef07};
    float fac2[4] = {coef08, coef08, coef10, coef11}, fac3[4] = {coef12, coef12, coef14, coef15};
    float fac4[4] = {coef16, coef16, coef18, coef19}, fac5[4] = {coef20, coef20, coef22, coef23};
    float vec0[4] = {m10, m00, m00, m00}, vec1[4] = {m11, m01, m01, m01};
    float vec2[4] = {m12, m02, m02, m02}, vec3[4] = {m13, m03, m03, m03};
    const float sign_a[4] = {1, -1, 1, -1}, sign_b[4] = {-1, 1, -1, 1};
    float inv[4][4];
    for (int k = 0; k < 4; ++k) {
        float inv0 = vec1[k] * fac0[k] - vec2[k] * fac1[k] + vec3[k] * fac2[k];
        float inv1 = vec0[k] * fac0[k] - vec2[k] * fac3[k] + vec3[k] * fac4[k];
        float inv2 = vec0[k] * fac1[k] - vec1[k] * fac3[k] + vec3[k] * fac5[k];
        float inv3 = vec0[k] * fac2[k] - vec1[k] * fac4[k] + vec2[k] * fac5[k];
        inv[0][k] = inv0 * sign_a[k]; inv[1][k] = inv1 * sign_b[k]; inv[2][k] = inv2 * sign_a[k]; inv[3][k] = inv3 * sign_b[k];
    }
    float dot0[4] = {m00 * inv[0][0], m01 * inv[1][0], m02 * inv[2][0], m03 * inv[3][0]};
    float dot1 = ((dot0[0] + dot0[1]) + dot0[2]) + dot0[3];
    float rcp_det = 1.0f / dot1;
    for (int c = 0; c < 4; ++c)
        for (int k = 0; k < 4; ++k) out[4 * c + k] = inv[c][k] * rcp_det;
}
float length3(const float a[3]) { return sqrtf((a[0] * a[0] + a[1] * a[1]) + a[2] * a[2]); }

// The alias-table cache rule of instance.rs:385-397, used both where prepare_instances decides whether to rebuild a light's table
// and where prepare_instance_transforms decides whether an update may stay on the device.
// glam Mat4::to_scale_rotation_translation().0 = (|x_axis| * det.signum(), |y_axis|, |z_axis|), with Rust's f32::signum: -1 for
// negative values and -0.0, +1 for positive values and +0.0, NaN for NaN.  det = the upper 3x3's, as the model is affine.
void scale_of(const float* m, float scale[3]) {
    const float det3 = m[0] * (m[5] * m[10] - m[6] * m[9]) - m[4] * (m[1] * m[10] - m[2] * m[9]) + m[8] * (m[1] * m[6] - m[2] * m[5]);
    const float signum = det3 != det3 ? det3 : copysignf(1.0f, det3);
    scale[0] = length3(m) * signum;
    scale[1] = length3(m + 4);
    scale[2] = length3(m + 8);
}
// Vec3::abs_diff_eq(other, 0.01): every |a - b| <= 0.01, so false when any component is NaN
bool scale_within(const float a[3], const float b[3]) {
    return fabsf(a[0] - b[0]) <= 0.01f && fabsf(a[1] - b[1]) <= 0.01f && fabsf(a[2] - b[2]) <= 0.01f;
}

}  // namespace

// ================================================================================================= GpuMesh
PrepareMeshError GpuMesh::try_from(const Mesh& mesh, GpuMesh* out, bool build_bvh) {  // mod.rs:379-467
    if (mesh.positions.empty()) return PrepareMeshError::MissingAttributePosition;
    if (mesh.normals.empty()) return PrepareMeshError::MissingAttributeNormal;
    if (mesh.uvs.empty()) return PrepareMeshError::MissingAttributeUV;
    size_t nv = std::min(mesh.positions.size(), std::min(mesh.normals.size(), mesh.uvs.size()));  // multizip
    out->vertices.resize(nv);
    for (size_t i = 0; i < nv; ++i) {
        hk_vertex& v = out->vertices[i];
        memcpy(v.position, mesh.positions[i].data(), 12);
        memcpy(v.normal, mesh.normals[i].data(), 12);
        v.u = mesh.uvs[i][0]; v.v = mesh.uvs[i][1];
    }
    std::vector<uint32_t> indices;
    if (mesh.has_indices) indices = mesh.indices;
    else { indices.resize(nv); for (size_t i = 0; i < nv; ++i) indices[i] = (uint32_t)i; }
    auto make = [&](uint32_t a, uint32_t b, uint32_t c) {
        hk_primitive p;
        const uint32_t id[3] = {a, b, c};
        for (int k = 0; k < 3; ++k) { memcpy(p.vertices[k].position, out->vertices[id[k]].position, 12); p.vertices[k].index = id[k]; }
        return p;
    };
    out->primitives.clear();
    if (mesh.topology == PrimitiveTopology::TriangleList) {
        for (size_t i = 0; i < indices.size(); i += 3) {
            if (i + 2 >= indices.size()) return PrepareMeshError::IncompatiblePrimitiveTopology;  // short chunk (mod.rs:417-420)
            out->primitives.push_back(make(indices[i], indices[i + 1], indices[i + 2]));
        }
    } else if (mesh.topology == PrimitiveTopology::TriangleStrip) {
        for (size_t i = 0; i + 2 < indices.size(); ++i) {
            uint32_t v0 = indices[i], v1 = indices[i + 1], v2 = indices[i + 2];
            out->primitives.push_back((i & 1) == 0 ? make(v0, v1, v2) : make(v1, v0, v2));
        }
    } else {
        return PrepareMeshError::IncompatiblePrimitiveTopology;
    }
    if (out->primitives.empty()) return PrepareMeshError::NoPrimitive;
    out->nodes.clear();
    if (!build_bvh) return PrepareMeshError::Ok;
    std::vector<std::array<float, 3>> mn(out->primitives.size()), mx(out->primitives.size());
    for (size_t i = 0; i < out->primitives.size(); ++i)
        for (int k = 0; k < 3; ++k) {
            const hk_primitive& p = out->primitives[i];
            mn[i][k] = std::min(std::min(p.vertices[0].position[k], p.vertices[1].position[k]), p.vertices[2].position[k]);
            mx[i][k] = std::max(std::max(p.vertices[0].position[k], p.vertices[1].position[k]), p.vertices[2].position[k]);
        }
    out->nodes = build_flat_bvh(mn, mx, nullptr);
    return PrepareMeshError::Ok;
}

std::vector<float> GpuMesh::transformed_primitive_areas(const float transform[16]) const {  // mod.rs:318-328
    std::vector<float> areas(primitives.size());
    for (size_t i = 0; i < primitives.size(); ++i) {
        float v[3][3];
        for (int k = 0; k < 3; ++k) transform_point3(transform, vertices[primitives[i].vertices[k].index].position, v[k]);
        float a[3] = {v[1][0] - v[0][0], v[1][1] - v[0][1], v[1][2] - v[0][2]};
        float b[3] = {v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2]};
        float c[3] = {a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]};  // glam cross
        areas[i] = 0.5f * fabsf(length3(c));
    }
    return areas;
}

std::vector<hk_alias_entry> GpuMesh::build_alias_table(const float transform[16]) const {  // mod.rs:330-376
    size_t primitive_count = primitives.size();
    std::vector<float> areas = transformed_primitive_areas(transform);
    float surface_area = 0.0f;
    for (float a : areas) surface_area += a;
    std::vector<hk_alias_entry> table;
    if (primitive_count == 0) return table;
    float mean_area = surface_area / (float)primitive_count;
    std::vector<std::pair<size_t, float>> over, under;
    for (size_t id = 0; id < primitive_count; ++id) {
        float prob = areas[id] / mean_area;
        if (prob > 1.0f) over.push_back({id, prob});
        if (prob < 1.0f) under.push_back({id, prob});
    }
    table.resize(primitive_count);
    for (size_t id = 0; id < primitive_count; ++id) { table[id].prob = 0.0f; table[id].index = (uint32_t)id; }
    while (!under.empty() && !over.empty()) {
        auto over_bucket = over.back(); over.pop_back();
        auto under_bucket = under.back(); under.pop_back();
        float delta = 1.0f - under_bucket.second;
        over_bucket.second -= delta;
        // assert!(over_bucket.1 >= 0.0) in the reference (mod.rs:360); no abort across the ABI here
        if (over_bucket.second > 1.0f) over.push_back(over_bucket);
        else if (over_bucket.second < 1.0f) under.push_back(over_bucket);
        table[under_bucket.first].prob = delta;
        table[under_bucket.first].index = (uint32_t)over_bucket.first;
    }
    return table;
}

// ======================================================================================= MeshMaterialWorld
uint32_t MeshMaterialWorld::add_mesh(const Mesh& mesh) {
    meshes_.push_back(mesh);
    device_mesh_.resize(meshes_.size(), false);
    return (uint32_t)meshes_.size() - 1;
}
uint32_t MeshMaterialWorld::add_device_mesh(const Mesh& mesh) {
    const uint32_t id = add_mesh(mesh);
    device_mesh_[id] = true;
    return id;
}
uint32_t MeshMaterialWorld::add_material(const StandardMaterial& m) { materials_in_.push_back(m); return (uint32_t)materials_in_.size() - 1; }
void MeshMaterialWorld::set_material(uint32_t id, const StandardMaterial& m) { if (id < materials_in_.size()) materials_in_[id] = m; }
uint32_t MeshMaterialWorld::add_instance(const InstanceDesc& i) { instances_in_.push_back(i); return (uint32_t)instances_in_.size() - 1; }
void MeshMaterialWorld::set_instance_transform(uint32_t instance, const float transform[16]) {
    if (instance < instances_in_.size()) memcpy(instances_in_[instance].transform, transform, 64);
}
void MeshMaterialWorld::set_instance_visible(uint32_t instance, bool visible) {
    if (instance < instances_in_.size()) instances_in_[instance].visible = visible;
}
void MeshMaterialWorld::previous_transform_system() {  // transform.rs:31-44
    for (InstanceDesc& d : instances_in_) {
        if (d.has_queue) memcpy(d.queue[1], d.queue[0], 64);
        else memcpy(d.queue[1], d.transform, 64);
        memcpy(d.queue[0], d.transform, 64);
        d.has_queue = true;
    }
}
uint32_t MeshMaterialWorld::add_texture(const hk_texture_desc& t, const uint8_t* pixels) {
    texture_pixels_.emplace_back(pixels, pixels + (size_t)t.width * t.height * 4);
    hk_texture_desc d = t;
    d.rgba8 = nullptr;  // fixed up in scene_desc()
    textures_.push_back(d);
    return (uint32_t)textures_.size() - 1;
}

void MeshMaterialWorld::prepare_mesh_assets() {  // mesh.rs:106-166
    mesh_aabb_ok_.clear();
    if (!universal_settings.build_mesh_acceleration_structure) return;
    gpu_meshes_.assign(meshes_.size(), GpuMesh());
    mesh_ok_.assign(meshes_.size(), false);
    mesh_errors_.assign(meshes_.size(), PrepareMeshError::Ok);
    mesh_index_.assign(meshes_.size(), hk_mesh_index{0, 0, 0, 0});
    vertices.clear(); primitives.clear(); asset_nodes.clear();
    device_mesh_.resize(meshes_.size(), false);
    bool any_device = false;
    uint32_t device_nodes = 0;          // BLAS records of the device meshes so far: they sit behind the host meshes' records
    host_vertex_count_ = host_primitive_count_ = 0;
    for (size_t i = 0; i < meshes_.size(); ++i) {
        const bool on_device = device_mesh_[i];
        PrepareMeshError e = GpuMesh::try_from(meshes_[i], &gpu_meshes_[i], !on_device);
        mesh_errors_[i] = e;
        if (e != PrepareMeshError::Ok) continue;  // silently dropped (mesh.rs:128-137)
        mesh_ok_[i] = true;
        const GpuMesh& g = gpu_meshes_[i];
        // hk_scene_add_meshes: 1 record for one primitive, 3 m - 2 for m >= 2 (bvh 0.7.1's flatten_custom)
        const size_t m = g.primitives.size();
        const uint32_t nodes = on_device ? (uint32_t)(m == 1 ? 1 : 3 * m - 2) : (uint32_t)g.nodes.size();
        mesh_index_[i] = hk_mesh_index{(uint32_t)vertices.size(), (uint32_t)primitives.size(), (uint32_t)asset_nodes.size() + device_nodes, nodes};
        if (!on_device && !any_device) { host_vertex_count_ += (uint32_t)g.vertices.size(); host_primitive_count_ += (uint32_t)m; }
        any_device = any_device || on_device;
        vertices.insert(vertices.end(), g.vertices.begin(), g.vertices.end());
        primitives.insert(primitives.end(), g.primitives.begin(), g.primitives.end());
        if (on_device) device_nodes += nodes;
        else asset_nodes.insert(asset_nodes.end(), g.nodes.begin(), g.nodes.end());
    }
}

void MeshMaterialWorld::prepare_material_assets() {  // material.rs:139-203
    materials.resize(materials_in_.size());
    for (size_t i = 0; i < materials_in_.size(); ++i) {
        const StandardMaterial& m = materials_in_[i];
        hk_material g;
        memset(&g, 0, sizeof(g));
        memcpy(g.base_color, m.base_color.data(), 16);
        memcpy(g.emissive, m.emissive.data(), 16);
        g.base_color_texture = m.base_color_texture;
        g.emissive_texture = m.emissive_texture;
        g.perceptual_roughness = m.perceptual_roughness;
        g.metallic = m.metallic;
        g.metallic_roughness_texture = m.metallic_roughness_texture;
        g.reflectance = m.reflectance;
        g.normal_map_texture = m.normal_map_texture;
        g.occlusion_texture = m.occlusion_texture;
        materials[i] = g;
    }
}

void MeshMaterialWorld::prepare_instances() {  // instance.rs:245-444
    if (!universal_settings.build_instance_acceleration_structure) return;
    instances.clear(); emissives.clear(); alias_table.clear(); instance_nodes.clear(); emissive_nodes.clear();
    previous_models.clear();
    alias_table_cache_.resize(instances_in_.size());
    std::vector<const InstanceDesc*> kept;
    for (const InstanceDesc& d : instances_in_) {
        if (!d.visible) continue;                                              // instance.rs:357
        if (d.mesh >= meshes_.size() || !mesh_ok_[d.mesh] || d.material >= materials.size()) continue;  // instance.rs:275-283
        kept.push_back(&d);
        const float* previous = d.has_queue ? d.queue[1] : d.transform;        // PreviousMeshUniform::transform = queue[1]
        previous_models.insert(previous_models.end(), previous, previous + 16);
    }
    kept_.clear();
    for (const InstanceDesc* d : kept) kept_.push_back({(uint32_t)(d - instances_in_.data()), d->mesh, d->material});
    for (const InstanceDesc* d : kept) {
        const GpuMesh& g = gpu_meshes_[d->mesh];
        // bevy Aabb of the mesh: from_min_max over the positions
        float mn[3] = {INF, INF, INF}, mx[3] = {-INF, -INF, -INF};
        for (const hk_vertex& v : g.vertices)
            for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], v.position[k]); mx[k] = std::max(mx[k], v.position[k]); }
        float center[3], half[3];
        for (int k = 0; k < 3; ++k) { center[k] = 0.5f * (mx[k] + mn[k]); half[k] = 0.5f * (mx[k] - mn[k]); }
        float c[3];
        transform_point3(d->transform, center, c);
        float lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};  // instance.rs:298-303 starts from ZERO
        for (int index = 0; index < 8; ++index) {
            float sgn[3] = {(float)(2 * (index & 1) - 1), (float)(2 * ((index >> 1) & 1) - 1), (float)(2 * ((index >> 2) & 1) - 1)};
            float vtx[3] = {half[0] * sgn[0], half[1] * sgn[1], half[2] * sgn[2]}, t[3];
            transform_vector3(d->transform, vtx, t);
            for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], t[k]); hi[k] = std::max(hi[k], t[k]); }
        }
        hk_instance inst;
        memset(&inst, 0, sizeof(inst));
        for (int k = 0; k < 3; ++k) { inst.min[k] = lo[k] + c[k]; inst.max[k] = hi[k] + c[k]; }
        memcpy(inst.model, d->transform, 64);
        float inv[16];
        mat4_inverse(d->transform, inv);
        for (int col = 0; col < 4; ++col)
            for (int row = 0; row < 4; ++row) inst.inverse_transpose_model[4 * col + row] = inv[4 * row + col];  // .transpose()
        inst.mesh = mesh_index_[d->mesh];
        inst.material = d->material;
        instances.push_back(inst);
    }
    if (!instances.empty()) {
        std::vector<std::array<float, 3>> mn(instances.size()), mx(instances.size());
        for (size_t i = 0; i < instances.size(); ++i)
            for (int k = 0; k < 3; ++k) { mn[i][k] = instances[i].min[k]; mx[i][k] = instances[i].max[k]; }
        std::vector<uint32_t> node_index;
        instance_nodes = build_flat_bvh(mn, mx, &node_index);
        for (size_t i = 0; i < instances.size(); ++i) instances[i].node_index = node_index[i];
    }
    for (size_t id = 0; id < instances.size(); ++id) {
        const hk_instance& inst = instances[id];
        const float* e = materials[inst.material].emissive;
        float intensity = 255.0f * e[3] * length3(e);
        if (intensity > 0.0f) {
            const GpuMesh& g = gpu_meshes_[kept[id]->mesh];
            // alias table cached per entity while the scale stays within 0.01 (instance.rs:385-397): a rotating or
            // translating light keeps the table computed for the transform it was first seen with
            float scale[3];
            scale_of(inst.model, scale);
            CachedAliasTable& cache = alias_table_cache_[(size_t)(kept[id] - instances_in_.data())];
            const bool cache_hit = cache.valid && scale_within(cache.scale, scale);
            if (!cache_hit) {
                cache.valid = true;
                memcpy(cache.scale, scale, 12);
                cache.table = g.build_alias_table(inst.model);
            }
            const std::vector<hk_alias_entry>& table = cache.table;
            hk_emissive em;
            memset(&em, 0, sizeof(em));
            em.alias_table_offset = (uint32_t)alias_table.size();
            em.alias_table_count = (uint32_t)table.size();
            alias_table.insert(alias_table.end(), table.begin(), table.end());
            float surface_area = 0.0f;
            for (float a : g.transformed_primitive_areas(inst.model)) surface_area += a;
            memcpy(em.emissive, e, 16);
            float ext[3];
            for (int k = 0; k < 3; ++k) { em.position[k] = 0.5f * (inst.max[k] + inst.min[k]); ext[k] = inst.max[k] - inst.min[k]; }
            em.radius = 0.5f * length3(ext) + sqrtf(intensity);
            em.instance = (uint32_t)id;
            em.surface_area = surface_area;
            emissives.push_back(em);
        }
    }
    if (!emissives.empty()) {
        std::vector<std::array<float, 3>> mn(emissives.size()), mx(emissives.size());
        for (size_t i = 0; i < emissives.size(); ++i)
            for (int k = 0; k < 3; ++k) { mn[i][k] = emissives[i].position[k] - emissives[i].radius; mx[i][k] = emissives[i].position[k] + emissives[i].radius; }
        std::vector<uint32_t> node_index;
        emissive_nodes = build_flat_bvh(mn, mx, &node_index);
        for (size_t i = 0; i < emissives.size(); ++i) emissives[i].node_index = node_index[i];
    }
}

bool MeshMaterialWorld::prepare_instance_transforms() {
    if (!universal_settings.build_instance_acceleration_structure) return false;
    std::vector<const InstanceDesc*> kept;
    for (const InstanceDesc& d : instances_in_) {
        if (!d.visible) continue;
        if (d.mesh >= meshes_.size() || !mesh_ok_[d.mesh] || d.material >= materials.size()) continue;
        kept.push_back(&d);
    }
    if (kept.size() != kept_.size() || kept.size() != instances.size()) return false;
    for (size_t i = 0; i < kept.size(); ++i)
        if ((uint32_t)(kept[i] - instances_in_.data()) != kept_[i].entity || kept[i]->mesh != kept_[i].mesh || kept[i]->material != kept_[i].material)
            return false;
    // an emissive whose scale left its cached alias table's range needs the table rebuilt: the full path
    for (const hk_emissive& em : emissives) {
        const InstanceDesc* d = kept[em.instance];
        const size_t entity = (size_t)(d - instances_in_.data());
        if (entity >= alias_table_cache_.size() || !alias_table_cache_[entity].valid) return false;
        float scale[3];
        scale_of(d->transform, scale);
        if (!scale_within(alias_table_cache_[entity].scale, scale)) return false;
    }
    mesh_aabb_.resize(meshes_.size());
    mesh_aabb_ok_.resize(meshes_.size(), false);
    transform_models.clear(); transform_previous.clear(); transform_aabbs.clear();
    for (const InstanceDesc* d : kept) {
        if (!mesh_aabb_ok_[d->mesh]) {   // bevy Aabb of the mesh: from_min_max over the positions, as prepare_instances computes it
            const GpuMesh& g = gpu_meshes_[d->mesh];
            float mn[3] = {INF, INF, INF}, mx[3] = {-INF, -INF, -INF};
            for (const hk_vertex& v : g.vertices)
                for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], v.position[k]); mx[k] = std::max(mx[k], v.position[k]); }
            for (int k = 0; k < 3; ++k) { mesh_aabb_[d->mesh][k] = 0.5f * (mx[k] + mn[k]); mesh_aabb_[d->mesh][3 + k] = 0.5f * (mx[k] - mn[k]); }
            mesh_aabb_ok_[d->mesh] = true;
        }
        const float* previous = d->has_queue ? d->queue[1] : d->transform;
        transform_models.insert(transform_models.end(), d->transform, d->transform + 16);
        transform_previous.insert(transform_previous.end(), previous, previous + 16);
        transform_aabbs.insert(transform_aabbs.end(), mesh_aabb_[d->mesh].begin(), mesh_aabb_[d->mesh].end());
    }
    return true;
}

void MeshMaterialWorld::prepare() { prepare_mesh_assets(); prepare_material_assets(); prepare_instances(); }

hk_scene_desc MeshMaterialWorld::scene_desc() const {
    hk_scene_desc d;
    memset(&d, 0, sizeof(d));
    // the host meshes only: the device meshes' records are built on the device (a world without them has every mesh here)
    const bool device = std::find(device_mesh_.begin(), device_mesh_.end(), true) != device_mesh_.end();
    d.vertices = vertices.data(); d.vertex_count = device ? host_vertex_count_ : (uint32_t)vertices.size();
    d.primitives = primitives.data(); d.primitive_count = device ? host_primitive_count_ : (uint32_t)primitives.size();
    d.asset_nodes = asset_nodes.data(); d.asset_node_count = (uint32_t)asset_nodes.size();
    d.alias_table = alias_table.data(); d.alias_count = (uint32_t)alias_table.size();
    d.instances = instances.data(); d.instance_count = (uint32_t)instances.size();
    d.instance_nodes = instance_nodes.data(); d.instance_node_count = (uint32_t)instance_nodes.size();
    d.materials = materials.data(); d.material_count = (uint32_t)materials.size();
    d.emissive_nodes = emissive_nodes.data(); d.emissive_node_count = (uint32_t)emissive_nodes.size();
    d.emissives = emissives.data(); d.emissive_count = (uint32_t)emissives.size();
    auto* self = const_cast<MeshMaterialWorld*>(this);
    for (size_t i = 0; i < textures_.size(); ++i) self->textures_[i].rgba8 = texture_pixels_[i].data();
    d.textures = textures_.data(); d.texture_count = (uint32_t)textures_.size();
    d.previous_instance_models = previous_models.size() == 16 * instances.size() && !instances.empty() ? previous_models.data() : nullptr;
    return d;
}

}  // namespace hikari
