// ORACLE — test infrastructure, not product code.  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may build, load or call this file.  The product (libhikari_b200.so) never does.
//
// CPU restatement (C++17 + OpenMP) of the reference's per-frame GPU path, pass by pass, texture format by texture
// format, exactly as LightNode::run (src/light.rs:590-702) and PostProcessNode::run (src/post_process.rs:1140-1234)
// dispatch it.  Every function cites the WGSL it follows (paths relative to /root/reference/src/shaders).
//
// PARITY: the compute passes below are PINNED against the reference's own shader text (and the ray-cast G-buffer is held, within a
// rasteriser's sub-pixel snapping, against prepass.wgsl executed behind a software rasteriser: tests/test_wgsl_prepass.py); the host-side scene build
// is not.  The reference ships no tests, golden vectors or fixtures for this path (SURVEY.md 4, 8(c)) and cannot be built
// here (no rustc / wgpu / Vulkan) — but its hot path IS text: oracle/wgsl/ translates src/shaders/{light,denoise,tone_mapping,smaa,taa}.wgsl
// (read in place under /root/reference) to C++, compiles one library per pipeline specialisation into oracle/_ref/wgsl/ and drives
// them with the bind-group wiring of src/light.rs / src/post_process.rs.  What that execution of the reference's text computes —
// every reservoir buffer, radiance / variance plane, albedo, denoised plane, tone-mapped image, SMAA / TAA / FSR image of every frame
// of twenty-three free-running sequences (FSR 1.0 from the GLSL of src/shaders/fsr/source.zip, oracle/wgsl/glsl2cpp.py) — is committed as fixtures (tests/golden/wgsl_*.npz, tools/make_wgsl_golden.py), and this file reproduces
// every one of them BIT FOR BIT (tests/test_wgsl_reference.py; the CUDA path likewise, tests/test_gpu_wgsl_golden.py).
// The G-buffer, which the reference rasterises and hko_prepass ray-casts, is held against prepass.wgsl executed behind a software
// rasteriser (oracle/wgsl/raster_prepass.py, tests/test_wgsl_prepass.py): same coverage, same ids up to edge pixels, values within a
// rasteriser's sub-pixel snapping.  Still a restatement, i.e. parity unpinned there: the BVH / alias-table build of the pinned crate
// bvh 0.7.1 and glam (host/hikari.cpp, restated from the published sources), and the ~110 lines of bevy_pbr 0.9.1 the shaders import
// (oracle/wgsl/prelude/, SURVEY App. D).  For those the evidence remains a second, independent restatement per pass
// (tests/test_*_numpy.py; table in DESIGN.md 2), the topology-invariance test and the physical anchors of tests/test_estimator.py.
// Deviations that are forced and documented:
//   * the G-buffer is ray-cast (hko_prepass) instead of rasterised (prepass.wgsl:40-100) — same five planes, same
//     formats, oracle-defined coverage;
//   * implementation-defined WGSL arithmetic (FMA contraction, sin/cos/exp/pow accuracy, NaN in min/max/clamp/pack)
//     is fixed by include/hk_math.h;
//   * the racy scatter store_previous_spatial_reservoir(previous_coords) (light.wgsl:1094,1201,1458) is resolved
//     in raster order, last writer wins.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <omp.h>

#include <algorithm>
#include <string>
#include <vector>

#include "hikari_b200.h"
#include "hk_math.h"

using namespace hk;

namespace {

// ------------------------------------------------------------------------------------------------ state
struct Texture {
    std::vector<vec4> texels;  // decoded (sRGB -> linear already applied per texel)
    uint32_t w = 0, h = 0, mode_u = 0, mode_v = 0, linear = 1;
};

struct Sample {  // light.wgsl:49-57
    vec4 radiance = v4(0.0f);
    vec4 random = v4(0.0f);
    vec4 visible_position = v4(0.0f);
    vec3 visible_normal = v3(0.0f);
    uint32_t visible_instance = 0;
    vec4 sample_position = v4(0.0f);
    vec3 sample_normal = v3(0.0f);
};
struct Reservoir {  // light.wgsl:59-66
    Sample s;
    float count = 0, lifetime = 0, w = 0, w_sum = 0, w2_sum = 0;
};
struct Ray { vec3 origin, direction, inv_direction; };
struct Aabb { vec3 min, max; };
struct Intersection { vec2 uv = v2(0, 0); float distance = 0; };
struct Hit { Intersection intersection; uint32_t instance_index = 0, primitive_index = 0; };
struct Surface { vec4 base_color, emissive; float reflectance, metallic, roughness, occlusion; };
struct HitInfo {
    vec4 position = v4(0.0f);
    vec3 normal = v3(0.0f);
    vec2 uv = v2(0, 0);
    uint32_t instance_index = 0, material_index = 0;
};
struct LightCandidate {
    vec3 direction = v3(0.0f);
    float max_distance = 0, min_distance = 0;
    uint32_t emissive_instance = 0;
    float p = 0;
};

struct ScatterWrite { int32_t index; hk_packed_reservoir value; };

}  // namespace

struct hko_context {
    int W = 0, H = 0;  // full (deferred) size; render size == full size at upscale ratio 1
    int RW = 0, RH = 0;
    int OW = 0, OH = 0;       // SMAA TU4x output extent: ceil(size * (2 / ratio)) in f32 (post_process.rs:663-667,711,717), <= 2 RW x 2 RH
    // scene (bind group 2)
    std::vector<hk_vertex> vertices;
    std::vector<hk_primitive> primitives;
    std::vector<hk_node> asset_nodes;
    std::vector<hk_alias_entry> alias_table;
    std::vector<hk_instance> instances;
    std::vector<float> previous_models;     // instance_count x 16, empty = no instance moved (prepass.wgsl:7-8 previous_mesh)
    std::vector<hk_node> instance_nodes;
    std::vector<hk_material> materials;
    std::vector<hk_node> emissive_nodes;
    std::vector<hk_emissive> emissives;
    std::vector<Texture> textures;
    bool scene_ready = false, noise_ready = false;
    std::vector<uint8_t> noise;  // 16 x 64 x 64 x 4
    // G-buffer (bind group 1), reference formats
    std::vector<vec4> position;            // Rgba32Float
    std::vector<uint32_t> normal;          // Rgba8Snorm
    std::vector<vec2> depth_gradient;      // Rg32Float
    std::vector<vec2> instance_material;   // Rg32Float
    std::vector<vec4> velocity_uv;         // Rgba32Float
    std::vector<vec4> previous_position, previous_velocity_uv;   // swapped with the current ones every frame (prepass.rs:312-321,427)
    // light textures (bind group 5) and reservoirs (bind group 6)
    std::vector<uvec2> albedo;             // Rgba16Float, full size
    std::vector<uvec2> render[3];          // Rgba16Float
    std::vector<float> variance[3];        // R32Float
    std::vector<hk_packed_reservoir> reservoir[10];
    // post process
    std::vector<uvec2> denoise_internal[4];
    std::vector<float> denoise_internal_variance;
    std::vector<uvec2> denoise_render[3];
    std::vector<uvec2> tone_mapping_output[2];   // [frame.number % 2] is written (post_process.rs:716,979)
    std::vector<uvec2> upscale_output;           // OW x OH <= 2 RW x 2 RH (post_process.rs:715-722); W x H under Upscale::Fsr1 (:723)
    std::vector<uvec2> upscale_sharpen_output;   // upscale_output[1], W x H: FSR RCAS result (post_process.rs:723,1079-1086)
    std::vector<uvec2> taa_output[2];            // OW x OH with SMAA TU4x, else RW x RH (post_process.rs:726-731)
    // per-frame
    hk_frame_inputs in;
    struct alignas(64) RayCounters { uint64_t primary = 0, tlas = 0, blas = 0; };
    std::vector<RayCounters> rays;   // one slot per OpenMP thread (no shared atomics on the timed path)
    RayCounters& cnt() { return rays[(size_t)omp_get_thread_num()]; }
    std::string error;
    int threads = 0;
};

namespace {

using Ctx = hko_context;

inline vec3 ld3(const float* p) { return v3(p[0], p[1], p[2]); }
inline vec4 ld4(const float* p) { return v4(p[0], p[1], p[2], p[3]); }
inline mat4 ldm(const float* p) { mat4 m; for (int c = 0; c < 4; ++c) m.c[c] = ld4(p + 4 * c); return m; }

inline vec2 coords_to_uv(ivec2 coords, ivec2 size) {  // utils.wgsl:37-39
    return (v2((float)coords.x, (float)coords.y) + 0.5f) / v2((float)size.x, (float)size.y);
}
inline vec2 clip_to_uv(vec4 clip) {  // utils.wgsl:30-35
    vec2 uv = v2(clip.x, clip.y) / clip.w;
    uv = (uv + 1.0f) * 0.5f;
    uv.y = 1.0f - uv.y;
    return uv;
}

// ------------------------------------------------------------------------------------------- reservoirs
Reservoir unpack_reservoir(const hk_packed_reservoir& packed) {  // light.wgsl:77-109
    Reservoir r;
    vec2 t0 = unpack2x16float(packed.reservoir[0]);
    vec2 t1 = unpack2x16float(packed.reservoir[1]);
    r.count = t0.x; r.w = t0.y; r.w_sum = t1.x; r.w2_sum = t1.y;
    t0 = unpack2x16float(packed.radiance[0]);
    t1 = unpack2x16float(packed.radiance[1]);
    r.s.radiance = v4(t0.x, t0.y, t1.x, t1.y);
    t0 = unpack2x16unorm(packed.random[0]);
    t1 = unpack2x16unorm(packed.random[1]);
    r.s.random = v4(t0.x, t0.y, t1.x, t1.y);
    vec4 t2 = unpack4x8snorm(packed.visible_normal);
    r.s.visible_position = ld4(packed.visible_position);
    r.s.visible_normal = normalize(xyz(t2));
    r.lifetime = 127.0f * (1.0f + t2.w);
    t2 = unpack4x8snorm(packed.sample_normal);
    r.s.sample_position = v4(packed.sample_position[0], packed.sample_position[1], packed.sample_position[2], t2.w);
    r.s.sample_normal = normalize(xyz(t2));
    r.s.visible_instance = f32_to_u32(packed.sample_position[3]);
    return r;
}
hk_packed_reservoir pack_reservoir(const Reservoir& r) {  // light.wgsl:111-136
    hk_packed_reservoir p;
    p.reservoir[0] = pack2x16float(r.count, r.w);
    p.reservoir[1] = pack2x16float(r.w_sum, r.w2_sum);
    p.radiance[0] = pack2x16float(r.s.radiance.x, r.s.radiance.y);
    p.radiance[1] = pack2x16float(r.s.radiance.z, r.s.radiance.w);
    p.random[0] = pack2x16unorm(r.s.random.x, r.s.random.y);
    p.random[1] = pack2x16unorm(r.s.random.z, r.s.random.w);
    p.visible_position[0] = r.s.visible_position.x; p.visible_position[1] = r.s.visible_position.y;
    p.visible_position[2] = r.s.visible_position.z; p.visible_position[3] = r.s.visible_position.w;
    p.sample_position[0] = r.s.sample_position.x; p.sample_position[1] = r.s.sample_position.y;
    p.sample_position[2] = r.s.sample_position.z; p.sample_position[3] = (float)r.s.visible_instance;
    p.visible_normal = pack4x8snorm(v4(r.s.visible_normal, r.lifetime / 127.0f - 1.0f));
    p.sample_normal = pack4x8snorm(v4(r.s.sample_normal, r.s.sample_position.w));
    return p;
}
void set_reservoir(Reservoir& r, const Sample& s, float w_new) {  // light.wgsl:138-144
    r.count = 1.0f; r.lifetime = 0.0f; r.w_sum = w_new; r.w2_sum = w_new * w_new; r.s = s;
}
void update_reservoir(Reservoir& r, const Sample& s, float w_new) {  // light.wgsl:146-173
    r.w_sum += w_new;
    r.w2_sum += w_new * w_new;
    r.count = r.count + 1.0f;
    float rand = fract(sum4(s.random));
    if (rand < w_new / r.w_sum) r.s = s;
}
void merge_reservoir(Reservoir& r, const Reservoir& other, float p) {  // light.wgsl:175-179
    float count = r.count;
    update_reservoir(r, other.s, p * other.w * other.count);
    r.count = count + other.count;
}
inline bool uv_inside(vec2 uv) { return fabsf(uv.x - 0.5f) < 0.5f && fabsf(uv.y - 0.5f) < 0.5f; }     // all(abs(uv-0.5) < 0.5)
inline bool uv_inside_eq(vec2 uv) { return fabsf(uv.x - 0.5f) <= 0.5f && fabsf(uv.y - 0.5f) <= 0.5f; }  // <=
inline int32_t uv_to_index(vec2 uv, ivec2 size) {
    ivec2 c; c.x = f32_to_i32(uv.x * (float)size.x); c.y = f32_to_i32(uv.y * (float)size.y);
    return c.x + size.x * c.y;
}
Reservoir load_previous(const std::vector<hk_packed_reservoir>& buf, vec2 uv, ivec2 size) {  // light.wgsl:181-190,201-210
    Reservoir r;
    if (uv_inside(uv)) r = unpack_reservoir(buf[uv_to_index(uv, size)]);
    return r;
}

// ---------------------------------------------------------------------------------------------- tracing
inline vec3 instance_position_world_to_local(const hk_instance& inst, vec3 p) {  // light.wgsl:306-310
    vec4 q = mul_transposed(ldm(inst.inverse_transpose_model), v4(p, 1.0f));
    return xyz(q) / q.w;
}
inline vec3 instance_direction_world_to_local(const hk_instance& inst, vec3 p) {  // light.wgsl:312-316
    return xyz(mul_transposed(ldm(inst.inverse_transpose_model), v4(p, 0.0f)));
}
inline vec3 instance_position_local_to_world(const hk_instance& inst, vec3 p) {  // light.wgsl:318-322
    vec4 q = mul(ldm(inst.model), v4(p, 1.0f));
    return xyz(q) / q.w;
}
inline vec3 instance_normal_local_to_world(const hk_instance& inst, vec3 n) {  // light.wgsl:324-338
    mat3 m;
    m.c[0] = ld3(inst.inverse_transpose_model + 0);
    m.c[1] = ld3(inst.inverse_transpose_model + 4);
    m.c[2] = ld3(inst.inverse_transpose_model + 8);
    return normalize(mul(m, n));
}
inline bool inside_aabb(vec3 p, const Aabb& a) {  // light.wgsl:340-342
    return p.x > a.min.x && p.y > a.min.y && p.z > a.min.z && p.x < a.max.x && p.y < a.max.y && p.z < a.max.z;
}
inline float intersects_aabb(const Ray& ray, const Aabb& aabb) {  // light.wgsl:344-362
    vec3 t1 = (aabb.min - ray.origin) * ray.inv_direction;
    vec3 t2 = (aabb.max - ray.origin) * ray.inv_direction;
    float t_min = fmin_(t1.x, t2.x);
    float t_max = fmax_(t1.x, t2.x);
    t_min = fmax_(t_min, fmin_(t1.y, t2.y));
    t_max = fmin_(t_max, fmax_(t1.y, t2.y));
    t_min = fmax_(t_min, fmin_(t1.z, t2.z));
    t_max = fmin_(t_max, fmax_(t1.z, t2.z));
    float t = F32_MAX;
    if (t_max >= t_min && t_max >= 0.0f) t = t_min;
    return t;
}
inline Intersection intersects_triangle(const Ray& ray, const hk_primitive& tri) {  // light.wgsl:364-398
    Intersection result;
    result.distance = F32_MAX;
    vec3 p0 = ld3(tri.vertices[0].position), p1 = ld3(tri.vertices[1].position), p2 = ld3(tri.vertices[2].position);
    vec3 ab = p1 - p0;
    vec3 ac = p2 - p0;
    vec3 u_vec = cross(ray.direction, ac);
    float det = dot(ab, u_vec);
    if (fabsf(det) < F32_EPSILON) return result;
    float inv_det = 1.0f / det;
    vec3 ao = ray.origin - p0;
    float u = dot(ao, u_vec) * inv_det;
    if (u < 0.0f || u > 1.0f) { result.uv = v2(u, 0.0f); return result; }
    vec3 v_vec = cross(ao, ab);
    float v = dot(ray.direction, v_vec) * inv_det;
    result.uv = v2(u, v);
    if (v < 0.0f || u + v > 1.0f) return result;
    float distance = dot(ac, v_vec) * inv_det;
    if (distance > F32_EPSILON) result.distance = distance;
    return result;
}
bool traverse_bottom(const Ctx& c, Hit& hit, const Ray& ray, const hk_mesh_index& mesh, float early_distance) {  // light.wgsl:400-440
    bool intersected = false;
    uint32_t index = 0;
    for (; index < mesh.node_count;) {
        uint32_t node_index = mesh.node_offset + index;
        const hk_node& node = c.asset_nodes[node_index];
        Aabb aabb;
        if (node.entry_index >= BVH_LEAF_FLAG) {
            uint32_t primitive_index = mesh.primitive + node.entry_index - BVH_LEAF_FLAG;
            const hk_primitive& prim = c.primitives[primitive_index];
            vec3 p0 = ld3(prim.vertices[0].position), p1 = ld3(prim.vertices[1].position), p2 = ld3(prim.vertices[2].position);
            aabb.min = vmin(p0, vmin(p1, p2));
            aabb.max = vmax(p0, vmax(p1, p2));
            if (intersects_aabb(ray, aabb) < hit.intersection.distance) {
                Intersection intersection = intersects_triangle(ray, prim);
                if (intersection.distance < hit.intersection.distance) {
                    hit.intersection = intersection;
                    hit.primitive_index = primitive_index;
                    intersected = true;
                    if (intersection.distance < early_distance) return intersected;
                }
            }
            index = node.exit_index;
        } else {
            aabb.min = ld3(node.min);
            aabb.max = ld3(node.max);
            index = (intersects_aabb(ray, aabb) < hit.intersection.distance) ? node.entry_index : node.exit_index;
        }
    }
    return intersected;
}
Hit traverse_top(const Ctx& c, const Ray& ray, float max_distance, float early_distance, uint32_t exclude_instance) {  // light.wgsl:442-486
    Hit hit;
    hit.intersection.distance = max_distance;
    hit.instance_index = U32_MAX;
    hit.primitive_index = U32_MAX;
    uint32_t index = 0;
    const uint32_t count = (uint32_t)c.instance_nodes.size();
    for (; index < count;) {
        const hk_node& node = c.instance_nodes[index];
        Aabb aabb;
        if (node.entry_index >= BVH_LEAF_FLAG) {
            uint32_t instance_index = node.entry_index - BVH_LEAF_FLAG;
            const hk_instance& instance = c.instances[instance_index];
            aabb.min = ld3(instance.min);
            aabb.max = ld3(instance.max);
            if (instance_index != exclude_instance && intersects_aabb(ray, aabb) < hit.intersection.distance) {
                Ray r;
                r.origin = instance_position_world_to_local(instance, ray.origin);
                r.direction = instance_direction_world_to_local(instance, ray.direction);
                r.inv_direction = 1.0f / r.direction;
                if (traverse_bottom(c, hit, r, instance.mesh, early_distance)) {
                    hit.instance_index = instance_index;
                    if (hit.intersection.distance < early_distance) return hit;
                }
            }
            index = node.exit_index;
        } else {
            aabb.min = ld3(node.min);
            aabb.max = ld3(node.max);
            index = (intersects_aabb(ray, aabb) < hit.intersection.distance) ? node.entry_index : node.exit_index;
        }
    }
    return hit;
}
HitInfo empty_hit_info(vec3 position, vec3 direction) {  // light.wgsl:488-494
    HitInfo info;
    info.instance_index = U32_MAX;
    info.material_index = U32_MAX;
    info.position = v4(position + direction * DISTANCE_MAX, 0.0f);
    return info;
}
HitInfo hit_info(const Ctx& c, const Ray& ray, const Hit& hit) {  // light.wgsl:496-523
    HitInfo info;
    info.instance_index = hit.instance_index;
    info.material_index = U32_MAX;
    if (hit.instance_index != U32_MAX) {
        const hk_instance& instance = c.instances[hit.instance_index];
        const hk_primitive& prim = c.primitives[hit.primitive_index];
        const hk_vertex& a = c.vertices[instance.mesh.vertex + prim.vertices[0].index];
        const hk_vertex& b = c.vertices[instance.mesh.vertex + prim.vertices[1].index];
        const hk_vertex& d = c.vertices[instance.mesh.vertex + prim.vertices[2].index];
        vec2 uv0 = v2(a.u, a.v), uv1 = v2(b.u, b.v), uv2 = v2(d.u, d.v);
        vec2 uv = hit.intersection.uv;
        info.uv = uv0 + uv.x * (uv1 - uv0) + uv.y * (uv2 - uv0);
        vec3 n0 = ld3(a.normal), n1 = ld3(b.normal), n2 = ld3(d.normal);
        info.normal = n0 + uv.x * (n1 - n0) + uv.y * (n2 - n0);
        info.normal = instance_normal_local_to_world(instance, info.normal);
        info.position = v4(ray.origin + ray.direction * hit.intersection.distance, 1.0f);
        info.material_index = instance.material;
    } else {
        info.position = v4(ray.origin + ray.direction * DISTANCE_MAX, 0.0f);
    }
    return info;
}
void occlude_hit_info(const Ray& ray, const Hit& hit, HitInfo& info) {  // light.wgsl:526-533
    if (hit.instance_index != U32_MAX) {
        info.instance_index = hit.instance_index;
        info.material_index = U32_MAX;
        info.position = v4(ray.origin + ray.direction * hit.intersection.distance, 1.0f);
        info.normal = v3(0.0f);
    }
}

// --------------------------------------------------------------------------------------------- sampling
inline vec2 sample_uniform_disk(vec2 rand) {  // light.wgsl:537-541
    float r = sqrtf(rand.x);
    float theta = 2.0f * PI * rand.y;
    float s, c; sincos_(theta, &s, &c);
    return v2(r * c, r * s);
}
inline vec4 sample_cosine_hemisphere(vec2 rand) {  // light.wgsl:544-549
    vec2 t = sample_uniform_disk(rand);
    vec3 direction = v3(t.x, t.y, sqrtf(1.0f - dot(t, t)));
    float pdf = 2.0f * INV_TAU * direction.z;
    return v4(direction, pdf);
}
inline vec4 sample_uniform_cone(vec2 rand, float cos_angle) {  // light.wgsl:552-559
    float z = 1.0f - (1.0f - cos_angle) * rand.x;
    float theta = TAU * rand.y;
    float r = sqrtf(1.0f - z * z);
    float s, c; sincos_(theta, &s, &c);
    vec3 direction = v3(r * c, r * s, z);
    float pdf = INV_TAU / (1.0f - cos_angle);
    return v4(direction, pdf);
}
inline vec2 sample_uniform_triangle_barycentric(vec2 rand) {  // light.wgsl:562-565
    float srx = sqrtf(rand.x);
    return v2(1.0f - srx, rand.y * srx);
}
inline vec4 compute_directional_cone(const Ctx& c) {  // light.wgsl:571-573
    float s, co; sincos_(c.in.frame.solar_angle, &s, &co);
    return v4(ld3(c.in.lights.direction_to_light), co);
}
inline vec3 compute_emissive_radiance(vec4 emissive) {  // light.wgsl:594-596
    return 255.0f * emissive.w * xyz(emissive);
}

LightCandidate select_light_candidate(Ctx& c, vec4 rand, vec3 position, vec3 normal, uint32_t instance, HitInfo& info) {  // light.wgsl:599-708
    LightCandidate candidate;
    candidate.max_distance = F32_MAX;
    candidate.min_distance = DISTANCE_MAX;
    candidate.emissive_instance = DONT_SAMPLE_EMISSIVE;

    vec4 cone = compute_directional_cone(c);
    vec3 rand_direction = mul(normal_basis(xyz(cone)), xyz(sample_uniform_cone(v2(rand.z, rand.w), cone.w)));
    candidate.direction = rand_direction;
    candidate.p = 1.0f;
    info = empty_hit_info(position, rand_direction);
    if (instance == DONT_SAMPLE_EMISSIVE) return candidate;

    hk_emissive emissive;
    memset(&emissive, 0, sizeof(emissive));
    float count = 0.0f;
    uint32_t index = 0;
    float rand_1d = rand.x;
    const uint32_t ncount = (uint32_t)c.emissive_nodes.size();
    for (; index < ncount;) {
        const hk_node& node = c.emissive_nodes[index];
        Aabb aabb;
        if (node.entry_index >= BVH_LEAF_FLAG) {
            uint32_t emissive_index = node.entry_index - BVH_LEAF_FLAG;
            const hk_emissive& cur = c.emissives[emissive_index];
            aabb.min = ld3(cur.position) - cur.radius;
            aabb.max = ld3(cur.position) + cur.radius;
            if (instance != cur.instance && inside_aabb(position, aabb)) {
                rand_1d = fract(rand_1d + GOLDEN_RATIO);
                count += 1.0f;
                if (rand_1d < 1.0f / count) {
                    candidate.emissive_instance = cur.instance;
                    emissive = cur;
                }
            }
            index = node.exit_index;
        } else {
            aabb.min = ld3(node.min);
            aabb.max = ld3(node.max);
            index = inside_aabb(position, aabb) ? node.entry_index : node.exit_index;
        }
    }

    if (candidate.emissive_instance != DONT_SAMPLE_EMISSIVE) {
        uint32_t alias_index = std::min(f32_to_u32(rand.x * (float)emissive.alias_table_count), emissive.alias_table_count - 1u);
        const hk_alias_entry& alias_entry = c.alias_table[emissive.alias_table_offset + alias_index];
        uint32_t primitive_index = (rand.y < alias_entry.prob) ? alias_entry.index : alias_index;

        const hk_instance& emissive_instance = c.instances[candidate.emissive_instance];
        const hk_primitive& prim = c.primitives[emissive_instance.mesh.primitive + primitive_index];
        vec2 b = sample_uniform_triangle_barycentric(v2(rand.z, rand.w));
        vec3 lp = b.x * ld3(prim.vertices[0].position) + b.y * ld3(prim.vertices[1].position) +
                  (1.0f - b.x - b.y) * ld3(prim.vertices[2].position);
        vec3 p = instance_position_local_to_world(emissive_instance, lp);

        Hit hit;
        hit.intersection.distance = F32_MAX;
        hit.instance_index = U32_MAX;
        hit.primitive_index = U32_MAX;

        Ray ray;
        ray.origin = position + normal * RAY_BIAS;
        ray.direction = normalize(p - position);
        ray.inv_direction = v3(0.0f);

        Ray r;
        r.origin = instance_position_world_to_local(emissive_instance, ray.origin);
        r.direction = instance_direction_world_to_local(emissive_instance, ray.direction);
        r.inv_direction = 1.0f / r.direction;

        candidate.direction = ray.direction;
        bool front = dot(candidate.direction, normal) > 0.0f;
        if (front) c.cnt().blas += 1;
        if (front && traverse_bottom(c, hit, r, emissive_instance.mesh, 0.0f)) {
            hit.instance_index = emissive.instance;
            info = hit_info(c, ray, hit);
            candidate.max_distance = hit.intersection.distance;
            candidate.min_distance = hit.intersection.distance - 0.1f;
            vec3 delta = xyz(info.position) - position;
            candidate.p = dot(delta, delta) / fabsf(dot(ray.direction, info.normal) * emissive.surface_area);
            candidate.p = candidate.p / count;
        } else {
            info = empty_hit_info(ray.origin, ray.direction);
            candidate.emissive_instance = DONT_SAMPLE_EMISSIVE;
            candidate.direction = rand_direction;
            candidate.p = 1.0f;
        }
    }
    return candidate;
}

// ---------------------------------------------------------------------------------------------- shading
inline vec3 calculate_view(const Ctx& c, vec4 world_position, bool is_orthographic) {  // light.wgsl:714-727
    if (is_orthographic) {
        const float* vp = c.in.view.view_proj;
        return normalize(v3(vp[0 * 4 + 2], vp[1 * 4 + 2], vp[2 * 4 + 2]));
    }
    return normalize(ld3(c.in.view.world_position) - xyz(world_position));
}
inline bool is_orthographic(const Ctx& c) { return c.in.view.projection[3 * 4 + 3] == 1.0f; }

vec4 sample_texture(const Texture& t, vec2 uv) {  // textureSampleLevel(textures[id], samplers[id], uv, 0.0)
    auto wrap = [](int i, int n, uint32_t mode) {
        if (mode == 0) { i %= n; if (i < 0) i += n; return i; }
        if (mode == 1) return std::min(std::max(i, 0), n - 1);
        int period = 2 * n; i %= period; if (i < 0) i += period;
        return (i < n) ? i : period - 1 - i;
    };
    if (!t.linear) {
        int x = (int)floorf(uv.x * (float)t.w), y = (int)floorf(uv.y * (float)t.h);
        return t.texels[(size_t)wrap(y, (int)t.h, t.mode_v) * t.w + wrap(x, (int)t.w, t.mode_u)];
    }
    float fx = uv.x * (float)t.w - 0.5f, fy = uv.y * (float)t.h - 0.5f;
    float x0f = floorf(fx), y0f = floorf(fy);
    float ax = fx - x0f, ay = fy - y0f;
    int x0 = (int)x0f, y0 = (int)y0f;
    int xa = wrap(x0, (int)t.w, t.mode_u), xb = wrap(x0 + 1, (int)t.w, t.mode_u);
    int ya = wrap(y0, (int)t.h, t.mode_v), yb = wrap(y0 + 1, (int)t.h, t.mode_v);
    vec4 t00 = t.texels[(size_t)ya * t.w + xa], t10 = t.texels[(size_t)ya * t.w + xb];
    vec4 t01 = t.texels[(size_t)yb * t.w + xa], t11 = t.texels[(size_t)yb * t.w + xb];
    vec4 top = t00 * (1.0f - ax) + t10 * ax;
    vec4 bot = t01 * (1.0f - ax) + t11 * ax;
    return top * (1.0f - ay) + bot * ay;
}

Surface retreive_surface(const Ctx& c, uint32_t material_index, vec2 uv) {  // light.wgsl:730-742 / 749-781
    Surface surface;
    const hk_material& material = c.materials[material_index];
    surface.base_color = ld4(material.base_color);
    surface.emissive = ld4(material.emissive);
    surface.metallic = material.metallic;
    surface.occlusion = 1.0f;
    if (!c.textures.empty()) {
        uint32_t id = material.base_color_texture;
        if (id != U32_MAX) surface.base_color = surface.base_color * sample_texture(c.textures[id], uv);
        id = material.emissive_texture;
        if (id != U32_MAX) surface.emissive = surface.emissive * sample_texture(c.textures[id], uv);
        id = material.metallic_roughness_texture;
        if (id != U32_MAX) surface.metallic *= sample_texture(c.textures[id], uv).x;
        id = material.occlusion_texture;
        if (id != U32_MAX) surface.occlusion = sample_texture(c.textures[id], uv).x;
    }
    surface.roughness = perceptualRoughnessToRoughness(material.perceptual_roughness);
    surface.reflectance = material.reflectance;
    return surface;
}
vec4 retreive_emissive(const Ctx& c, uint32_t material_index, vec2 uv) {  // light.wgsl:744-747 / 783-793
    const hk_material& material = c.materials[material_index];
    vec4 emissive = ld4(material.emissive);
    if (!c.textures.empty()) {
        uint32_t id = material.emissive_texture;
        if (id != U32_MAX) emissive = emissive * sample_texture(c.textures[id], uv);
    }
    return emissive;
}
vec3 lit(vec3 radiance, vec3 diffuse_color, float roughness, vec3 F0, vec3 Lv, vec3 N, vec3 V) {  // light.wgsl:796-818
    vec3 Hv = normalize(Lv + V);
    float NoL = saturate(dot(N, Lv));
    float NoH = saturate(dot(N, Hv));
    float LoH = saturate(dot(Lv, Hv));
    float NdotV = fmax_(dot(N, V), 0.0001f);
    vec3 diffuse = diffuse_color * Fd_Burley(roughness, NdotV, NoL, LoH);
    float specular_intensity = 1.0f;
    vec3 specular_light = specular(F0, roughness, NdotV, NoL, NoH, LoH, specular_intensity);
    return (specular_light + diffuse) * radiance * NoL;
}
vec3 ambient(const Ctx& c, vec3 diffuse_color, float roughness, float occlusion, vec3 F0, vec3 N, vec3 V) {  // light.wgsl:820-833
    float NdotV = fmax_(dot(N, V), 0.0001f);
    vec3 diffuse_ambient = EnvBRDFApprox(diffuse_color, 1.0f, NdotV);
    vec3 specular_ambient = EnvBRDFApprox(F0, roughness, NdotV);
    return occlusion * (diffuse_ambient + specular_ambient) * xyz(ld4(c.in.lights.ambient_color));
}
vec4 input_radiance(const Ctx& c, const Ray& ray, const HitInfo& info, bool sample_directional, uint32_t sample_emissive,
                    bool sample_ambient) {  // light.wgsl:835-867
    vec3 radiance = v3(0.0f);
    float amb = 0.0f;
    if (info.instance_index == U32_MAX) {
        vec4 cone = compute_directional_cone(c);
        bool hit_directional = dot(ray.direction, xyz(cone)) >= cone.w;
        if (sample_directional && hit_directional) {
            radiance = xyz(ld4(c.in.lights.directional_color));
            amb = 0.0f;
        } else {
            radiance = sample_ambient ? xyz(ld4(c.in.lights.ambient_color)) : v3(0.0f);
            amb = 1.0f;
        }
    } else {
        if (sample_emissive == info.instance_index) {
            vec4 emissive = retreive_emissive(c, info.material_index, info.uv);
            radiance = compute_emissive_radiance(emissive);
        }
    }
    return v4(radiance, 1.0f - amb);
}
vec3 shading(const Ctx& c, vec3 V, vec3 N, vec3 Lv, const Surface& surface, vec4 in_radiance) {  // light.wgsl:869-888
    vec3 base_color = xyz(surface.base_color);
    float reflectance = surface.reflectance, roughness = surface.roughness, metallic = surface.metallic;
    float occlusion = surface.occlusion;
    vec3 F0 = v3(0.16f * reflectance * reflectance * (1.0f - metallic)) + base_color * metallic;
    vec3 diffuse_color = base_color * (1.0f - metallic);
    vec3 lit_radiance = lit(xyz(in_radiance), diffuse_color, roughness, F0, Lv, N, V);
    vec3 ambient_radiance = ambient(c, diffuse_color, roughness, occlusion, F0, N, V);
    return mix(lit_radiance, ambient_radiance, 1.0f - in_radiance.w);
}
vec3 env_brdf(vec3 V, vec3 N, const Surface& surface) {  // light.wgsl:890-908
    vec3 base_color = xyz(surface.base_color);
    float reflectance = surface.reflectance, roughness = surface.roughness, metallic = surface.metallic;
    float occlusion = surface.occlusion;
    float NdotV = fmax_(dot(N, V), 0.0001f);
    vec3 F0 = v3(0.16f * reflectance * reflectance * (1.0f - metallic)) + base_color * metallic;
    vec3 diffuse_color = base_color * (1.0f - metallic);
    vec3 diffuse_ambient = EnvBRDFApprox(diffuse_color, 1.0f, NdotV);
    vec3 specular_ambient = EnvBRDFApprox(F0, roughness, NdotV);
    return occlusion * (diffuse_ambient + specular_ambient);
}

// ----------------------------------------------------------------------------------------------- restir
inline float reservoir_lifetime(const Ctx& c) {  // light.wgsl:913-915
    return (c.in.frame.max_reservoir_lifetime <= 1.0f) ? F32_MAX : c.in.frame.max_reservoir_lifetime;
}
bool check_previous_reservoir(Reservoir& r, const Sample& s) {  // light.wgsl:917-935
    float depth_ratio = r.s.visible_position.w / s.visible_position.w;
    depth_ratio = (depth_ratio < 1.0f) ? 1.0f / depth_ratio : depth_ratio;
    bool depth_miss = depth_ratio > 1.05f * (1.0f + 0.5f * s.random.x);
    bool instance_miss = r.s.visible_instance != s.visible_instance;
    bool normal_miss = dot(s.visible_normal, r.s.visible_normal) < 0.9f;
    if (depth_miss || normal_miss || instance_miss) { r = Reservoir(); return false; }
    return true;
}
void temporal_restir(Reservoir& r, const Sample& s, float w_new, uint32_t max_sample_count) {  // light.wgsl:937-952
    update_reservoir(r, s, w_new);
    float m = (float)max_sample_count;
    if (r.count > m) {
        r.w_sum *= m / r.count;
        r.w2_sum *= m / r.count;
        r.count = m;
    }
}
float compute_jacobian(const Sample& q, const Sample& r) {  // light.wgsl:985-1004
    vec3 normal = q.sample_normal;
    float cos_phi_1 = fabsf(dot(normalize(xyz(r.visible_position) - xyz(q.sample_position)), normal));
    float cos_phi_2 = fabsf(dot(normalize(xyz(q.visible_position) - xyz(q.sample_position)), normal));
    float term_1 = cos_phi_1 / fmax_(0.0001f, cos_phi_2);
    float num = length(xyz(q.visible_position) - xyz(q.sample_position));
    num *= num;
    float denom = length(xyz(r.visible_position) - xyz(q.sample_position));
    denom *= denom;
    float term_2 = num / fmax_(denom, 0.0001f);
    float jacobian = term_1 * term_2;
    return clampf(jacobian, 1.0f, 50.0f);
}
inline float variance_of(const Reservoir& r) {  // light.wgsl:1224-1226
    float variance = r.w2_sum / r.count - sq(r.w_sum / r.count);
    variance = (r.count < 1.0f) ? variance : variance / r.count;
    return fmin_(variance, MAX_VARIANCE);
}

// ------------------------------------------------------------------------------------------ G-buffer I/O
struct Deferred {
    const Ctx& c;
    explicit Deferred(const Ctx& ctx) : c(ctx) {}
    ivec2 size() const { ivec2 s; s.x = c.W; s.y = c.H; return s; }
    vec2 jittered_uv(vec2 uv, float amount) const {  // light.wgsl:1007-1011 (0.25) / denoise.wgsl:37-41 (0.5)
        vec2 texel_size = v2(1.0f, 1.0f) / v2((float)c.W, (float)c.H);
        float ratio = c.in.frame.upscale_ratio - 1.0f;
        float sgn = ((c.in.frame.number & 1u) == 0u) ? -amount : amount;
        return uv + sgn * texel_size * ratio;
    }
    ivec2 jittered_coords(vec2 uv) const {  // light.wgsl:1013-1017
        vec2 d = jittered_uv(uv, 0.25f);
        ivec2 r; r.x = f32_to_i32(d.x * (float)c.W); r.y = f32_to_i32(d.y * (float)c.H);
        return r;
    }
    bool in_bounds(ivec2 p) const { return p.x >= 0 && p.y >= 0 && p.x < c.W && p.y < c.H; }
    // textureLoad out of bounds returns zero (robust access)
    vec4 position(ivec2 p) const { return in_bounds(p) ? c.position[(size_t)p.y * c.W + p.x] : v4(0.0f); }
    vec4 normal(ivec2 p) const { return in_bounds(p) ? unpack4x8snorm(c.normal[(size_t)p.y * c.W + p.x]) : v4(0.0f); }
    vec2 depth_gradient(ivec2 p) const { return in_bounds(p) ? c.depth_gradient[(size_t)p.y * c.W + p.x] : v2(0, 0); }
    vec2 instance_material(ivec2 p) const { return in_bounds(p) ? c.instance_material[(size_t)p.y * c.W + p.x] : v2(0, 0); }
    vec4 velocity_uv(ivec2 p) const { return in_bounds(p) ? c.velocity_uv[(size_t)p.y * c.W + p.x] : v4(0.0f); }
    // textureSampleLevel(..., nearest_sampler, uv, 0.0): clamp-to-edge nearest
    ivec2 nearest(vec2 uv) const {
        ivec2 p; p.x = (int)floorf(uv.x * (float)c.W); p.y = (int)floorf(uv.y * (float)c.H);
        p.x = std::min(std::max(p.x, 0), c.W - 1); p.y = std::min(std::max(p.y, 0), c.H - 1);
        return p;
    }
};

inline vec4 noise_random(const Ctx& c, ivec2 coords) {  // light.wgsl:1075-1079
    uint32_t number = c.in.frame.number;
    uint32_t noise_id = number % NOISE_TEXTURE_COUNT;
    vec2 noise_uv = (v2((float)coords.x, (float)coords.y) + (float)number + 0.5f) / v2(64.0f, 64.0f);
    // nearest + repeat
    int tx = (int)floorf(fract(noise_uv.x) * 64.0f), ty = (int)floorf(fract(noise_uv.y) * 64.0f);
    tx = std::min(tx, 63); ty = std::min(ty, 63);
    const uint8_t* t = &c.noise[(((size_t)noise_id * 64 + ty) * 64 + tx) * 4];
    vec4 rnd = v4(unorm8(t[0]), unorm8(t[1]), unorm8(t[2]), unorm8(t[3]));
    return fract(rnd + (float)number * GOLDEN_RATIO);
}

template <class F>
void for_pixels(Ctx& c, int w, int h, F f) {
#pragma omp parallel for schedule(dynamic, 4) num_threads(c.threads)
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) f(x, y);
}

// ------------------------------------------------------------------------------- P0: G-buffer (ray cast)
// Replaces the raster prepass (prepass.wgsl:40-100, prepass.rs:760-852): same five planes, cleared to 0.
vec2 frame_jitter(const Ctx& c) {  // prepass.wgsl:30-38
    uint32_t index = c.in.smaa_tu4x ? ((c.in.frame.number >> 1u) & 15u) : (c.in.frame.number & 15u);
    const float* h = c.in.frame.halton[index >> 1u];
    return ((index & 1u) == 0u) ? v2(h[0], h[1]) : v2(h[2], h[3]);
}
Ray primary_ray(const Ctx& c, float px, float py, vec2 jitter_ndc) {
    vec2 uv = v2(px + 0.5f, py + 0.5f) / v2((float)c.W, (float)c.H);
    vec2 ndc = v2(uv.x * 2.0f - 1.0f, (1.0f - uv.y) * 2.0f - 1.0f) - jitter_ndc;
    vec4 p = mul(ldm(c.in.view.inverse_view_proj), v4(ndc.x, ndc.y, 1.0f, 1.0f));
    vec3 near_point = xyz(p) / p.w;
    Ray ray;
    if (is_orthographic(c)) {
        // parallel projection (what the raster prepass draws for an OrthographicProjection): the line of sight of the pixel
        // runs from its point on the near plane (NDC z = 1, reverse Z) towards its point on the far plane (NDC z = 0)
        vec4 q = mul(ldm(c.in.view.inverse_view_proj), v4(ndc.x, ndc.y, 0.0f, 1.0f));
        ray.origin = near_point;
        ray.direction = normalize(xyz(q) / q.w - near_point);
    } else {
        ray.origin = ld3(c.in.view.world_position);
        ray.direction = normalize(near_point - ray.origin);
    }
    ray.inv_direction = 1.0f / ray.direction;
    return ray;
}
void pass_prepass(Ctx& c) {
    // prepass_textures_system swaps current <-> previous every frame before the pass renders (prepass.rs:427)
    c.position.swap(c.previous_position);
    c.velocity_uv.swap(c.previous_velocity_uv);
    const mat4 view_proj = ldm(c.in.view.view_proj);
    const mat4 prev_view_proj = ldm(c.in.previous_view.view_proj);
    vec2 jitter_ndc = v2(0.0f, 0.0f);
    if (c.in.taa_jitter) {  // prepass.wgsl:52-54,71: clip.xy += (jx, -jy) * w with j = 2 * halton * texel
        vec2 j = 2.0f * frame_jitter(c) * (v2(1.0f, 1.0f) / v2(c.in.view.viewport[2], c.in.view.viewport[3]));
        jitter_ndc = v2(j.x, -j.y);
    }
    for_pixels(c, c.W, c.H, [&](int x, int y) {
        size_t idx = (size_t)y * c.W + x;
        Ray ray = primary_ray(c, (float)x, (float)y, jitter_ndc);
        c.cnt().primary += 1;
        Hit hit = traverse_top(c, ray, F32_MAX, 0.0f, DONT_EXCLUDE);
        if (hit.instance_index == U32_MAX) {
            c.position[idx] = v4(0.0f); c.normal[idx] = 0u; c.depth_gradient[idx] = v2(0, 0);
            c.instance_material[idx] = v2(0, 0); c.velocity_uv[idx] = v4(0.0f);
            return;
        }
        const hk_instance& inst = c.instances[hit.instance_index];
        const hk_primitive& prim = c.primitives[hit.primitive_index];
        const hk_vertex& a = c.vertices[inst.mesh.vertex + prim.vertices[0].index];
        const hk_vertex& b = c.vertices[inst.mesh.vertex + prim.vertices[1].index];
        const hk_vertex& d = c.vertices[inst.mesh.vertex + prim.vertices[2].index];
        float u = hit.intersection.uv.x, v = hit.intersection.uv.y;
        vec3 world_position = ray.origin + ray.direction * hit.intersection.distance;
        vec4 clip = mul(view_proj, v4(world_position, 1.0f));
        float depth = clip.z / clip.w;
        // vertex stage: world_normal = mesh_normal_local_to_world(vertex.normal) (normalised per vertex), interpolated
        vec3 n0 = instance_normal_local_to_world(inst, ld3(a.normal));
        vec3 n1 = instance_normal_local_to_world(inst, ld3(b.normal));
        vec3 n2 = instance_normal_local_to_world(inst, ld3(d.normal));
        vec3 world_normal = n0 + u * (n1 - n0) + v * (n2 - n0);
        vec2 uv0 = v2(a.u, a.v), uv1 = v2(b.u, b.v), uv2 = v2(d.u, d.v);
        vec2 tex_uv = uv0 + u * (uv1 - uv0) + v * (uv2 - uv0);
        // dpdx / dpdy of clip_position.z: NDC depth is affine in screen space on a planar triangle
        const mat4 model = ldm(inst.model);
        vec3 P0 = xyz(mul(model, v4(ld3(prim.vertices[0].position), 1.0f)));
        vec3 P1 = xyz(mul(model, v4(ld3(prim.vertices[1].position), 1.0f)));
        vec3 P2 = xyz(mul(model, v4(ld3(prim.vertices[2].position), 1.0f)));
        vec3 Ng = cross(P1 - P0, P2 - P0);
        auto plane_depth = [&](float px, float py) {
            Ray r2 = primary_ray(c, px, py, jitter_ndc);
            float t = dot(P0 - r2.origin, Ng) / dot(r2.direction, Ng);
            vec4 cl = mul(view_proj, v4(r2.origin + r2.direction * t, 1.0f));
            return cl.z / cl.w;
        };
        vec2 grad = v2(plane_depth((float)x + 1.0f, (float)y) - depth, plane_depth((float)x, (float)y + 1.0f) - depth);
        // prepass.wgsl:52,99: previous_world_position = previous_mesh.model * vertex position, interpolated.  Here: the model
        // of the previous frame applied to the hit's object-space point when the instance moved, else the hit point itself.
        vec3 previous_world_position = world_position;
        if (!c.previous_models.empty()) {
            const float* pm = &c.previous_models[16 * (size_t)hit.instance_index];
            if (memcmp(pm, inst.model, 64) != 0) {
                vec3 p0 = ld3(prim.vertices[0].position), p1 = ld3(prim.vertices[1].position), p2 = ld3(prim.vertices[2].position);
                vec3 local_position = p0 + u * (p1 - p0) + v * (p2 - p0);
                previous_world_position = xyz(mul(ldm(pm), v4(local_position, 1.0f)));
            }
        }
        vec2 velocity = clip_to_uv(clip) - clip_to_uv(mul(prev_view_proj, v4(previous_world_position, 1.0f)));
        c.position[idx] = v4(world_position, depth);
        c.normal[idx] = pack4x8snorm(v4(world_normal, 1.0f));
        c.depth_gradient[idx] = grad;
        c.instance_material[idx] = v2((float)hit.instance_index + 0.5f, (float)inst.material + 0.5f);
        c.velocity_uv[idx] = v4(velocity.x, velocity.y, tex_uv.x, tex_uv.y);
    });
}

// ------------------------------------------------------------------------------ P1: full_screen_albedo
void pass_albedo(Ctx& c) {  // light.wgsl:1019-1042
    Deferred g(c);
    for_pixels(c, c.W, c.H, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        size_t idx = (size_t)y * c.W + x;
        vec4 position_depth = g.position(coords);
        vec4 position = v4(xyz(position_depth), 1.0f);
        float depth = position_depth.w;
        if (depth < F32_EPSILON) { c.albedo[idx] = pack_rgba16f(v4(0.0f)); return; }
        vec3 normal = xyz(g.normal(coords));
        vec2 im = g.instance_material(coords);
        vec4 velocity_uv = g.velocity_uv(coords);
        Surface surface = retreive_surface(c, f32_to_u32(im.y), v2(velocity_uv.z, velocity_uv.w));
        vec3 view_direction = calculate_view(c, position, is_orthographic(c));
        c.albedo[idx] = pack_rgba16f(v4(env_brdf(view_direction, normal, surface), 1.0f));
    });
}

// ------------------------------------------------------------------------------------- P2: direct_lit
struct PassBuffers {  // bind group 6 (light.rs:518-546) + bind group 5
    std::vector<hk_packed_reservoir>* previous_reservoir;           // binding 0
    std::vector<hk_packed_reservoir>* reservoir;                    // binding 1
    std::vector<hk_packed_reservoir>* previous_spatial_reservoir;   // binding 2
    std::vector<hk_packed_reservoir>* spatial_reservoir;            // binding 3
    std::vector<float>* variance;
    std::vector<uvec2>* render;
};
PassBuffers bind(Ctx& c, int signal) {
    static const int temporal[3] = {0, 2, 6}, spatial[3] = {4, 4, 8};
    int current = (int)(c.in.frame.number % 2u), previous = 1 - current;
    PassBuffers b;
    b.previous_reservoir = &c.reservoir[current + temporal[signal]];
    b.reservoir = &c.reservoir[previous + temporal[signal]];
    b.previous_spatial_reservoir = &c.reservoir[current + spatial[signal]];
    b.spatial_reservoir = &c.reservoir[previous + spatial[signal]];
    b.variance = &c.variance[signal];
    b.render = &c.render[signal];
    return b;
}
// deferred scatter log: writes to previous_spatial_reservoir applied in raster order of the writer
struct ScatterLog {
    std::vector<std::vector<ScatterWrite>> rows;
    explicit ScatterLog(int h) : rows(h) {}
    void push(int y, int32_t index, const hk_packed_reservoir& v) { rows[y].push_back({index, v}); }
    void apply(std::vector<hk_packed_reservoir>& buf) {
        // a previous uv of 1.0 in y, or in x on the last row, indexes past the buffer: WGSL's robust buffer access may discard the
        // store, as the kernels do
        for (auto& row : rows)
            for (auto& w : row)
                if (w.index >= 0 && (size_t)w.index < buf.size()) buf[w.index] = w.value;
    }
};

template <bool EMISSIVE_LIT, bool RENDER_EMISSIVE>
void pass_direct_lit(Ctx& c, int signal) {  // light.wgsl:1044-1261
    Deferred g(c);
    PassBuffers B = bind(c, signal);
    ScatterLog scatter(c.RH);
    const hk_frame_uniform& frame = c.in.frame;
    ivec2 render_size; render_size.x = c.RW; render_size.y = c.RH;
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        vec2 uv = coords_to_uv(coords, render_size);
        int32_t idx = coords.x + render_size.x * coords.y;
        Sample s;
        ivec2 deferred_coords = g.jittered_coords(uv);
        vec4 position_depth = g.position(deferred_coords);
        vec4 position = v4(xyz(position_depth), 1.0f);
        float depth = position_depth.w;
        if (depth < F32_EPSILON) {
            Reservoir r;
            set_reservoir(r, s, 0.0f);
            hk_packed_reservoir p = pack_reservoir(r);
            (*B.reservoir)[idx] = p;
            (*B.spatial_reservoir)[idx] = p;
            scatter.push(y, idx, p);
            (*B.variance)[idx] = 0.0f;
            (*B.render)[idx] = pack_rgba16f(v4(0.0f));
            return;
        }
        vec3 normal = xyz(g.normal(deferred_coords));
        vec2 imf = g.instance_material(deferred_coords);
        uint32_t instance_id = f32_to_u32(imf.x), material_id = f32_to_u32(imf.y);
        vec4 velocity_uv = g.velocity_uv(deferred_coords);

        s.random = noise_random(c, coords);
        s.visible_position = v4(xyz(position), depth);
        s.visible_normal = normal;
        s.visible_instance = instance_id;

        Ray ray; ray.origin = ray.direction = ray.inv_direction = v3(0.0f);
        Hit hit;
        HitInfo info;

        vec2 previous_uv = g.jittered_uv(uv, 0.25f) - v2(velocity_uv.x, velocity_uv.y);
        Reservoir r = load_previous(*B.previous_reservoir, previous_uv, render_size);
        if (!check_previous_reservoir(r, s) && uv_inside_eq(previous_uv))
            scatter.push(y, uv_to_index(previous_uv, render_size), pack_reservoir(r));

        const uint32_t validate_interval = EMISSIVE_LIT ? frame.emissive_validate_interval : frame.direct_validate_interval;
        const uint32_t select_light_instance = EMISSIVE_LIT ? instance_id : DONT_SAMPLE_EMISSIVE;

        if (frame.number % validate_interval != 0u || r.count < 4.0f) {
            LightCandidate candidate = select_light_candidate(c, s.random, xyz(s.visible_position), s.visible_normal,
                                                              select_light_instance, info);
            ray.origin = xyz(position) + normal * RAY_BIAS;
            ray.direction = candidate.direction;
            ray.inv_direction = 1.0f / ray.direction;
            bool trace_condition = dot(candidate.direction, normal) > 0.0f;
            trace_condition = trace_condition && candidate.p > 0.0f;
            if (EMISSIVE_LIT) trace_condition = trace_condition && candidate.emissive_instance != DONT_SAMPLE_EMISSIVE;
            if (trace_condition) {
                c.cnt().tlas += 1;
                hit = traverse_top(c, ray, candidate.max_distance, candidate.min_distance, candidate.emissive_instance);
                occlude_hit_info(ray, hit, info);
                if (EMISSIVE_LIT) s.radiance = input_radiance(c, ray, info, false, candidate.emissive_instance, false);
                else s.radiance = input_radiance(c, ray, info, true, DONT_SAMPLE_EMISSIVE, false);
            }
            s.sample_position = info.position;
            s.sample_normal = info.normal;
            float w_new = (candidate.p > 0.0f) ? luminance(xyz(s.radiance)) / candidate.p : 0.0f;
            temporal_restir(r, s, w_new, frame.max_temporal_reuse_count);
        }

        if (frame.number % validate_interval == 0u) {
            LightCandidate candidate = select_light_candidate(c, r.s.random, xyz(r.s.visible_position), r.s.visible_normal,
                                                              select_light_instance, info);
            ray.origin = xyz(s.visible_position) + s.visible_normal * RAY_BIAS;
            ray.direction = normalize(xyz(r.s.sample_position) - xyz(s.visible_position));
            ray.inv_direction = 1.0f / ray.direction;
            vec4 validate_radiance = v4(0.0f);
            bool trace_condition = dot(candidate.direction, r.s.visible_normal) > 0.0f;
            trace_condition = trace_condition && candidate.p > 0.0f;
            if (EMISSIVE_LIT) trace_condition = trace_condition && candidate.emissive_instance != DONT_SAMPLE_EMISSIVE;
            if (trace_condition) {
                c.cnt().tlas += 1;
                hit = traverse_top(c, ray, candidate.max_distance, candidate.min_distance, candidate.emissive_instance);
                occlude_hit_info(ray, hit, info);
                if (EMISSIVE_LIT) validate_radiance = input_radiance(c, ray, info, false, candidate.emissive_instance, false);
                else validate_radiance = input_radiance(c, ray, info, true, DONT_SAMPLE_EMISSIVE, false);
            }
            if (r.count >= 4.0f) {
                s.random = r.s.random;
                s.sample_position = info.position;
                s.sample_normal = info.normal;
                s.radiance = validate_radiance;
            }
            float luminance_ratio = luminance(xyz(validate_radiance)) / fmax_(luminance(xyz(r.s.radiance)), 0.0001f);
            if (luminance_ratio > 1.25f || luminance_ratio < 0.8f) {
                if (uv_inside_eq(previous_uv)) scatter.push(y, uv_to_index(previous_uv, render_size), pack_reservoir(r));
                float w_new = (candidate.p > 0.0f) ? luminance(xyz(s.radiance)) / candidate.p : 0.0f;
                set_reservoir(r, s, w_new);
            }
        }

        float total_lum = r.count * luminance(xyz(r.s.radiance));
        r.w = (total_lum > 0.0f) ? r.w_sum / total_lum : 0.0f;
        r.s.visible_position = s.visible_position;
        r.s.visible_normal = s.visible_normal;
        r.lifetime += 1.0f;
        (*B.variance)[idx] = variance_of(r);
        if (frame.temporal_reuse > 0u) (*B.reservoir)[idx] = pack_reservoir(r);

        Surface surface = retreive_surface(c, material_id, v2(velocity_uv.z, velocity_uv.w));
        vec3 view_direction = calculate_view(c, position, is_orthographic(c));
        vec3 out_radiance = shading(c, view_direction, r.s.visible_normal,
                                    normalize(xyz(r.s.sample_position) - xyz(r.s.visible_position)), surface, r.s.radiance);
        out_radiance = out_radiance * r.w;
        vec3 out_color = RENDER_EMISSIVE ? out_radiance + compute_emissive_radiance(surface.emissive) : out_radiance;
        (*B.render)[idx] = pack_rgba16f(v4(out_color, 1.0f));
    });
    scatter.apply(*B.previous_spatial_reservoir);
}

// ----------------------------------------------------------------------------- P3: indirect_lit_ambient
template <bool MULTIPLE_BOUNCES>
void pass_indirect(Ctx& c) {  // light.wgsl:1263-1498
    Deferred g(c);
    PassBuffers B = bind(c, 2);
    ScatterLog scatter(c.RH);
    const hk_frame_uniform& frame = c.in.frame;
    ivec2 render_size; render_size.x = c.RW; render_size.y = c.RH;
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        vec2 uv = coords_to_uv(coords, render_size);
        int32_t idx = coords.x + render_size.x * coords.y;
        ivec2 deferred_coords = g.jittered_coords(uv);
        vec4 position_depth = g.position(deferred_coords);
        vec4 position = v4(xyz(position_depth), 1.0f);
        float depth = position_depth.w;
        Sample s;
        Reservoir r;
        if (frame.indirect_bounces == 0u || depth < F32_EPSILON) {
            hk_packed_reservoir p = pack_reservoir(r);
            (*B.reservoir)[idx] = p;
            (*B.spatial_reservoir)[idx] = p;
            scatter.push(y, idx, p);
            (*B.variance)[idx] = 0.0f;
            (*B.render)[idx] = pack_rgba16f(v4(0.0f));
            return;
        }
        vec3 normal = normalize(xyz(g.normal(deferred_coords)));
        vec2 imf = g.instance_material(deferred_coords);
        uint32_t instance_id = f32_to_u32(imf.x), material_id = f32_to_u32(imf.y);
        vec4 velocity_uv = g.velocity_uv(deferred_coords);

        s.random = noise_random(c, coords);
        s.visible_position = v4(xyz(position), depth);
        s.visible_normal = normal;
        s.visible_instance = instance_id;

        Ray ray;
        Hit hit;
        HitInfo info;
        float pdf = 0.0f;
        Surface surface;

        if (MULTIPLE_BOUNCES) {
            Sample bounce_sample = s;
            vec3 color_transport = v3(1.0f);
            for (uint32_t n = 0u; n < frame.indirect_bounces &&
                                  (color_transport.x > 0.01f || color_transport.y > 0.01f || color_transport.z > 0.01f); n += 1u) {
                vec4 rand_sample = sample_cosine_hemisphere(v2(bounce_sample.random.x, bounce_sample.random.y));
                ray.origin = xyz(bounce_sample.visible_position) + bounce_sample.visible_normal * RAY_BIAS;
                ray.direction = mul(normal_basis(bounce_sample.visible_normal), xyz(rand_sample));
                ray.inv_direction = 1.0f / ray.direction;
                c.cnt().tlas += 1;
                hit = traverse_top(c, ray, F32_MAX, 0.0f, DONT_EXCLUDE);
                info = hit_info(c, ray, hit);
                if (n == 0u) {
                    s.sample_position = info.position;
                    s.sample_normal = info.normal;
                    pdf = rand_sample.w;
                }
                bounce_sample.sample_position = info.position;
                bounce_sample.sample_normal = info.normal;
                if (hit.instance_index != U32_MAX) {
                    vec3 out_radiance = v3(0.0f);
                    surface = retreive_surface(c, info.material_index, info.uv);
                    surface.roughness = 1.0f;
                    LightCandidate candidate = select_light_candidate(c, bounce_sample.random, xyz(bounce_sample.sample_position),
                                                                      bounce_sample.sample_normal, info.instance_index, info);
                    bool sample_directional = (candidate.emissive_instance == DONT_SAMPLE_EMISSIVE);
                    vec3 bounce_view_direction = normalize(xyz(bounce_sample.visible_position) - xyz(bounce_sample.sample_position));
                    if (dot(candidate.direction, bounce_sample.sample_normal) > 0.0f && candidate.p > 0.0f) {
                        ray.origin = xyz(bounce_sample.sample_position) + bounce_sample.sample_normal * RAY_BIAS;
                        ray.direction = candidate.direction;
                        ray.inv_direction = 1.0f / ray.direction;
                        c.cnt().tlas += 1;
                        hit = traverse_top(c, ray, candidate.max_distance, candidate.min_distance, candidate.emissive_instance);
                        occlude_hit_info(ray, hit, info);
                        vec4 in_radiance = input_radiance(c, ray, info, sample_directional, candidate.emissive_instance, false);
                        out_radiance = shading(c, bounce_view_direction, bounce_sample.sample_normal, ray.direction, surface, in_radiance);
                        out_radiance = out_radiance / candidate.p;
                        if (n > 0u) out_radiance = (rand_sample.w < 0.01f) ? v3(0.0f) : out_radiance / rand_sample.w;
                        float out_luminance = luminance(out_radiance);
                        if (out_luminance > frame.max_indirect_luminance)
                            out_radiance = out_radiance * frame.max_indirect_luminance / out_luminance;
                        s.radiance = s.radiance + v4(color_transport * out_radiance, 1.0f);
                    }
                    color_transport = color_transport * env_brdf(bounce_view_direction, bounce_sample.sample_normal, surface);
                    bounce_sample.random = fract(bounce_sample.random + (float)frame.number * GOLDEN_RATIO);
                    bounce_sample.visible_position = bounce_sample.sample_position;
                    bounce_sample.visible_normal = bounce_sample.sample_normal;
                } else {
                    vec3 out_radiance = xyz(input_radiance(c, ray, info, false, DONT_SAMPLE_EMISSIVE, true));
                    s.radiance = s.radiance + v4(color_transport * out_radiance, 0.0f);
                    break;
                }
            }
        } else {
            vec4 rand_sample = sample_cosine_hemisphere(v2(s.random.x, s.random.y));
            ray.origin = xyz(s.visible_position) + s.visible_normal * RAY_BIAS;
            ray.direction = mul(normal_basis(s.visible_normal), xyz(rand_sample));
            ray.inv_direction = 1.0f / ray.direction;
            c.cnt().tlas += 1;
            hit = traverse_top(c, ray, F32_MAX, 0.0f, DONT_EXCLUDE);
            info = hit_info(c, ray, hit);
            s.sample_position = info.position;
            s.sample_normal = info.normal;
            pdf = rand_sample.w;
            if (hit.instance_index != U32_MAX) {
                vec3 out_radiance = v3(0.0f);
                surface = retreive_surface(c, info.material_index, info.uv);
                surface.roughness = 1.0f;
                LightCandidate candidate = select_light_candidate(c, s.random, xyz(s.sample_position), s.sample_normal,
                                                                  info.instance_index, info);
                bool sample_directional = (candidate.emissive_instance == DONT_SAMPLE_EMISSIVE);
                if (dot(candidate.direction, s.sample_normal) > 0.0f && candidate.p > 0.0f) {
                    ray.origin = xyz(s.sample_position) + s.sample_normal * RAY_BIAS;
                    ray.direction = candidate.direction;
                    ray.inv_direction = 1.0f / ray.direction;
                    c.cnt().tlas += 1;
                    hit = traverse_top(c, ray, candidate.max_distance, candidate.min_distance, candidate.emissive_instance);
                    occlude_hit_info(ray, hit, info);
                    vec4 in_radiance = input_radiance(c, ray, info, sample_directional, candidate.emissive_instance, false);
                    out_radiance = shading(c, normalize(xyz(s.visible_position) - xyz(s.sample_position)), s.sample_normal,
                                           ray.direction, surface, in_radiance);
                    out_radiance = out_radiance / candidate.p;
                    s.radiance = s.radiance + v4(out_radiance, 1.0f);
                }
            } else {
                vec3 out_radiance = xyz(input_radiance(c, ray, info, false, DONT_SAMPLE_EMISSIVE, true));
                s.radiance = s.radiance + v4(out_radiance, 0.0f);
            }
        }

        // ReSTIR: temporal
        vec2 previous_uv = g.jittered_uv(uv, 0.25f) - v2(velocity_uv.x, velocity_uv.y);
        r = load_previous(*B.previous_reservoir, previous_uv, render_size);
        if (!check_previous_reservoir(r, s) && uv_inside_eq(previous_uv))
            scatter.push(y, uv_to_index(previous_uv, render_size), pack_reservoir(r));

        surface = retreive_surface(c, material_id, v2(velocity_uv.z, velocity_uv.w));
        vec3 view_direction = calculate_view(c, position, is_orthographic(c));
        vec3 sample_radiance = shading(c, view_direction, s.visible_normal,
                                       normalize(xyz(s.sample_position) - xyz(s.visible_position)), surface, s.radiance);
        float w_new = (pdf > 0.0f) ? luminance(sample_radiance) / pdf : 0.0f;
        temporal_restir(r, s, w_new, frame.max_temporal_reuse_count);

        vec3 out_radiance = shading(c, view_direction, r.s.visible_normal,
                                    normalize(xyz(r.s.sample_position) - xyz(r.s.visible_position)), surface, r.s.radiance);
        float total_lum = r.count * luminance(out_radiance);
        r.w = (total_lum > 0.0f) ? r.w_sum / total_lum : 0.0f;
        r.s.visible_position = s.visible_position;
        r.s.visible_normal = s.visible_normal;
        r.lifetime += 1.0f;
        (*B.variance)[idx] = variance_of(r);
        if (frame.temporal_reuse > 0u) (*B.reservoir)[idx] = pack_reservoir(r);
        (*B.render)[idx] = pack_rgba16f(v4(out_radiance * r.w, 1.0f));
    });
    scatter.apply(*B.previous_spatial_reservoir);
}

// ----------------------------------------------------------------------------------- P4: spatial_reuse
// Neighbour i of the pixel at `coords` (light.wgsl:1566-1575): its offset, its radius and its pixel
inline ivec2 spatial_neighbour(ivec2 coords, uint32_t i, uint32_t count, float range, float rotation, float random_frame,
                               float& rad, vec2& offset) {
    float ang = TAU * fract((float)i * GOLDEN_RATIO + rotation + random_frame);
    rad = sqrtf((float)i / (float)count) * range;
    float sn, cs; sincos_(ang, &sn, &cs);
    offset = rad * v2(cs, sn);
    ivec2 sample_coords;
    sample_coords.x = f32_to_i32(offset.x + (float)coords.x);
    sample_coords.y = f32_to_i32(offset.y + (float)coords.y);
    return sample_coords;
}
// uv of the depth-march tap at distance tap_dist towards that neighbour (light.wgsl:1617-1619)
inline vec2 spatial_tap_uv(vec2 uv, vec2 offset, float tap_dist, ivec2 render_size) {
    vec2 tap_offset = tap_dist * normalize(offset);
    return uv + tap_offset / v2((float)render_size.x, (float)render_size.y);
}

template <bool EMISSIVE_LIT, bool RENDER_EMISSIVE>
void pass_spatial_reuse(Ctx& c, int signal) {  // light.wgsl:1500-1684
    Deferred g(c);
    PassBuffers B = bind(c, signal);
    const hk_frame_uniform& frame = c.in.frame;
    const uint32_t SPATIAL_REUSE_COUNT = EMISSIVE_LIT ? 8u : 16u;       // light.wgsl:246-252
    const float SPATIAL_REUSE_RANGE = EMISSIVE_LIT ? 10.0f : 20.0f;
    const uint32_t SPATIAL_REUSE_TAPS = 4u;
    ivec2 render_size; render_size.x = c.RW; render_size.y = c.RH;
    // The 8x8 workgroup cache (light.wgsl:1500-1501,1584-1591) holds unpack(reservoir_buffer[..]) of the same dispatch's
    // inputs, so reading the buffer directly is value-identical; the oracle reads the buffer.
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        vec2 uv = coords_to_uv(coords, render_size);
        int32_t idx = coords.x + render_size.x * coords.y;
        ivec2 deferred_coords = g.jittered_coords(uv);
        vec4 position_depth = g.position(deferred_coords);
        vec4 position = v4(xyz(position_depth), 1.0f);
        float depth = position_depth.w;
        Reservoir r = unpack_reservoir((*B.reservoir)[idx]);
        if (depth < F32_EPSILON) {
            (*B.spatial_reservoir)[idx] = pack_reservoir(r);
            (*B.render)[idx] = pack_rgba16f(v4(0.0f));
            return;
        }
        vec2 imf = g.instance_material(deferred_coords);
        uint32_t material_id = f32_to_u32(imf.y);
        vec4 velocity_uv = g.velocity_uv(deferred_coords);
        Surface surface = retreive_surface(c, material_id, v2(velocity_uv.z, velocity_uv.w));
        bool use_spatial_variance = r.count <= 4.0f;
        vec2 previous_uv = g.jittered_uv(uv, 0.25f) - v2(velocity_uv.x, velocity_uv.y);
        Reservoir q = r;
        const Sample s = q.s;
        if (r.lifetime <= reservoir_lifetime(c)) r = load_previous(*B.previous_spatial_reservoir, previous_uv, render_size);
        vec3 view_direction = calculate_view(c, position, is_orthographic(c));
        if (EMISSIVE_LIT) {
            merge_reservoir(r, q, luminance(xyz(q.s.radiance)));
        } else {
            vec3 out_radiance = shading(c, view_direction, s.visible_normal,
                                        normalize(xyz(s.sample_position) - xyz(s.visible_position)), surface, s.radiance);
            merge_reservoir(r, q, luminance(out_radiance));
        }
        r.s.visible_position = s.visible_position;
        r.s.visible_normal = s.visible_normal;

        for (uint32_t i = 1u; i <= SPATIAL_REUSE_COUNT; i += 1u) {
            float rad;
            vec2 offset;
            ivec2 sample_coords = spatial_neighbour(coords, i, SPATIAL_REUSE_COUNT, SPATIAL_REUSE_RANGE, sum4(s.random),
                                                    random_float(frame.number), rad, offset);
            vec2 sample_uv = coords_to_uv(sample_coords, render_size);
            ivec2 sample_deferred_coords = g.jittered_coords(sample_uv);
            if (sample_uv.x < 0.0f || sample_uv.y < 0.0f || sample_uv.x > 1.0f || sample_uv.y > 1.0f) continue;

            float sample_depth = g.position(sample_deferred_coords).w;
            q = unpack_reservoir((*B.reservoir)[sample_coords.x + render_size.x * sample_coords.y]);

            float depth_ratio = depth / sample_depth;
            if (depth_ratio < 0.9f || depth_ratio > 1.1f) continue;
            bool normal_miss = dot(s.visible_normal, q.s.visible_normal) < 0.866f;
            if (q.count < F32_EPSILON || normal_miss) continue;
            vec3 sample_direction = normalize(xyz(q.s.sample_position) - xyz(s.visible_position));
            if (dot(sample_direction, s.visible_normal) < 0.0f) continue;

            float tap_interval = fmax_(1.0f, rad / (float)(SPATIAL_REUSE_TAPS + 1u));
            uint32_t tap_count = f32_to_u32(rad / tap_interval);
            bool occluded = false;
            for (uint32_t j = 1u; j <= tap_count; j += 1u) {
                ivec2 tap_deferred_coords = g.jittered_coords(spatial_tap_uv(uv, offset, (float)j * tap_interval, render_size));
                float tap_depth = g.position(tap_deferred_coords).w;
                float ref_depth = mixf(depth, sample_depth, (float)j / (float)(tap_count + 1u));
                if (tap_depth > ref_depth + 0.00001f) { occluded = true; break; }
            }
            if (occluded) continue;

            float jacobian = (q.s.sample_position.w > 0.5f) ? compute_jacobian(q.s, s) : 1.0f;
            if (EMISSIVE_LIT) {
                merge_reservoir(r, q, luminance(xyz(q.s.radiance)) / jacobian);
            } else {
                vec3 out_radiance = shading(c, view_direction, s.visible_normal, sample_direction, surface, q.s.radiance);
                merge_reservoir(r, q, luminance(out_radiance) / jacobian);
            }
        }

        float m = (float)frame.max_spatial_reuse_count;
        if (r.count > m) {
            r.w_sum *= m / r.count;
            r.w2_sum *= m / r.count;
            r.count = m;
        }
        vec3 out_radiance = shading(c, view_direction, s.visible_normal,
                                    normalize(xyz(r.s.sample_position) - xyz(s.visible_position)), surface, r.s.radiance);
        float total_lum = EMISSIVE_LIT ? r.count * luminance(xyz(r.s.radiance)) : r.count * luminance(out_radiance);
        r.w = (total_lum > 0.0f) ? r.w_sum / total_lum : 0.0f;
        r.lifetime += 1.0f;
        (*B.spatial_reservoir)[idx] = pack_reservoir(r);
        if (use_spatial_variance) (*B.variance)[idx] = variance_of(r);
        vec3 out_color = RENDER_EMISSIVE ? r.w * out_radiance + compute_emissive_radiance(surface.emissive) : r.w * out_radiance;
        (*B.render)[idx] = pack_rgba16f(v4(out_color, 1.0f));
    });
}

// ------------------------------------------------------------------------------------------ P5/P6: denoise
inline vec4 tex16(const std::vector<uvec2>& t, int w, int h, ivec2 p) {  // textureLoad on a storage texture
    if (p.x < 0 || p.y < 0 || p.x >= w || p.y >= h) return v4(0.0f);
    return unpack_rgba16f(t[(size_t)p.y * w + p.x]);
}
inline float kernel_at(const hk_frame_uniform& f, int col, int row) { return f.kernel[col][row]; }  // frame.kernel[a][b]

void pass_demodulation(Ctx& c, int signal) {  // denoise.wgsl:135-162
    Deferred g(c);
    const hk_frame_uniform& frame = c.in.frame;
    ivec2 output_size; output_size.x = c.RW; output_size.y = c.RH;
    ivec2 input_size = output_size;
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        size_t idx = (size_t)y * c.RW + x;
        vec2 uv = coords_to_uv(coords, output_size);
        vec2 deferred_uv = g.jittered_uv(uv, 0.5f);
        ivec2 ap = g.nearest(deferred_uv);
        vec3 albedo = xyz(unpack_rgba16f(c.albedo[(size_t)ap.y * c.W + ap.x]));
        ivec2 rp; rp.x = std::min(std::max((int)floorf(uv.x * (float)c.RW), 0), c.RW - 1);
        rp.y = std::min(std::max((int)floorf(uv.y * (float)c.RH), 0), c.RH - 1);
        vec3 irradiance = xyz(unpack_rgba16f(c.render[signal][(size_t)rp.y * c.RW + rp.x]));
        vec3 q = irradiance / albedo;
        irradiance = v3(albedo.x < 0.01f ? 0.0f : q.x, albedo.y < 0.01f ? 0.0f : q.y, albedo.z < 0.01f ? 0.0f : q.z);
        c.denoise_internal[0][idx] = pack_rgba16f(v4(irradiance, 1.0f));

        float sum_variance = 0.0f;
        auto accumulate_variance = [&](int ox, int oy) {  // denoise.wgsl:116-133
            vec2 sample_uv = uv + v2((float)ox, (float)oy) / v2((float)input_size.x, (float)input_size.y);
            if (sample_uv.x < 0.0f || sample_uv.y < 0.0f || sample_uv.x > 1.0f || sample_uv.y > 1.0f) return;
            ivec2 p; p.x = std::min(std::max((int)floorf(sample_uv.x * (float)c.RW), 0), c.RW - 1);
            p.y = std::min(std::max((int)floorf(sample_uv.y * (float)c.RH), 0), c.RH - 1);
            float variance = c.variance[signal][(size_t)p.y * c.RW + p.x];
            if (variance > F32_MAX) return;
            sum_variance += kernel_at(frame, oy + 1, ox + 1) * fmax_(variance, 0.0f);
        };
        accumulate_variance(-1, -1); accumulate_variance(-1, 0); accumulate_variance(-1, 1);
        accumulate_variance(0, -1);  accumulate_variance(0, 0);  accumulate_variance(0, 1);
        accumulate_variance(1, -1);  accumulate_variance(1, 0);  accumulate_variance(1, 1);
        c.denoise_internal_variance[idx] = sum_variance;
    });
}

template <int LEVEL, bool FIREFLY_FILTERING>
void pass_denoise(Ctx& c, int signal) {  // denoise.wgsl:164-319
    Deferred g(c);
    const hk_frame_uniform& frame = c.in.frame;
    const int step_size = 8 >> LEVEL;  // denoise.wgsl:101-114
    const std::vector<uvec2>& input = c.denoise_internal[LEVEL];
    std::vector<uvec2>& output = (LEVEL == 3) ? c.denoise_render[signal] : c.denoise_internal[LEVEL + 1];
    ivec2 output_size; output_size.x = c.RW; output_size.y = c.RH;
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        size_t idx = (size_t)y * c.RW + x;
        vec2 uv = coords_to_uv(coords, output_size);
        vec2 deferred_uv = g.jittered_uv(uv, 0.5f);
        ivec2 dp = g.nearest(deferred_uv);
        float depth = g.position(dp).w;
        vec2 depth_gradient = g.depth_gradient(dp);
        vec3 normal = normalize(xyz(g.normal(dp)));
        float instance = g.instance_material(dp).x;
        if (depth < F32_EPSILON) { output[idx] = pack_rgba16f(v4(0.0f)); return; }

        float variance = c.denoise_internal_variance[idx];
        vec3 irradiance = xyz(tex16(input, c.RW, c.RH, coords));
        vec3 sum_irradiance = irradiance * kernel_at(frame, 1, 1);
        float sum_w = kernel_at(frame, 1, 1);
        auto bad = [](vec3 v) { return is_nan(v.x) || is_nan(v.y) || is_nan(v.z) || v.x > F32_MAX || v.y > F32_MAX || v.z > F32_MAX; };
        if (bad(irradiance)) { irradiance = v3(0.0f); sum_irradiance = v3(0.0f); sum_w = 0.0f; }
        float lum = luminance(irradiance);
        float ff_moment_1 = 0.0f, ff_moment_2 = 0.0f, ff_count = 0.0f;

        auto accumulate_irradiance = [&](int ox, int oy) {  // denoise.wgsl:164-213
            ivec2 sample_coords; sample_coords.x = coords.x + ox * step_size; sample_coords.y = coords.y + oy * step_size;
            vec2 sample_uv = coords_to_uv(sample_coords, output_size);
            vec2 sample_deferred_uv = g.jittered_uv(sample_uv, 0.5f);
            if (sample_uv.x < 0.0f || sample_uv.y < 0.0f || sample_uv.x > 1.0f || sample_uv.y > 1.0f) return;
            vec3 irr = xyz(tex16(input, c.RW, c.RH, sample_coords));
            if (bad(irr)) return;
            ivec2 sp = g.nearest(sample_deferred_uv);
            vec3 sample_normal = normalize(xyz(g.normal(sp)));
            float sample_depth = g.position(sp).w;
            float sample_instance = g.instance_material(sp).x;
            float sample_luminance = luminance(irr);
            float w_normal = pow16(fmax_(0.0f, dot(normal, sample_normal)));                                    // :44-47
            float w_depth = exp_((-fabsf(depth - sample_depth)) /
                                 (fabsf(dot(depth_gradient, v2((float)ox, (float)oy))) + 0.01f));               // :50-53
            float w_instance = fmax_(0.0f, 1.0f - fabsf(instance - sample_instance));                           // :63-65
            float w_luminance = exp_((-fabsf(lum - sample_luminance)) / (4.0f * pow025(variance) + 0.001f));    // :56-61
            float w = clampf(w_normal * w_depth * w_instance * w_luminance, 0.0f, 1.0f) * kernel_at(frame, oy + 1, ox + 1);
            sum_irradiance = sum_irradiance + irr * w;
            sum_w += w;
            if (FIREFLY_FILTERING) {
                ff_moment_1 += sample_luminance;
                ff_moment_2 += sample_luminance * sample_luminance;
                ff_count += 1.0f;
            }
        };
        accumulate_irradiance(-1, -1); accumulate_irradiance(0, -1); accumulate_irradiance(1, -1);
        accumulate_irradiance(-1, 0);  accumulate_irradiance(1, 0);
        accumulate_irradiance(-1, 1);  accumulate_irradiance(0, 1);  accumulate_irradiance(1, 1);

        irradiance = (sum_w < 0.0001f) ? v3(0.0f) : sum_irradiance / sum_w;
        if (FIREFLY_FILTERING) {
            float ff_mean = ff_moment_1 / ff_count;
            float ff_var = ff_moment_2 / ff_count - ff_mean * ff_mean;
            if (lum > ff_mean + 3.0f * sqrtf(ff_var)) irradiance = ff_mean / lum * irradiance;
        }
        vec4 color = v4(irradiance, 1.0f);
        if (LEVEL == 3) {
            ivec2 ap = g.nearest(deferred_uv);
            vec4 albedo = unpack_rgba16f(c.albedo[(size_t)ap.y * c.W + ap.x]);
            color = color * albedo;
        }
        output[idx] = pack_rgba16f(color);
    });
}

void pass_tone_mapping(Ctx& c) {  // tone_mapping.wgsl:21-32 ; inputs per post_process.rs:940-954
    const bool dn = c.in.denoise != 0;
    const std::vector<uvec2>& direct = dn ? c.denoise_render[0] : c.render[0];
    const std::vector<uvec2>& emissive = dn ? c.denoise_render[1] : c.render[1];
    const std::vector<uvec2>* indirect = dn ? &c.denoise_render[2] : &c.render[2];
    const bool no_indirect = c.in.frame.indirect_bounces == 0;  // fallback 1x1 texture: only texel (0,0) is in bounds
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        size_t idx = (size_t)y * c.RW + x;
        vec4 color = unpack_rgba16f(direct[idx]);
        color = color + unpack_rgba16f(emissive[idx]);
        if (!no_indirect) color = color + unpack_rgba16f((*indirect)[idx]);
        vec3 rgb = reinhard_luminance(vmax(xyz(color), 0.0039f));
        color = v4(rgb, color.w);
        if (!(color.w > 0.0f)) color = ld4(c.in.frame.clear_color);
        c.tone_mapping_output[c.in.frame.number % 2u][idx] = pack_rgba16f(color);
    });
}


// ----------------------------------------------------------------------------- K11/K12: SMAA TU4x and TAA
// Texture addressing used by smaa.wgsl / taa.wgsl, both samplers clamp-to-edge (post_process.rs:697-708):
//   nearest: texel floor(uv * size);  linear: bilinear around uv * size - 0.5 with fp32 weights;
//   textureGather: the 2x2 bilinear footprint as (x: (i0,j1), y: (i1,j1), z: (i1,j0), w: (i0,j0)).
struct Image16 {   // an Rgba16Float texture
    const std::vector<uvec2>* t; int w, h;
    vec4 texel(int x, int y) const {
        x = std::min(std::max(x, 0), w - 1); y = std::min(std::max(y, 0), h - 1);
        return unpack_rgba16f((*t)[(size_t)y * w + x]);
    }
    vec4 load(ivec2 p) const { return (p.x < 0 || p.y < 0 || p.x >= w || p.y >= h) ? v4(0.0f) : unpack_rgba16f((*t)[(size_t)p.y * w + p.x]); }
    vec4 nearest(vec2 uv) const { return texel((int)floorf(uv.x * (float)w), (int)floorf(uv.y * (float)h)); }
    vec4 linear(vec2 uv) const {
        float fx = uv.x * (float)w - 0.5f, fy = uv.y * (float)h - 0.5f;
        float x0 = floorf(fx), y0 = floorf(fy), ax = fx - x0, ay = fy - y0;
        vec4 t00 = texel((int)x0, (int)y0), t10 = texel((int)x0 + 1, (int)y0), t01 = texel((int)x0, (int)y0 + 1), t11 = texel((int)x0 + 1, (int)y0 + 1);
        vec4 top = t00 * (1.0f - ax) + t10 * ax, bot = t01 * (1.0f - ax) + t11 * ax;
        return top * (1.0f - ay) + bot * ay;
    }
    void gather(vec2 uv, vec4 out[4]) const {   // out[k] = texel k of the footprint in gather order
        float fx = uv.x * (float)w - 0.5f, fy = uv.y * (float)h - 0.5f;
        int i0 = (int)floorf(fx), j0 = (int)floorf(fy);
        out[0] = texel(i0, j0 + 1); out[1] = texel(i0 + 1, j0 + 1); out[2] = texel(i0 + 1, j0); out[3] = texel(i0, j0);
    }
};
struct Image32 {   // an Rgba32Float texture (position / velocity_uv planes)
    const std::vector<vec4>* t; int w, h;
    vec4 texel(int x, int y) const {
        x = std::min(std::max(x, 0), w - 1); y = std::min(std::max(y, 0), h - 1);
        return (*t)[(size_t)y * w + x];
    }
    vec4 nearest(vec2 uv) const { return texel((int)floorf(uv.x * (float)w), (int)floorf(uv.y * (float)h)); }
    vec4 gather_w(vec2 uv) const {
        float fx = uv.x * (float)w - 0.5f, fy = uv.y * (float)h - 0.5f;
        int i0 = (int)floorf(fx), j0 = (int)floorf(fy);
        return v4(texel(i0, j0 + 1).w, texel(i0 + 1, j0 + 1).w, texel(i0 + 1, j0).w, texel(i0, j0).w);
    }
};
inline vec3 RGB_to_YCoCg(vec3 rgb) {  // smaa.wgsl:23-28
    float y = (rgb.x / 4.0f) + (rgb.y / 2.0f) + (rgb.z / 4.0f);
    float co = (rgb.x / 2.0f) - (rgb.z / 2.0f);
    float cg = (-rgb.x / 4.0f) + (rgb.y / 2.0f) - (rgb.z / 4.0f);
    return v3(y, co, cg);
}
inline vec3 clamp01(vec3 v) { return v3(clampf(v.x, 0.0f, 1.0f), clampf(v.y, 0.0f, 1.0f), clampf(v.z, 0.0f, 1.0f)); }
inline vec3 YCoCg_to_RGB(vec3 c) {  // smaa.wgsl:30-35
    return clamp01(v3(c.x + c.y - c.z, c.x + c.z, c.x - c.y - c.z));
}
inline vec3 vabs(vec3 a) { return v3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }
inline vec3 vsqrt(vec3 a) { return v3(sqrtf(a.x), sqrtf(a.y), sqrtf(a.z)); }
inline vec3 clip_towards_aabb_center(vec3 previous_color, vec3 current_color, vec3 aabb_min, vec3 aabb_max) {  // smaa.wgsl:37-45
    (void)current_color;
    vec3 p_clip = 0.5f * (aabb_max + aabb_min);
    vec3 e_clip = 0.5f * (aabb_max - aabb_min);
    vec3 v_clip = previous_color - p_clip;
    vec3 v_unit = v_clip / e_clip;
    vec3 a_unit = vabs(v_unit);
    float ma_unit = fmax_(a_unit.x, fmax_(a_unit.y, a_unit.z));
    return (ma_unit > 1.0f) ? p_clip + v_clip / ma_unit : previous_color;
}
// smaa.wgsl:52-72 / taa.wgsl:57-77; `texel_size` differs between the two callers
vec2 nearest_velocity(const Image32& position, const Image32& velocity_uv, vec2 uv, vec2 texel_size) {
    vec4 depths;
    depths.x = position.nearest(uv + v2(texel_size.x, texel_size.y)).w;
    depths.y = position.nearest(uv + v2(-texel_size.x, texel_size.y)).w;
    depths.z = position.nearest(uv + v2(texel_size.x, -texel_size.y)).w;
    depths.w = position.nearest(uv + v2(-texel_size.x, -texel_size.y)).w;
    float max_depth = fmax_(fmax_(depths.x, depths.y), fmax_(depths.z, depths.w));
    float depth = position.nearest(uv).w;
    vec2 offset = v2(0.0f, 0.0f);
    if (depth < max_depth) {
        vec4 sx = v4(depths.x == max_depth ? 1.0f : 0.0f, depths.y == max_depth ? -1.0f : 0.0f, depths.z == max_depth ? 1.0f : 0.0f,
                     depths.w == max_depth ? -1.0f : 0.0f);
        vec4 sy = v4(depths.x == max_depth ? 1.0f : 0.0f, depths.y == max_depth ? 1.0f : 0.0f, depths.z == max_depth ? -1.0f : 0.0f,
                     depths.w == max_depth ? -1.0f : 0.0f);
        offset = v2(dot(v4(texel_size.x), sx), dot(v4(texel_size.y), sy));
    }
    vec4 v = velocity_uv.nearest(uv + offset);
    return v2(v.x, v.y);
}
inline float distance4(vec4 a, vec4 b) { vec4 d = a - b; return sqrtf(dot(d, d)); }
inline float distance2(vec2 a, vec2 b) { vec2 d = a - b; return sqrtf(dot(d, d)); }
inline bool any_lt(vec4 a, float t) { return a.x < t || a.y < t || a.z < t || a.w < t; }

void pass_smaa_tu4x(Ctx& c) {  // smaa.wgsl:81-199
    const uint32_t cur = c.in.frame.number % 2u, prev = 1u - cur;
    Image16 render{&c.tone_mapping_output[cur], c.RW, c.RH}, previous_render{&c.tone_mapping_output[prev], c.RW, c.RH};
    Image32 position{&c.position, c.W, c.H}, previous_position{&c.previous_position, c.W, c.H};
    Image32 velocity_uv{&c.velocity_uv, c.W, c.H}, previous_velocity_uv{&c.previous_velocity_uv, c.W, c.H};
    const int OW = c.OW, OH = c.OH;                                          // textureDimensions(output_texture)
    ivec2 input_size; input_size.x = c.RW; input_size.y = c.RH;
    ivec2 output_size; output_size.x = OW; output_size.y = OH;
    const int current_jitter = ((c.in.frame.number & 1u) == 0u) ? 0 : 1;     // current_smaa_jitter :74-76
    const int previous_jitter = ((c.in.frame.number & 1u) == 0u) ? 1 : 0;    // previous_smaa_jitter :78-80
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        vec2 uv = coords_to_uv(coords, input_size);
        vec2 texel_size = v2(1.0f, 1.0f) / v2((float)OW, (float)OH);
        vec2 uv_biases[5] = {v2(0.0f, 0.0f), v2(2.5f, 2.5f) * texel_size, v2(-2.5f, 2.5f) * texel_size, v2(2.5f, -2.5f) * texel_size,
                             v2(-2.5f, -2.5f) * texel_size};
        ivec2 current_output_coords; current_output_coords.x = 2 * x + current_jitter; current_output_coords.y = 2 * y + current_jitter;
        vec3 current_color = xyz(render.nearest(uv));
        ivec2 previous_output_coords; previous_output_coords.x = 2 * x + previous_jitter; previous_output_coords.y = 2 * y + previous_jitter;
        vec2 previous_output_uv = coords_to_uv(previous_output_coords, output_size);
        vec2 deferred_texel = v2(1.0f, 1.0f) / v2((float)c.W, (float)c.H);
        vec2 velocity = nearest_velocity(position, velocity_uv, previous_output_uv, deferred_texel);
        vec2 previous_reprojected_uv = previous_output_uv - velocity;
        vec3 previous_color = xyz(previous_render.nearest(previous_reprojected_uv));
        bool boundary_miss = fabsf(previous_reprojected_uv.x - 0.5f) > 0.5f || fabsf(previous_reprojected_uv.y - 0.5f) > 0.5f;
        Image32 instance_material_dummy{nullptr, 0, 0}; (void)instance_material_dummy;
        auto instance_at = [&](vec2 u) {
            int px = std::min(std::max((int)floorf(u.x * (float)c.W), 0), c.W - 1), py = std::min(std::max((int)floorf(u.y * (float)c.H), 0), c.H - 1);
            return c.instance_material[(size_t)py * c.W + px].x;
        };
        float current_instance = instance_at(previous_output_uv);
        bool instance_miss = false;
        float current_depth = position.nearest(previous_output_uv).w;
        bool depth_miss = current_depth == 0.0f;
        for (uint32_t i = 0u; i < 5u; i += 1u) {
            vec4 previous_depths = previous_position.gather_w(previous_reprojected_uv + uv_biases[i]);
            vec4 q = v4(current_depth) ;
            vec4 depth_ratio = v4(previous_depths.x == 0.0f ? 1.0f : q.x / previous_depths.x, previous_depths.y == 0.0f ? 1.0f : q.y / previous_depths.y,
                                  previous_depths.z == 0.0f ? 1.0f : q.z / previous_depths.z, previous_depths.w == 0.0f ? 1.0f : q.w / previous_depths.w);
            depth_miss = depth_miss || any_lt(depth_ratio, 0.95f);
            float previous_instance = instance_at(previous_reprojected_uv + uv_biases[i]);
            instance_miss = instance_miss || (any_lt(depth_ratio, 0.95f) && fabsf(previous_instance - current_instance) > 1.0f);
        }
        vec4 pv = previous_velocity_uv.nearest(previous_reprojected_uv);
        bool velocity_miss = distance2(velocity, v2(pv.x, pv.y)) > 0.0001f;
        if (boundary_miss || ((depth_miss || instance_miss) && velocity_miss)) {
            vec2 uv_bias = v2(0.0f, 0.0f);
            float min_ds = 10.0f;
            for (uint32_t i = 0u; i < 5u; i += 1u) {
                vec4 ds = position.gather_w(previous_output_uv + uv_biases[i]);
                float dds = distance4(v4(current_depth), ds);
                if (dds < min_ds) uv_bias = uv_biases[i];
                min_ds = fmin_(min_ds, dds);
            }
            vec4 g[4];
            render.gather(previous_output_uv + uv_bias, g);
            vec3 s1 = RGB_to_YCoCg(xyz(g[0])), s2 = RGB_to_YCoCg(xyz(g[1])), s3 = RGB_to_YCoCg(xyz(g[2])), s4 = RGB_to_YCoCg(xyz(g[3]));
            vec3 s_mm = RGB_to_YCoCg(current_color);
            vec3 moment_1 = s1 + s2 + s3 + s4;
            vec3 moment_2 = s1 * s1 + s2 * s2 + s3 * s3 + s4 * s4;
            vec3 mean = moment_1 / 4.0f;
            vec3 variance = vsqrt((moment_2 / 4.0f) - (mean * mean));
            previous_color = RGB_to_YCoCg(previous_color);
            previous_color = clip_towards_aabb_center(previous_color, s_mm, mean - variance, mean + variance);
            previous_color = YCoCg_to_RGB(previous_color);
        }
        vec2 sv = velocity / (2.0f * texel_size);
        vec2 subpixel_velocity = v2(fract(sv.x), fract(sv.y));
        float blend_factor = fmax_(subpixel_velocity.x, subpixel_velocity.y);
        float sn, cs; sincos_(blend_factor * TAU, &sn, &cs);
        blend_factor = clampf(-cs, 0.0f, 1.0f);
        vec3 remix_color = xyz(render.linear(previous_output_uv));
        previous_color = mix(previous_color, remix_color, blend_factor);
        auto store = [&](ivec2 p, vec4 v) {   // textureStore outside the texture is dropped
            if (p.x < OW && p.y < OH) c.upscale_output[(size_t)p.y * OW + p.x] = pack_rgba16f(v);
        };
        store(current_output_coords, v4(current_color, 1.0f));
        store(previous_output_coords, v4(previous_color, 1.0f));
    });
}

void pass_smaa_tu4x_extrapolate(Ctx& c) {  // smaa.wgsl:201-271
    const int OW = c.OW, OH = c.OH;
    Image16 out{&c.upscale_output, OW, OH};
    auto lum3 = [](vec4 a, vec4 b) { return luminance(vabs(xyz(a) - xyz(b))); };
    for_pixels(c, c.RW, c.RH, [&](int x, int y) {
        auto L = [&](int dx, int dy) { ivec2 p; p.x = 2 * x + dx; p.y = 2 * y + dy; return out.load(p); };
        vec4 t = L(0, 0), b = L(1, 1), n = L(1, -1), e = L(2, 0), s_ = L(0, 2), w = L(-1, 1);
        // differential_blend_factor :201-222
        vec2 dh = v2(lum3(w, b), lum3(t, e));
        vec2 dv = v2(lum3(t, s_), lum3(n, b));
        vec2 factor_xy = v2(fmax_(dv.x, 0.001f) * fmax_(dv.y, 0.001f), fmax_(dh.x, 0.001f) * fmax_(dh.y, 0.001f));
        float factor_z = 1.0f / (factor_xy.x + factor_xy.y);
        auto blend = [&](vec4 tt, vec4 bb, vec4 ll, vec4 rr) {  // differential_blend :224-235
            vec4 color = v4(0.0f);
            color = color + (ll + rr) * factor_xy.x;
            color = color + (tt + bb) * factor_xy.y;
            return color * (0.5f * factor_z);
        };
        vec4 x_color = blend(t, s_, w, b);
        vec4 y_color = blend(n, b, t, e);
        if (2 * x < OW && 2 * y + 1 < OH) c.upscale_output[(size_t)(2 * y + 1) * OW + 2 * x] = pack_rgba16f(x_color);
        if (2 * x + 1 < OW && 2 * y < OH) c.upscale_output[(size_t)(2 * y) * OW + 2 * x + 1] = pack_rgba16f(y_color);
    });
}

// ----------------------------------------------------------------------------- FSR 1.0 (Upscale::Fsr1), SURVEY 8(f) rank 4
// The reference ships EASU and RCAS as SPIR-V built from AMD's FidelityFX sources, which sit next to the blobs
// (src/shaders/fsr/source.zip: FSR_Pass.glsl, ffx_fsr1.h, ffx_a.h, texture_gather.glsl; compile.bat).  This restates the
// variant that build selects: SAMPLE_SLOW_FALLBACK = 1 -> the 32-bit paths FsrEasuF / FsrRcasF, no FSR_RCAS_DENOISE, no alpha
// pass-through, `hdr == 0` (post_process.rs:531), constants computed per invocation from FsrConstantsUniform
// (post_process.rs:518-534: viewport = input size = scaled_size, output = the camera target).
// Texture access: texture_gather.glsl emulates textureGather by four bilinear taps half a texel around the gather point,
// i.e. exactly at the centres of the four texels (linear sampler, clamp-to-edge, post_process.rs:703-708,879) — restated as
// four clamped texel fetches; FsrRcasLoadF is texelFetch, zero outside the image like every textureLoad here.

// FsrEasuSetF, ffx_fsr1.h:275-313: one corner's contribution to gradient direction and edge length
inline void fsr_easu_set(vec2& dir, float& len, float w, float lA, float lB, float lC, float lD, float lE) {
    float dc = lD - lC, cb = lC - lB;
    float lenX = fmax_(fabsf(dc), fabsf(cb));
    lenX = fsr_rcp_lo(lenX);
    float dirX = lD - lB;
    dir.x += dirX * w;
    lenX = clampf(fabsf(dirX) * lenX, 0.0f, 1.0f);
    lenX *= lenX;
    len += lenX * w;
    float ec = lE - lC, ca = lC - lA;
    float lenY = fmax_(fabsf(ec), fabsf(ca));
    lenY = fsr_rcp_lo(lenY);
    float dirY = lE - lA;
    dir.y += dirY * w;
    lenY = clampf(fabsf(dirY) * lenY, 0.0f, 1.0f);
    lenY *= lenY;
    len += lenY * w;
}
// FsrEasuTapF, ffx_fsr1.h:239-273
inline void fsr_easu_tap(vec3& aC, float& aW, vec2 off, vec2 dir, vec2 len, float lob, float clp, vec3 col) {
    vec2 v;
    v.x = (off.x * dir.x) + (off.y * dir.y);
    v.y = (off.x * (-dir.y)) + (off.y * dir.x);
    v = v * len;
    float d2 = v.x * v.x + v.y * v.y;
    d2 = fmin_(d2, clp);
    float wB = (2.0f / 5.0f) * d2 + -1.0f;
    float wA = lob * d2 + -1.0f;
    wB *= wB;
    wA *= wA;
    wB = (25.0f / 16.0f) * wB + (-(25.0f / 16.0f - 1.0f));
    float w = wB * wA;
    aC = aC + col * w;
    aW += w;
}
inline vec3 min3v(vec3 a, vec3 b) { return v3(fmin_(a.x, b.x), fmin_(a.y, b.y), fmin_(a.z, b.z)); }
inline vec3 max3v(vec3 a, vec3 b) { return v3(fmax_(a.x, b.x), fmax_(a.y, b.y), fmax_(a.z, b.z)); }

void pass_fsr_easu(Ctx& c) {   // FSR_Pass.glsl main + CurrFilter (SAMPLE_EASU), FsrEasuF ffx_fsr1.h:315-437
    const uint32_t cur = c.in.frame.number % 2u;
    // upscale_input_texture, post_process.rs:1037-1040; both are scaled_size textures under Fsr1 (post_process.rs:716,726-729)
    Image16 input{c.in.taa_jitter ? &c.taa_output[cur] : &c.tone_mapping_output[cur], c.RW, c.RH};
    const FsrEasuConstants con = fsr_easu_constants((float)c.RW, (float)c.RH, (float)c.W, (float)c.H);
    for_pixels(c, c.W, c.H, [&](int x, int y) {
        vec2 pp = v2((float)x * con.scale_x + con.offset_x, (float)y * con.scale_y + con.offset_y);
        vec2 fp = v2(floorf(pp.x), floorf(pp.y));
        pp = pp - fp;
        const int fx = (int)fp.x, fy = (int)fp.y;
        auto T = [&](int dx, int dy) { return xyz(input.texel(fx + dx, fy + dy)); };
        //    b c
        //  e f g h
        //  i j k l
        //    n o
        vec3 b = T(0, -1), cc = T(1, -1), e = T(-1, 0), f = T(0, 0), g = T(1, 0), h = T(2, 0);
        vec3 i = T(-1, 1), j = T(0, 1), k = T(1, 1), l = T(2, 1), n = T(0, 2), o = T(1, 2);
        auto luma2 = [](vec3 t) { return t.z * 0.5f + (t.x * 0.5f + t.y); };
        float bL = luma2(b), cL = luma2(cc), eL = luma2(e), fL = luma2(f), gL = luma2(g), hL = luma2(h);
        float iL = luma2(i), jL = luma2(j), kL = luma2(k), lL = luma2(l), nL = luma2(n), oL = luma2(o);
        vec2 dir = v2(0.0f, 0.0f);
        float len = 0.0f;
        fsr_easu_set(dir, len, (1.0f - pp.x) * (1.0f - pp.y), bL, eL, fL, gL, jL);
        fsr_easu_set(dir, len, pp.x * (1.0f - pp.y), cL, fL, gL, hL, kL);
        fsr_easu_set(dir, len, (1.0f - pp.x) * pp.y, fL, iL, jL, kL, nL);
        fsr_easu_set(dir, len, pp.x * pp.y, gL, jL, kL, lL, oL);
        vec2 dir2 = dir * dir;
        float dirR = dir2.x + dir2.y;
        const bool zro = dirR < (1.0f / 32768.0f);
        dirR = fsr_rsq_lo(dirR);
        dirR = zro ? 1.0f : dirR;
        dir.x = zro ? 1.0f : dir.x;
        dir = dir * dirR;
        len = len * 0.5f;
        len *= len;
        float stretch = (dir.x * dir.x + dir.y * dir.y) * fsr_rcp_lo(fmax_(fabsf(dir.x), fabsf(dir.y)));
        vec2 len2 = v2(1.0f + (stretch - 1.0f) * len, 1.0f + -0.5f * len);
        float lob = 0.5f + ((1.0f / 4.0f - 0.04f) - 0.5f) * len;
        float clp = fsr_rcp_lo(lob);
        vec3 min4 = min3v(min3v(f, min3v(g, j)), k);
        vec3 max4 = max3v(max3v(f, max3v(g, j)), k);
        vec3 aC = v3(0.0f, 0.0f, 0.0f);
        float aW = 0.0f;
        fsr_easu_tap(aC, aW, v2(0.0f, -1.0f) - pp, dir, len2, lob, clp, b);
        fsr_easu_tap(aC, aW, v2(1.0f, -1.0f) - pp, dir, len2, lob, clp, cc);
        fsr_easu_tap(aC, aW, v2(-1.0f, 1.0f) - pp, dir, len2, lob, clp, i);
        fsr_easu_tap(aC, aW, v2(0.0f, 1.0f) - pp, dir, len2, lob, clp, j);
        fsr_easu_tap(aC, aW, v2(0.0f, 0.0f) - pp, dir, len2, lob, clp, f);
        fsr_easu_tap(aC, aW, v2(-1.0f, 0.0f) - pp, dir, len2, lob, clp, e);
        fsr_easu_tap(aC, aW, v2(1.0f, 1.0f) - pp, dir, len2, lob, clp, k);
        fsr_easu_tap(aC, aW, v2(2.0f, 1.0f) - pp, dir, len2, lob, clp, l);
        fsr_easu_tap(aC, aW, v2(2.0f, 0.0f) - pp, dir, len2, lob, clp, h);
        fsr_easu_tap(aC, aW, v2(1.0f, 0.0f) - pp, dir, len2, lob, clp, g);
        fsr_easu_tap(aC, aW, v2(1.0f, 2.0f) - pp, dir, len2, lob, clp, o);
        fsr_easu_tap(aC, aW, v2(0.0f, 2.0f) - pp, dir, len2, lob, clp, n);
        vec3 pix = min3v(max4, max3v(min4, aC * (1.0f / aW)));
        c.upscale_output[(size_t)y * c.W + x] = pack_rgba16f(v4(pix, 1.0f));   // imageStore(OutputTexture, pos, AF4(c, 1))
    });
}

void pass_fsr_rcas(Ctx& c) {   // FSR_Pass.glsl CurrFilter (SAMPLE_RCAS), FsrRcasF ffx_fsr1.h:684-772
    Image16 input{&c.upscale_output, c.W, c.H};
    const float sharp = fsr_rcas_constant(c.in.fsr_sharpness);
    for_pixels(c, c.W, c.H, [&](int x, int y) {
        auto Ld = [&](int dx, int dy) { ivec2 p; p.x = x + dx; p.y = y + dy; return xyz(input.load(p)); };
        //    b
        //  d e f
        //    h
        vec3 b = Ld(0, -1), d = Ld(-1, 0), e = Ld(0, 0), f = Ld(1, 0), h = Ld(0, 1);
        auto min4f = [](float p, float q, float r, float s_) { return fmin_(fmin_(p, fmin_(q, r)), s_); };   // min(AMin3F1(b,d,f),h)
        auto max4f = [](float p, float q, float r, float s_) { return fmax_(fmax_(p, fmax_(q, r)), s_); };
        vec3 mn4 = v3(min4f(b.x, d.x, f.x, h.x), min4f(b.y, d.y, f.y, h.y), min4f(b.z, d.z, f.z, h.z));
        vec3 mx4 = v3(max4f(b.x, d.x, f.x, h.x), max4f(b.y, d.y, f.y, h.y), max4f(b.z, d.z, f.z, h.z));
        auto lobe_of = [](float mn, float mx, float ec) {
            float hitMin = fmin_(mn, ec) * (1.0f / (4.0f * mx));
            float hitMax = (1.0f - fmax_(mx, ec)) * (1.0f / (4.0f * mn + -4.0f));
            return fmax_(-hitMin, hitMax);
        };
        float lobeR = lobe_of(mn4.x, mx4.x, e.x), lobeG = lobe_of(mn4.y, mx4.y, e.y), lobeB = lobe_of(mn4.z, mx4.z, e.z);
        float lobe = fmax_(-FSR_RCAS_LIMIT, fmin_(fmax_(lobeR, fmax_(lobeG, lobeB)), 0.0f)) * sharp;
        float rcpL = fsr_rcp_med(4.0f * lobe + 1.0f);
        vec3 pix = v3((lobe * b.x + lobe * d.x + lobe * h.x + lobe * f.x + e.x) * rcpL,
                      (lobe * b.y + lobe * d.y + lobe * h.y + lobe * f.y + e.y) * rcpL,
                      (lobe * b.z + lobe * d.z + lobe * h.z + lobe * f.z + e.z) * rcpL);
        c.upscale_sharpen_output[(size_t)y * c.W + x] = pack_rgba16f(v4(pix, 1.0f));
    });
}

void pass_taa_jasmine(Ctx& c) {  // taa.wgsl:79-170
    const uint32_t cur = c.in.frame.number % 2u, prev = 1u - cur;
    const bool smaa = c.in.smaa_tu4x != 0;
    const int OW = smaa ? c.OW : c.RW, OH = smaa ? c.OH : c.RH;              // post_process.rs:717,726-731; the dispatch over 2 RW x 2 RH (:1258)
                                                                             // stores nothing outside the texture
    Image16 render{smaa ? &c.upscale_output : &c.tone_mapping_output[cur], OW, OH};   // taa_input_texture, post_process.rs:1011-1014
    Image16 previous_render{&c.taa_output[prev], OW, OH};
    Image32 position{&c.position, c.W, c.H}, previous_position{&c.previous_position, c.W, c.H};
    Image32 velocity_uv{&c.velocity_uv, c.W, c.H}, previous_velocity_uv{&c.previous_velocity_uv, c.W, c.H};
    ivec2 output_size; output_size.x = OW; output_size.y = OH;
    auto sample_previous = [&](vec2 u) { return clamp01(xyz(previous_render.linear(u))); };          // :47-50
    auto sample_render = [&](vec2 u) { return RGB_to_YCoCg(clamp01(xyz(render.nearest(u)))); };      // :52-55
    for_pixels(c, OW, OH, [&](int x, int y) {
        ivec2 coords; coords.x = x; coords.y = y;
        vec2 size = v2((float)OW, (float)OH);
        vec2 texel_size = v2(1.0f, 1.0f) / size;
        vec2 uv = coords_to_uv(coords, output_size);
        vec4 original_color = render.nearest(uv);
        vec3 current_color = xyz(original_color);
        vec2 velocity = nearest_velocity(position, velocity_uv, uv, texel_size);   // texel of render_texture here (taa.wgsl:58)
        vec2 previous_uv = uv - velocity;
        bool boundary_miss = fabsf(previous_uv.x - 0.5f) > 0.5f || fabsf(previous_uv.y - 0.5f) > 0.5f;
        vec2 uv_biases[5] = {v2(0.0f, 0.0f), v2(1.5f, 1.5f) * texel_size, v2(-1.5f, 1.5f) * texel_size, v2(1.5f, -1.5f) * texel_size,
                             v2(-1.5f, -1.5f) * texel_size};
        vec4 current_position_depth = position.nearest(uv);
        bool has_content = current_position_depth.w > 0.0f;
        bool depth_miss = current_position_depth.w == 0.0f;
        bool position_miss = current_position_depth.w == 0.0f;
        for (uint32_t i = 0u; i < 5u; i += 1u) {
            vec4 pd = previous_position.gather_w(previous_uv + uv_biases[i]);
            float cd = current_position_depth.w;
            vec4 depth_ratio = v4(pd.x == 0.0f ? 1.0f : cd / pd.x, pd.y == 0.0f ? 1.0f : cd / pd.y, pd.z == 0.0f ? 1.0f : cd / pd.z,
                                  pd.w == 0.0f ? 1.0f : cd / pd.w);
            has_content = has_content || pd.x > 0.0f || pd.y > 0.0f || pd.z > 0.0f || pd.w > 0.0f;
            depth_miss = depth_miss || any_lt(depth_ratio, 0.95f);
            vec3 previous_pos = xyz(previous_position.nearest(previous_uv + uv_biases[i]));
            position_miss = position_miss || length(xyz(current_position_depth) - previous_pos) > 0.5f;
        }
        size_t oidx = (size_t)y * OW + x;
        if (!has_content) { c.taa_output[cur][oidx] = pack_rgba16f(ld4(c.in.frame.clear_color)); return; }
        vec4 pv = previous_velocity_uv.nearest(previous_uv);
        bool velocity_miss = distance2(velocity, v2(pv.x, pv.y)) > 0.00005f;
        // 5-tap Catmull-Rom (taa.wgsl:121-139)
        vec2 sample_position = (uv - velocity) * size;
        vec2 tp1 = v2(floorf(sample_position.x - 0.5f), floorf(sample_position.y - 0.5f)) + 0.5f;
        vec2 f = sample_position - tp1;
        auto W0 = [](float f_) { return f_ * (-0.5f + f_ * (1.0f - 0.5f * f_)); };
        auto W1 = [](float f_) { return 1.0f + f_ * f_ * (-2.5f + 1.5f * f_); };
        auto W2 = [](float f_) { return f_ * (0.5f + f_ * (2.0f - 1.5f * f_)); };
        auto W3 = [](float f_) { return f_ * f_ * (-0.5f + 0.5f * f_); };
        vec2 w0 = v2(W0(f.x), W0(f.y)), w1 = v2(W1(f.x), W1(f.y)), w2 = v2(W2(f.x), W2(f.y)), w3 = v2(W3(f.x), W3(f.y));
        vec2 w12 = w1 + w2;
        vec2 offset12 = w2 / (w1 + w2);
        vec2 tp0 = (tp1 - 1.0f) * texel_size;
        vec2 tp3 = (tp1 + 2.0f) * texel_size;
        vec2 tp12 = (tp1 + offset12) * texel_size;
        vec3 previous_color = v3(0.0f);
        previous_color = previous_color + sample_previous(v2(tp12.x, tp0.y)) * w12.x * w0.y;
        previous_color = previous_color + sample_previous(v2(tp0.x, tp12.y)) * w0.x * w12.y;
        previous_color = previous_color + sample_previous(v2(tp12.x, tp12.y)) * w12.x * w12.y;
        previous_color = previous_color + sample_previous(v2(tp3.x, tp12.y)) * w3.x * w12.y;
        previous_color = previous_color + sample_previous(v2(tp12.x, tp3.y)) * w12.x * w3.y;
        if (boundary_miss || (position_miss && velocity_miss && depth_miss)) {
            vec3 s_tl = sample_render(uv + v2(-texel_size.x, texel_size.y));
            vec3 s_tm = sample_render(uv + v2(0.0f, texel_size.y));
            vec3 s_tr = sample_render(uv + texel_size);
            vec3 s_ml = sample_render(uv - v2(texel_size.x, 0.0f));
            vec3 s_mm = RGB_to_YCoCg(current_color);
            vec3 s_mr = sample_render(uv + v2(texel_size.x, 0.0f));
            vec3 s_bl = sample_render(uv - texel_size);
            vec3 s_bm = sample_render(uv - v2(0.0f, texel_size.y));
            vec3 s_br = sample_render(uv + v2(texel_size.x, -texel_size.y));
            vec3 moment_1 = s_tl + s_tm + s_tr + s_ml + s_mm + s_mr + s_bl + s_bm + s_br;
            vec3 moment_2 = (s_tl * s_tl) + (s_tm * s_tm) + (s_tr * s_tr) + (s_ml * s_ml) + (s_mm * s_mm) + (s_mr * s_mr) + (s_bl * s_bl) +
                            (s_bm * s_bm) + (s_br * s_br);
            vec3 mean = moment_1 / 9.0f;
            vec3 variance = vsqrt((moment_2 / 9.0f) - (mean * mean));
            previous_color = RGB_to_YCoCg(previous_color);
            previous_color = clip_towards_aabb_center(previous_color, s_mm, mean - variance, mean + variance);
            previous_color = YCoCg_to_RGB(previous_color);
        }
        vec3 output = mix(previous_color, current_color, 0.1f / c.in.frame.upscale_ratio);
        c.taa_output[cur][oidx] = pack_rgba16f(v4(output, original_color.w));
    });
}

// ----------------------------------------------------------------------------------------- node drivers
void light_node(Ctx& c) {  // LightNode::run, light.rs:590-702
    pass_albedo(c);
    pass_direct_lit<false, true>(c, 0);                       // direct_lit + RENDER_EMISSIVE (light.rs:409-414)
    pass_direct_lit<true, false>(c, 1);                       // direct_emissive: EMISSIVE_LIT (light.rs:415-420)
    if (c.in.frame.emissive_spatial_reuse) pass_spatial_reuse<true, false>(c, 1);
    if (c.in.frame.indirect_bounces < 2) pass_indirect<false>(c); else pass_indirect<true>(c);
    if (c.in.frame.indirect_spatial_reuse) pass_spatial_reuse<false, false>(c, 2);
}
void post_process_node(Ctx& c) {  // PostProcessNode::run, post_process.rs:1140-1234
    if (c.in.denoise) {
        int signals = (c.in.frame.indirect_bounces == 0) ? 2 : 3;  // post_process.rs:949-954
        for (int sgl = 0; sgl < signals; ++sgl) {
            pass_demodulation(c, sgl);
            if (sgl == 0) {  // denoise_direct: no FIREFLY_FILTERING (post_process.rs:1193-1197)
                pass_denoise<0, false>(c, sgl); pass_denoise<1, false>(c, sgl);
                pass_denoise<2, false>(c, sgl); pass_denoise<3, false>(c, sgl);
            } else {
                pass_denoise<0, true>(c, sgl); pass_denoise<1, true>(c, sgl);
                pass_denoise<2, true>(c, sgl); pass_denoise<3, true>(c, sgl);
            }
        }
    }
    pass_tone_mapping(c);
    if (c.in.temporal_upscalers) {   // post_process.rs:1236-1308 (K11/K12 and FSR1, SURVEY.md 8(f) ranks 1 and 4)
        if (c.in.smaa_tu4x) { pass_smaa_tu4x(c); pass_smaa_tu4x_extrapolate(c); }
        if (c.in.taa_jitter) pass_taa_jasmine(c);
        if (c.in.fsr1 && !c.in.smaa_tu4x) { pass_fsr_easu(c); pass_fsr_rcas(c); }
    }
}

int fail(Ctx* c, int code, const char* msg) { if (c) c->error = msg; return code; }

template <class T>
void assign(std::vector<T>& dst, const T* src, uint32_t n) { dst.assign(src, src + n); }

}  // namespace

// ================================================================================================ C API
extern "C" {

int hko_context_create(hko_context** out, uint32_t width, uint32_t height, int threads) {
    if (!out || !width || !height) return HK_ERR_INVALID_ARGUMENT;
    Ctx* c = new Ctx();
    c->W = c->RW = (int)width;
    c->H = c->RH = (int)height;
    c->threads = threads > 0 ? threads : 1;
    c->rays.assign((size_t)c->threads + 1, hko_context::RayCounters());
    size_t n = (size_t)width * height;
    c->position.assign(n, v4(0.0f)); c->normal.assign(n, 0u); c->depth_gradient.assign(n, v2(0, 0));
    c->instance_material.assign(n, v2(0, 0)); c->velocity_uv.assign(n, v4(0.0f));
    uvec2 z2; z2.x = z2.y = 0;
    c->albedo.assign(n, z2);
    hk_packed_reservoir zr; memset(&zr, 0, sizeof(zr));
    for (int i = 0; i < 3; ++i) { c->render[i].assign(n, z2); c->variance[i].assign(n, 0.0f); c->denoise_render[i].assign(n, z2); }
    for (int i = 0; i < 10; ++i) c->reservoir[i].assign(n, zr);
    for (int i = 0; i < 4; ++i) c->denoise_internal[i].assign(n, z2);
    c->denoise_internal_variance.assign(n, 0.0f);
    for (int i = 0; i < 2; ++i) { c->tone_mapping_output[i].assign(n, z2); c->taa_output[i].assign(4 * n, z2); }
    c->upscale_output.assign(4 * n, z2);
    c->upscale_sharpen_output.assign(n, z2);
    c->previous_position.assign(n, v4(0.0f)); c->previous_velocity_uv.assign(n, v4(0.0f));
    memset(&c->in, 0, sizeof(c->in));
    *out = c;
    return HK_OK;
}
void hko_context_destroy(hko_context* c) { delete c; }
int hko_reset_temporal_state(hko_context* c) {
    hk_packed_reservoir zr; memset(&zr, 0, sizeof(zr));
    for (int i = 0; i < 10; ++i) std::fill(c->reservoir[i].begin(), c->reservoir[i].end(), zr);
    return HK_OK;
}
int hko_scene_update_instances(hko_context* c, const hk_scene_desc* s) {   // instance.rs:427-435 (set + write_buffer)
    if (!c || !s) return HK_ERR_INVALID_ARGUMENT;
    assign(c->alias_table, s->alias_table, s->alias_count);
    assign(c->instances, s->instances, s->instance_count);
    assign(c->instance_nodes, s->instance_nodes, s->instance_node_count);
    assign(c->emissive_nodes, s->emissive_nodes, s->emissive_node_count);
    assign(c->emissives, s->emissives, s->emissive_count);
    if (s->materials && s->material_count) assign(c->materials, s->materials, s->material_count);   // material.rs:139-203
    c->previous_models.clear();
    if (s->previous_instance_models) c->previous_models.assign(s->previous_instance_models, s->previous_instance_models + 16 * (size_t)s->instance_count);
    return HK_OK;
}
int hko_scene_upload(hko_context* c, const hk_scene_desc* s) {
    if (!c || !s) return HK_ERR_INVALID_ARGUMENT;
    assign(c->vertices, s->vertices, s->vertex_count);
    assign(c->primitives, s->primitives, s->primitive_count);
    assign(c->asset_nodes, s->asset_nodes, s->asset_node_count);
    assign(c->materials, s->materials, s->material_count);
    hko_scene_update_instances(c, s);
    c->textures.clear();
    float srgb_lut[256], lin_lut[256];
    for (int i = 0; i < 256; ++i) {
        double v = i / 255.0;
        lin_lut[i] = (float)v;
        srgb_lut[i] = (float)(v <= 0.04045 ? v / 12.92 : pow((v + 0.055) / 1.055, 2.4));
    }
    for (uint32_t t = 0; t < s->texture_count; ++t) {
        const hk_texture_desc& d = s->textures[t];
        Texture tex;
        tex.w = d.width; tex.h = d.height; tex.mode_u = d.address_mode_u; tex.mode_v = d.address_mode_v; tex.linear = d.filter_linear;
        tex.texels.resize((size_t)d.width * d.height);
        const float* lut = d.srgb ? srgb_lut : lin_lut;
        for (size_t i = 0; i < tex.texels.size(); ++i)
            tex.texels[i] = v4(lut[d.rgba8[4 * i]], lut[d.rgba8[4 * i + 1]], lut[d.rgba8[4 * i + 2]], lin_lut[d.rgba8[4 * i + 3]]);
        c->textures.push_back(std::move(tex));
    }
    c->scene_ready = true;
    return HK_OK;
}
int hko_set_noise(hko_context* c, const uint8_t* rgba) {
    c->noise.assign(rgba, rgba + 16 * 64 * 64 * 4);
    c->noise_ready = true;
    return HK_OK;
}
static int begin(hko_context* c, const hk_frame_inputs* in) {
    if (!c || !in) return HK_ERR_INVALID_ARGUMENT;
    if (!c->scene_ready || !c->noise_ready) return fail(c, HK_ERR_NOT_READY, "scene or noise not uploaded");
    c->in = *in;
    // scaled_size = (ratio.recip() * size.as_vec2()).ceil() (light.rs:622-624)
    const float scale = 1.0f / in->frame.upscale_ratio;
    c->RW = (int)ceilf(scale * (float)c->W);
    c->RH = (int)ceilf(scale * (float)c->H);
    const float scale2 = scale * 2.0f;                 // `scale *= 2.0` before upscale_output / taa_output are created
    c->OW = (int)ceilf((float)c->W * scale2);
    c->OH = (int)ceilf((float)c->H * scale2);
    if (c->RW < 1 || c->RH < 1 || c->RW > c->W || c->RH > c->H) return fail(c, HK_ERR_INVALID_ARGUMENT, "upscale_ratio out of range");
    return HK_OK;
}
int hko_prepass_run(hko_context* c, const hk_frame_inputs* in) { int e = begin(c, in); if (e) return e; pass_prepass(*c); return HK_OK; }
int hko_light_run(hko_context* c, const hk_frame_inputs* in) { int e = begin(c, in); if (e) return e; light_node(*c); return HK_OK; }
int hko_post_process_run(hko_context* c, const hk_frame_inputs* in) { int e = begin(c, in); if (e) return e; post_process_node(*c); return HK_OK; }
int hko_render_frame(hko_context* c, const hk_frame_inputs* in) {
    int e = begin(c, in); if (e) return e;
    pass_prepass(*c); light_node(*c); post_process_node(*c);
    return HK_OK;
}
// single passes, for per-pass parity from identical inputs.  pass ids: 0 albedo, 1 direct(sun), 2 direct(emissive),
// 3 spatial(emissive), 4 indirect, 5 spatial(indirect), 6 denoise chain of signal `arg`, 7 tone mapping, 8 FSR EASU, 9 FSR RCAS
int hko_run_pass(hko_context* c, const hk_frame_inputs* in, int pass, int arg) {
    int e = begin(c, in); if (e) return e;
    switch (pass) {
        case 0: pass_albedo(*c); break;
        case 1: pass_direct_lit<false, true>(*c, 0); break;
        case 2: pass_direct_lit<true, false>(*c, 1); break;
        case 3: pass_spatial_reuse<true, false>(*c, 1); break;
        case 4: if (c->in.frame.indirect_bounces < 2) pass_indirect<false>(*c); else pass_indirect<true>(*c); break;
        case 5: pass_spatial_reuse<false, false>(*c, 2); break;
        case 6:
            pass_demodulation(*c, arg);
            if (arg == 0) { pass_denoise<0, false>(*c, arg); pass_denoise<1, false>(*c, arg); pass_denoise<2, false>(*c, arg); pass_denoise<3, false>(*c, arg); }
            else { pass_denoise<0, true>(*c, arg); pass_denoise<1, true>(*c, arg); pass_denoise<2, true>(*c, arg); pass_denoise<3, true>(*c, arg); }
            break;
        case 7: pass_tone_mapping(*c); break;
        case 8: pass_fsr_easu(*c); break;
        case 9: pass_fsr_rcas(*c); break;
        default: return HK_ERR_INVALID_ARGUMENT;
    }
    return HK_OK;
}
static void* plane(hko_context* c, int which, size_t* bytes) {
    size_t n = (size_t)c->W * c->H;                   // deferred (full) size planes
    const size_t nr = (size_t)c->RW * c->RH;          // render-size planes (row stride RW, so the first RW*RH entries)
    const bool smaa = c->in.smaa_tu4x != 0;
    auto R = [&](void* p, size_t b) { *bytes = b * n; return p; };
    auto RR = [&](void* p, size_t b, size_t count) { *bytes = b * count; return p; };
    switch (which) {
        case HK_OUT_TONE_MAPPED: return RR(c->tone_mapping_output[c->in.frame.number % 2u].data(), 8, nr);
        case HK_OUT_UPSCALED: return RR(c->upscale_output.data(), 8, c->in.fsr1 ? n : (size_t)c->OW * c->OH);
        case HK_OUT_FSR_SHARPENED: return RR(c->upscale_sharpen_output.data(), 8, n);
        case HK_OUT_TAA: return RR(c->taa_output[c->in.frame.number % 2u].data(), 8, smaa ? (size_t)c->OW * c->OH : nr);
        case HK_OUT_RENDER_DIRECT: case HK_OUT_RENDER_EMISSIVE: case HK_OUT_RENDER_INDIRECT:
            return RR(c->render[which - HK_OUT_RENDER_DIRECT].data(), 8, nr);
        case HK_OUT_VARIANCE_DIRECT: case HK_OUT_VARIANCE_EMISSIVE: case HK_OUT_VARIANCE_INDIRECT:
            return RR(c->variance[which - HK_OUT_VARIANCE_DIRECT].data(), 4, nr);
        case HK_OUT_ALBEDO: return R(c->albedo.data(), 8);
        case HK_OUT_DENOISED_DIRECT: case HK_OUT_DENOISED_EMISSIVE: case HK_OUT_DENOISED_INDIRECT:
            return RR(c->denoise_render[which - HK_OUT_DENOISED_DIRECT].data(), 8, nr);
        case HK_OUT_GBUFFER_POSITION: return R(c->position.data(), 16);
        case HK_OUT_GBUFFER_NORMAL: return R(c->normal.data(), 4);
        case HK_OUT_GBUFFER_DEPTH_GRADIENT: return R(c->depth_gradient.data(), 8);
        case HK_OUT_GBUFFER_INSTANCE_MATERIAL: return R(c->instance_material.data(), 8);
        case HK_OUT_GBUFFER_VELOCITY_UV: return R(c->velocity_uv.data(), 16);
        default:
            if (which >= HK_OUT_RESERVOIR_0 && which < HK_OUT_RESERVOIR_0 + 10) return RR(c->reservoir[which - HK_OUT_RESERVOIR_0].data(), 64, nr);
    }
    return nullptr;
}
int hko_output_extent(hko_context* c, int which, uint32_t* width, uint32_t* height) {   // pixels of a read-back plane, last frame's settings
    size_t b = 0;
    if (!plane(c, which, &b)) return fail(c, HK_ERR_INVALID_ARGUMENT, "bad plane id");
    const bool deferred = which == HK_OUT_ALBEDO || (which >= HK_OUT_GBUFFER_POSITION && which <= HK_OUT_GBUFFER_VELOCITY_UV);
    const bool fsr = c->in.fsr1 && (which == HK_OUT_UPSCALED || which == HK_OUT_FSR_SHARPENED);   // the camera target size
    const int k = ((which == HK_OUT_UPSCALED && !c->in.fsr1) || (which == HK_OUT_TAA && c->in.smaa_tu4x)) ? 2 : 1;
    *width = (uint32_t)((deferred || fsr) ? c->W : (k == 2 ? c->OW : c->RW)); *height = (uint32_t)((deferred || fsr) ? c->H : (k == 2 ? c->OH : c->RH));
    return HK_OK;
}
int hko_readback(hko_context* c, int which, void* host, size_t bytes) {
    size_t b = 0; void* p = plane(c, which, &b);
    if (!p || bytes != b) return fail(c, HK_ERR_INVALID_ARGUMENT, "bad plane id or size");
    memcpy(host, p, b);
    return HK_OK;
}
int hko_upload_state(hko_context* c, int which, const void* host, size_t bytes) {
    size_t b = 0; void* p = plane(c, which, &b);
    if (!p || bytes != b) return fail(c, HK_ERR_INVALID_ARGUMENT, "bad plane id or size");
    memcpy(p, host, b);
    return HK_OK;
}
int hko_trace_rays(hko_context* c, const hk_ray* rays, size_t n, hk_hit* hits) {
    if (!c->scene_ready) return fail(c, HK_ERR_NOT_READY, "scene not uploaded");
#pragma omp parallel for num_threads(c->threads)
    for (long long i = 0; i < (long long)n; ++i) {
        Ray r;
        r.origin = ld3(rays[i].origin); r.direction = ld3(rays[i].direction); r.inv_direction = 1.0f / r.direction;
        Hit h = traverse_top(*c, r, rays[i].max_distance, rays[i].early_distance, rays[i].exclude_instance);
        hits[i].u = h.intersection.uv.x; hits[i].v = h.intersection.uv.y; hits[i].distance = h.intersection.distance;
        hits[i].instance_index = h.instance_index; hits[i].primitive_index = h.primitive_index;
    }
    return HK_OK;
}
// Diagnostic for kernel design (not a pass of the reference): number of TLAS and BLAS records each ray touches.
static void count_steps(const Ctx& c, const Ray& ray, float max_distance, float early_distance, uint32_t exclude, uint32_t* out3) {
    float best = max_distance;
    uint32_t tlas = 0, blas = 0, leaves = 0;
    uint32_t index = 0;
    const uint32_t count = (uint32_t)c.instance_nodes.size();
    bool done = false;
    for (; index < count && !done;) {
        const hk_node& node = c.instance_nodes[index];
        ++tlas;
        Aabb aabb;
        if (node.entry_index >= BVH_LEAF_FLAG) {
            uint32_t ii = node.entry_index - BVH_LEAF_FLAG;
            const hk_instance& inst = c.instances[ii];
            aabb.min = ld3(inst.min); aabb.max = ld3(inst.max);
            if (ii != exclude && intersects_aabb(ray, aabb) < best) {
                Ray r;
                r.origin = instance_position_world_to_local(inst, ray.origin);
                r.direction = instance_direction_world_to_local(inst, ray.direction);
                r.inv_direction = 1.0f / r.direction;
                uint32_t bi = 0;
                while (bi < inst.mesh.node_count) {
                    const hk_node& bn = c.asset_nodes[inst.mesh.node_offset + bi];
                    ++blas;
                    if (bn.entry_index >= BVH_LEAF_FLAG) {
                        ++leaves;
                        const hk_primitive& prim = c.primitives[inst.mesh.primitive + bn.entry_index - BVH_LEAF_FLAG];
                        Intersection is = intersects_triangle(r, prim);
                        if (is.distance < best) { best = is.distance; if (is.distance < early_distance) { done = true; break; } }
                        bi = bn.exit_index;
                    } else {
                        aabb.min = ld3(bn.min); aabb.max = ld3(bn.max);
                        bi = (intersects_aabb(r, aabb) < best) ? bn.entry_index : bn.exit_index;
                    }
                }
            }
            index = node.exit_index;
        } else {
            aabb.min = ld3(node.min); aabb.max = ld3(node.max);
            index = (intersects_aabb(ray, aabb) < best) ? node.entry_index : node.exit_index;
        }
    }
    out3[0] = tlas; out3[1] = blas; out3[2] = leaves;
}
int hko_trace_steps(hko_context* c, const hk_ray* rays, size_t n, uint32_t* steps3) {
#pragma omp parallel for num_threads(c->threads)
    for (long long i = 0; i < (long long)n; ++i) {
        Ray r;
        r.origin = ld3(rays[i].origin); r.direction = ld3(rays[i].direction); r.inv_direction = 1.0f / r.direction;
        count_steps(*c, r, rays[i].max_distance, rays[i].early_distance, rays[i].exclude_instance, steps3 + 3 * i);
    }
    return HK_OK;
}
int hko_get_stats(hko_context* c, hk_frame_stats* out) {
    memset(out, 0, sizeof(*out));
    for (auto& r : c->rays) {
        out->primary_rays += r.primary; out->tlas_rays += r.tlas; out->blas_rays += r.blas;
        r = hko_context::RayCounters();
    }
    return HK_OK;
}
const char* hko_last_error(hko_context* c) { return c ? c->error.c_str() : ""; }

// scalar primitives exported for known-answer tests of include/hk_math.h
float hko_math_exp2(float x) { return exp2_(x); }
float hko_math_exp(float x) { return exp_(x); }
void hko_math_sincos(float x, float* s, float* c) { sincos_(x, s, c); }
uint32_t hko_math_pack2x16float(float a, float b) { return pack2x16float(a, b); }
float hko_math_f16_to_f32(uint16_t h) { return f16_bits_to_f32(h); }
uint32_t hko_math_pack4x8snorm(float x, float y, float z, float w) { return pack4x8snorm(v4(x, y, z, w)); }
uint32_t hko_math_pack2x16unorm(float a, float b) { return pack2x16unorm(a, b); }
uint32_t hko_math_hash(uint32_t v) { return hash_u32(v); }
float hko_math_unsnorm8(uint32_t b) { return unsnorm8(b); }
float hko_math_unorm8(uint32_t b) { return unorm8(b); }
float hko_math_unorm16(uint32_t u) { return unpack2x16unorm(u).x; }
// BRDF pieces of light.wgsl:796-833 (imported from bevy_pbr::pbr_lighting) for tests/test_math.py, which checks them
// against a float64 restatement of the published Filament / Karis formulas
void hko_math_lit(const float* radiance, const float* diffuse_color, float roughness, const float* F0, const float* Lv, const float* N,
                  const float* V, float* out3) {
    vec3 r = lit(ld3(radiance), ld3(diffuse_color), roughness, ld3(F0), ld3(Lv), ld3(N), ld3(V));
    out3[0] = r.x; out3[1] = r.y; out3[2] = r.z;
}
void hko_math_env_brdf_approx(const float* f0, float perceptual_roughness, float NoV, float* out3) {
    vec3 r = EnvBRDFApprox(ld3(f0), perceptual_roughness, NoV);
    out3[0] = r.x; out3[1] = r.y; out3[2] = r.z;
}
float hko_math_perceptual_roughness_to_roughness(float pr) { return perceptualRoughnessToRoughness(pr); }
void hko_math_normal_basis(const float* n, float* out9) {
    mat3 m = normal_basis(v3(n[0], n[1], n[2]));
    for (int i = 0; i < 3; ++i) { out9[3 * i] = m.c[i].x; out9[3 * i + 1] = m.c[i].y; out9[3 * i + 2] = m.c[i].z; }
}
void hko_pack_reservoir_roundtrip(const hk_packed_reservoir* in, hk_packed_reservoir* out) { *out = pack_reservoir(unpack_reservoir(*in)); }

// Batch forms of the primitives for tests/test_gpu_device_math.py, which compares them with tests/cuda/math_probe.cu (the same
// header compiled for the device): fn numbers as there.  hko_math_batch reads n inputs (2n for the two-operand functions);
// hko_math_batch_range evaluates the bit patterns first .. first + n - 1.  fn 40 and above take and give several words per element
// (normalize, the lighting functions, the reservoir record and its unpacked state).
static uint32_t math_probe1(int fn, uint32_t u) {
    const float x = u2f(u);
    switch (fn) {
        case 0: return f32_to_u32(x);
        case 1: return (uint32_t)f32_to_i32(x);
        case 2: return f32_to_f16_bits(x);
        case 3: return snorm8(x);
        case 4: return pack2x16unorm(x, 0.0f) & 0xFFFFu;
        case 5: return f2u(fract(x));
        case 6: return f2u(pow5(x));
        case 7: return f2u(pow16(x));
        case 8: return hash_u32(u);
        case 9: { float s, c; sincos_(x, &s, &c); return f2u(s); }
        case 10: { float s, c; sincos_(x, &s, &c); return f2u(c); }
        case 11: return f2u(pow025(x));
        case 12: return f2u(random_float(u));
        case 13: return f2u(exp2_(x));
        case 14: return f2u(exp_(x));
        case 15: return f2u(saturate(x));
        case 16: return f2u(f16_bits_to_f32((uint16_t)u));
        case 17: return f2u(unsnorm8(u));
        case 18: return f2u(unorm8(u));
        case 19: return f2u(unpack2x16unorm(u).x);
        default: return 0xDEADBEEFu;
    }
}
static uint32_t math_probe2(int fn, uint32_t ua, uint32_t ub) {
    const float a = u2f(ua), b = u2f(ub);
    switch (fn) {
        case 32: return f2u(fmin_(a, b));
        case 33: return f2u(fmax_(a, b));
        case 34: return f2u(clampf(a, b, 1.0f));
        case 35: return f2u(clampf(a, -1.0f, b));
        default: return 0xDEADBEEFu;
    }
}
// fn 40..: several words in and out, as tests/cuda/math_probe.cu probe_words()
static void math_probe_words(int fn, int& in, int& out) {
    in = fn >= 32 ? 2 : 1; out = 1;
    switch (fn) {
        case 40: case 45: in = 3; out = 3; break;
        case 41: in = 2; out = 2; break;
        case 42: in = 2; break;
        case 43: in = 3; break;
        case 44: in = 5; out = 3; break;
        case 50: in = 16; out = 16; break;
        case 51: in = 16; out = 32; break;
        case 52: in = 32; out = 16; break;
        default: break;
    }
}
static void math_probe_n(int fn, const uint32_t* a, uint32_t* o) {
    auto f = [&](int k) { return u2f(a[k]); };
    auto put3 = [&](vec3 r) { o[0] = f2u(r.x); o[1] = f2u(r.y); o[2] = f2u(r.z); };
    hk_packed_reservoir p;
    switch (fn) {
        case 40: put3(normalize(v3(f(0), f(1), f(2)))); break;
        case 41: { vec2 r = normalize(v2(f(0), f(1))); o[0] = f2u(r.x); o[1] = f2u(r.y); break; }
        case 42: o[0] = f2u(D_GGX(f(0), f(1))); break;
        case 43: o[0] = f2u(V_SmithGGXCorrelated(f(0), f(1), f(2))); break;
        case 44: put3(EnvBRDFApprox(v3(f(0), f(1), f(2)), f(3), f(4))); break;
        case 45: put3(reinhard_luminance(v3(f(0), f(1), f(2)))); break;
        case 50: memcpy(&p, a, 64); p = pack_reservoir(unpack_reservoir(p)); memcpy(o, &p, 64); break;
        case 51: {      // the unpacked state as 32 words (math_probe.cu P_UNPACK_RESERVOIR)
            memcpy(&p, a, 64);
            const Reservoir r = unpack_reservoir(p);
            const float v[32] = {r.s.radiance.x, r.s.radiance.y, r.s.radiance.z, r.s.radiance.w, r.s.random.x, r.s.random.y, r.s.random.z,
                                 r.s.random.w, r.s.visible_position.x, r.s.visible_position.y, r.s.visible_position.z, r.s.visible_position.w,
                                 r.s.visible_normal.x, r.s.visible_normal.y, r.s.visible_normal.z, 0.0f, r.s.sample_position.x,
                                 r.s.sample_position.y, r.s.sample_position.z, r.s.sample_position.w, r.s.sample_normal.x, r.s.sample_normal.y,
                                 r.s.sample_normal.z, r.count, r.lifetime, r.w, r.w_sum, r.w2_sum, 0.0f, 0.0f, 0.0f, 0.0f};
            for (int k = 0; k < 32; ++k) o[k] = f2u(v[k]);
            o[15] = r.s.visible_instance;
            break;
        }
        case 52: {
            Reservoir r;
            r.s.radiance = v4(f(0), f(1), f(2), f(3)); r.s.random = v4(f(4), f(5), f(6), f(7));
            r.s.visible_position = v4(f(8), f(9), f(10), f(11)); r.s.visible_normal = v3(f(12), f(13), f(14));
            r.s.visible_instance = a[15];
            r.s.sample_position = v4(f(16), f(17), f(18), f(19)); r.s.sample_normal = v3(f(20), f(21), f(22));
            r.count = f(23); r.lifetime = f(24); r.w = f(25); r.w_sum = f(26); r.w2_sum = f(27);
            p = pack_reservoir(r);
            memcpy(o, &p, 64);
            break;
        }
        default: o[0] = 0xDEADBEEFu; break;
    }
}
void hko_math_batch(int fn, const uint32_t* in, uint32_t* out, size_t n) {
    int win, wout;
    math_probe_words(fn, win, wout);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) {
        if (fn >= 40) math_probe_n(fn, in + i * win, out + i * wout);
        else out[i] = fn >= 32 ? math_probe2(fn, in[2 * i], in[2 * i + 1]) : math_probe1(fn, in[i]);
    }
}
void hko_math_batch_range(int fn, uint32_t first, uint32_t* out, size_t n) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = math_probe1(fn, first + (uint32_t)i);
}
// Per pixel of a w x h frame at upscale ratio 1: an FNV-1a digest over the pixel of every spatial neighbour and the pixels of its
// depth-march taps, as pass_spatial_reuse computes them (spatial_neighbour, spatial_tap_uv), for the rotation math_probe.cu draws
void hko_spatial_digest(uint32_t count, float range, int w, int h, uint32_t frame, uint32_t* out) {
    ivec2 size; size.x = w; size.y = h;
    const float random_frame = random_float(frame);
    const float tap_count_f = 4.0f + 1.0f;          // SPATIAL_REUSE_TAPS + 1
#pragma omp parallel for schedule(static)
    for (int64_t p = 0; p < (int64_t)w * h; ++p) {
        ivec2 coords; coords.x = (int)(p % w); coords.y = (int)(p / w);
        vec4 r;
        float* c = &r.x;
        for (uint32_t k = 0; k < 4u; ++k) c[k] = f16_bits_to_f32((uint16_t)(hash_u32((uint32_t)p * 4u + k + frame * 0x9E3779B9u) % 0x3C00u));
        const float rotation = sum4(r);
        const vec2 uv = coords_to_uv(coords, size);
        uint32_t d = 2166136261u;
        for (uint32_t i = 1u; i <= count; ++i) {
            float rad;
            vec2 offset;
            ivec2 sc = spatial_neighbour(coords, i, count, range, rotation, random_frame, rad, offset);
            d = (d ^ (uint32_t)sc.x) * 16777619u;
            d = (d ^ (uint32_t)sc.y) * 16777619u;
            float tap_interval = fmax_(1.0f, rad / tap_count_f);
            uint32_t tap_count = f32_to_u32(rad / tap_interval);
            for (uint32_t j = 1u; j <= tap_count; j += 1u) {
                vec2 t = spatial_tap_uv(uv, offset, (float)j * tap_interval, size);   // jittered_coords at ratio 1: uv + 0
                d = (d ^ (uint32_t)f32_to_i32(t.x * (float)w)) * 16777619u;
                d = (d ^ (uint32_t)f32_to_i32(t.y * (float)h)) * 16777619u;
            }
        }
        out[p] = d;
    }
}
// Per render pixel of a w x h frame at upscale ratio `ratio` in (1, 2]: four FNV-1a digests (math_probe.cu k_deferred_digest) of
//   [0] the light passes' G-buffer texel, Deferred::jittered_coords of coords_to_uv,
//   [1] the denoise passes' texel, Deferred::nearest of jittered_uv(uv, 0.5),
//   [2] load_previous's pixel of jittered_uv(uv, 0.25) - velocity, with the all(< 0.5) and the all(<= 0.5) test (scatter), for
//       velocity 0 and for the velocity math_probe.cu draws: the index, or ~0 outside.  The index is the reference's
//       coords.x + size.x * coords.y: a uv of exactly 1 in x is column 0 of the next row, one past the buffer counts as outside,
//   [3] for both tables, pass_spatial_reuse's neighbour pixels (spatial_neighbour), the texel of each one inside the frame and of each
//       of its depth-march taps (spatial_tap_uv).
void hko_deferred_digest(int w, int h, float ratio, uint32_t frame, uint32_t* out) {
    hko_context c;                  // what Deferred reads: the G-buffer size and the frame's upscale ratio and number
    c.W = w; c.H = h;
    memset(&c.in, 0, sizeof(c.in));
    c.in.frame.upscale_ratio = ratio;
    c.in.frame.number = frame;
    const float scale = 1.0f / ratio;       // begin()
    c.RW = (int)ceilf(scale * (float)c.W);
    c.RH = (int)ceilf(scale * (float)c.H);
    const Deferred g(c);
    ivec2 size; size.x = c.RW; size.y = c.RH;
    const float random_frame = random_float(frame);
    const float tap_count_f = 4.0f + 1.0f;          // SPATIAL_REUSE_TAPS + 1
    auto fnv = [](uint32_t d, uint32_t v) { return (d ^ v) * 16777619u; };
#pragma omp parallel for schedule(static)
    for (int64_t p = 0; p < (int64_t)size.x * size.y; ++p) {
        ivec2 coords; coords.x = (int)(p % size.x); coords.y = (int)(p / size.x);
        const vec2 uv = coords_to_uv(coords, size);
        uint32_t d[4] = {2166136261u, 2166136261u, 2166136261u, 2166136261u};
        ivec2 t = g.jittered_coords(uv);
        d[0] = fnv(fnv(d[0], (uint32_t)t.x), (uint32_t)t.y);
        t = g.nearest(g.jittered_uv(uv, 0.5f));
        d[1] = fnv(fnv(d[1], (uint32_t)t.x), (uint32_t)t.y);
        const uint32_t hv = hash_u32((uint32_t)p * 2u + frame * 0x85EBCA6Bu), gv = hash_u32(hv);       // math_probe.cu probe_velocity
        const vec2 velocities[2] = {v2(0.0f, 0.0f), v2((float)((int)(hv & 0x3FFFu) - 0x2000) * 0x1p-16f,
                                                       (float)((int)(gv & 0x3FFFu) - 0x2000) * 0x1p-16f)};
        for (const vec2& velocity : velocities) {
            const vec2 previous_uv = g.jittered_uv(uv, 0.25f) - v2(velocity.x, velocity.y);
            for (int inclusive = 0; inclusive < 2; ++inclusive) {
                uint32_t index = 0xFFFFFFFFu;
                if (inclusive ? uv_inside_eq(previous_uv) : uv_inside(previous_uv)) {
                    const int32_t i = uv_to_index(previous_uv, size);
                    if (i < size.x * size.y) index = (uint32_t)i;
                }
                d[2] = fnv(d[2], index);
            }
        }
        vec4 r;
        float* rc = &r.x;
        for (uint32_t k = 0; k < 4u; ++k) rc[k] = f16_bits_to_f32((uint16_t)(hash_u32((uint32_t)p * 4u + k + frame * 0x9E3779B9u) % 0x3C00u));
        const float rotation = sum4(r);
        const uint32_t counts[2] = {16u, 8u};
        const float ranges[2] = {20.0f, 10.0f};
        for (int table = 0; table < 2; ++table) {
            for (uint32_t i = 1u; i <= counts[table]; ++i) {
                float rad;
                vec2 offset;
                const ivec2 sc = spatial_neighbour(coords, i, counts[table], ranges[table], rotation, random_frame, rad, offset);
                d[3] = fnv(fnv(d[3], (uint32_t)sc.x), (uint32_t)sc.y);
                const vec2 sample_uv = coords_to_uv(sc, size);
                if (sample_uv.x < 0.0f || sample_uv.y < 0.0f || sample_uv.x > 1.0f || sample_uv.y > 1.0f) continue;
                t = g.jittered_coords(sample_uv);
                d[3] = fnv(fnv(d[3], (uint32_t)t.x), (uint32_t)t.y);
                const float tap_interval = fmax_(1.0f, rad / tap_count_f);
                const uint32_t tap_count = f32_to_u32(rad / tap_interval);
                for (uint32_t j = 1u; j <= tap_count; j += 1u) {
                    t = g.jittered_coords(spatial_tap_uv(uv, offset, (float)j * tap_interval, size));
                    d[3] = fnv(fnv(d[3], (uint32_t)t.x), (uint32_t)t.y);
                }
            }
        }
        for (int k = 0; k < 4; ++k) out[4 * p + k] = d[k];
    }
}

}  // extern "C"
