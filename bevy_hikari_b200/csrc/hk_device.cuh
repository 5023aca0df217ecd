// hk_device.cuh — device-side building blocks of the CUDA path: memory layout in HBM, 128-bit record loads,
// skip-link TLAS/BLAS traversal, light sampling, BRDF and ReSTIR state handling.
//
// Data layout (all per-pixel state is planar, row-major over the context's band of rows, so that a warp that owns an
// 8x4 pixel tile touches whole 32-byte sectors):
//   G-buffer      pos_depth float4 | normal snorm8x4 | depth_gradient float2 | instance_material float2 | velocity_uv float4
//   reservoirs    10 buffers x 4 planes of uint4 (the 64-byte PackedReservoir of light.wgsl:35-43 split in 16-byte
//                 quarters: q0 = radiance|random, q1 = visible_position, q2 = sample_position, q3 = normals|reservoir)
//   radiance      render[3], albedo, denoise scratch, output: Rgba16Float as uint2; variance[3]: float
// Scene records keep the reference's std430 layouts (include/hk_layout.h) and are fetched with 16-byte read-only loads.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "hikari_b200.h"
#include "hk_math.h"

// Inlining policy of the large device functions (code size vs call overhead; see DESIGN.md 4: the light kernels are
// instruction-fetch bound).  Override per function group with -DHK_INL_<GROUP>=__noinline__.
#ifndef HK_INL_PACK
#define HK_INL_PACK __forceinline__
#endif
#ifndef HK_INL_TRAVERSE
#define HK_INL_TRAVERSE __forceinline__
#endif
#ifndef HK_INL_HITINFO
#define HK_INL_HITINFO __forceinline__
#endif
#ifndef HK_INL_TEXTURE
#define HK_INL_TEXTURE __forceinline__
#endif
#ifndef HK_SURFACE_LOOP
#define HK_SURFACE_LOOP 0
#endif
#ifndef HK_INL_SURFACE
#define HK_INL_SURFACE __forceinline__
#endif
#ifndef HK_INL_SHADE
#define HK_INL_SHADE __forceinline__
#endif
#ifndef HK_INL_RADIANCE
#define HK_INL_RADIANCE __forceinline__
#endif
#ifndef HK_INL_SELECT
#define HK_INL_SELECT __forceinline__
#endif

namespace hkd {
using namespace hk;

// Compact per-instance record of the BVH walk: the 80 bytes of hk_instance (176 B) a TLAS leaf needs once the navigator's box
// test has passed — transpose(inverse_transpose_model) as stored (light.wgsl:306-316) and the mesh index.  Built at upload
// (context.cu) so that one TMA bulk copy stages all of them into shared memory (hk_pool.cuh).
struct hk_instance_trav {
    float inverse_transpose_model[16];
    uint32_t mesh[4];          // vertex, primitive, node_offset, node_count
};
static_assert(sizeof(hk_instance_trav) == 80, "5 float4 per instance");

// Where each staged scene array lives inside the pooled kernels' shared-memory stage, in float4 units; decided on the host per
// scene (context.cu).  A count of 0 means "not staged: read from global memory".
#define HK_STAGE_F4 1024               // float4 slots (16 KB) of staged scene records per CTA
struct StagePlan {
    uint32_t tlas_f4, tlas_count;      // instance_nodes: 2 float4 per record
    uint32_t itrav_f4, itrav_count;    // hk_instance_trav: 5 float4 per instance
    uint32_t blas_f4, blas_count;      // asset_nodes (whole buffer): 2 float4 per record
    uint32_t prim_f4, prim_count;      // primitives (whole buffer): 3 float4 per triangle
};

struct hk_wide_node;     // hk_wide.cuh: 4-wide BVH node of the image-exact traversal mode

struct DeviceScene {
    const hk_vertex* vertices;
    const hk_primitive* primitives;
    const hk_node* asset_nodes;
    const hk_alias_entry* alias_table;
    const hk_instance* instances;
    const hk_node* instance_nodes;
    const hk_material* materials;
    const hk_node* emissive_nodes;
    const hk_emissive* emissives;
    const cudaTextureObject_t* textures;   // unused by the NO_TEXTURE variant
    const float4* texture_texels;          // decoded texels of all textures, concatenated
    const uint4* texture_info;             // per texture: (offset, width, height, flags: bit0-1 mode_u, 2-3 mode_v, 4 linear)
    uint32_t instance_node_count, emissive_node_count, texture_count;
    uint32_t leaf_boxes_match;   // 1 = every leaf's navigator box equals the shape's own AABB (validated at upload)
    // previous-frame model matrices (4 float4 columns per instance) and a per-instance "moved" flag (previous != current,
    // compared bitwise on the host); both nullptr when no instance moved
    const float4* previous_models;
    const uint32_t* instance_moved;
    const hk_instance_trav* instance_trav;   // one per instance
    StagePlan stage;
    // image-exact traversal mode (hk_wide.cuh, built by wide_build.h at upload): 4-wide trees derived from the flat arrays above
    const hk_wide_node* wide_tlas;           // tree over the instances
    const hk_wide_node* wide_blas;           // the trees of all meshes, one after the other
    const uint2* wide_instance;              // per instance: first node of its mesh's tree in wide_blas | root reference
    const uint32_t* wide_instance_rank;      // per instance: position of its leaf in instance_nodes (array order = the reference's visit order)
    const uint32_t* wide_primitive_rank;     // per primitive: position of its leaf in its mesh's asset_nodes range
    uint32_t wide_tlas_root;
    uint32_t wide_ready;                     // 1 = every tree could be derived and fits the walk's stack
};

struct ReservoirPlanes {  // one PackedReservoir buffer as 4 planes
    uint4* q[4];
};

struct Planes {
    float4* pos_depth;          // current frame (= pos_depth_db[gbuffer_current]); previous frame = the other one (prepass.rs:312-321)
    uint32_t* normal;
    float2* depth_gradient;
    float2* instance_material;
    float4* velocity_uv;
    float* depth;               // pos_depth.w of the current frame as a plane of its own: what the TMA tile loads of kc_spatial stage
    float4* pos_depth_db[2];
    float4* velocity_uv_db[2];
    uint2* albedo;
    uint2* render[3];
    float* variance[3];
    ReservoirPlanes reservoir[10];
    // deterministic resolution of store_previous_spatial_reservoir(previous_coords) (light.wgsl:1094,1201,1458): writers
    // race for a target pixel in the reference; here the winner is the last writer in raster order (= the oracle's rule)
    uint32_t* scatter_key;          // per target pixel: max over writers of ((writer_linear_index + 1) << 2 | kind), 0 = none
    ReservoirPlanes scatter_value;  // per writer pixel: the reservoir a kind-2 (validation miss) write carries
    float4* dn_geometry;        // normalize(unpack(normal)).xyz | depth : what every a-trous tap needs, prepared once per frame
    float* dn_instance;         // instance id + 0.5 (instance_material.x)
    uint2* dn_internal[4][3];   // [level][signal]; level 0 = demodulated input
    float* dn_variance[3];
    uint2* dn_render[3];
    uint2* tone_mapped;         // owned rectangle only, tightly packed; = tone_mapped_db[frame.number % 2] (post_process.rs:716,979)
    uint2* tone_mapped_db[2];
    uint2* tone_ring_db[2];     // tiles with upscalers: the tone-mapped image over the tile's allocation (owned + 4-px ring + halo)
    uint2* upscale_output;      // Band::OW x OH (SMAA TU4x: ceil(size * 2 / ratio), <= 2 RW x 2 RH); tiles: 2 x the allocation.  W x H under Upscale::Fsr1 (the EASU result)
    uint2* upscale_sharpen_output;   // W x H, full-frame contexts: the RCAS result (post_process.rs:723 upscale_output[1])
    uint2* taa_output[2];       // [frame.number % 2] is written
};

// Row pitch (in pixels) of every per-pixel plane of an allocation `w` pixels wide: a multiple of 4, so that the pitch of a 4-byte
// plane is a multiple of 16 bytes (what a TMA tensor map requires of its strides, hk_tile.cuh).  The padding columns are never
// part of a launch rectangle.
__host__ __device__ inline int hk_plane_pitch(int w) { return (w + 3) & ~3; }

struct Band {             // the tile of the frame one context renders (whole frame: everything 0..W, 0..H)
    int W, H;             // full image
    int ax0, ax1, a0, a1; // allocated rectangle: columns [ax0,ax1), rows [a0,a1) = owned +- ghost, clamped to the image
    int cx0, cx1, r0, r1; // owned rectangle: columns [cx0,cx1), rows [r0,r1)
    int AW;               // hk_plane_pitch(ax1 - ax0): row stride of the deferred-size planes (G-buffer, albedo)
    // render size = ceil(size / upscale_ratio) (light.rs:622-624).  At ratio 1 (every tiled / benchmark configuration)
    // render space == deferred space and RS == AW; at ratio > 1 (full-frame contexts only) render-size planes use stride RW.
    int RW, RH, RS;
    // extent of the SMAA TU4x output (and of the TAA images that follow it): ceil(size * (2 / ratio)) in f32 as create_texture computes it
    // (post_process.rs:663-667,715-721) — 2 RW x 2 RH except where the two ceilings disagree (ratio 2 on an odd width: W, not W + 1)
    int OW, OH;
};

struct Counters { unsigned long long primary, tlas, blas; };

// Per-neighbour constants of spatial_reuse (light.wgsl:1566-1572,1609-1620): they depend only on the neighbour index i,
// so they are evaluated once on the host (same IEEE sqrt / division as the shader expression) instead of per pixel.
struct SpatialTable {
    float phase[17];        // f32(i) * GOLDEN_RATIO
    float radius[17];       // sqrt(f32(i) / f32(COUNT)) * RANGE
    uint32_t tap_count[17]; // u32(radius / max(1, radius / (TAPS + 1)))
    float tap_dist[17][6];  // f32(j) * tap_interval, j = 1..tap_count  (tap_count is 5 when radius >= 5: r / (r/5))
    float tap_ratio[17][6]; // f32(j) / f32(tap_count + 1)
};

struct KParams {
    hk_frame_inputs in;
    DeviceScene scene;
    Planes planes;
    Band band;
    Counters* counters;     // nullptr = counting compiled in but disabled at run time
    const uint8_t* noise;   // 16 x 64 x 64 x 4
    int row_lo, row_hi;     // rows this launch covers (global)
    int col_lo, col_hi;     // columns this launch covers (global)
    float cos_solar_angle;  // cos(frame.solar_angle), hk::sincos_ evaluated once on the host with the same routine
    float random_frame;     // random_float(frame.number)
    const SpatialTable* spatial_tables;   // [0] = indirect (16 neighbours, 20 px), [1] = emissive (8 neighbours, 10 px)
    int ratio1;             // upscale_ratio == 1: deferred coordinates are the render coordinates
    float jitter_sign;      // -1 on even frames, +1 on odd frames (light.wgsl:1010, denoise.wgsl:40)
    float ratio_m1;         // upscale_ratio - 1
    int gbuffer_current;    // which of the double-buffered position / velocity_uv planes is "current" this frame
    // frame assembly (hk_set_frame_target): a full-frame Rgba16Float image, possibly in a peer GPU's memory (NVLink), that
    // receives this context's owned pixels at their global position; nullptr = none
    uint2* frame_target;
    uint32_t frame_pitch;   // pixels
    float inv_rw, inv_rh;   // RN(1 / RW), RN(1 / RH), computed on the host (HK_SPATIAL_FAST_DIV)
    int tile_images;        // 1 = tile context with the temporal upscalers enabled: render-size images are stored over the allocation
};

// --------------------------------------------------------------------------------------------- raw loads
__device__ __forceinline__ float4 ldg4(const void* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ uint4 ldg4u(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ vec3 f4xyz(float4 a) { return v3(a.x, a.y, a.z); }
__device__ __forceinline__ vec4 f4v(float4 a) { return v4(a.x, a.y, a.z, a.w); }
__device__ __forceinline__ float4 vf4(vec4 a) { return make_float4(a.x, a.y, a.z, a.w); }

struct Ray { vec3 origin, direction, inv_direction; };
struct Hit { float u, v, distance; uint32_t instance_index, primitive_index; };
struct HitInfo { vec4 position; vec3 normal; vec2 uv; uint32_t instance_index, material_index; };
struct Surface { vec4 base_color, emissive; float reflectance, metallic, roughness, occlusion; };
struct LightCandidate { vec3 direction; float max_distance, min_distance; uint32_t emissive_instance; float p; };

struct Sample {
    vec4 radiance, random, visible_position;
    vec3 visible_normal;
    uint32_t visible_instance;
    vec4 sample_position;
    vec3 sample_normal;
};
struct Reservoir { Sample s; float count, lifetime, w, w_sum, w2_sum; };

__device__ __forceinline__ Sample zero_sample() {
    Sample s;
    s.radiance = v4(0.0f); s.random = v4(0.0f); s.visible_position = v4(0.0f); s.visible_normal = v3(0.0f);
    s.visible_instance = 0u; s.sample_position = v4(0.0f); s.sample_normal = v3(0.0f);
    return s;
}
__device__ __forceinline__ Reservoir zero_reservoir() {
    Reservoir r;
    r.s = zero_sample(); r.count = 0.0f; r.lifetime = 0.0f; r.w = 0.0f; r.w_sum = 0.0f; r.w2_sum = 0.0f;
    return r;
}

// ------------------------------------------------------------------------------ reservoir quarters <-> state
// light.wgsl:77-136 on the planar layout.
struct PackedQuarters { uint4 q0, q1, q2, q3; };

static __device__ HK_INL_PACK Reservoir unpack_reservoir(const PackedQuarters& p) {
    Reservoir r;
    vec2 t0 = unpack2x16float(p.q3.z), t1 = unpack2x16float(p.q3.w);
    r.count = t0.x; r.w = t0.y; r.w_sum = t1.x; r.w2_sum = t1.y;
    t0 = unpack2x16float(p.q0.x); t1 = unpack2x16float(p.q0.y);
    r.s.radiance = v4(t0.x, t0.y, t1.x, t1.y);
    t0 = unpack2x16unorm(p.q0.z); t1 = unpack2x16unorm(p.q0.w);
    r.s.random = v4(t0.x, t0.y, t1.x, t1.y);
    vec4 t2 = unpack4x8snorm(p.q3.x);
    r.s.visible_position = v4(__uint_as_float(p.q1.x), __uint_as_float(p.q1.y), __uint_as_float(p.q1.z), __uint_as_float(p.q1.w));
    r.s.visible_normal = normalize(xyz(t2));
    r.lifetime = 127.0f * (1.0f + t2.w);
    t2 = unpack4x8snorm(p.q3.y);
    r.s.sample_position = v4(__uint_as_float(p.q2.x), __uint_as_float(p.q2.y), __uint_as_float(p.q2.z), t2.w);
    r.s.sample_normal = normalize(xyz(t2));
    r.s.visible_instance = f32_to_u32(__uint_as_float(p.q2.w));
    return r;
}
static __device__ HK_INL_PACK PackedQuarters pack_reservoir(const Reservoir& r) {
    PackedQuarters p;
    p.q0.x = pack2x16float(r.s.radiance.x, r.s.radiance.y);
    p.q0.y = pack2x16float(r.s.radiance.z, r.s.radiance.w);
    p.q0.z = pack2x16unorm(r.s.random.x, r.s.random.y);
    p.q0.w = pack2x16unorm(r.s.random.z, r.s.random.w);
    p.q1 = make_uint4(__float_as_uint(r.s.visible_position.x), __float_as_uint(r.s.visible_position.y),
                      __float_as_uint(r.s.visible_position.z), __float_as_uint(r.s.visible_position.w));
    p.q2 = make_uint4(__float_as_uint(r.s.sample_position.x), __float_as_uint(r.s.sample_position.y),
                      __float_as_uint(r.s.sample_position.z), __float_as_uint((float)r.s.visible_instance));
    p.q3.x = pack4x8snorm(v4(r.s.visible_normal, add_rn(div_rn(r.lifetime, 127.0f), -1.0f)));   // IEEE in a tolerance unit too
    p.q3.y = pack4x8snorm(v4(r.s.sample_normal, r.s.sample_position.w));
    p.q3.z = pack2x16float(r.count, r.w);
    p.q3.w = pack2x16float(r.w_sum, r.w2_sum);
    return p;
}
__device__ __forceinline__ PackedQuarters load_quarters(const ReservoirPlanes& b, size_t i) {
    PackedQuarters p;
    p.q0 = b.q[0][i]; p.q1 = b.q[1][i]; p.q2 = b.q[2][i]; p.q3 = b.q[3][i];
    return p;
}
__device__ __forceinline__ void store_quarters(const ReservoirPlanes& b, size_t i, const PackedQuarters& p) {
    b.q[0][i] = p.q0; b.q[1][i] = p.q1; b.q[2][i] = p.q2; b.q[3][i] = p.q3;
}

// light.wgsl:138-179
__device__ __forceinline__ void set_reservoir(Reservoir& r, const Sample& s, float w_new) {
    r.count = 1.0f; r.lifetime = 0.0f; r.w_sum = w_new; r.w2_sum = w_new * w_new; r.s = s;
}
__device__ __forceinline__ void update_reservoir(Reservoir& r, const Sample& s, float w_new) {
    r.w_sum += w_new;
    r.w2_sum += w_new * w_new;
    r.count = r.count + 1.0f;
    float rnd = fract(sum4(s.random));
    if (rnd < w_new / r.w_sum) r.s = s;
}
__device__ __forceinline__ void merge_reservoir(Reservoir& r, const Reservoir& other, float p) {
    float count = r.count;
    update_reservoir(r, other.s, p * other.w * other.count);
    r.count = count + other.count;
}
// light.wgsl:917-952
__device__ __forceinline__ bool check_previous_reservoir(Reservoir& r, const Sample& s) {
    float depth_ratio = r.s.visible_position.w / s.visible_position.w;
    depth_ratio = (depth_ratio < 1.0f) ? 1.0f / depth_ratio : depth_ratio;
    bool depth_miss = depth_ratio > 1.05f * (1.0f + 0.5f * s.random.x);
    bool instance_miss = r.s.visible_instance != s.visible_instance;
    bool normal_miss = dot(s.visible_normal, r.s.visible_normal) < 0.9f;
    if (depth_miss || normal_miss || instance_miss) { r = zero_reservoir(); return false; }
    return true;
}
__device__ __forceinline__ void temporal_restir(Reservoir& r, const Sample& s, float w_new, uint32_t max_sample_count) {
    update_reservoir(r, s, w_new);
    float m = (float)max_sample_count;
    if (r.count > m) {
        r.w_sum *= m / r.count;
        r.w2_sum *= m / r.count;
        r.count = m;
    }
}
__device__ __forceinline__ float variance_of(const Reservoir& r) {  // light.wgsl:1224-1226
    float variance = r.w2_sum / r.count - sq(r.w_sum / r.count);
    variance = (r.count < 1.0f) ? variance : variance / r.count;
    return fmin_(variance, MAX_VARIANCE);
}
__device__ __forceinline__ float compute_jacobian(const Sample& q, const Sample& r) {  // light.wgsl:985-1004
    vec3 normal = q.sample_normal;
    vec3 qs = xyz(q.sample_position);
    float cos_phi_1 = fabsf(dot(normalize(xyz(r.visible_position) - qs), normal));
    float cos_phi_2 = fabsf(dot(normalize(xyz(q.visible_position) - qs), normal));
    float term_1 = cos_phi_1 / fmax_(0.0001f, cos_phi_2);
    float num = length(xyz(q.visible_position) - qs);
    num *= num;
    float denom = length(xyz(r.visible_position) - qs);
    denom *= denom;
    float term_2 = num / fmax_(denom, 0.0001f);
    return clampf(term_1 * term_2, 1.0f, 50.0f);
}

// --------------------------------------------------------------------------------------------- traversal
// Slab test, light.wgsl:344-362.  Returns t_min or F32_MAX.
__device__ __forceinline__ float slab(const Ray& ray, vec3 bmin, vec3 bmax) {
    vec3 t1 = (bmin - ray.origin) * ray.inv_direction;
    vec3 t2 = (bmax - ray.origin) * ray.inv_direction;
    float t_min = fmin_(t1.x, t2.x);
    float t_max = fmax_(t1.x, t2.x);
    t_min = fmax_(t_min, fmin_(t1.y, t2.y));
    t_max = fmin_(t_max, fmax_(t1.y, t2.y));
    t_min = fmax_(t_min, fmin_(t1.z, t2.z));
    t_max = fmin_(t_max, fmax_(t1.z, t2.z));
    return (t_max >= t_min && t_max >= 0.0f) ? t_min : F32_MAX;
}

// Moeller-Trumbore, light.wgsl:364-398.  Returns distance (F32_MAX on miss) and the (u,v) the reference would leave
// in Intersection.uv for every exit path (they are stored only on a hit, but keep the exact values anyway).
__device__ __forceinline__ float triangle(const Ray& ray, vec3 p0, vec3 p1, vec3 p2, float& u_out, float& v_out) {
    vec3 ab = p1 - p0;
    vec3 ac = p2 - p0;
    vec3 u_vec = cross(ray.direction, ac);
    float det = dot(ab, u_vec);
    u_out = 0.0f; v_out = 0.0f;
    if (fabsf(det) < F32_EPSILON) return F32_MAX;
    float inv_det = 1.0f / det;
    vec3 ao = ray.origin - p0;
    float u = dot(ao, u_vec) * inv_det;
    u_out = u;
    if (u < 0.0f || u > 1.0f) return F32_MAX;
    vec3 v_vec = cross(ao, ab);
    float v = dot(ray.direction, v_vec) * inv_det;
    v_out = v;
    if (v < 0.0f || u + v > 1.0f) return F32_MAX;
    float distance = dot(ac, v_vec) * inv_det;
    return (distance > F32_EPSILON) ? distance : F32_MAX;
}

// BLAS walk, light.wgsl:400-440.  Visit order and the strict '<' updates are the reference's, so ties between
// equidistant triangles and the any-hit winner (early_distance) resolve identically.
__device__ __forceinline__ bool traverse_bottom(const DeviceScene& sc, Hit& hit, const Ray& ray, uint32_t mesh_primitive,
                                                uint32_t node_offset, uint32_t node_count, float early_distance) {
    bool intersected = false;
    const hk_node* nodes = sc.asset_nodes + node_offset;
    uint32_t index = 0;
    while (index < node_count) {
        const float4 n0 = ldg4(&nodes[index]);                                           // min.xyz | entry_index
        const float4 n1 = ldg4(reinterpret_cast<const float4*>(&nodes[index]) + 1);      // max.xyz | exit_index
        const uint32_t entry = __float_as_uint(n0.w);
        if (entry >= BVH_LEAF_FLAG) {
            const bool via_navigator = index != 0u && sc.leaf_boxes_match != 0u;         // see traverse_top
            const uint32_t primitive_index = mesh_primitive + entry - BVH_LEAF_FLAG;
            const hk_primitive* prim = sc.primitives + primitive_index;
            const float4 a = ldg4(&prim->vertices[0]), b = ldg4(&prim->vertices[1]), c = ldg4(&prim->vertices[2]);
            const vec3 p0 = f4xyz(a), p1 = f4xyz(b), p2 = f4xyz(c);
            if (via_navigator || slab(ray, vmin(p0, vmin(p1, p2)), vmax(p0, vmax(p1, p2))) < hit.distance) {
                float u, v;
                const float distance = triangle(ray, p0, p1, p2, u, v);
                if (distance < hit.distance) {
                    hit.u = u; hit.v = v; hit.distance = distance;
                    hit.primitive_index = primitive_index;
                    intersected = true;
                    if (distance < early_distance) return true;
                }
            }
            index = __float_as_uint(n1.w);
        } else {
            index = (slab(ray, f4xyz(n0), f4xyz(n1)) < hit.distance) ? entry : __float_as_uint(n1.w);
        }
    }
    return intersected;
}

// world -> object space with transpose(inverse_transpose_model), light.wgsl:306-316
__device__ __forceinline__ void instance_ray(const hk_instance* inst, const Ray& ray, Ray& r) {
    const float4* m = reinterpret_cast<const float4*>(inst->inverse_transpose_model);
    vec4 c0 = f4v(ldg4(m)), c1 = f4v(ldg4(m + 1)), c2 = f4v(ldg4(m + 2)), c3 = f4v(ldg4(m + 3));
    vec4 o = v4(ray.origin, 1.0f), d = v4(ray.direction, 0.0f);
    vec4 po = v4(dot(c0, o), dot(c1, o), dot(c2, o), dot(c3, o));
    r.origin = (po.w == 1.0f) ? xyz(po) : xyz(po) / po.w;     // x / 1 == x exactly: affine instances skip three divisions
    r.direction = v3(dot(c0, d), dot(c1, d), dot(c2, d));
    r.inv_direction = 1.0f / r.direction;
}

// TLAS + BLAS walk, light.wgsl:442-486 with traverse_bottom (:400-440) inlined as ONE loop ("if-if" instead of
// "while-while"): every iteration performs one node step of whichever level the lane is in.  TLAS and BLAS records share
// one format and one slab test, so lanes that are inside different instances' BLASes and lanes that are still walking
// the TLAS execute the same interior-node code together instead of serialising inner against outer loop, where the nested
// form leaves most lanes of a warp idle on secondary rays.  Visit order, the strict '<'
// updates and both early-outs are unchanged, so hits are bit-identical to the nested walk.
// Ending phase 1 on a warp vote (as soon as at most 1/2 .. 1/8 of the lanes are still on interior records) instead of waiting for
// the last lane was tried and not kept: the votes and the per-lane state machine cost what the shorter waits save.
static __device__ HK_INL_TRAVERSE Hit traverse_top(const DeviceScene& sc, const Ray& ray, float max_distance, float early_distance,
                                            uint32_t exclude_instance) {
    Hit hit;
    hit.u = 0.0f; hit.v = 0.0f; hit.distance = max_distance;
    hit.instance_index = U32_MAX; hit.primitive_index = U32_MAX;
    const hk_node* nodes = sc.instance_nodes;
    uint32_t count = sc.instance_node_count;
    uint32_t index = 0;
    Ray cur = ray;                 // world-space ray while in the TLAS, object-space ray while in a BLAS
    bool in_blas = false, blas_hit = false;
    uint32_t tlas_resume = 0, instance_index = 0, mesh_primitive = 0;
    for (;;) {
        // phase 1 — every lane steps over interior (navigator) records until it stands on a leaf record or its level is
        // exhausted.  Lanes reconverge after this loop, so the expensive leaf work below (instance transform, triangle
        // test) runs with all lanes that have a leaf pending instead of the 3-4 that happen to be in phase with each other.
        uint32_t entry = 0, exit_index = 0;
        while (index < count) {
            // both halves of the record in one round trip (a leaf record only needs .w of each)
            const float4 n0 = ldg4(&nodes[index]);                                           // min.xyz | entry_index
            const float4 n1 = ldg4(reinterpret_cast<const float4*>(&nodes[index]) + 1);      // max.xyz | exit_index
            entry = __float_as_uint(n0.w);
            exit_index = __float_as_uint(n1.w);
            if (entry >= BVH_LEAF_FLAG) break;
            index = (slab(cur, f4xyz(n0), f4xyz(n1)) < hit.distance) ? entry : exit_index;
        }
        if (index >= count) {
            if (!in_blas) break;
            // traverse_bottom returned: back to the TLAS record after the instance leaf
            in_blas = false;
            if (blas_hit) {
                hit.instance_index = instance_index;
                if (hit.distance < early_distance) break;
            }
            nodes = sc.instance_nodes; count = sc.instance_node_count; index = tlas_resume;
            cur = ray;
            continue;
        }
        // phase 2 — leaf record.  A leaf record is only ever reached through its navigator (the record before it), whose
        // box is the shape's own AABB (bvh 0.7.1 stores the child's joint AABB = min/max of the triangle's vertices, resp.
        // the instance's min/max) and whose slab test against the same ray and the same hit.distance has just passed.
        // The reference repeats that test on the re-derived box (light.wgsl:411-414, 456-459); it cannot fail, so it is
        // skipped — except for the root of a single-shape BVH (index 0), which has no navigator.
        const bool via_navigator = index != 0u && sc.leaf_boxes_match != 0u;
        index = exit_index;
        if (!in_blas) {
            const uint32_t candidate = entry - BVH_LEAF_FLAG;
            if (candidate != exclude_instance) {
                const hk_instance* inst = sc.instances + candidate;
                bool pass = via_navigator;
                if (!pass) {
                    const float4 imin = ldg4(inst->min), imax = ldg4(inst->max);
                    pass = slab(ray, f4xyz(imin), f4xyz(imax)) < hit.distance;
                }
                if (pass) {
                    instance_ray(inst, ray, cur);
                    const uint4 mesh = ldg4u(&inst->mesh);     // vertex, primitive, node_offset, node_count
                    in_blas = true; blas_hit = false;
                    tlas_resume = exit_index; instance_index = candidate; mesh_primitive = mesh.y;
                    nodes = sc.asset_nodes + mesh.z; count = mesh.w; index = 0;
                }
            }
        } else {
            const uint32_t primitive_index = mesh_primitive + entry - BVH_LEAF_FLAG;
            const hk_primitive* prim = sc.primitives + primitive_index;
            const float4 a = ldg4(&prim->vertices[0]), b = ldg4(&prim->vertices[1]), c = ldg4(&prim->vertices[2]);
            const vec3 p0 = f4xyz(a), p1 = f4xyz(b), p2 = f4xyz(c);
            if (via_navigator || slab(cur, vmin(p0, vmin(p1, p2)), vmax(p0, vmax(p1, p2))) < hit.distance) {
                float u, v;
                const float distance = triangle(cur, p0, p1, p2, u, v);
                if (distance < hit.distance) {
                    hit.u = u; hit.v = v; hit.distance = distance;
                    hit.primitive_index = primitive_index;
                    blas_hit = true;
                    if (distance < early_distance) {           // traverse_bottom returns, traverse_top returns
                        hit.instance_index = instance_index;
                        break;
                    }
                }
            }
        }
    }
    return hit;
}

__device__ __forceinline__ vec3 instance_normal_local_to_world(const hk_instance* inst, vec3 n) {  // light.wgsl:324-338
    const float4* m = reinterpret_cast<const float4*>(inst->inverse_transpose_model);
    mat3 t;
    t.c[0] = f4xyz(ldg4(m)); t.c[1] = f4xyz(ldg4(m + 1)); t.c[2] = f4xyz(ldg4(m + 2));
    return normalize(mul(t, n));
}
__device__ __forceinline__ HitInfo empty_hit_info(vec3 position, vec3 direction) {  // light.wgsl:488-494
    HitInfo info;
    info.instance_index = U32_MAX; info.material_index = U32_MAX;
    info.position = v4(position + direction * DISTANCE_MAX, 0.0f);
    info.normal = v3(0.0f); info.uv = v2(0.0f, 0.0f);
    return info;
}
static __device__ HK_INL_HITINFO HitInfo hit_info(const DeviceScene& sc, const Ray& ray, const Hit& hit) {  // light.wgsl:496-523
    HitInfo info;
    info.instance_index = hit.instance_index;
    info.material_index = U32_MAX;
    info.normal = v3(0.0f); info.uv = v2(0.0f, 0.0f);
    if (hit.instance_index != U32_MAX) {
        const hk_instance* inst = sc.instances + hit.instance_index;
        const hk_primitive* prim = sc.primitives + hit.primitive_index;
        uint32_t vbase = __ldg(&inst->mesh.vertex);
        const hk_vertex* va = sc.vertices + vbase + __ldg(&prim->vertices[0].index);
        const hk_vertex* vb = sc.vertices + vbase + __ldg(&prim->vertices[1].index);
        const hk_vertex* vc = sc.vertices + vbase + __ldg(&prim->vertices[2].index);
        float4 a0 = ldg4(va), a1 = ldg4(reinterpret_cast<const float4*>(va) + 1);  // pos|u , normal|v
        float4 b0 = ldg4(vb), b1 = ldg4(reinterpret_cast<const float4*>(vb) + 1);
        float4 c0 = ldg4(vc), c1 = ldg4(reinterpret_cast<const float4*>(vc) + 1);
        vec2 uv0 = v2(a0.w, a1.w), uv1 = v2(b0.w, b1.w), uv2 = v2(c0.w, c1.w);
        info.uv = uv0 + hit.u * (uv1 - uv0) + hit.v * (uv2 - uv0);
        vec3 n0 = f4xyz(a1), n1 = f4xyz(b1), n2 = f4xyz(c1);
        vec3 n = n0 + hit.u * (n1 - n0) + hit.v * (n2 - n0);
        info.normal = instance_normal_local_to_world(inst, n);
        info.position = v4(ray.origin + ray.direction * hit.distance, 1.0f);
        info.material_index = __ldg(&inst->material);
    } else {
        info.position = v4(ray.origin + ray.direction * DISTANCE_MAX, 0.0f);
    }
    return info;
}
__device__ __forceinline__ void occlude_hit_info(const Ray& ray, const Hit& hit, HitInfo& info) {  // light.wgsl:526-533
    if (hit.instance_index != U32_MAX) {
        info.instance_index = hit.instance_index;
        info.material_index = U32_MAX;
        info.position = v4(ray.origin + ray.direction * hit.distance, 1.0f);
        info.normal = v3(0.0f);
    }
}

// ---------------------------------------------------------------------------------------------- sampling
__device__ __forceinline__ vec4 sample_cosine_hemisphere(float rx, float ry) {  // light.wgsl:537-549
    float r = sqrtf(rx);
    float s, c;
    sincos_(2.0f * PI * ry, &s, &c);
    float tx = r * c, ty = r * s;
    float z = sqrtf(1.0f - dot(v2(tx, ty), v2(tx, ty)));
    return v4(tx, ty, z, 2.0f * INV_TAU * z);
}
__device__ __forceinline__ vec3 sample_uniform_cone_dir(float rx, float ry, float cos_angle) {  // light.wgsl:552-559
    float z = 1.0f - (1.0f - cos_angle) * rx;
    float s, c;
    sincos_(TAU * ry, &s, &c);
    float r = sqrtf(1.0f - z * z);
    return v3(r * c, r * s, z);
}
__device__ __forceinline__ vec3 compute_emissive_radiance(vec4 emissive) { return 255.0f * emissive.w * xyz(emissive); }

// Texture fetch for the textured variant (light.wgsl:756): manual bilinear on pre-decoded float4 texels so that the
// weights are fp32 like the oracle's (CUDA texture units filter with 9-bit weights).
__device__ __forceinline__ int wrap_coord(int i, int n, uint32_t mode) {
    // texel coordinates of uv in [0, 1) are already inside the texture: every addressing mode is the identity there, and the
    // integer modulo by a run-time size (an emulated division on the GPU) is only needed for coordinates that really wrap
    if ((unsigned)i < (unsigned)n) return i;
    if (mode == 0u) { i %= n; if (i < 0) i += n; return i; }
    if (mode == 1u) return min(max(i, 0), n - 1);
    int period = 2 * n; i %= period; if (i < 0) i += period;
    return (i < n) ? i : period - 1 - i;
}
static __device__ HK_INL_TEXTURE vec4 sample_texture(const DeviceScene& sc, uint32_t id, vec2 uv) {
    uint4 ti = __ldg(&sc.texture_info[id]);
    const float4* tex = sc.texture_texels + ti.x;
    int w = (int)ti.y, h = (int)ti.z;
    uint32_t mu = ti.w & 3u, mv = (ti.w >> 2) & 3u;
    if (!(ti.w & 16u)) {
        int x = (int)floorf(uv.x * (float)w), y = (int)floorf(uv.y * (float)h);
        return f4v(__ldg(&tex[(size_t)wrap_coord(y, h, mv) * w + wrap_coord(x, w, mu)]));
    }
    float fx = uv.x * (float)w - 0.5f, fy = uv.y * (float)h - 0.5f;
    float x0f = floorf(fx), y0f = floorf(fy);
    float ax = fx - x0f, ay = fy - y0f;
    int x0 = (int)x0f, y0 = (int)y0f;
    int xa = wrap_coord(x0, w, mu), xb = wrap_coord(x0 + 1, w, mu);
    int ya = wrap_coord(y0, h, mv), yb = wrap_coord(y0 + 1, h, mv);
    vec4 t00 = f4v(__ldg(&tex[(size_t)ya * w + xa])), t10 = f4v(__ldg(&tex[(size_t)ya * w + xb]));
    vec4 t01 = f4v(__ldg(&tex[(size_t)yb * w + xa])), t11 = f4v(__ldg(&tex[(size_t)yb * w + xb]));
    vec4 top = t00 * (1.0f - ax) + t10 * ax;
    vec4 bot = t01 * (1.0f - ax) + t11 * ax;
    return top * (1.0f - ay) + bot * ay;
}

// retreive_surface, light.wgsl:730-742 (NO_TEXTURE) / 749-781
static __device__ HK_INL_SURFACE Surface retreive_surface(const DeviceScene& sc, uint32_t material_index, vec2 uv) {
    const float4* m = reinterpret_cast<const float4*>(sc.materials + material_index);
    float4 base = ldg4(m), t0 = ldg4(m + 1), emis = ldg4(m + 2), t1 = ldg4(m + 3), t2 = ldg4(m + 4);
    Surface s;
    s.base_color = f4v(base);
    s.emissive = f4v(emis);
    s.metallic = t1.z;
    s.occlusion = 1.0f;
    if (sc.texture_count != 0u) {
#if HK_SURFACE_LOOP
        // Tuning variant (off by default; validated on the emulated kernels, not yet timed): ONE inlined copy of the sampler
        // in a rolled loop over the four texture slots instead of four copies — the same look-ups and products in the same
        // order, 1 458 -> ~500 SASS instructions per retreive_surface site of the textured kernels (city, scene.rs)
        const uint32_t id0 = __float_as_uint(t0.x), id1 = __float_as_uint(t1.x), id2 = __float_as_uint(t1.w), id3 = __float_as_uint(t2.z);
#pragma unroll 1
        for (int k = 0; k < 4; ++k) {
            const uint32_t id = k == 0 ? id0 : (k == 1 ? id1 : (k == 2 ? id2 : id3));
            if (id == U32_MAX) continue;
            const vec4 t = sample_texture(sc, id, uv);
            if (k == 0) s.base_color = s.base_color * t;
            else if (k == 1) s.emissive = s.emissive * t;
            else if (k == 2) s.metallic *= t.x;
            else s.occlusion = t.x;
        }
#else
        uint32_t id = __float_as_uint(t0.x);
        if (id != U32_MAX) s.base_color = s.base_color * sample_texture(sc, id, uv);
        id = __float_as_uint(t1.x);
        if (id != U32_MAX) s.emissive = s.emissive * sample_texture(sc, id, uv);
        id = __float_as_uint(t1.w);
        if (id != U32_MAX) s.metallic *= sample_texture(sc, id, uv).x;
        id = __float_as_uint(t2.z);
        if (id != U32_MAX) s.occlusion = sample_texture(sc, id, uv).x;
#endif
    }
    s.roughness = perceptualRoughnessToRoughness(t1.y);
    s.reflectance = t2.x;
    return s;
}
static __device__ HK_INL_SURFACE vec4 retreive_emissive(const DeviceScene& sc, uint32_t material_index, vec2 uv) {  // light.wgsl:744-747 / 783-793
    const float4* m = reinterpret_cast<const float4*>(sc.materials + material_index);
    vec4 emissive = f4v(ldg4(m + 2));
    if (sc.texture_count != 0u) {
        uint32_t id = __float_as_uint(ldg4(m + 3).x);
        if (id != U32_MAX) emissive = emissive * sample_texture(sc, id, uv);
    }
    return emissive;
}

// ----------------------------------------------------------------------------------------------- shading
struct ShadeEnv {  // per-frame lighting constants pulled once into registers
    vec3 sun_dir; float cos_solar; vec3 sun_color; vec3 ambient; vec3 eye; bool ortho; vec3 ortho_dir;
};
__device__ __forceinline__ ShadeEnv make_env(const KParams& P) {
    ShadeEnv e;
    e.sun_dir = v3(P.in.lights.direction_to_light[0], P.in.lights.direction_to_light[1], P.in.lights.direction_to_light[2]);
    e.cos_solar = P.cos_solar_angle;
    e.sun_color = v3(P.in.lights.directional_color[0], P.in.lights.directional_color[1], P.in.lights.directional_color[2]);
    e.ambient = v3(P.in.lights.ambient_color[0], P.in.lights.ambient_color[1], P.in.lights.ambient_color[2]);
    e.eye = v3(P.in.view.world_position[0], P.in.view.world_position[1], P.in.view.world_position[2]);
    e.ortho = P.in.view.projection[15] == 1.0f;                       // light.wgsl:1040
    e.ortho_dir = v3(P.in.view.view_proj[2], P.in.view.view_proj[6], P.in.view.view_proj[10]);
    return e;
}
__device__ __forceinline__ vec3 calculate_view(const ShadeEnv& e, vec3 world_position) {  // light.wgsl:714-727
    return e.ortho ? normalize(e.ortho_dir) : normalize(e.eye - world_position);
}
__device__ __forceinline__ vec3 env_terms(vec3 diffuse_color, vec3 F0, float roughness, float NdotV) {
    return EnvBRDFApprox(diffuse_color, 1.0f, NdotV) + EnvBRDFApprox(F0, roughness, NdotV);
}
static __device__ HK_INL_SHADE vec3 env_brdf(vec3 V, vec3 N, const Surface& s) {  // light.wgsl:890-908
    vec3 base_color = xyz(s.base_color);
    float NdotV = fmax_(dot(N, V), 0.0001f);
    vec3 F0 = v3(0.16f * s.reflectance * s.reflectance * (1.0f - s.metallic)) + base_color * s.metallic;
    vec3 diffuse_color = base_color * (1.0f - s.metallic);
    return s.occlusion * env_terms(diffuse_color, F0, s.roughness, NdotV);
}
// shading = mix(lit, ambient, 1 - a), light.wgsl:796-888, split in the part that depends only on (V, N, surface) and
// the part that depends on the light direction and radiance: the spatial-reuse kernel shades up to 18 samples against
// the same surface point, so the first part (two EnvBRDFApprox with an exp2 each, F0, f90, N.V) is evaluated once.
// Operations and their order are exactly those of the single-call form, so results are bit-identical.
struct ShadeCtx {
    vec3 V, N, F0, diffuse_color, ambient_radiance;
    float roughness, NdotV, f90;
};
__device__ __forceinline__ ShadeCtx make_shade_ctx(const ShadeEnv& e, vec3 V, vec3 N, const Surface& s) {
    ShadeCtx c;
    vec3 base_color = xyz(s.base_color);
    c.V = V; c.N = N;
    c.F0 = v3(0.16f * s.reflectance * s.reflectance * (1.0f - s.metallic)) + base_color * s.metallic;
    c.diffuse_color = base_color * (1.0f - s.metallic);
    c.roughness = s.roughness;
    c.NdotV = fmax_(dot(N, V), 0.0001f);
    c.f90 = saturate(dot(c.F0, v3(50.0f * 0.33f)));                                                  // fresnel()
    c.ambient_radiance = s.occlusion * env_terms(c.diffuse_color, c.F0, s.roughness, c.NdotV) * e.ambient;  // ambient()
    return c;
}
__device__ __forceinline__ vec3 shade(const ShadeCtx& c, vec3 Lv, vec4 in_radiance) {
    // lit()
    vec3 Hv = normalize(Lv + c.V);
    float NoL = saturate(dot(c.N, Lv));
    float NoH = saturate(dot(c.N, Hv));
    float LoH = saturate(dot(Lv, Hv));
    vec3 diffuse = c.diffuse_color * Fd_Burley(c.roughness, c.NdotV, NoL, LoH);
    float D = D_GGX(c.roughness, NoH);
    float Vis = V_SmithGGXCorrelated(c.roughness, c.NdotV, NoL);
    vec3 F = F_Schlick_vec(c.F0, c.f90, LoH);
    vec3 specular_light = (1.0f * D * Vis) * F;                                                       // specular(), intensity 1
    vec3 lit_radiance = (specular_light + diffuse) * xyz(in_radiance) * NoL;
    return mix(lit_radiance, c.ambient_radiance, 1.0f - in_radiance.w);
}
static __device__ HK_INL_SHADE vec3 shading(const ShadeEnv& e, vec3 V, vec3 N, vec3 Lv, const Surface& s, vec4 in_radiance) {
    return shade(make_shade_ctx(e, V, N, s), Lv, in_radiance);
}
// input_radiance, light.wgsl:835-867
static __device__ HK_INL_RADIANCE vec4 input_radiance(const DeviceScene& sc, const ShadeEnv& e, vec3 ray_direction, const HitInfo& info,
                                               bool sample_directional, uint32_t sample_emissive, bool sample_ambient) {
    vec3 radiance = v3(0.0f);
    float amb = 0.0f;
    if (info.instance_index == U32_MAX) {
        bool hit_directional = dot(ray_direction, e.sun_dir) >= e.cos_solar;
        if (sample_directional && hit_directional) {
            radiance = e.sun_color;
        } else {
            radiance = sample_ambient ? e.ambient : v3(0.0f);
            amb = 1.0f;
        }
    } else if (sample_emissive == info.instance_index) {
        radiance = compute_emissive_radiance(retreive_emissive(sc, info.material_index, info.uv));
    }
    return v4(radiance, 1.0f - amb);
}

// hk_wide.cuh (defined there; only the WIDE instantiations of the light kernels need the definition)
#ifndef HK_INL_WIDE
#define HK_INL_WIDE __forceinline__
#endif
template <bool BOTTOM>
static __device__ HK_INL_WIDE Hit wide_walk(const DeviceScene& sc, const Ray& ray, float max_distance, float early_distance,
                                            uint32_t exclude_instance, uint32_t instance);

// select_light_candidate, light.wgsl:599-708.  COUNT_RAYS adds the stand-alone BLAS ray to *blas_rays.  WIDE: the BLAS ray towards
// the light walks the mesh's 4-wide tree (hk_wide.cuh) instead of its flat array.
template <bool COUNT_RAYS, bool WIDE = false>
static __device__ HK_INL_SELECT LightCandidate select_light_candidate(const DeviceScene& sc, const ShadeEnv& e, vec4 rnd, vec3 position,
                                                                 vec3 normal, uint32_t instance, HitInfo& info, uint32_t& blas_rays) {
    LightCandidate cand;
    cand.max_distance = F32_MAX;
    cand.min_distance = DISTANCE_MAX;
    cand.emissive_instance = DONT_SAMPLE_EMISSIVE;
    vec3 rand_direction = mul(normal_basis(e.sun_dir), sample_uniform_cone_dir(rnd.z, rnd.w, e.cos_solar));
    cand.direction = rand_direction;
    cand.p = 1.0f;
    info = empty_hit_info(position, rand_direction);
    if (instance == DONT_SAMPLE_EMISSIVE) return cand;

    // stackless walk of the emissive BVH with a streaming 1/count pick (light.wgsl:623-657)
    uint32_t picked = U32_MAX;
    float count = 0.0f;
    float rand_1d = rnd.x;
    uint32_t index = 0;
    while (index < sc.emissive_node_count) {
        float4 n0 = ldg4(&sc.emissive_nodes[index]);
        uint32_t entry = __float_as_uint(n0.w);
        if (entry >= BVH_LEAF_FLAG) {
            uint32_t emissive_index = entry - BVH_LEAF_FLAG;
            float4 pr = ldg4(sc.emissives[emissive_index].position);  // position | radius
            uint32_t em_instance = __ldg(&sc.emissives[emissive_index].instance);
            vec3 c = f4xyz(pr);
            vec3 bmin = c - pr.w, bmax = c + pr.w;
            bool inside = position.x > bmin.x && position.y > bmin.y && position.z > bmin.z &&
                          position.x < bmax.x && position.y < bmax.y && position.z < bmax.z;
            if (instance != em_instance && inside) {
                rand_1d = fract(rand_1d + GOLDEN_RATIO);
                count += 1.0f;
                if (rand_1d < 1.0f / count) { cand.emissive_instance = em_instance; picked = emissive_index; }
            }
            index = __ldg(&sc.emissive_nodes[index].exit_index);
        } else {
            float4 n1 = ldg4(reinterpret_cast<const float4*>(&sc.emissive_nodes[index]) + 1);
            bool inside = position.x > n0.x && position.y > n0.y && position.z > n0.z &&
                          position.x < n1.x && position.y < n1.y && position.z < n1.z;
            index = inside ? entry : __float_as_uint(n1.w);
        }
    }

    if (cand.emissive_instance != DONT_SAMPLE_EMISSIVE) {
        const hk_emissive* em = sc.emissives + picked;
        uint4 e2 = ldg4u(&em->instance);      // instance | pad | alias offset | alias count
        float surface_area = __ldg(&em->surface_area);
        uint32_t alias_index = min(f32_to_u32(rnd.x * (float)e2.w), e2.w - 1u);
        uint2 ae = __ldg(reinterpret_cast<const uint2*>(sc.alias_table + e2.z + alias_index));  // prob | index
        uint32_t primitive_index = (rnd.y < __uint_as_float(ae.x)) ? ae.y : alias_index;

        const hk_instance* einst = sc.instances + cand.emissive_instance;
        uint4 mesh = ldg4u(&einst->mesh);
        const hk_primitive* prim = sc.primitives + mesh.y + primitive_index;
        vec3 p0 = f4xyz(ldg4(&prim->vertices[0])), p1 = f4xyz(ldg4(&prim->vertices[1])), p2 = f4xyz(ldg4(&prim->vertices[2]));
        float srx = sqrtf(rnd.z);                       // sample_uniform_triangle_barycentric, light.wgsl:562-565
        float bx = 1.0f - srx, by = rnd.w * srx;
        vec3 lp = bx * p0 + by * p1 + (1.0f - bx - by) * p2;
        const float4* mm = reinterpret_cast<const float4*>(einst->model);
        mat4 model;
        model.c[0] = f4v(ldg4(mm)); model.c[1] = f4v(ldg4(mm + 1)); model.c[2] = f4v(ldg4(mm + 2)); model.c[3] = f4v(ldg4(mm + 3));
        vec4 wp = mul(model, v4(lp, 1.0f));
        vec3 p = xyz(wp) / wp.w;

        Hit hit;
        hit.u = 0.0f; hit.v = 0.0f; hit.distance = F32_MAX; hit.instance_index = U32_MAX; hit.primitive_index = U32_MAX;
        Ray ray;
        ray.origin = position + normal * RAY_BIAS;
        ray.direction = normalize(p - position);
        ray.inv_direction = v3(0.0f);
        cand.direction = ray.direction;
        bool found = false;
        if (dot(cand.direction, normal) > 0.0f) {
            if (COUNT_RAYS) blas_rays += 1u;
            Ray r;
            instance_ray(einst, ray, r);
            if constexpr (WIDE) {
                hit = wide_walk<true>(sc, r, F32_MAX, 0.0f, DONT_EXCLUDE, cand.emissive_instance);
                found = hit.primitive_index != U32_MAX;
            } else {
                found = traverse_bottom(sc, hit, r, mesh.y, mesh.z, mesh.w, 0.0f);
            }
        }
        if (found) {
            hit.instance_index = e2.x;
            info = hit_info(sc, ray, hit);
            cand.max_distance = hit.distance;
            cand.min_distance = hit.distance - 0.1f;
            vec3 delta = xyz(info.position) - position;
            cand.p = dot(delta, delta) / fabsf(dot(ray.direction, info.normal) * surface_area);
            cand.p = cand.p / count;
        } else {
            info = empty_hit_info(ray.origin, ray.direction);
            cand.emissive_instance = DONT_SAMPLE_EMISSIVE;
            cand.direction = rand_direction;
            cand.p = 1.0f;
        }
    }
    return cand;
}

// -------------------------------------------------------------------------------------------- pixel helpers
__device__ __forceinline__ size_t band_index(const Band& b, int x, int y) { return (size_t)(y - b.a0) * (size_t)b.AW + (size_t)(x - b.ax0); }
__device__ __forceinline__ bool band_allocated(const Band& b, int x, int y) { return x >= b.ax0 && x < b.ax1 && y >= b.a0 && y < b.a1; }
__device__ __forceinline__ bool band_owned(const Band& b, int x, int y) { return x >= b.cx0 && x < b.cx1 && y >= b.r0 && y < b.r1; }
__device__ __forceinline__ size_t render_index(const Band& b, int x, int y) { return (size_t)(y - b.a0) * (size_t)b.RS + (size_t)(x - b.ax0); }
__device__ __forceinline__ size_t owned_index(const Band& b, int x, int y) { return (size_t)(y - b.r0) * (size_t)(b.cx1 - b.cx0) + (size_t)(x - b.cx0); }

// blue-noise fetch, light.wgsl:1075-1079 (nearest + repeat on a 64x64 texture == integer wrap)
__device__ __forceinline__ vec4 noise_random(const KParams& P, int x, int y) {
    uint32_t number = P.in.frame.number;
    uint32_t noise_id = number % NOISE_TEXTURE_COUNT;
    uint32_t tx = ((uint32_t)x + number) & 63u, ty = ((uint32_t)y + number) & 63u;
    uchar4 t = __ldg(reinterpret_cast<const uchar4*>(P.noise) + ((noise_id * 64u + ty) * 64u + tx));
    vec4 rnd = v4(unorm8(t.x), unorm8(t.y), unorm8(t.z), unorm8(t.w));
    return fract(rnd + (float)number * GOLDEN_RATIO);
}

// ---- render space <-> deferred (G-buffer) space, light.wgsl:1007-1017 and denoise.wgsl:37-41
// These end in an integer texel, and at upscale ratio 1.5 (sizes divisible by 3) half the columns and rows sit exactly on a texel
// edge, so one rounding step picks another texel.  Every product, sum and quotient is therefore written as a correctly rounded operation (mul_rn /
// add_rn / div_rn / rcp_rn): the operations the exact build emits anyway, never contracted or approximated in the tolerance build
// (kernels_spatial.cu, kernels_post.cu), whose texels are then the oracle's too (tests/test_gpu_device_math.py).
__device__ __forceinline__ vec2 render_uv(const KParams& P, int x, int y) {   // coords_to_uv(coords, render_size)
    return v2(div_rn(add_rn((float)x, 0.5f), (float)P.band.RW), div_rn(add_rn((float)y, 0.5f), (float)P.band.RH));
}
__device__ __forceinline__ vec2 jittered_deferred_uv(const KParams& P, vec2 uv, float amount) {
    if (P.ratio1) return uv;   // + (+-amount) * texel * 0
    const float s = mul_rn(P.jitter_sign, amount);     // uv + (+-amount) * texel_size * (ratio - 1), texel_size = 1 / size
    return v2(add_rn(uv.x, mul_rn(mul_rn(s, rcp_rn((float)P.band.W)), P.ratio_m1)),
              add_rn(uv.y, mul_rn(mul_rn(s, rcp_rn((float)P.band.H)), P.ratio_m1)));
}
// jittered_deferred_coords (light passes: +-0.25 texel, truncation) of any uv: a pixel's, a neighbour's or a depth-march tap's
__device__ __forceinline__ void jittered_deferred_coords(const KParams& P, vec2 uv, int& dx, int& dy) {
    const vec2 d = jittered_deferred_uv(P, uv, 0.25f);
    dx = f32_to_i32(mul_rn(d.x, (float)P.band.W)); dy = f32_to_i32(mul_rn(d.y, (float)P.band.H));
}
// the same for the render pixel (x, y) whose uv is `uv`
__device__ __forceinline__ void light_deferred_coords(const KParams& P, vec2 uv, int x, int y, int& dx, int& dy) {
    if (P.ratio1) { dx = x; dy = y; return; }   // trunc(((x + 0.5) / W) * W) == x
    jittered_deferred_coords(P, uv, dx, dy);
}
// textureSampleLevel(<deferred texture>, nearest_sampler, jittered_deferred_uv(uv)) of the denoise passes: +-0.5 texel, floor, clamp
__device__ __forceinline__ void denoise_deferred_coords(const KParams& P, vec2 uv, int x, int y, int& dx, int& dy) {
    if (P.ratio1) { dx = x; dy = y; return; }
    vec2 d = jittered_deferred_uv(P, uv, 0.5f);
    dx = min(max((int)floorf(mul_rn(d.x, (float)P.band.W)), 0), P.band.W - 1);
    dy = min(max((int)floorf(mul_rn(d.y, (float)P.band.H)), 0), P.band.H - 1);
}
__device__ __forceinline__ bool render_allocated(const KParams& P, int x, int y) {
    return P.ratio1 ? band_allocated(P.band, x, y) : (x >= 0 && x < P.band.RW && y >= 0 && y < P.band.RH);
}

// ------------------------------------------------------------------------------------- shared pass plumbing
struct PassBuffers {  // bind group 6 (light.rs:518-546)
    ReservoirPlanes previous_reservoir, reservoir, previous_spatial_reservoir, spatial_reservoir;
};
__device__ __forceinline__ PassBuffers bind(const KParams& P, int signal) {
    const int temporal = (signal == 0) ? 0 : (signal == 1 ? 2 : 6);
    const int spatial = (signal == 2) ? 8 : 4;
    const int current = (int)(P.in.frame.number & 1u), previous = 1 - current;
    PassBuffers b;
    b.previous_reservoir = P.planes.reservoir[current + temporal];
    b.reservoir = P.planes.reservoir[previous + temporal];
    b.previous_spatial_reservoir = P.planes.reservoir[current + spatial];
    b.spatial_reservoir = P.planes.reservoir[previous + spatial];
    return b;
}
// reprojected pixel of `previous_uv` (light.wgsl:181-190): returns false when outside [0,1) or outside the band.  Correctly rounded
// like the deferred coordinates above (uv - 0.5 == uv + -0.5 exactly)
__device__ __forceinline__ bool previous_pixel(const KParams& P, vec2 previous_uv, bool inclusive, size_t& pidx) {
    float ax = fabsf(add_rn(previous_uv.x, -0.5f)), ay = fabsf(add_rn(previous_uv.y, -0.5f));
    bool inside = inclusive ? (ax <= 0.5f && ay <= 0.5f) : (ax < 0.5f && ay < 0.5f);
    if (!inside) return false;
    int px = f32_to_i32(mul_rn(previous_uv.x, (float)P.band.RW)), py = f32_to_i32(mul_rn(previous_uv.y, (float)P.band.RH));
    if (!render_allocated(P, px, py)) return false;
    pidx = render_index(P.band, px, py);
    return true;
}
__device__ __forceinline__ vec2 pixel_uv(const KParams& P, int x, int y) { return render_uv(P, x, y); }  // coords_to_uv, utils.wgsl:37-39
// index of the G-buffer texel a light pass reads for render pixel (x, y): jittered_deferred_coords(uv)
__device__ __forceinline__ size_t light_gbuffer_index(const KParams& P, int x, int y, size_t render_idx) {
    if (P.ratio1) return render_idx;
    int dx, dy;
    light_deferred_coords(P, render_uv(P, x, y), x, y, dx, dy);
    return band_index(P.band, dx, dy);
}

// kinds of writes to the previous-spatial buffer, in the order one pixel can issue them
constexpr uint32_t SCATTER_BACKGROUND = 0u, SCATTER_MISS = 1u, SCATTER_VALIDATION = 2u;
__device__ __forceinline__ void scatter_claim(const KParams& P, size_t target, int x, int y, uint32_t kind) {
    uint32_t writer = (uint32_t)y * (uint32_t)P.band.RW + (uint32_t)x;   // global raster index in render space
    atomicMax(&P.planes.scatter_key[target], ((writer + 1u) << 2) | kind);
}

// 8x4-pixel tiles per warp, 4 warps per CTA (16x8 pixels): ray coherence + whole-sector plane accesses.
// HK_CTA_WARPS (2 / 4 / 8; tuning builds): warps of a CTA sit side by side in pairs, so the CTA's tile is 16 x (2 x warps) pixels.  A CTA
// gives its registers and warp slots back only when its slowest warp ends, and the light kernels' warps end at very different times;
// the HK_MINB_* values are CTAs per SM and must be scaled with the CTA size by such a build.
#ifndef HK_CTA_WARPS
#define HK_CTA_WARPS 4
#endif
static_assert(HK_CTA_WARPS == 2 || HK_CTA_WARPS == 4 || HK_CTA_WARPS == 8, "tile_pixel places warps in pairs");
constexpr int TILE_W = 16, TILE_H = 2 * HK_CTA_WARPS, CTA_THREADS = 32 * HK_CTA_WARPS;
#ifndef HK_MINB_INDIRECT
#define HK_MINB_INDIRECT 8   // these kernels are latency / instruction-fetch bound and want warps, not registers.  H100 SXM, ms/frame of
                             // cornell 1080p (the benchmark) / city 4K / scene.rs 1080p (profiles/h100_tune_defaults.jsonl, "default"):
                             // 8 CTAs/SM (64 registers) 2.87 / 27.2 / 15.7, 12 (40 registers, spills) 2.95 / 26.0 / 15.3, 16 (32 registers)
                             // 3.31 / 25.4 / 15.6.  8 is chosen for the benchmark workload; deeper scenes want more warps (DESIGN.md 6b)
#endif
#ifndef HK_MINB_INDIRECT_RESTIR
#define HK_MINB_INDIRECT_RESTIR 5   // k_indirect_restir, the ReSTIR-GI tail of the indirect pass: 8 CTAs/SM (64 registers) spill 120 B, 5 take 94 without spills
#endif
#ifndef HK_MINB_DIRECT
#define HK_MINB_DIRECT 8
#endif
#ifndef HK_MINB_DIRECT_UNTEXTURED
#define HK_MINB_DIRECT_UNTEXTURED 5   // k_direct's TEX = false instantiations (untextured scenes).  H100 SXM 700 W, direct + emissive ms
                                      // on cornell 1080p at 5 / 6 / 7 / 8 CTAs/SM: 0.497 / 0.514 / 0.540 / 0.570; the textured city 4K and
                                      // scene.rs 1080p frames are 1-2 % slower below 8 (profiles/h100_ab_direct_bounds.json, DESIGN.md 4a-5)
#endif
#ifndef HK_MINB_GBUFFER
#define HK_MINB_GBUFFER 8    // 64 registers instead of the 66-78 an uncapped build takes
#endif
#ifndef HK_MINB_INDIRECT_WIDE
#define HK_MINB_INDIRECT_WIDE 6   // the 4-wide walk holds a node's seven 16-byte loads in flight: 80 registers instead of 64
#endif
#ifndef HK_MINB_DIRECT_WIDE
#define HK_MINB_DIRECT_WIDE 6
#endif
#ifndef HK_MINB_DENOISE
#define HK_MINB_DENOISE 8
#endif
#ifndef HK_MINB_SPATIAL
#define HK_MINB_SPATIAL 8
#endif
__device__ __forceinline__ void tile_pixel(int& x, int& y, const KParams& P) {
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    x = P.col_lo + blockIdx.x * TILE_W + (warp & 1) * 8 + (lane & 7);
    y = P.row_lo + blockIdx.y * TILE_H + (warp >> 1) * 4 + (lane >> 3);
}
__device__ __forceinline__ bool tile_active(const KParams& P, int x, int y) { return x < P.col_hi && y < P.row_hi; }

}  // namespace hkd
