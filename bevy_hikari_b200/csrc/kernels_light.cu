// kernels_light.cu — the light node of the CUDA path: G-buffer generation by primary rays (+ albedo), sun / emissive
// direct lighting with temporal ReSTIR, N-bounce indirect lighting with temporal ReSTIR-GI, and spatial reuse.
// Replaces the compute entry points of src/shaders/light.wgsl dispatched by LightNode::run (src/light.rs:590-702)
// and the raster prepass (src/shaders/prepass.wgsl, src/prepass.rs:769-851).
#include "hk_device.cuh"
#include "hk_wide.cuh"
#include "hk_kernels.h"

// NO_TEXTURE specialisation (light.rs:141-143: the reference compiles its light shaders with NO_TEXTURE when the scene has no
// texture at all, light.wgsl:729-747 vs :749-793).  TEX = false instantiations see texture_count == 0 as a compile-time constant,
// so the bilinear sampler, the wrap modes and the four texture look-ups per retreive_surface are not in the kernel at all; the
// launchers pick them when the uploaded scene has no textures (cornell).  Values are identical by construction — the same
// `if (sc.texture_count != 0u)` decides, at compile time instead of at run time.  -DHK_NO_TEXTURE_VARIANT=0 keeps one variant.
#ifndef HK_NO_TEXTURE_VARIANT
#define HK_NO_TEXTURE_VARIANT 1
#endif
#ifndef HK_NOVAL_VARIANT
#define HK_NOVAL_VARIANT 1          // 0: k_direct always uses the instantiation that tests for a validation frame at run time
#endif

namespace hkd {

template <bool COUNT>
__device__ __forceinline__ void flush_counters(const KParams& P, uint32_t primary, uint32_t tlas, uint32_t blas) {
    if (!COUNT || P.counters == nullptr) return;
    for (int o = 16; o > 0; o >>= 1) {
        primary += __shfl_xor_sync(0xffffffffu, primary, o);
        tlas += __shfl_xor_sync(0xffffffffu, tlas, o);
        blas += __shfl_xor_sync(0xffffffffu, blas, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (primary) atomicAdd(&P.counters->primary, (unsigned long long)primary);
        if (tlas) atomicAdd(&P.counters->tlas, (unsigned long long)tlas);
        if (blas) atomicAdd(&P.counters->blas, (unsigned long long)blas);
    }
}

// traverse_top in the launch's traversal mode: WIDE = the image-exact 4-wide walk (hk_wide.cuh), else the reference's fixed-order walk
template <bool WIDE>
__device__ __forceinline__ Hit trace_top(const DeviceScene& sc, const Ray& ray, float max_distance, float early_distance, uint32_t exclude_instance) {
    if constexpr (WIDE) return wide_walk<false>(sc, ray, max_distance, early_distance, exclude_instance, 0u);
    else return traverse_top(sc, ray, max_distance, early_distance, exclude_instance);
}

__device__ __forceinline__ mat4 load_mat4(const float* m) {
    mat4 r;
    for (int c = 0; c < 4; ++c) r.c[c] = v4(m[4 * c], m[4 * c + 1], m[4 * c + 2], m[4 * c + 3]);
    return r;
}

// ----------------------------------------------------------------------------------- P0 + P1: G-buffer, albedo
__device__ __forceinline__ Ray primary_ray(const KParams& P, const mat4& inv_view_proj, float px, float py, vec2 jitter_ndc) {
    vec2 uv = v2(px + 0.5f, py + 0.5f) / v2((float)P.band.W, (float)P.band.H);
    vec2 ndc = v2(uv.x * 2.0f - 1.0f, (1.0f - uv.y) * 2.0f - 1.0f) - jitter_ndc;
    vec4 p = mul(inv_view_proj, v4(ndc.x, ndc.y, 1.0f, 1.0f));
    vec3 near_point = xyz(p) / p.w;
    Ray ray;
    if (P.in.view.projection[15] == 1.0f) {   // orthographic (light.wgsl:1040): parallel lines of sight, near plane -> far plane
        vec4 q = mul(inv_view_proj, v4(ndc.x, ndc.y, 0.0f, 1.0f));
        ray.origin = near_point;
        ray.direction = normalize(xyz(q) / q.w - near_point);
    } else {
        ray.origin = v3(P.in.view.world_position[0], P.in.view.world_position[1], P.in.view.world_position[2]);
        ray.direction = normalize(near_point - ray.origin);
    }
    ray.inv_direction = 1.0f / ray.direction;
    return ray;
}

template <bool TEX>
__device__ __forceinline__ DeviceScene scene_variant(const DeviceScene& scene) {
    DeviceScene sc = scene;
    if (!TEX) sc.texture_count = 0u;     // constant-folds every `sc.texture_count != 0u` below it
    return sc;
}

template <bool COUNT, bool TEX = true, bool WIDE = false>
__global__ void __launch_bounds__(CTA_THREADS, HK_MINB_GBUFFER) k_gbuffer(const __grid_constant__ KParams P) {
    int x, y;
    tile_pixel(x, y, P);
    const bool active = tile_active(P, x, y);
    uint32_t n_primary = 0;
    if (active) {
        const size_t idx = band_index(P.band, x, y);
        const mat4 view_proj = load_mat4(P.in.view.view_proj);
        const mat4 inv_view_proj = load_mat4(P.in.view.inverse_view_proj);
        vec2 jitter_ndc = v2(0.0f, 0.0f);
        if (P.in.taa_jitter) {  // prepass.wgsl:30-38,52-54,71
            uint32_t index = P.in.smaa_tu4x ? ((P.in.frame.number >> 1u) & 15u) : (P.in.frame.number & 15u);
            const float* h = P.in.frame.halton[index >> 1u];
            vec2 hj = ((index & 1u) == 0u) ? v2(h[0], h[1]) : v2(h[2], h[3]);
            vec2 j = 2.0f * hj * (v2(1.0f, 1.0f) / v2(P.in.view.viewport[2], P.in.view.viewport[3]));
            jitter_ndc = v2(j.x, -j.y);
        }
        Ray ray = primary_ray(P, inv_view_proj, (float)x, (float)y, jitter_ndc);
        n_primary = 1;
        Hit hit = trace_top<WIDE>(P.scene, ray, F32_MAX, 0.0f, DONT_EXCLUDE);
        if (hit.instance_index == U32_MAX) {
            P.planes.pos_depth[idx] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            P.planes.depth[idx] = 0.0f;
            P.planes.normal[idx] = 0u;
            P.planes.depth_gradient[idx] = make_float2(0.0f, 0.0f);
            P.planes.instance_material[idx] = make_float2(0.0f, 0.0f);
            P.planes.velocity_uv[idx] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            P.planes.albedo[idx] = make_uint2(0u, 0u);
        } else {
            const DeviceScene sc = scene_variant<TEX>(P.scene);
            const hk_instance* inst = sc.instances + hit.instance_index;
            const hk_primitive* prim = sc.primitives + hit.primitive_index;
            uint32_t vbase = __ldg(&inst->mesh.vertex);
            uint32_t material = __ldg(&inst->material);
            float4 pa = ldg4(&prim->vertices[0]), pb = ldg4(&prim->vertices[1]), pc = ldg4(&prim->vertices[2]);
            const hk_vertex* va = sc.vertices + vbase + __float_as_uint(pa.w);
            const hk_vertex* vb = sc.vertices + vbase + __float_as_uint(pb.w);
            const hk_vertex* vc = sc.vertices + vbase + __float_as_uint(pc.w);
            float4 a0 = ldg4(va), a1 = ldg4(reinterpret_cast<const float4*>(va) + 1);
            float4 b0 = ldg4(vb), b1 = ldg4(reinterpret_cast<const float4*>(vb) + 1);
            float4 c0 = ldg4(vc), c1 = ldg4(reinterpret_cast<const float4*>(vc) + 1);
            vec3 world_position = ray.origin + ray.direction * hit.distance;
            vec4 clip = mul(view_proj, v4(world_position, 1.0f));
            float depth = clip.z / clip.w;
            vec3 n0 = instance_normal_local_to_world(inst, f4xyz(a1));
            vec3 n1 = instance_normal_local_to_world(inst, f4xyz(b1));
            vec3 n2 = instance_normal_local_to_world(inst, f4xyz(c1));
            vec3 world_normal = n0 + hit.u * (n1 - n0) + hit.v * (n2 - n0);
            vec2 uv0 = v2(a0.w, a1.w), uv1 = v2(b0.w, b1.w), uv2 = v2(c0.w, c1.w);
            vec2 tex_uv = uv0 + hit.u * (uv1 - uv0) + hit.v * (uv2 - uv0);
            // screen-space derivatives of NDC depth on the triangle's plane (dpdx/dpdy of clip_position.z)
            const mat4 model = load_mat4(inst->model);
            vec3 P0 = xyz(mul(model, v4(f4xyz(pa), 1.0f)));
            vec3 P1 = xyz(mul(model, v4(f4xyz(pb), 1.0f)));
            vec3 P2 = xyz(mul(model, v4(f4xyz(pc), 1.0f)));
            vec3 Ng = cross(P1 - P0, P2 - P0);
            Ray rx = primary_ray(P, inv_view_proj, (float)x + 1.0f, (float)y, jitter_ndc);
            float tx = dot(P0 - rx.origin, Ng) / dot(rx.direction, Ng);
            vec4 cx = mul(view_proj, v4(rx.origin + rx.direction * tx, 1.0f));
            Ray ry = primary_ray(P, inv_view_proj, (float)x, (float)y + 1.0f, jitter_ndc);
            float ty = dot(P0 - ry.origin, Ng) / dot(ry.direction, Ng);
            vec4 cy = mul(view_proj, v4(ry.origin + ry.direction * ty, 1.0f));
            vec2 grad = v2(cx.z / cx.w - depth, cy.z / cy.w - depth);
            // velocity = clip_to_uv(view_proj * world_position) - clip_to_uv(previous_view_proj * previous_world_position)
            // (prepass.wgsl:52,99): previous_world_position = previous_mesh.model * local position for instances whose
            // model matrix changed since the last frame, the world position itself otherwise
            vec3 previous_world_position = world_position;
            if (sc.instance_moved != nullptr && __ldg(&sc.instance_moved[hit.instance_index]) != 0u) {
                const float4* pm = sc.previous_models + 4u * (size_t)hit.instance_index;
                mat4 previous_model;
                for (int c = 0; c < 4; ++c) previous_model.c[c] = f4v(ldg4(pm + c));
                vec3 local_position = f4xyz(pa) + hit.u * (f4xyz(pb) - f4xyz(pa)) + hit.v * (f4xyz(pc) - f4xyz(pa));
                previous_world_position = xyz(mul(previous_model, v4(local_position, 1.0f)));
            }
            vec4 pclip = mul(load_mat4(P.in.previous_view.view_proj), v4(previous_world_position, 1.0f));
            vec2 uva = v2(clip.x, clip.y) / clip.w; uva = (uva + 1.0f) * 0.5f; uva.y = 1.0f - uva.y;
            vec2 uvb = v2(pclip.x, pclip.y) / pclip.w; uvb = (uvb + 1.0f) * 0.5f; uvb.y = 1.0f - uvb.y;
            vec2 velocity = uva - uvb;
            uint32_t packed_normal = pack4x8snorm(v4(world_normal, 1.0f));
            P.planes.pos_depth[idx] = make_float4(world_position.x, world_position.y, world_position.z, depth);
            P.planes.depth[idx] = depth;
            P.planes.normal[idx] = packed_normal;
            P.planes.depth_gradient[idx] = make_float2(grad.x, grad.y);
            P.planes.instance_material[idx] = make_float2((float)hit.instance_index + 0.5f, (float)material + 0.5f);
            P.planes.velocity_uv[idx] = make_float4(velocity.x, velocity.y, tex_uv.x, tex_uv.y);
            // full_screen_albedo (light.wgsl:1019-1042) fused: it reads back exactly what was just written
            uvec2 alb; alb.x = 0u; alb.y = 0u;
            if (!(depth < F32_EPSILON)) {
                ShadeEnv env = make_env(P);
                vec3 normal = xyz(unpack4x8snorm(packed_normal));
                Surface surface = retreive_surface(sc, f32_to_u32((float)material + 0.5f), tex_uv);
                vec3 view_direction = calculate_view(env, world_position);
                alb = pack_rgba16f(v4(env_brdf(view_direction, normal, surface), 1.0f));
            }
            P.planes.albedo[idx] = make_uint2(alb.x, alb.y);
        }
    }
    if (!band_owned(P.band, x, y)) n_primary = 0;   // ghost pixels are redundant work: not counted
    flush_counters<COUNT>(P, n_primary, 0u, 0u);
}

// stand-alone full_screen_albedo for externally supplied G-buffers
__global__ void __launch_bounds__(CTA_THREADS) k_albedo(const __grid_constant__ KParams P) {
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const size_t idx = band_index(P.band, x, y);
    float4 pd = P.planes.pos_depth[idx];
    P.planes.depth[idx] = pd.w;                        // the planar copy of the depth follows an externally supplied G-buffer too
    if (pd.w < F32_EPSILON) { P.planes.albedo[idx] = make_uint2(0u, 0u); return; }
    ShadeEnv env = make_env(P);
    vec3 normal = xyz(unpack4x8snorm(P.planes.normal[idx]));
    float2 im = P.planes.instance_material[idx];
    float4 vu = P.planes.velocity_uv[idx];
    Surface surface = retreive_surface(P.scene, f32_to_u32(im.y), v2(vu.z, vu.w));
    uvec2 alb = pack_rgba16f(v4(env_brdf(calculate_view(env, f4xyz(pd)), normal, surface), 1.0f));
    P.planes.albedo[idx] = make_uint2(alb.x, alb.y);
}

// --------------------------------------------------------------------------------------- P2: direct_lit
// light.wgsl:1044-1261.  EMISSIVE_LIT=false is the sun pass (+RENDER_EMISSIVE), true is the emissive pass.
// NOVAL = true: instantiation for the frames that are NOT validation frames (frame.number % validate_interval != 0, a launch-wide
// fact the launcher knows): the whole validation block — a second select_light_candidate with its own emissive-BVH walk and BLAS
// traversal, a second TLAS traversal, the reset logic — is not in the kernel (2 of 3 sun frames, 4 of 5 emissive frames at the
// default intervals).  The generic instantiation decides the same thing at run time; values are identical.
template <bool EMISSIVE_LIT, bool COUNT, bool TEX = true, bool NOVAL = false, bool WIDE = false>
__global__ void __launch_bounds__(CTA_THREADS, WIDE ? HK_MINB_DIRECT_WIDE : (TEX ? HK_MINB_DIRECT : HK_MINB_DIRECT_UNTEXTURED))
k_direct(const __grid_constant__ KParams P) {
    constexpr int SIGNAL = EMISSIVE_LIT ? 1 : 0;
    constexpr bool RENDER_EMISSIVE = !EMISSIVE_LIT;
    int x, y;
    tile_pixel(x, y, P);
    const bool active = tile_active(P, x, y);
    uint32_t n_tlas = 0, n_blas = 0;
    if (active) {
        const DeviceScene sc = scene_variant<TEX>(P.scene);
        const hk_frame_uniform& frame = P.in.frame;
        const size_t idx = render_index(P.band, x, y);
        const size_t gidx = light_gbuffer_index(P, x, y, idx);
        const PassBuffers B = bind(P, SIGNAL);
        const float4 pd = P.planes.pos_depth[gidx];
        const float depth = pd.w;
        if (depth < F32_EPSILON) {
            Reservoir r = zero_reservoir();
            set_reservoir(r, zero_sample(), 0.0f);
            PackedQuarters q = pack_reservoir(r);
            store_quarters(B.reservoir, idx, q);
            store_quarters(B.spatial_reservoir, idx, q);
            scatter_claim(P, idx, x, y, SCATTER_BACKGROUND);
            P.planes.variance[SIGNAL][idx] = 0.0f;
            P.planes.render[SIGNAL][idx] = make_uint2(0u, 0u);
        } else {
            const ShadeEnv env = make_env(P);
            const vec3 position = f4xyz(pd);
            const vec3 normal = xyz(unpack4x8snorm(P.planes.normal[gidx]));  // NOT normalised (light.wgsl:1071)
            const float2 imf = P.planes.instance_material[gidx];
            const uint32_t instance_id = f32_to_u32(imf.x), material_id = f32_to_u32(imf.y);
            const float4 vu = P.planes.velocity_uv[gidx];

            Sample s = zero_sample();
            s.random = noise_random(P, x, y);
            s.visible_position = v4(position, depth);
            s.visible_normal = normal;
            s.visible_instance = instance_id;

            HitInfo info = empty_hit_info(v3(0.0f), v3(0.0f));
            info.instance_index = 0u; info.material_index = 0u; info.position = v4(0.0f);

            const vec2 previous_uv = jittered_deferred_uv(P, pixel_uv(P, x, y), 0.25f) - v2(vu.x, vu.y);
            size_t pidx = 0;
            Reservoir r = zero_reservoir();
            if (previous_pixel(P, previous_uv, false, pidx)) r = unpack_reservoir(load_quarters(B.previous_reservoir, pidx));
            if (!check_previous_reservoir(r, s)) {   // r is now the zero reservoir: the write carries a constant
                size_t sidx;
                if (previous_pixel(P, previous_uv, true, sidx)) scatter_claim(P, sidx, x, y, SCATTER_MISS);
            }

            const uint32_t validate_interval = EMISSIVE_LIT ? frame.emissive_validate_interval : frame.direct_validate_interval;
            const uint32_t select_light_instance = EMISSIVE_LIT ? instance_id : DONT_SAMPLE_EMISSIVE;
            const bool validation_frame = NOVAL ? false : (frame.number % validate_interval) == 0u;

            if (!validation_frame || r.count < 4.0f) {
                LightCandidate cand = select_light_candidate<COUNT, WIDE>(sc, env, s.random, position, normal, select_light_instance, info, n_blas);
                Ray ray;
                ray.origin = position + normal * RAY_BIAS;
                ray.direction = cand.direction;
                ray.inv_direction = 1.0f / ray.direction;
                bool trace_condition = dot(cand.direction, normal) > 0.0f && cand.p > 0.0f;
                if (EMISSIVE_LIT) trace_condition = trace_condition && cand.emissive_instance != DONT_SAMPLE_EMISSIVE;
                if (trace_condition) {
                    if (COUNT) n_tlas += 1u;
                    Hit hit = trace_top<WIDE>(sc, ray, cand.max_distance, cand.min_distance, cand.emissive_instance);
                    occlude_hit_info(ray, hit, info);
                    s.radiance = EMISSIVE_LIT ? input_radiance(sc, env, ray.direction, info, false, cand.emissive_instance, false)
                                              : input_radiance(sc, env, ray.direction, info, true, DONT_SAMPLE_EMISSIVE, false);
                }
                s.sample_position = info.position;
                s.sample_normal = info.normal;
                float w_new = (cand.p > 0.0f) ? luminance(xyz(s.radiance)) / cand.p : 0.0f;
                temporal_restir(r, s, w_new, frame.max_temporal_reuse_count);
            }

            if (validation_frame) {
                LightCandidate cand = select_light_candidate<COUNT, WIDE>(sc, env, r.s.random, xyz(r.s.visible_position), r.s.visible_normal,
                                                                    select_light_instance, info, n_blas);
                Ray ray;
                ray.origin = position + normal * RAY_BIAS;
                ray.direction = normalize(xyz(r.s.sample_position) - position);
                ray.inv_direction = 1.0f / ray.direction;
                vec4 validate_radiance = v4(0.0f);
                bool trace_condition = dot(cand.direction, r.s.visible_normal) > 0.0f && cand.p > 0.0f;
                if (EMISSIVE_LIT) trace_condition = trace_condition && cand.emissive_instance != DONT_SAMPLE_EMISSIVE;
                if (trace_condition) {
                    if (COUNT) n_tlas += 1u;
                    Hit hit = trace_top<WIDE>(sc, ray, cand.max_distance, cand.min_distance, cand.emissive_instance);
                    occlude_hit_info(ray, hit, info);
                    validate_radiance = EMISSIVE_LIT ? input_radiance(sc, env, ray.direction, info, false, cand.emissive_instance, false)
                                                     : input_radiance(sc, env, ray.direction, info, true, DONT_SAMPLE_EMISSIVE, false);
                }
                if (r.count >= 4.0f) {
                    s.random = r.s.random;
                    s.sample_position = info.position;
                    s.sample_normal = info.normal;
                    s.radiance = validate_radiance;
                }
                float luminance_ratio = luminance(xyz(validate_radiance)) / fmax_(luminance(xyz(r.s.radiance)), 0.0001f);
                if (luminance_ratio > 1.25f || luminance_ratio < 0.8f) {
                    size_t sidx;
                    if (previous_pixel(P, previous_uv, true, sidx)) {
                        store_quarters(P.planes.scatter_value, idx, pack_reservoir(r));
                        scatter_claim(P, sidx, x, y, SCATTER_VALIDATION);
                    }
                    float w_new = (cand.p > 0.0f) ? luminance(xyz(s.radiance)) / cand.p : 0.0f;
                    set_reservoir(r, s, w_new);
                }
            }

            float total_lum = r.count * luminance(xyz(r.s.radiance));
            r.w = (total_lum > 0.0f) ? r.w_sum / total_lum : 0.0f;
            r.s.visible_position = s.visible_position;
            r.s.visible_normal = s.visible_normal;
            r.lifetime += 1.0f;
            P.planes.variance[SIGNAL][idx] = variance_of(r);
            if (frame.temporal_reuse > 0u) store_quarters(B.reservoir, idx, pack_reservoir(r));

            Surface surface = retreive_surface(sc, material_id, v2(vu.z, vu.w));
            vec3 view_direction = calculate_view(env, position);
            vec3 out_radiance = shading(env, view_direction, r.s.visible_normal,
                                        normalize(xyz(r.s.sample_position) - xyz(r.s.visible_position)), surface, r.s.radiance);
            out_radiance = out_radiance * r.w;
            vec3 out_color = RENDER_EMISSIVE ? out_radiance + compute_emissive_radiance(surface.emissive) : out_radiance;
            uvec2 o = pack_rgba16f(v4(out_color, 1.0f));
            P.planes.render[SIGNAL][idx] = make_uint2(o.x, o.y);
        }
    }
    if (!band_owned(P.band, x, y)) { n_tlas = 0; n_blas = 0; }   // ghost pixels are redundant work: not counted
    flush_counters<COUNT>(P, 0u, n_tlas, n_blas);
}

// ----------------------------------------------------------------------------- P3: indirect_lit_ambient
// light.wgsl:1263-1498 as two kernels over the same pixels.  k_indirect_path traces the path of every surface pixel and keeps
// alive only what the walk needs; k_indirect_restir then runs the temporal ReSTIR-GI tail with coherent warps and no ray.
// Between them the path's four results travel at full f32 precision through the scatter_value planes: those carry a reservoir
// only from a validation write of k_direct to the k_scatter_resolve of the same pass, which has run before this pass starts.
struct PathResult { vec4 radiance, sample_position; vec3 sample_normal; float pdf; };
// the first bounce's hit is stored as soon as it is known, so that it is not carried through the later bounces
__device__ __forceinline__ void store_path_sample(const KParams& P, size_t idx, vec4 sample_position, vec3 sample_normal, float pdf) {
    P.planes.scatter_value.q[1][idx] = make_uint4(__float_as_uint(sample_position.x), __float_as_uint(sample_position.y),
                                                  __float_as_uint(sample_position.z), __float_as_uint(sample_position.w));
    P.planes.scatter_value.q[2][idx] = make_uint4(__float_as_uint(sample_normal.x), __float_as_uint(sample_normal.y),
                                                  __float_as_uint(sample_normal.z), __float_as_uint(pdf));
}
__device__ __forceinline__ void store_path_radiance(const KParams& P, size_t idx, vec4 radiance) {
    P.planes.scatter_value.q[0][idx] = make_uint4(__float_as_uint(radiance.x), __float_as_uint(radiance.y),
                                                  __float_as_uint(radiance.z), __float_as_uint(radiance.w));
}
__device__ __forceinline__ PathResult load_path(const KParams& P, size_t idx) {
    const uint4 a = P.planes.scatter_value.q[0][idx], b = P.planes.scatter_value.q[1][idx], c = P.planes.scatter_value.q[2][idx];
    PathResult r;
    r.radiance = v4(__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(a.w));
    r.sample_position = v4(__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(b.w));
    r.sample_normal = v3(__uint_as_float(c.x), __uint_as_float(c.y), __uint_as_float(c.z));
    r.pdf = __uint_as_float(c.w);
    return r;
}
__device__ __forceinline__ bool indirect_background(const KParams& P, float depth) {
    return P.in.frame.indirect_bounces == 0u || depth < F32_EPSILON;
}

// The bounce loop.  One kernel covers both the single-bounce and the MULTIPLE_BOUNCES variants: the reference's single-bounce
// body is the loop body for n == 0 without the luminance clamp, so MULTI only switches those two bits.
template <bool MULTI, bool COUNT, bool TEX = true, bool WIDE = false>
__global__ void __launch_bounds__(CTA_THREADS, WIDE ? HK_MINB_INDIRECT_WIDE : HK_MINB_INDIRECT) k_indirect_path(const __grid_constant__ KParams P) {
    int x, y;
    tile_pixel(x, y, P);
    const bool active = tile_active(P, x, y);
    uint32_t n_tlas = 0, n_blas = 0;
    if (active) {
        const size_t idx = render_index(P.band, x, y);
        const size_t gidx = light_gbuffer_index(P, x, y, idx);
        const float4 pd = P.planes.pos_depth[gidx];
        if (!indirect_background(P, pd.w)) {
            const DeviceScene sc = scene_variant<TEX>(P.scene);
            const hk_frame_uniform& frame = P.in.frame;
            const ShadeEnv env = make_env(P);
            vec4 radiance = v4(0.0f);
            // bounce state: the vertex we are leaving
            vec3 b_position = f4xyz(pd), b_normal = normalize(xyz(unpack4x8snorm(P.planes.normal[gidx])));  // normalised here (light.wgsl:1289)
            vec4 b_random = noise_random(P, x, y);
            vec3 color_transport = v3(1.0f);
            const uint32_t bounces = MULTI ? frame.indirect_bounces : 1u;
            for (uint32_t n = 0u; n < bounces && (color_transport.x > 0.01f || color_transport.y > 0.01f || color_transport.z > 0.01f); n += 1u) {
                vec4 rand_sample = sample_cosine_hemisphere(b_random.x, b_random.y);
                Ray ray;
                ray.origin = b_position + b_normal * RAY_BIAS;
                ray.direction = mul(normal_basis(b_normal), xyz(rand_sample));
                ray.inv_direction = 1.0f / ray.direction;
                if (COUNT) n_tlas += 1u;
                Hit hit = trace_top<WIDE>(sc, ray, F32_MAX, 0.0f, DONT_EXCLUDE);
                HitInfo info = hit_info(sc, ray, hit);
                if (n == 0u) store_path_sample(P, idx, info.position, info.normal, rand_sample.w);
                const vec3 h_position = xyz(info.position), h_normal = info.normal;
                if (hit.instance_index != U32_MAX) {
                    vec3 out_radiance = v3(0.0f);
                    Surface surface = retreive_surface(sc, info.material_index, info.uv);
                    surface.roughness = 1.0f;
                    LightCandidate cand = select_light_candidate<COUNT, WIDE>(sc, env, b_random, h_position, h_normal, info.instance_index, info, n_blas);
                    const bool sample_directional = (cand.emissive_instance == DONT_SAMPLE_EMISSIVE);
                    const vec3 bounce_view_direction = normalize(b_position - h_position);
                    if (dot(cand.direction, h_normal) > 0.0f && cand.p > 0.0f) {
                        ray.origin = h_position + h_normal * RAY_BIAS;
                        ray.direction = cand.direction;
                        ray.inv_direction = 1.0f / ray.direction;
                        if (COUNT) n_tlas += 1u;
                        hit = trace_top<WIDE>(sc, ray, cand.max_distance, cand.min_distance, cand.emissive_instance);
                        occlude_hit_info(ray, hit, info);
                        vec4 in_radiance = input_radiance(sc, env, ray.direction, info, sample_directional, cand.emissive_instance, false);
                        out_radiance = shading(env, bounce_view_direction, h_normal, ray.direction, surface, in_radiance);
                        out_radiance = out_radiance / cand.p;
                        if (MULTI) {
                            if (n > 0u) out_radiance = (rand_sample.w < 0.01f) ? v3(0.0f) : out_radiance / rand_sample.w;
                            float out_luminance = luminance(out_radiance);
                            if (out_luminance > frame.max_indirect_luminance)
                                out_radiance = out_radiance * frame.max_indirect_luminance / out_luminance;
                            radiance = radiance + v4(color_transport * out_radiance, 1.0f);
                        } else {
                            radiance = radiance + v4(out_radiance, 1.0f);
                        }
                    }
                    if (MULTI) {
                        color_transport = color_transport * env_brdf(bounce_view_direction, h_normal, surface);
                        b_random = fract(b_random + (float)frame.number * GOLDEN_RATIO);
                        b_position = h_position;
                        b_normal = h_normal;
                    }
                } else {
                    vec3 out_radiance = xyz(input_radiance(sc, env, ray.direction, info, false, DONT_SAMPLE_EMISSIVE, true));
                    radiance = MULTI ? radiance + v4(color_transport * out_radiance, 0.0f) : radiance + v4(out_radiance, 0.0f);
                    break;
                }
            }
            store_path_radiance(P, idx, radiance);
        }
    }
    if (!band_owned(P.band, x, y)) { n_tlas = 0; n_blas = 0; }   // ghost pixels are redundant work: not counted
    flush_counters<COUNT>(P, 0u, n_tlas, n_blas);
}

// The temporal ReSTIR-GI tail over k_indirect_path's results: reservoir reuse, shading, variance and the scatter claims.
template <bool TEX = true>
__global__ void __launch_bounds__(CTA_THREADS, HK_MINB_INDIRECT_RESTIR) k_indirect_restir(const __grid_constant__ KParams P) {
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const DeviceScene sc = scene_variant<TEX>(P.scene);
    const hk_frame_uniform& frame = P.in.frame;
    const size_t idx = render_index(P.band, x, y);
    const size_t gidx = light_gbuffer_index(P, x, y, idx);
    const PassBuffers B = bind(P, 2);
    const float4 pd = P.planes.pos_depth[gidx];
    const float depth = pd.w;
    if (indirect_background(P, depth)) {
        PackedQuarters q = pack_reservoir(zero_reservoir());
        store_quarters(B.reservoir, idx, q);
        store_quarters(B.spatial_reservoir, idx, q);
        scatter_claim(P, idx, x, y, SCATTER_BACKGROUND);
        P.planes.variance[2][idx] = 0.0f;
        P.planes.render[2][idx] = make_uint2(0u, 0u);
    } else {
        const ShadeEnv env = make_env(P);
        const vec3 position = f4xyz(pd);
        const vec3 normal = normalize(xyz(unpack4x8snorm(P.planes.normal[gidx])));  // normalised here (light.wgsl:1289)
        const float2 imf = P.planes.instance_material[gidx];
        const uint32_t instance_id = f32_to_u32(imf.x), material_id = f32_to_u32(imf.y);
        const float4 vu = P.planes.velocity_uv[gidx];

        const PathResult path = load_path(P, idx);
        Sample s = zero_sample();
        s.random = noise_random(P, x, y);
        s.visible_position = v4(position, depth);
        s.visible_normal = normal;
        s.visible_instance = instance_id;
        s.radiance = path.radiance;
        s.sample_position = path.sample_position;
        s.sample_normal = path.sample_normal;
        const float pdf = path.pdf;

        // ReSTIR: temporal
        const vec2 previous_uv = jittered_deferred_uv(P, pixel_uv(P, x, y), 0.25f) - v2(vu.x, vu.y);
        size_t pidx = 0;
        Reservoir r = zero_reservoir();
        if (previous_pixel(P, previous_uv, false, pidx)) r = unpack_reservoir(load_quarters(B.previous_reservoir, pidx));
        if (!check_previous_reservoir(r, s)) {
            size_t sidx;
            if (previous_pixel(P, previous_uv, true, sidx)) scatter_claim(P, sidx, x, y, SCATTER_MISS);
        }
        Surface surface = retreive_surface(sc, material_id, v2(vu.z, vu.w));
        vec3 view_direction = calculate_view(env, position);
        vec3 sample_radiance = shading(env, view_direction, s.visible_normal,
                                       normalize(xyz(s.sample_position) - xyz(s.visible_position)), surface, s.radiance);
        float w_new = (pdf > 0.0f) ? luminance(sample_radiance) / pdf : 0.0f;
        temporal_restir(r, s, w_new, frame.max_temporal_reuse_count);

        vec3 out_radiance = shading(env, view_direction, r.s.visible_normal,
                                    normalize(xyz(r.s.sample_position) - xyz(r.s.visible_position)), surface, r.s.radiance);
        float total_lum = r.count * luminance(out_radiance);
        r.w = (total_lum > 0.0f) ? r.w_sum / total_lum : 0.0f;
        r.s.visible_position = s.visible_position;
        r.s.visible_normal = s.visible_normal;
        r.lifetime += 1.0f;
        P.planes.variance[2][idx] = variance_of(r);
        if (frame.temporal_reuse > 0u) store_quarters(B.reservoir, idx, pack_reservoir(r));
        uvec2 o = pack_rgba16f(v4(out_radiance * r.w, 1.0f));
        P.planes.render[2][idx] = make_uint2(o.x, o.y);
    }
}

// depth plane <- pos_depth.w (after hk_upload_state of the position plane)
__global__ void __launch_bounds__(CTA_THREADS) k_extract_depth(const __grid_constant__ KParams P) {
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const size_t idx = band_index(P.band, x, y);
    P.planes.depth[idx] = P.planes.pos_depth[idx].w;
}

// ------------------------------------------------------------------------------------------- scatter resolve
// Applies the winning write of each target pixel to the previous-spatial buffer of `signal` (see Planes::scatter_key).
__global__ void __launch_bounds__(CTA_THREADS) k_scatter_resolve(const __grid_constant__ KParams P, int signal) {
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const size_t idx = render_index(P.band, x, y);
    const uint32_t key = P.planes.scatter_key[idx];
    if (key == 0u) return;
    P.planes.scatter_key[idx] = 0u;   // leave the plane clean for the next pass
    const uint32_t kind = key & 3u, writer = (key >> 2) - 1u;
    const PassBuffers B = bind(P, signal);
    PackedQuarters q;
    if (kind == SCATTER_VALIDATION) {
        const int wy = (int)(writer / (uint32_t)P.band.RW), wx = (int)(writer % (uint32_t)P.band.RW);
        q = load_quarters(P.planes.scatter_value, render_index(P.band, wx, wy));
    } else {
        Reservoir r = zero_reservoir();
        if (kind == SCATTER_BACKGROUND && signal != 2) set_reservoir(r, zero_sample(), 0.0f);   // light.wgsl:1059-1063 vs :1279-1282
        q = pack_reservoir(r);
    }
    store_quarters(B.previous_spatial_reservoir, idx, q);
}

// ---------------------------------------------------------------------------------------------- ray-dump hook
template <bool WIDE>
__global__ void k_trace_rays(DeviceScene sc, const hk_ray* rays, size_t n, hk_hit* hits) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Ray r;
    r.origin = v3(rays[i].origin[0], rays[i].origin[1], rays[i].origin[2]);
    r.direction = v3(rays[i].direction[0], rays[i].direction[1], rays[i].direction[2]);
    r.inv_direction = 1.0f / r.direction;
    Hit h = trace_top<WIDE>(sc, r, rays[i].max_distance, rays[i].early_distance, rays[i].exclude_instance);
    hits[i].u = h.u; hits[i].v = h.v; hits[i].distance = h.distance;
    hits[i].instance_index = h.instance_index; hits[i].primitive_index = h.primitive_index;
}

// ------------------------------------------------------------------------------------------------ launchers
static dim3 grid_for(const KParams& P) {
    int rows = P.row_hi - P.row_lo, cols = P.col_hi - P.col_lo;
    return dim3((unsigned)((cols + TILE_W - 1) / TILE_W), (unsigned)((rows + TILE_H - 1) / TILE_H), 1u);
}

}  // namespace hkd

using namespace hkd;

static inline bool no_texture(const KParams& P) { return HK_NO_TEXTURE_VARIANT && P.scene.texture_count == 0u; }
// the image-exact traversal mode is a launch-wide choice (hk_set_tuning(HK_TUNE_WIDE_TRAVERSAL)) and needs the derived trees
static inline bool wide_mode(const KParams& P, bool wide) { return wide && P.scene.wide_ready != 0u; }

void hk_launch_gbuffer(const KParams& P, bool count, bool wide, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    const dim3 g = grid_for(P);
    if (wide_mode(P, wide)) {
        if (count) k_gbuffer<true, true, true><<<g, CTA_THREADS, 0, st>>>(P);
        else if (no_texture(P)) k_gbuffer<false, false, true><<<g, CTA_THREADS, 0, st>>>(P);
        else k_gbuffer<false, true, true><<<g, CTA_THREADS, 0, st>>>(P);
        return;
    }
    if (count) k_gbuffer<true><<<g, CTA_THREADS, 0, st>>>(P);
    else if (no_texture(P)) k_gbuffer<false, false><<<g, CTA_THREADS, 0, st>>>(P);
    else k_gbuffer<false><<<g, CTA_THREADS, 0, st>>>(P);
}
void hk_launch_extract_depth(const KParams& P, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    k_extract_depth<<<grid_for(P), CTA_THREADS, 0, st>>>(P);
}
void hk_launch_albedo(const KParams& P, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    k_albedo<<<grid_for(P), CTA_THREADS, 0, st>>>(P);
}
template <bool WIDE>
static void launch_direct(const KParams& P, bool emissive, bool count, cudaStream_t st) {
    dim3 g = grid_for(P);
    const uint32_t interval = emissive ? P.in.frame.emissive_validate_interval : P.in.frame.direct_validate_interval;
    const bool noval = HK_NOVAL_VARIANT && !count && (P.in.frame.number % interval) != 0u;
    if (noval) {                         // not a validation frame: the lean instantiation
        if (no_texture(P)) {
            if (emissive) k_direct<true, false, false, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
            else k_direct<false, false, false, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
        } else {
            if (emissive) k_direct<true, false, true, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
            else k_direct<false, false, true, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
        }
        return;
    }
    if (!count && no_texture(P)) {       // the timed variants of an untextured scene
        if (emissive) k_direct<true, false, false, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
        else k_direct<false, false, false, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
        return;
    }
    if (emissive) { if (count) k_direct<true, true, true, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P); else k_direct<true, false, true, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P); }
    else { if (count) k_direct<false, true, true, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P); else k_direct<false, false, true, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P); }
}
void hk_launch_direct(const KParams& P, bool emissive, bool count, bool wide, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    if (wide_mode(P, wide)) launch_direct<true>(P, emissive, count, st);
    else launch_direct<false>(P, emissive, count, st);
}
template <bool WIDE>
static void launch_indirect(const KParams& P, bool multi, bool count, cudaStream_t st) {
    dim3 g = grid_for(P);
    if (!count && no_texture(P)) {
        if (multi) k_indirect_path<true, false, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
        else k_indirect_path<false, false, false, WIDE><<<g, CTA_THREADS, 0, st>>>(P);
        k_indirect_restir<false><<<g, CTA_THREADS, 0, st>>>(P);
        return;
    }
    if (multi) { if (count) k_indirect_path<true, true, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P); else k_indirect_path<true, false, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P); }
    else { if (count) k_indirect_path<false, true, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P); else k_indirect_path<false, false, true, WIDE><<<g, CTA_THREADS, 0, st>>>(P); }
    k_indirect_restir<true><<<g, CTA_THREADS, 0, st>>>(P);
}
void hk_launch_indirect(const KParams& P, bool multi, bool count, bool wide, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    if (wide_mode(P, wide)) launch_indirect<true>(P, multi, count, st);
    else launch_indirect<false>(P, multi, count, st);
}
void hk_launch_scatter_resolve(const KParams& P, int signal, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    k_scatter_resolve<<<grid_for(P), CTA_THREADS, 0, st>>>(P, signal);
}
void hk_launch_trace_rays(const DeviceScene& sc, const hk_ray* rays, size_t n, hk_hit* hits, bool wide, cudaStream_t st) {
    if (n == 0) return;
    if (wide && sc.wide_ready != 0u) k_trace_rays<true><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(sc, rays, n, hits);
    else k_trace_rays<false><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(sc, rays, n, hits);
}
