// kernels_pool.cu — the cooperative (kc_*) light kernels: per-pixel shading in the owner thread's registers, every ray of the CTA
// traced through the shared-memory ray pool of hk_pool.cuh (dynamic fetch by a few traversal warps, scene records staged with TMA).
//
//   kc_indirect<MULTI, COUNT, TEX>    indirect_lit_ambient, light.wgsl:1263-1498 — replaces round 1's k_indirect
//
// The arithmetic of every pixel is statement for statement that of the per-pixel kernels in kernels_light.cu (which it shares
// through hk_device.cuh), so outputs are bit-identical; what changed is WHO walks a ray and WHEN: the kernel is a sequence of
// shading stages separated by pool_traverse() calls, three per bounce (bounce ray, light-sample ray, shadow ray).
#include "hk_pool.cuh"
#include "hk_kernels.h"

namespace hkd {

// ---------------------------------------------------------------- select_light_candidate (light.wgsl:599-708) in two halves
// Half A: everything up to the stand-alone BLAS walk towards the sampled light point (:599-686).  `want_ray` says whether that
// walk is needed; the caller queues it as a RAY_KIND_BLAS ray of instance `emissive_instance`.
struct LightPick {
    vec3 rand_direction;       // the sun-cone direction (fallback)
    vec3 ray_origin, ray_direction;
    float count, surface_area;
    uint32_t emissive_instance;   // DONT_SAMPLE_EMISSIVE when no emissive is in range
    bool want_ray;
};
static __device__ __forceinline__ LightPick light_pick(const DeviceScene& sc, const ShadeEnv& e, vec4 rnd, vec3 position, vec3 normal, uint32_t instance) {
    LightPick L;
    L.rand_direction = mul(normal_basis(e.sun_dir), sample_uniform_cone_dir(rnd.z, rnd.w, e.cos_solar));
    L.ray_origin = v3(0.0f); L.ray_direction = v3(0.0f);
    L.count = 0.0f; L.surface_area = 0.0f;
    L.emissive_instance = DONT_SAMPLE_EMISSIVE;
    L.want_ray = false;
    if (instance == DONT_SAMPLE_EMISSIVE) return L;

    uint32_t picked = U32_MAX;
    float count = 0.0f;
    float rand_1d = rnd.x;
    uint32_t index = 0;
    while (index < sc.emissive_node_count) {          // stackless walk of the emissive BVH with a streaming 1/count pick (:623-657)
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
                if (rand_1d < 1.0f / count) { L.emissive_instance = em_instance; picked = emissive_index; }
            }
            index = __ldg(&sc.emissive_nodes[index].exit_index);
        } else {
            float4 n1 = ldg4(reinterpret_cast<const float4*>(&sc.emissive_nodes[index]) + 1);
            bool inside = position.x > n0.x && position.y > n0.y && position.z > n0.z &&
                          position.x < n1.x && position.y < n1.y && position.z < n1.z;
            index = inside ? entry : __float_as_uint(n1.w);
        }
    }
    L.count = count;
    if (L.emissive_instance != DONT_SAMPLE_EMISSIVE) {
        const hk_emissive* em = sc.emissives + picked;
        uint4 e2 = ldg4u(&em->instance);      // instance | pad | alias offset | alias count
        L.surface_area = __ldg(&em->surface_area);
        uint32_t alias_index = min(f32_to_u32(rnd.x * (float)e2.w), e2.w - 1u);
        uint2 ae = __ldg(reinterpret_cast<const uint2*>(sc.alias_table + e2.z + alias_index));  // prob | index
        uint32_t primitive_index = (rnd.y < __uint_as_float(ae.x)) ? ae.y : alias_index;

        const hk_instance* einst = sc.instances + L.emissive_instance;
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
        L.ray_origin = position + normal * RAY_BIAS;
        L.ray_direction = normalize(p - position);
        L.want_ray = dot(L.ray_direction, normal) > 0.0f;
    }
    return L;
}
// Half B (:687-707): the candidate and the light's HitInfo from the result of that walk.  `hit` is only read when L.want_ray.
static __device__ __forceinline__ LightCandidate light_resolve(const DeviceScene& sc, const LightPick& L, vec3 position, Hit hit, HitInfo& info) {
    LightCandidate cand;
    cand.max_distance = F32_MAX;
    cand.min_distance = DISTANCE_MAX;
    cand.emissive_instance = DONT_SAMPLE_EMISSIVE;
    cand.direction = L.rand_direction;
    cand.p = 1.0f;
    info = empty_hit_info(position, L.rand_direction);
    if (L.emissive_instance == DONT_SAMPLE_EMISSIVE) return cand;
    Ray ray;
    ray.origin = L.ray_origin; ray.direction = L.ray_direction; ray.inv_direction = v3(0.0f);
    const bool found = L.want_ray && hit.instance_index != U32_MAX;
    if (found) {
        hit.instance_index = L.emissive_instance;
        info = hit_info(sc, ray, hit);
        cand.emissive_instance = L.emissive_instance;
        cand.direction = ray.direction;
        cand.max_distance = hit.distance;
        cand.min_distance = hit.distance - 0.1f;
        vec3 delta = xyz(info.position) - position;
        cand.p = dot(delta, delta) / fabsf(dot(ray.direction, info.normal) * L.surface_area);
        cand.p = cand.p / L.count;
    } else {
        info = empty_hit_info(ray.origin, ray.direction);
    }
    return cand;
}

template <bool COUNT>
__device__ __forceinline__ void pool_flush_counters(const KParams& P, uint32_t tlas, uint32_t blas) {
    if (!COUNT || P.counters == nullptr) return;
    for (int o = 16; o > 0; o >>= 1) {
        tlas += __shfl_xor_sync(FULL_MASK, tlas, o);
        blas += __shfl_xor_sync(FULL_MASK, blas, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (tlas) atomicAdd(&P.counters->tlas, (unsigned long long)tlas);
        if (blas) atomicAdd(&P.counters->blas, (unsigned long long)blas);
    }
}

// ----------------------------------------------------------------------------- P3: indirect_lit_ambient, pooled
template <bool MULTI, bool COUNT, bool TEX>
__global__ void __launch_bounds__(POOL_THREADS, HK_POOL_MINB) kc_indirect(const __grid_constant__ KParams P) {
    __shared__ PoolShared S;
    pool_stage_begin(S, P.scene, P.scene.stage);
    __syncthreads();                                   // mbarrier + queue counters initialised

    int x, y;
    pool_pixel(x, y, P);
    const bool in_launch = tile_active(P, x, y);
    const DeviceScene sc = scene_variant<TEX>(P.scene);
    const hk_frame_uniform& frame = P.in.frame;
    const ShadeEnv env = make_env(P);
    const size_t idx = in_launch ? render_index(P.band, x, y) : 0;
    const size_t gidx = in_launch ? light_gbuffer_index(P, x, y, idx) : 0;
    const PassBuffers B = bind(P, 2);
    uint32_t n_tlas = 0, n_blas = 0;

    float4 pd = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (in_launch) pd = P.planes.pos_depth[gidx];
    const float depth = pd.w;
    // pixels that trace: inside the launch rectangle, on a surface, with at least one bounce asked for
    const bool surface_pixel = in_launch && !(frame.indirect_bounces == 0u || depth < F32_EPSILON);
    if (in_launch && !surface_pixel) {                 // light.wgsl:1279-1287
        PackedQuarters q = pack_reservoir(zero_reservoir());
        store_quarters(B.reservoir, idx, q);
        store_quarters(B.spatial_reservoir, idx, q);
        scatter_claim(P, idx, x, y, SCATTER_BACKGROUND);
        P.planes.variance[2][idx] = 0.0f;
        P.planes.render[2][idx] = make_uint2(0u, 0u);
    }

    vec3 position = v3(0.0f), normal = v3(0.0f);
    Sample s = zero_sample();
    if (surface_pixel) {
        position = f4xyz(pd);
        normal = normalize(xyz(unpack4x8snorm(P.planes.normal[gidx])));  // normalised here (light.wgsl:1289)
        s.random = noise_random(P, x, y);
        s.visible_position = v4(position, depth);
        s.visible_normal = normal;
        s.visible_instance = f32_to_u32(P.planes.instance_material[gidx].x);
    }

    const WalkScene W = pool_stage_wait(S, P.scene, P.scene.stage);   // the staged records have landed

    float pdf = 0.0f;
    vec3 b_position = position, b_normal = normal;     // the path vertex we are leaving
    vec4 b_random = s.random;
    vec3 color_transport = v3(1.0f);
    const uint32_t bounces = MULTI ? frame.indirect_bounces : 1u;
    bool alive = surface_pixel;                        // still extending its path
    int phase = 0;
    for (uint32_t n = 0u; n < bounces; n += 1u) {
        alive = alive && (color_transport.x > 0.01f || color_transport.y > 0.01f || color_transport.z > 0.01f);
        if (!__syncthreads_or(alive)) break;           // every path of the CTA has ended

        // ---- stage A: the bounce ray (closest hit)
        vec4 rand_sample = v4(0.0f);
        Ray ray;
        ray.origin = ray.direction = ray.inv_direction = v3(0.0f);
        if (alive) {
            rand_sample = sample_cosine_hemisphere(b_random.x, b_random.y);
            ray.origin = b_position + b_normal * RAY_BIAS;
            ray.direction = mul(normal_basis(b_normal), xyz(rand_sample));
            if (COUNT) n_tlas += 1u;
        }
        pool_push(S, phase, alive, RAY_KIND_TLAS, ray.origin, ray.direction, F32_MAX, 0.0f, DONT_EXCLUDE);
        pool_traverse(S, W, phase); ++phase;

        // ---- stage B: the hit; pick a light for it (first half of select_light_candidate)
        HitInfo info = empty_hit_info(v3(0.0f), v3(0.0f));
        vec3 h_position = v3(0.0f), h_normal = v3(0.0f);
        vec2 h_uv = v2(0.0f, 0.0f);
        uint32_t h_material = 0u;
        bool on_surface = false;
        LightPick pick;
        pick.rand_direction = pick.ray_origin = pick.ray_direction = v3(0.0f);
        pick.count = pick.surface_area = 0.0f; pick.emissive_instance = DONT_SAMPLE_EMISSIVE; pick.want_ray = false;
        if (alive) {
            const Hit hit = pool_result(S);
            info = hit_info(sc, ray, hit);
            if (n == 0u) {
                s.sample_position = info.position;
                s.sample_normal = info.normal;
                pdf = rand_sample.w;
            }
            h_position = xyz(info.position); h_normal = info.normal;
            if (hit.instance_index != U32_MAX) {
                on_surface = true;
                h_uv = info.uv; h_material = info.material_index;
                pick = light_pick(sc, env, b_random, h_position, h_normal, info.instance_index);
                if (COUNT && pick.want_ray) n_blas += 1u;
            } else {                                   // escaped: ambient, path ends (light.wgsl:1391-1397)
                vec3 out_radiance = xyz(input_radiance(sc, env, ray.direction, info, false, DONT_SAMPLE_EMISSIVE, true));
                s.radiance = MULTI ? s.radiance + v4(color_transport * out_radiance, 0.0f) : s.radiance + v4(out_radiance, 0.0f);
                alive = false;
            }
        }
        pool_push(S, phase, on_surface && pick.want_ray, RAY_KIND_BLAS, pick.ray_origin, pick.ray_direction, F32_MAX, 0.0f, pick.emissive_instance);
        pool_traverse(S, W, phase); ++phase;

        // ---- stage C: the light candidate (second half); the shadow ray towards it
        LightCandidate cand;
        cand.direction = v3(0.0f); cand.max_distance = cand.min_distance = 0.0f; cand.emissive_instance = DONT_SAMPLE_EMISSIVE; cand.p = 0.0f;
        bool shadow = false;
        if (on_surface) {
            Hit light_hit;
            light_hit.u = light_hit.v = light_hit.distance = 0.0f; light_hit.instance_index = light_hit.primitive_index = U32_MAX;
            if (pick.want_ray) light_hit = pool_result(S);
            cand = light_resolve(sc, pick, h_position, light_hit, info);
            shadow = dot(cand.direction, h_normal) > 0.0f && cand.p > 0.0f;
            if (shadow) {
                ray.origin = h_position + h_normal * RAY_BIAS;
                ray.direction = cand.direction;
                if (COUNT) n_tlas += 1u;
            }
        }
        pool_push(S, phase, shadow, RAY_KIND_TLAS, ray.origin, ray.direction, cand.max_distance, cand.min_distance, cand.emissive_instance);
        pool_traverse(S, W, phase); ++phase;

        // ---- stage D: shade the vertex, extend the path
        if (on_surface) {
            Surface surface = retreive_surface(sc, h_material, h_uv);
            surface.roughness = 1.0f;
            const bool sample_directional = (cand.emissive_instance == DONT_SAMPLE_EMISSIVE);
            const vec3 bounce_view_direction = normalize(b_position - h_position);
            if (shadow) {
                const Hit hit = pool_result(S);
                occlude_hit_info(ray, hit, info);
                vec4 in_radiance = input_radiance(sc, env, ray.direction, info, sample_directional, cand.emissive_instance, false);
                vec3 out_radiance = shading(env, bounce_view_direction, h_normal, ray.direction, surface, in_radiance);
                out_radiance = out_radiance / cand.p;
                if (MULTI) {
                    if (n > 0u) out_radiance = (rand_sample.w < 0.01f) ? v3(0.0f) : out_radiance / rand_sample.w;
                    float out_luminance = luminance(out_radiance);
                    if (out_luminance > frame.max_indirect_luminance)
                        out_radiance = out_radiance * frame.max_indirect_luminance / out_luminance;
                    s.radiance = s.radiance + v4(color_transport * out_radiance, 1.0f);
                } else {
                    s.radiance = s.radiance + v4(out_radiance, 1.0f);
                }
            }
            if (MULTI) {
                color_transport = color_transport * env_brdf(bounce_view_direction, h_normal, surface);
                b_random = fract(b_random + (float)frame.number * GOLDEN_RATIO);
                b_position = h_position;
                b_normal = h_normal;
            }
        }
    }

    if (surface_pixel) {
        // ReSTIR: temporal (light.wgsl:1400-1498); the G-buffer values are re-read instead of being kept alive across the walks
        const float4 vu = P.planes.velocity_uv[gidx];
        const uint32_t material_id = f32_to_u32(P.planes.instance_material[gidx].y);
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
    if (!in_launch || !band_owned(P.band, x, y)) { n_tlas = 0; n_blas = 0; }   // ghost pixels are redundant work: not counted
    pool_flush_counters<COUNT>(P, n_tlas, n_blas);
}

static dim3 pool_grid_for(const KParams& P) {
    int rows = P.row_hi - P.row_lo, cols = P.col_hi - P.col_lo;
    return dim3((unsigned)((cols + POOL_TILE_W - 1) / POOL_TILE_W), (unsigned)((rows + POOL_TILE_H - 1) / POOL_TILE_H), 1u);
}

}  // namespace hkd

using namespace hkd;

void hk_launch_indirect_pool(const KParams& P, bool multi, bool count, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    const dim3 g = pool_grid_for(P);
    const bool tex = P.scene.texture_count != 0u;
    if (count) {
        if (multi) kc_indirect<true, true, true><<<g, POOL_THREADS, 0, st>>>(P);
        else kc_indirect<false, true, true><<<g, POOL_THREADS, 0, st>>>(P);
    } else if (tex) {
        if (multi) kc_indirect<true, false, true><<<g, POOL_THREADS, 0, st>>>(P);
        else kc_indirect<false, false, true><<<g, POOL_THREADS, 0, st>>>(P);
    } else {
        if (multi) kc_indirect<true, false, false><<<g, POOL_THREADS, 0, st>>>(P);
        else kc_indirect<false, false, false><<<g, POOL_THREADS, 0, st>>>(P);
    }
}
