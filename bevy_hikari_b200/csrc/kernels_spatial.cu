// kernels_spatial.cu — spatial reuse of the ReSTIR reservoirs (light.wgsl:1500-1684), both pipelines.  In its own translation unit
// because it traces no rays: nothing in here decides visibility or an id, so the product build compiles it (like kernels_post.cu)
// with the tolerance flags of build.py (FMA contraction, approximate division / square root / exp), while the kernels that walk the
// BVH stay on exact arithmetic.  The exact build compiles it like everything else and is bit-identical to the oracle.
#include "hk_tile.cuh"
#include "hk_kernels.h"

#ifndef HK_NO_TEXTURE_VARIANT
#define HK_NO_TEXTURE_VARIANT 1
#endif
// Requesting a neighbour's reservoir together with its depth, and dividing by the frame size with a host-computed reciprocal (exact
// whenever the quotient is normal); =0 restores the two-step load / the division for A/B runs.
#ifndef HK_SPATIAL_EAGER_LOAD
#define HK_SPATIAL_EAGER_LOAD 1
#endif
#ifndef HK_SPATIAL_FAST_DIV
#define HK_SPATIAL_FAST_DIV 1
#endif

// CTAs of 256 threads per SM of the tiled kernel: 74 KB of shared memory each for the indirect pipeline (at most 3 fit), 32 KB for the
// emissive one.  2 CTAs/SM = 127 registers without spills rather than 3 CTAs/SM = 80 registers with spills (slower on the H100)
#ifndef HK_SPATIAL_TILED_MINB_INDIRECT
#define HK_SPATIAL_TILED_MINB_INDIRECT 2
#endif
#ifndef HK_SPATIAL_TILED_MINB_EMISSIVE
#define HK_SPATIAL_TILED_MINB_EMISSIVE 2
#endif
// kc_spatial stages its tiles only when one of its pixels is a surface pixel (=0: every CTA stages them, for A/B runs)
#ifndef HK_SPATIAL_SKIP_EMPTY_TILES
#define HK_SPATIAL_SKIP_EMPTY_TILES 1
#endif
// Surviving neighbours whose gathers kc_spatial keeps in flight ahead of the one it merges.  Each holds 12 registers: 2 spills at the
// 127-register cap of 2 CTAs/SM and was slower on the H100 (cornell 1080p)
#ifndef HK_SPATIAL_GATHER_AHEAD
#define HK_SPATIAL_GATHER_AHEAD 1
#endif

namespace hkd {

template <bool TEX>
__device__ __forceinline__ DeviceScene scene_variant(const DeviceScene& scene) {
    DeviceScene sc = scene;
    if (!TEX) sc.texture_count = 0u;     // constant-folds every `sc.texture_count != 0u` below it
    return sc;
}

// ----------------------------------------------------------------------------------- P4: spatial_reuse
// light.wgsl:1500-1684.  The reference's 8x8 workgroup cache holds unpack(reservoir_buffer[..]) of this dispatch's
// read-only input, so gathering neighbours straight from the planes (L1/L2-resident) is value-identical.
template <bool EMISSIVE_LIT, bool TEX = true>
__global__ void __launch_bounds__(CTA_THREADS, HK_MINB_SPATIAL) k_spatial(const __grid_constant__ KParams P) {
    constexpr int SIGNAL = EMISSIVE_LIT ? 1 : 2;
    constexpr uint32_t SPATIAL_REUSE_COUNT = EMISSIVE_LIT ? 8u : 16u;   // light.wgsl:246-252
    constexpr float SPATIAL_REUSE_RANGE = EMISSIVE_LIT ? 10.0f : 20.0f;
    constexpr uint32_t SPATIAL_REUSE_TAPS = 4u;
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const DeviceScene sc = scene_variant<TEX>(P.scene);
    const hk_frame_uniform& frame = P.in.frame;
    const size_t idx = render_index(P.band, x, y);
    const size_t gidx = light_gbuffer_index(P, x, y, idx);
    const PassBuffers B = bind(P, SIGNAL);
    const float4 pd = P.planes.pos_depth[gidx];
    const float depth = pd.w;
    const PackedQuarters own = load_quarters(B.reservoir, idx);
    if (depth < F32_EPSILON) {
        // store_spatial_reservoir(pack(unpack(x))): keep the re-pack, it is not the identity for every bit pattern
        store_quarters(B.spatial_reservoir, idx, pack_reservoir(unpack_reservoir(own)));
        P.planes.render[SIGNAL][idx] = make_uint2(0u, 0u);
        return;
    }
    Reservoir r = unpack_reservoir(own);
    const ShadeEnv env = make_env(P);
    const vec3 position = f4xyz(pd);
    const float2 imf = P.planes.instance_material[gidx];
    const float4 vu = P.planes.velocity_uv[gidx];
    const Surface surface = retreive_surface(sc, f32_to_u32(imf.y), v2(vu.z, vu.w));
    const bool use_spatial_variance = r.count <= 4.0f;
    const vec2 uv = pixel_uv(P, x, y);
    const vec2 previous_uv = jittered_deferred_uv(P, uv, 0.25f) - v2(vu.x, vu.y);

    Reservoir q = r;
    const Sample s = q.s;
    const float lifetime_limit = (frame.max_reservoir_lifetime <= 1.0f) ? F32_MAX : frame.max_reservoir_lifetime;  // light.wgsl:913-915
    if (r.lifetime <= lifetime_limit) {
        size_t pidx;
        r = zero_reservoir();
        if (previous_pixel(P, previous_uv, false, pidx)) r = unpack_reservoir(load_quarters(B.previous_spatial_reservoir, pidx));
    }
    const vec3 view_direction = calculate_view(env, position);
    const ShadeCtx shade_ctx = make_shade_ctx(env, view_direction, s.visible_normal, surface);   // shared by every shading below
    if (EMISSIVE_LIT) {
        merge_reservoir(r, q, luminance(xyz(q.s.radiance)));
    } else {
        vec3 out_radiance = shade(shade_ctx, normalize(xyz(s.sample_position) - xyz(s.visible_position)), s.radiance);
        merge_reservoir(r, q, luminance(out_radiance));
    }
    r.s.visible_position = s.visible_position;
    r.s.visible_normal = s.visible_normal;

    const vec2 size_f = v2((float)P.band.RW, (float)P.band.RH);
    const SpatialTable& T = P.spatial_tables[EMISSIVE_LIT ? 1 : 0];
    const float rotation = sum4(s.random);
    for (uint32_t i = 1u; i <= SPATIAL_REUSE_COUNT; i += 1u) {
        float ang = TAU * fract(T.phase[i] + rotation + P.random_frame);
        const float rad = T.radius[i];
        float sn, cs;
        sincos_(ang, &sn, &cs);
        vec2 offset = rad * v2(cs, sn);
        int sx = f32_to_i32(offset.x + (float)x), sy = f32_to_i32(offset.y + (float)y);
        // light.wgsl:1577-1580 tests sample_uv = (coords + 0.5) / size against [0, 1].  For integer coords and size < 2^22
        // the correctly rounded quotient is < 0 iff coords < 0 and > 1 iff coords >= size ((size - 0.5) / size < 1 and
        // (size + 0.5) / size >= 1 + 2^-23 survive rounding), so the two IEEE divisions per neighbour are not needed.
        if (sx < 0 || sy < 0 || sx >= P.band.RW || sy >= P.band.RH) continue;
        const size_t sidx = render_index(P.band, sx, sy);
#if HK_SPATIAL_EAGER_LOAD
        // Default (-DHK_SPATIAL_EAGER_LOAD=0 restores the two-step form): the neighbour's reservoir
        // is requested together with its depth instead of after the depth test, so a neighbour exposes one load latency
        // instead of two; rejected neighbours cost 64 bytes of L1/L2 traffic more.
        const float* depth_ptr = &P.planes.pos_depth[light_gbuffer_index(P, sx, sy, sidx)].w;
        const float sample_depth = __ldg(depth_ptr);
        PackedQuarters packed;
        packed.q0 = __ldg(&B.reservoir.q[0][sidx]); packed.q1 = __ldg(&B.reservoir.q[1][sidx]);
        packed.q2 = __ldg(&B.reservoir.q[2][sidx]); packed.q3 = __ldg(&B.reservoir.q[3][sidx]);
        float depth_ratio = depth / sample_depth;
        if (depth_ratio < 0.9f || depth_ratio > 1.1f) continue;
        q = unpack_reservoir(packed);
#else
        const float sample_depth = P.planes.pos_depth[light_gbuffer_index(P, sx, sy, sidx)].w;
        float depth_ratio = depth / sample_depth;
        if (depth_ratio < 0.9f || depth_ratio > 1.1f) continue;
        q = unpack_reservoir(load_quarters(B.reservoir, sidx));
#endif
        bool normal_miss = dot(s.visible_normal, q.s.visible_normal) < 0.866f;
        if (q.count < F32_EPSILON || normal_miss) continue;
        vec3 sample_direction = normalize(xyz(q.s.sample_position) - xyz(s.visible_position));
        if (dot(sample_direction, s.visible_normal) < 0.0f) continue;

        // screen-space depth march towards the neighbour (light.wgsl:1608-1628)
        const uint32_t tap_count = T.tap_count[i];
        bool occluded = false;
        vec2 unit = normalize(offset);
        for (uint32_t j = 1u; j <= tap_count; j += 1u) {
            float tap_dist = T.tap_dist[i][j - 1u];
#if HK_SPATIAL_FAST_DIV
            // Default since round 2 (-DHK_SPATIAL_FAST_DIV=0 restores the IEEE division): x / C for the frame constant C as q = x * y, r = fma(-q, C, x), fma(r, y, q)
            // with y = RN(1 / C) from the host — the correctly rounded quotient whenever it is a normal number
            // (tools/check_runtime_division.cpp: all 2^32 inputs for the benchmark extents); a subnormal quotient is absorbed
            // by the addition to uv >= 0.5 / size.
            const vec2 tap_offset = tap_dist * unit;
            const float qx = tap_offset.x * P.inv_rw, qy = tap_offset.y * P.inv_rh;
            vec2 tap_uv = uv + v2(fmaf(fmaf(-qx, size_f.x, tap_offset.x), P.inv_rw, qx), fmaf(fmaf(-qy, size_f.y, tap_offset.y), P.inv_rh, qy));
#else
            vec2 tap_uv = uv + (tap_dist * unit) / size_f;
#endif
            vec2 tap_deferred_uv = jittered_deferred_uv(P, tap_uv, 0.25f);
            int tx = f32_to_i32(tap_deferred_uv.x * (float)P.band.W), ty = f32_to_i32(tap_deferred_uv.y * (float)P.band.H);
            float tap_depth = 0.0f;  // out-of-bounds textureLoad -> 0
            if (tx >= 0 && tx < P.band.W && ty >= 0 && ty < P.band.H) tap_depth = P.planes.pos_depth[band_index(P.band, tx, ty)].w;
            float ref_depth = mixf(depth, sample_depth, T.tap_ratio[i][j - 1u]);
            if (tap_depth > ref_depth + 0.00001f) { occluded = true; break; }
        }
        if (occluded) continue;

        float jacobian = (q.s.sample_position.w > 0.5f) ? compute_jacobian(q.s, s) : 1.0f;
        if (EMISSIVE_LIT) {
            merge_reservoir(r, q, luminance(xyz(q.s.radiance)) / jacobian);
        } else {
            vec3 out_radiance = shade(shade_ctx, sample_direction, q.s.radiance);
            merge_reservoir(r, q, luminance(out_radiance) / jacobian);
        }
    }

    float m = (float)frame.max_spatial_reuse_count;
    if (r.count > m) {
        r.w_sum *= m / r.count;
        r.w2_sum *= m / r.count;
        r.count = m;
    }
    vec3 out_radiance = shade(shade_ctx, normalize(xyz(r.s.sample_position) - xyz(s.visible_position)), r.s.radiance);
    float total_lum = EMISSIVE_LIT ? r.count * luminance(xyz(r.s.radiance)) : r.count * luminance(out_radiance);
    r.w = (total_lum > 0.0f) ? r.w_sum / total_lum : 0.0f;
    r.lifetime += 1.0f;
    store_quarters(B.spatial_reservoir, idx, pack_reservoir(r));
    if (use_spatial_variance) P.planes.variance[SIGNAL][idx] = variance_of(r);
    vec3 out_color = r.w * out_radiance;   // RENDER_EMISSIVE is never set on the spatial pipelines (light.rs:433-442)
    uvec2 o = pack_rgba16f(v4(out_color, 1.0f));
    P.planes.render[SIGNAL][idx] = make_uint2(o.x, o.y);
}


// Frame pixel (tx, ty) of tap j (1-based) of neighbour i's screen-space depth march (light.wgsl:1608-1628) at upscale ratio 1
__device__ __forceinline__ void march_tap(const KParams& P, const SpatialTable& T, uint32_t i, uint32_t j, vec2 uv, vec2 size_f, vec2 unit,
                                          int& tx, int& ty) {
    float tap_dist = T.tap_dist[i][j - 1u];
#if HK_SPATIAL_FAST_DIV
    const vec2 tap_offset = tap_dist * unit;
    const float qx = tap_offset.x * P.inv_rw, qy = tap_offset.y * P.inv_rh;
    vec2 tap_uv = uv + v2(fmaf(fmaf(-qx, size_f.x, tap_offset.x), P.inv_rw, qx), fmaf(fmaf(-qy, size_f.y, tap_offset.y), P.inv_rh, qy));
#else
    vec2 tap_uv = uv + (tap_dist * unit) / size_f;
#endif
    tx = f32_to_i32(tap_uv.x * (float)P.band.W); ty = f32_to_i32(tap_uv.y * (float)P.band.H);
}
// The depth march of neighbour i with every tap read from the G-buffer instead of the staged tile: kc_spatial's fallback when a tap
// lies in the frame but outside the tile (a tap lies between the pixel and its neighbour, hence inside it; a float coordinate that
// rounds one pixel out of it has never been observed) or when the table holds more taps than kc_spatial unrolls
static __device__ HK_NOINLINE bool march_occluded_from_plane(const KParams& P, const SpatialTable& T, uint32_t i, vec2 uv, vec2 size_f,
                                                              vec2 unit, float depth, float sample_depth) {
    for (uint32_t j = 1u; j <= T.tap_count[i]; j += 1u) {
        int tx, ty;
        march_tap(P, T, i, j, uv, size_f, unit, tx, ty);
        float tap_depth = 0.0f;  // out-of-bounds textureLoad -> 0
        if (tx >= 0 && tx < P.band.W && ty >= 0 && ty < P.band.H) tap_depth = P.planes.pos_depth[band_index(P.band, tx, ty)].w;
        if (tap_depth > mixf(depth, sample_depth, T.tap_ratio[i][j - 1u]) + 0.00001f) return true;
    }
    return false;
}

// ------------------------------------------------------------------------- P4 with TMA-staged neighbourhood tiles
// kc_spatial: the same pass for upscale ratio 1 (render space == G-buffer space: every benchmark and every tiled configuration).
// A CTA of 16 x 16 pixels stages, with two TMA tile loads (cp.async.bulk.tensor.2d, hk_tile.cuh), the part of the frame its
// neighbours can lie in — its own tile grown by the reuse radius (20 px indirect, 10 px emissive):
//   * the G-buffer depth plane                          (4 B / px):  the neighbour's depth and every tap of the depth march
//   * quarter 3 of the temporal reservoir being reused (16 B / px):  count + visible normal, i.e. the cheap rejections
// 60 x 56 x 20 B = 66 KB (indirect) / 40 x 36 x 20 B = 28 KB (emissive) of shared memory, plus 2 bytes per neighbour and thread for
// the hand-over between the two stages below.  Per pixel that replaces 16 (8) scattered depth fetches, up to 80 (40) scattered
// depth-march taps and the 64-byte reservoir fetches of the neighbours that the depth, count, normal and march tests reject by reads
// from shared memory.  Stage A runs those tests for every neighbour; stage B gathers the three remaining quarters of the survivors
// only (about 9 of 16 indirect and 5 of 8 emissive neighbours of a surface pixel on cornell 1080p) and merges them.
// Arithmetic and merge order are those of k_spatial: same bytes out (exact flavour).
template <bool EMISSIVE_LIT> struct SpatialTile {
    static constexpr int R = EMISSIVE_LIT ? 10 : 20;
    static constexpr int BH = POOL_TILE_H + 2 * R;                    // rows of the neighbourhood
    static constexpr int BW = tile_box_width(POOL_TILE_W + 2 * R);     // columns: + slack for the 16-byte alignment of the box start
    // every TMA destination starts on a 128-byte boundary
    static constexpr size_t DEPTH_BYTES = ((size_t)BW * BH * 4 + 127) & ~(size_t)127, Q3_BYTES = ((size_t)BW * BH * 16 + 127) & ~(size_t)127;
    static constexpr uint32_t TX_BYTES = (uint32_t)((size_t)BW * BH * 20);     // what the two copies deliver
    static constexpr uint32_t COUNT = EMISSIVE_LIT ? 8u : 16u;
    static constexpr size_t CELL_BYTES = (size_t)COUNT * POOL_THREADS * 2;    // stage A -> B: each survivor's cell, u16 per neighbour and thread
    static constexpr size_t SMEM_BYTES = DEPTH_BYTES + Q3_BYTES + CELL_BYTES + 16;       // + the mbarrier
    static_assert((size_t)BW * BH <= 65536, "cells fit in 16 bits");
};

template <bool EMISSIVE_LIT, bool TEX = true>
__global__ void __launch_bounds__(POOL_THREADS, EMISSIVE_LIT ? HK_SPATIAL_TILED_MINB_EMISSIVE : HK_SPATIAL_TILED_MINB_INDIRECT) kc_spatial(const __grid_constant__ KParams P, const __grid_constant__ TileMap depth_map,
                                                                                   const __grid_constant__ TileMap q3_map, const __grid_constant__ SpatialTable T) {
    using ST = SpatialTile<EMISSIVE_LIT>;
    constexpr int SIGNAL = EMISSIVE_LIT ? 1 : 2;
    constexpr uint32_t SPATIAL_REUSE_COUNT = EMISSIVE_LIT ? 8u : 16u;   // light.wgsl:246-252
    constexpr int R = ST::R, BW = ST::BW, BH = ST::BH;
    HK_DYNAMIC_SMEM(smem);
    float* s_depth = reinterpret_cast<float*>(smem);
    uint4* s_q3 = reinterpret_cast<uint4*>(smem + ST::DEPTH_BYTES);
    uint16_t* s_cell = reinterpret_cast<uint16_t*>(smem + ST::DEPTH_BYTES + ST::Q3_BYTES);
    uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem + ST::DEPTH_BYTES + ST::Q3_BYTES + ST::CELL_BYTES);
    // tile origin in frame coordinates, and in plane (allocation) coordinates for the copy engine
    const int px0 = tile_origin_x(P.col_lo + (int)blockIdx.x * POOL_TILE_W - R - P.band.ax0);       // plane column of the tile's first cell
    const int tx0 = px0 + P.band.ax0, ty0 = P.row_lo + (int)blockIdx.y * POOL_TILE_H - R;
    auto stage_tiles = [&]() {
        mbar_expect_tx(s_bar, ST::TX_BYTES);
        tile_load_2d(s_depth, &depth_map, px0, ty0 - P.band.a0, s_bar);
        tile_load_2d(s_q3, &q3_map, 4 * px0, ty0 - P.band.a0, s_bar);      // the plane as rows of u32: 4 per pixel
        mbar_complete_emulated(s_bar);
    };
    if (threadIdx.x == 0) {
        mbar_init(s_bar, 1u);
        if (!HK_SPATIAL_SKIP_EMPTY_TILES) stage_tiles();
    }
    if (!HK_SPATIAL_SKIP_EMPTY_TILES) __syncthreads();      // the barrier is initialised before anybody waits on it

    int x, y;
    pool_pixel(x, y, P);
    const bool in_launch = tile_active(P, x, y);
    // everything that does not need the tiles first: the copies run meanwhile
    const DeviceScene sc = scene_variant<TEX>(P.scene);
    const hk_frame_uniform& frame = P.in.frame;
    const size_t idx = in_launch ? render_index(P.band, x, y) : 0;
    const PassBuffers Bf = bind(P, SIGNAL);
    float4 pd = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    PackedQuarters own;
    own.q0 = own.q1 = own.q2 = own.q3 = make_uint4(0u, 0u, 0u, 0u);
    if (in_launch) { pd = P.planes.pos_depth[idx]; own = load_quarters(Bf.reservoir, idx); }
    const float depth = pd.w;
    const bool surface_pixel = in_launch && !(depth < F32_EPSILON);
    if (in_launch && !surface_pixel) {
        store_quarters(Bf.spatial_reservoir, idx, pack_reservoir(unpack_reservoir(own)));
        P.planes.render[SIGNAL][idx] = make_uint2(0u, 0u);
    }
#if HK_SPATIAL_SKIP_EMPTY_TILES
    // A CTA of background pixels only (around the model) needs no neighbourhood: it stages nothing and leaves at once.  Otherwise
    // its background threads leave without waiting: the surface threads wait for the copies before the CTA's memory can go away.
    if (!__syncthreads_or(surface_pixel)) return;       // (also orders the barrier's initialisation before any wait on it)
    if (threadIdx.x == 0) stage_tiles();
    if (!surface_pixel) return;
#else
    if (!surface_pixel) { mbar_wait(s_bar, 0u); return; }      // (every thread observes the copies before the CTA's memory can go away)
#endif

    Reservoir r = unpack_reservoir(own);
    const ShadeEnv env = make_env(P);
    const vec3 position = f4xyz(pd);
    const float2 imf = P.planes.instance_material[idx];
    const float4 vu = P.planes.velocity_uv[idx];
    const Surface surface = retreive_surface(sc, f32_to_u32(imf.y), v2(vu.z, vu.w));
    const bool use_spatial_variance = r.count <= 4.0f;
    const vec2 uv = pixel_uv(P, x, y);
    const vec2 previous_uv = uv - v2(vu.x, vu.y);       // jittered_deferred_uv is the identity at ratio 1

    Reservoir q = r;
    const Sample s = q.s;
    const float lifetime_limit = (frame.max_reservoir_lifetime <= 1.0f) ? F32_MAX : frame.max_reservoir_lifetime;  // light.wgsl:913-915
    if (r.lifetime <= lifetime_limit) {
        size_t pidx;
        r = zero_reservoir();
        if (previous_pixel(P, previous_uv, false, pidx)) r = unpack_reservoir(load_quarters(Bf.previous_spatial_reservoir, pidx));
    }
    const vec3 view_direction = calculate_view(env, position);
    const ShadeCtx shade_ctx = make_shade_ctx(env, view_direction, s.visible_normal, surface);   // shared by every shading below
    if (EMISSIVE_LIT) {
        merge_reservoir(r, q, luminance(xyz(q.s.radiance)));
    } else {
        vec3 out_radiance = shade(shade_ctx, normalize(xyz(s.sample_position) - xyz(s.visible_position)), s.radiance);
        merge_reservoir(r, q, luminance(out_radiance));
    }
    r.s.visible_position = s.visible_position;
    r.s.visible_normal = s.visible_normal;

    const vec2 size_f = v2((float)P.band.RW, (float)P.band.RH);
    const float rotation = sum4(s.random);
    mbar_wait(s_bar, 0u);                               // the tiles have landed

    // Stage A, shared memory only: every test that rejects a neighbour without its gathered quarters — bounds, depth ratio, count
    // and visible normal (staged quarter 3) and the screen-space depth march (light.wgsl:1608-1628).  The march runs before the
    // hemisphere test of stage B instead of after it: every test is a pure rejection, so the set of merged neighbours is the same.
    // Unrolled, so that the independent neighbours' shared-memory chains interleave.  Each survivor's cell goes to s_cell.
    uint32_t survivors = 0u;                            // bit i: neighbour i passed stage A
#pragma unroll
    for (uint32_t i = 1u; i <= SPATIAL_REUSE_COUNT; i += 1u) {
        float ang = TAU * fract(T.phase[i] + rotation + P.random_frame);
        const float rad = T.radius[i];
        float sn, cs;
        sincos_(ang, &sn, &cs);
        const vec2 offset = rad * v2(cs, sn);
        int sx = f32_to_i32(offset.x + (float)x), sy = f32_to_i32(offset.y + (float)y);
        if (sx < 0 || sy < 0 || sx >= P.band.RW || sy >= P.band.RH) continue;      // see k_spatial
        const int tcell = (sy - ty0) * BW + (sx - tx0);
        const float sample_depth = s_depth[tcell];
        float depth_ratio = depth / sample_depth;
        if (depth_ratio < 0.9f || depth_ratio > 1.1f) continue;
        // count and visible normal from the staged quarter: the same values unpack_reservoir derives from it in stage B
        const uint4 n_q3 = s_q3[tcell];
        const float n_count = unpack2x16float(n_q3.z).x;
        const vec3 n_normal = normalize(xyz(unpack4x8snorm(n_q3.x)));
        if (n_count < F32_EPSILON || dot(s.visible_normal, n_normal) < 0.866f) continue;

        // screen-space depth march towards the neighbour, every tap out of the staged depth tile.  No exit at the first occluding tap
        // and no branch per tap: "some tap lies in front" is the same outcome, and the taps' shared-memory reads overlap instead of
        // forming a chain of dependent reads and branches (the march was the costliest part of the pass).  tap_count <= 5:
        // u32(radius / max(1, radius / 5)).
        const uint32_t tap_count = T.tap_count[i];
        bool occluded = false, from_plane = tap_count > 5u;
        vec2 unit = normalize(offset);
#pragma unroll
        for (uint32_t j = 1u; j <= 5u; j += 1u) {
            int tx, ty;
            march_tap(P, T, i, j, uv, size_f, unit, tx, ty);
            const bool in_frame = tx >= 0 && tx < P.band.W && ty >= 0 && ty < P.band.H;      // out-of-bounds textureLoad -> 0
            const int cxl = tx - tx0, cyl = ty - ty0;
            const bool in_tile = (unsigned)cxl < (unsigned)BW && (unsigned)cyl < (unsigned)BH;
            const float staged = s_depth[in_tile ? cyl * BW + cxl : 0];
            const float tap_depth = in_frame ? staged : 0.0f;
            const bool live = j <= tap_count;
            from_plane |= live && in_frame && !in_tile;
            occluded |= live && tap_depth > mixf(depth, sample_depth, T.tap_ratio[i][j - 1u]) + 0.00001f;
        }
        if (from_plane) occluded = march_occluded_from_plane(P, T, i, uv, size_f, unit, depth, sample_depth);
        if (occluded) continue;
        survivors |= 1u << i;
        s_cell[(i - 1u) * POOL_THREADS + threadIdx.x] = (uint16_t)tcell;
    }

    // Stage B, survivors only, in neighbour order: the three quarters not staged are gathered from the planes while the survivor
    // before them is unpacked, tested against the hemisphere and merged.  Rejected neighbours no longer sit between two gathers.
    struct Gather { bool valid; int cell; uint4 q0, q1, q2; };
    auto gather_next = [&]() -> Gather {
        Gather g;
        g.valid = survivors != 0u; g.cell = 0;
        g.q0 = g.q1 = g.q2 = make_uint4(0u, 0u, 0u, 0u);
        if (!g.valid) return g;
        const uint32_t i = (uint32_t)__ffs(survivors) - 1u;
        survivors &= survivors - 1u;
        g.cell = s_cell[(i - 1u) * POOL_THREADS + threadIdx.x];
        const size_t sidx = render_index(P.band, tx0 + g.cell % BW, ty0 + g.cell / BW);
        g.q0 = __ldg(&Bf.reservoir.q[0][sidx]); g.q1 = __ldg(&Bf.reservoir.q[1][sidx]); g.q2 = __ldg(&Bf.reservoir.q[2][sidx]);
        return g;
    };
    Gather ahead[HK_SPATIAL_GATHER_AHEAD + 1];
#pragma unroll
    for (int k = 0; k <= HK_SPATIAL_GATHER_AHEAD; ++k) ahead[k] = gather_next();
    while (ahead[0].valid) {
        const Gather cur = ahead[0];
#pragma unroll
        for (int k = 0; k < HK_SPATIAL_GATHER_AHEAD; ++k) ahead[k] = ahead[k + 1];
        ahead[HK_SPATIAL_GATHER_AHEAD] = gather_next();
        PackedQuarters packed;
        packed.q0 = cur.q0; packed.q1 = cur.q1; packed.q2 = cur.q2; packed.q3 = s_q3[cur.cell];
        q = unpack_reservoir(packed);
        vec3 sample_direction = normalize(xyz(q.s.sample_position) - xyz(s.visible_position));
        if (dot(sample_direction, s.visible_normal) < 0.0f) continue;

        float jacobian = (q.s.sample_position.w > 0.5f) ? compute_jacobian(q.s, s) : 1.0f;
        if (EMISSIVE_LIT) {
            merge_reservoir(r, q, luminance(xyz(q.s.radiance)) / jacobian);
        } else {
            vec3 out_radiance = shade(shade_ctx, sample_direction, q.s.radiance);
            merge_reservoir(r, q, luminance(out_radiance) / jacobian);
        }
    }

    float m = (float)frame.max_spatial_reuse_count;
    if (r.count > m) {
        r.w_sum *= m / r.count;
        r.w2_sum *= m / r.count;
        r.count = m;
    }
    vec3 out_radiance = shade(shade_ctx, normalize(xyz(r.s.sample_position) - xyz(s.visible_position)), r.s.radiance);
    float total_lum = EMISSIVE_LIT ? r.count * luminance(xyz(r.s.radiance)) : r.count * luminance(out_radiance);
    r.w = (total_lum > 0.0f) ? r.w_sum / total_lum : 0.0f;
    r.lifetime += 1.0f;
    store_quarters(Bf.spatial_reservoir, idx, pack_reservoir(r));
    if (use_spatial_variance) P.planes.variance[SIGNAL][idx] = variance_of(r);
    vec3 out_color = r.w * out_radiance;   // RENDER_EMISSIVE is never set on the spatial pipelines (light.rs:433-442)
    uvec2 o = pack_rgba16f(v4(out_color, 1.0f));
    P.planes.render[SIGNAL][idx] = make_uint2(o.x, o.y);
}

static dim3 grid_for(const KParams& P) {
    int rows = P.row_hi - P.row_lo, cols = P.col_hi - P.col_lo;
    return dim3((unsigned)((cols + TILE_W - 1) / TILE_W), (unsigned)((rows + TILE_H - 1) / TILE_H), 1u);
}

}  // namespace hkd

using namespace hkd;

static inline bool no_texture(const KParams& P) { return HK_NO_TEXTURE_VARIANT && P.scene.texture_count == 0u; }

template <bool EMISSIVE_LIT, bool TEX>
static void launch_tiled(const KParams& P, const TileMap& depth_map, const TileMap& q3_map, const SpatialTable& table, cudaStream_t st) {
    const size_t smem = SpatialTile<EMISSIVE_LIT>::SMEM_BYTES;
    static bool configured[64] = {};     // per instantiation AND per device: the attribute belongs to the function on one device
    int dev = 0;
    cudaGetDevice(&dev);
    if (!configured[dev & 63]) { cudaFuncSetAttribute(kc_spatial<EMISSIVE_LIT, TEX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); configured[dev & 63] = true; }
    const int rows = P.row_hi - P.row_lo, cols = P.col_hi - P.col_lo;
    const dim3 g((unsigned)((cols + POOL_TILE_W - 1) / POOL_TILE_W), (unsigned)((rows + POOL_TILE_H - 1) / POOL_TILE_H), 1u);
    kc_spatial<EMISSIVE_LIT, TEX><<<g, POOL_THREADS, smem, st>>>(P, depth_map, q3_map, table);
}

// `depth_map` / `q3_map`: TMA descriptors of the depth plane and of quarter 3 of the temporal reservoir this launch reuses, boxed for
// this variant's radius (context.cu); nullptr (or an upscale ratio above 1) selects the gather-from-global form.  `table`: host copy
// of this pipeline's P.spatial_tables entry, which the tiled form takes as a kernel parameter.
void hk_launch_spatial(const KParams& P, bool emissive, const TileMap* depth_map, const TileMap* q3_map, const SpatialTable& table, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    if (depth_map && q3_map && P.ratio1) {
        if (no_texture(P)) { if (emissive) launch_tiled<true, false>(P, *depth_map, *q3_map, table, st); else launch_tiled<false, false>(P, *depth_map, *q3_map, table, st); }
        else { if (emissive) launch_tiled<true, true>(P, *depth_map, *q3_map, table, st); else launch_tiled<false, true>(P, *depth_map, *q3_map, table, st); }
        return;
    }
    if (no_texture(P)) {
        if (emissive) k_spatial<true, false><<<grid_for(P), CTA_THREADS, 0, st>>>(P);
        else k_spatial<false, false><<<grid_for(P), CTA_THREADS, 0, st>>>(P);
        return;
    }
    if (emissive) k_spatial<true><<<grid_for(P), CTA_THREADS, 0, st>>>(P);
    else k_spatial<false><<<grid_for(P), CTA_THREADS, 0, st>>>(P);
}
