// kernels_post.cu — the post-process node of the CUDA path: demodulation, 4-level edge-stopping a-trous denoise and
// tone mapping.  Replaces src/shaders/denoise.wgsl + tone_mapping.wgsl as dispatched by PostProcessNode::run
// (src/post_process.rs:1140-1234): 3 x (1 + 4) + 1 = 16 dispatches there, 5 launches here —
//   * the three signals (sun / emissive / indirect) are filtered by the same thread: the geometric edge-stopping
//     weights (normal^16, depth/gradient, instance) depend only on the G-buffer and are computed once per tap instead
//     of three times; only the luminance weight is per signal.  Per signal the arithmetic and its order are the
//     reference's, so results are bit-identical to running the passes one signal at a time;
//   * level 3 re-modulates with albedo, and (optionally) sums the signals and applies Reinhard tone mapping in the
//     same thread, so denoise_render[3] never has to be re-read.
#include "hk_tile.cuh"
#include "hk_kernels.h"

namespace hkd {

__device__ __forceinline__ vec4 load16(const uint2* plane, size_t i) {
    uint2 u = plane[i];
    uvec2 w; w.x = u.x; w.y = u.y;
    return unpack_rgba16f(w);
}
__device__ __forceinline__ void store16(uint2* plane, size_t i, vec4 v) {
    uvec2 w = pack_rgba16f(v);
    plane[i] = make_uint2(w.x, w.y);
}
// the tone-mapped pixel: into the context's own tile and, when a frame target is set, into the assembled frame — for a
// remote target this store over NVLink *is* the transfer (no gather kernel, no collective on the data path)
__device__ __forceinline__ void store_final(const KParams& P, int x, int y, vec4 color) {
    uvec2 w = pack_rgba16f(color);
    const uint2 bits = make_uint2(w.x, w.y);
    if (P.tile_images) P.planes.tone_ring_db[P.in.frame.number % 2u][band_index(P.band, x, y)] = bits;   // incl. the ring the upscalers sample
    if (!band_owned(P.band, x, y)) return;
    P.planes.tone_mapped[owned_index(P.band, x, y)] = bits;
    if (P.frame_target) P.frame_target[(size_t)y * P.frame_pitch + (size_t)x] = bits;
}
__device__ __forceinline__ bool bad3(vec3 v) {  // any_is_nan_vec3(v) || any(v > F32_MAX), denoise.wgsl:190,239
    return is_nan(v.x) || is_nan(v.y) || is_nan(v.z) || v.x > F32_MAX || v.y > F32_MAX || v.z > F32_MAX;
}
__device__ __forceinline__ float kernel_at(const KParams& P, int a, int b) { return P.in.frame.kernel[a][b]; }

// ----------------------------------------------------------------------------------------- demodulation
// denoise.wgsl:135-162 for all signals of a pixel.
__global__ void __launch_bounds__(CTA_THREADS) k_demodulation(const __grid_constant__ KParams P, int signals) {
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const size_t idx = render_index(P.band, x, y);
    size_t gidx = idx;   // the G-buffer / albedo texel this render pixel samples (nearest at the +-0.5-texel jittered uv)
    if (!P.ratio1) {
        int dx, dy;
        denoise_deferred_coords(P, render_uv(P, x, y), x, y, dx, dy);
        gidx = band_index(P.band, dx, dy);
    }
    // Every input of this kernel is read-only here, so all loads are issued before the first store (ld.global.nc): the
    // kernel is a chain of dependent global-load latencies otherwise.
    const uint32_t packed_normal = __ldg(&P.planes.normal[gidx]);
    const float depth = __ldg(&P.planes.pos_depth[gidx].w);
    const float instance = __ldg(&P.planes.instance_material[gidx].x);
    const uint2 albedo_bits = __ldg(&P.planes.albedo[gidx]);
    uint2 render_bits[3];
    float variance[3][9];
    bool tap_inside[9];
#pragma unroll
    for (int ox = -1; ox <= 1; ++ox)
#pragma unroll
        for (int oy = -1; oy <= 1; ++oy) {
            const int sx = x + ox, sy = y + oy;
            tap_inside[(ox + 1) * 3 + (oy + 1)] = !(sx < 0 || sy < 0 || sx >= P.band.RW || sy >= P.band.RH);
        }
#pragma unroll
    for (int sgl = 0; sgl < 3; ++sgl) {
        if (sgl >= signals) continue;
        render_bits[sgl] = __ldg(&P.planes.render[sgl][idx]);
#pragma unroll
        for (int ox = -1; ox <= 1; ++ox)
#pragma unroll
            for (int oy = -1; oy <= 1; ++oy) {
                const int t = (ox + 1) * 3 + (oy + 1);
                variance[sgl][t] = tap_inside[t] ? __ldg(&P.planes.variance[sgl][render_index(P.band, x + ox, y + oy)]) : 0.0f;
            }
    }
    {   // tap geometry for the four a-trous levels: the normalised normal, depth and instance id of this pixel are read
        // by up to 36 taps; normalise once here instead of 36 times there (same operations, same values)
        const vec3 n = normalize(xyz(unpack4x8snorm(packed_normal)));
        P.planes.dn_geometry[idx] = make_float4(n.x, n.y, n.z, depth);
        P.planes.dn_instance[idx] = instance;
    }
    uvec2 ab; ab.x = albedo_bits.x; ab.y = albedo_bits.y;
    const vec3 albedo = xyz(unpack_rgba16f(ab));
#pragma unroll
    for (int sgl = 0; sgl < 3; ++sgl) {
        if (sgl >= signals) continue;
        uvec2 rb; rb.x = render_bits[sgl].x; rb.y = render_bits[sgl].y;
        vec3 irradiance = xyz(unpack_rgba16f(rb));
        vec3 q = irradiance / albedo;
        irradiance = v3(albedo.x < 0.01f ? 0.0f : q.x, albedo.y < 0.01f ? 0.0f : q.y, albedo.z < 0.01f ? 0.0f : q.z);
        store16(P.planes.dn_internal[0][sgl], idx, v4(irradiance, 1.0f));
        float sum_variance = 0.0f;
        // accumulate_variance order of denoise.wgsl:152-160: x outer (-1,0,1), y inner (-1,0,1)
#pragma unroll
        for (int ox = -1; ox <= 1; ++ox) {
#pragma unroll
            for (int oy = -1; oy <= 1; ++oy) {
                const int t = (ox + 1) * 3 + (oy + 1);
                if (!tap_inside[t]) continue;
                const float v = variance[sgl][t];
                if (v > F32_MAX) continue;
                sum_variance += kernel_at(P, oy + 1, ox + 1) * fmax_(v, 0.0f);
            }
        }
        P.planes.dn_variance[sgl][idx] = sum_variance;
    }
}

// --------------------------------------------------------------------------------------------- denoise level
struct SignalAcc {
    vec3 irradiance, sum_irradiance;
    float sum_w, lum, lum_denominator, ff_moment_1, ff_moment_2, ff_count;
};

template <int LEVEL, bool FUSE_TONE_MAPPING>
__global__ void __launch_bounds__(CTA_THREADS, HK_MINB_DENOISE) k_denoise(const __grid_constant__ KParams P, int signals, int keep_denoised) {
    constexpr int STEP = 8 >> LEVEL;  // denoise.wgsl:101-114: coarse to fine
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const size_t idx = render_index(P.band, x, y);
    size_t gidx = idx;
    if (!P.ratio1) {
        int dx, dy;
        denoise_deferred_coords(P, render_uv(P, x, y), x, y, dx, dy);
        gidx = band_index(P.band, dx, dy);
    }
    const float4 geometry = P.planes.dn_geometry[idx];
    const float depth = geometry.w;
    vec4 result[3];
    result[0] = result[1] = result[2] = v4(0.0f);
    if (!(depth < F32_EPSILON)) {
        const float2 dg = P.planes.depth_gradient[gidx];
        const vec2 depth_gradient = v2(dg.x, dg.y);
        const vec3 normal = f4xyz(geometry);
        const float instance = P.planes.dn_instance[idx];

        SignalAcc acc[3];
#pragma unroll
        for (int sgl = 0; sgl < 3; ++sgl) {
            if (sgl >= signals) continue;
            SignalAcc& a = acc[sgl];
            // denominator of luminance_weight (denoise.wgsl:56-61) depends on the centre pixel only: two sqrt per pixel
            // instead of two per tap
            a.lum_denominator = 4.0f * pow025(P.planes.dn_variance[sgl][idx]) + 0.001f;
            a.irradiance = xyz(load16(P.planes.dn_internal[LEVEL][sgl], idx));
            a.sum_irradiance = a.irradiance * kernel_at(P, 1, 1);
            a.sum_w = kernel_at(P, 1, 1);
            if (bad3(a.irradiance)) { a.irradiance = v3(0.0f); a.sum_irradiance = v3(0.0f); a.sum_w = 0.0f; }
            a.lum = luminance(a.irradiance);
            a.ff_moment_1 = 0.0f; a.ff_moment_2 = 0.0f; a.ff_count = 0.0f;
        }

        // tap order of denoise.wgsl:252-268
        const int OX[8] = {-1, 0, 1, -1, 1, -1, 0, 1};
        const int OY[8] = {-1, -1, -1, 0, 0, 1, 1, 1};
        // Every tap's loads are unconditional (out-of-frame taps read a clamped, valid address) and go through the read-only path, so
        // nothing but register pressure keeps the compiler from issuing the loads of later taps during the arithmetic of earlier
        // ones; only the accumulation is predicated.  Same operations on the same values for every tap that counts.
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            const int ox = OX[t], oy = OY[t];
            const int sx = x + ox * STEP, sy = y + oy * STEP;
            const bool valid = !(sx < 0 || sy < 0 || sx >= P.band.RW || sy >= P.band.RH);
            const size_t sidx = render_index(P.band, min(max(sx, 0), P.band.RW - 1), min(max(sy, 0), P.band.RH - 1));
            const float4 sample_geometry = __ldg(&P.planes.dn_geometry[sidx]);
            const float sample_instance = __ldg(&P.planes.dn_instance[sidx]);
            uint2 bits[3];
#pragma unroll
            for (int sgl = 0; sgl < 3; ++sgl) bits[sgl] = (sgl < signals) ? __ldg(&P.planes.dn_internal[LEVEL][sgl][sidx]) : make_uint2(0u, 0u);
            const vec3 sample_normal = f4xyz(sample_geometry);
            const float sample_depth = sample_geometry.w;
            const float w_normal = pow16(fmax_(0.0f, dot(normal, sample_normal)));                                       // :44-47
            const float w_depth = exp_((-fabsf(depth - sample_depth)) / (fabsf(dot(depth_gradient, v2((float)ox, (float)oy))) + 0.01f));  // :50-53
            const float w_instance = fmax_(0.0f, 1.0f - fabsf(instance - sample_instance));                              // :63-65
            const float w_geometry = w_normal * w_depth * w_instance;
            const float k = kernel_at(P, oy + 1, ox + 1);
#pragma unroll
            for (int sgl = 0; sgl < 3; ++sgl) {
                if (sgl >= signals) continue;
                SignalAcc& a = acc[sgl];
                uvec2 q; q.x = bits[sgl].x; q.y = bits[sgl].y;
                vec3 irr = xyz(unpack_rgba16f(q));
                float sample_luminance = luminance(irr);
                float w_luminance = exp_((-fabsf(a.lum - sample_luminance)) / a.lum_denominator);                       // :56-61
                float w = clampf(w_geometry * w_luminance, 0.0f, 1.0f) * k;
                if (valid && !bad3(irr)) {
                    a.sum_irradiance = a.sum_irradiance + irr * w;
                    a.sum_w += w;
                    if (sgl != 0) {  // FIREFLY_FILTERING: emissive + indirect only (post_process.rs:1193-1197)
                        a.ff_moment_1 += sample_luminance;
                        a.ff_moment_2 += sample_luminance * sample_luminance;
                        a.ff_count += 1.0f;
                    }
                }
            }
        }

        vec4 albedo = v4(1.0f);
        if (LEVEL == 3) albedo = load16(P.planes.albedo, gidx);
#pragma unroll
        for (int sgl = 0; sgl < 3; ++sgl) {
            if (sgl >= signals) continue;
            SignalAcc& a = acc[sgl];
            vec3 irradiance = (a.sum_w < 0.0001f) ? v3(0.0f) : a.sum_irradiance / a.sum_w;
            if (sgl != 0) {
                float ff_mean = a.ff_moment_1 / a.ff_count;
                float ff_var = a.ff_moment_2 / a.ff_count - ff_mean * ff_mean;
                if (a.lum > ff_mean + 3.0f * sqrtf(ff_var)) irradiance = ff_mean / a.lum * irradiance;
            }
            vec4 color = v4(irradiance, 1.0f);
            if (LEVEL == 3) color = color * albedo;  // denoise.wgsl:314-315
            result[sgl] = color;
        }
    }

    if (LEVEL < 3) {
#pragma unroll
        for (int sgl = 0; sgl < 3; ++sgl)
            if (sgl < signals) store16(P.planes.dn_internal[LEVEL + 1][sgl], idx, result[sgl]);
        return;
    }
    // level 3 -> denoise_render (Rgba16Float), then tone_mapping.wgsl:21-32 on the f16-rounded values
    vec4 color = v4(0.0f);
#pragma unroll
    for (int sgl = 0; sgl < 3; ++sgl) {
        if (sgl >= signals) continue;
        uvec2 w = pack_rgba16f(result[sgl]);
        if (!FUSE_TONE_MAPPING || keep_denoised) P.planes.dn_render[sgl][idx] = make_uint2(w.x, w.y);
        if (FUSE_TONE_MAPPING) color = color + unpack_rgba16f(w);
    }
    if (FUSE_TONE_MAPPING && (P.tile_images || band_owned(P.band, x, y))) {
        vec3 rgb = reinhard_luminance(vmax(xyz(color), 0.0039f));
        color = v4(rgb, color.w);
        if (!(color.w > 0.0f))
            color = v4(P.in.frame.clear_color[0], P.in.frame.clear_color[1], P.in.frame.clear_color[2], P.in.frame.clear_color[3]);
        store_final(P, x, y, color);
    }
}

// ------------------------------------------------------------------------------- denoise level, TMA-staged taps
// kc_denoise: the same level for upscale ratio 1.  A CTA of 16 x 16 pixels stages its tile grown by the level's tap distance with
// five TMA tile loads — tap geometry (16 B/px), instance (4 B/px) and the three signals (8 B/px each) — and every one of the 9 x 5
// tap fetches of a pixel is a shared-memory read: 36 x 32 x 44 B = 50 KB at STEP 8, 24 x 18 x 44 B = 19 KB at STEP 1, instead of
// 45 scattered requests per pixel to L1 / L2.  Arithmetic and tap order are k_denoise's.
template <int LEVEL> struct DenoiseTile {
    static constexpr int STEP = 8 >> LEVEL;
    static constexpr int BH = POOL_TILE_H + 2 * STEP;                    // 32, 24, 20, 18 rows
    static constexpr int BW = tile_box_width(POOL_TILE_W + 2 * STEP);     // 36, 28, 24, 24 columns (slack for the 16-byte alignment of the box start)
    // sizes rounded up so that every TMA destination starts on a 128-byte boundary
    static constexpr size_t GEO = ((size_t)BW * BH * 16 + 127) & ~(size_t)127, INST = ((size_t)BW * BH * 4 + 127) & ~(size_t)127, SIG = ((size_t)BW * BH * 8 + 127) & ~(size_t)127;
    static constexpr size_t SMEM_BYTES = GEO + INST + 3 * SIG + 16;
};
struct DenoiseMaps { TileMap geometry, instance, signal[3]; };

template <int LEVEL, bool FUSE_TONE_MAPPING>
__global__ void __launch_bounds__(POOL_THREADS, 4) kc_denoise(const __grid_constant__ KParams P, const __grid_constant__ DenoiseMaps M, int signals, int keep_denoised) {
    using DT = DenoiseTile<LEVEL>;
    constexpr int STEP = DT::STEP, BW = DT::BW, BH = DT::BH;
    HK_DYNAMIC_SMEM(smem);
    float4* s_geo = reinterpret_cast<float4*>(smem);
    float* s_inst = reinterpret_cast<float*>(smem + DT::GEO);
    uint2* s_sig[3] = {reinterpret_cast<uint2*>(smem + DT::GEO + DT::INST), reinterpret_cast<uint2*>(smem + DT::GEO + DT::INST + DT::SIG),
                       reinterpret_cast<uint2*>(smem + DT::GEO + DT::INST + 2 * DT::SIG)};
    uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem + DT::GEO + DT::INST + 3 * DT::SIG);
    const int px = tile_origin_x(P.col_lo + (int)blockIdx.x * POOL_TILE_W - STEP - P.band.ax0);     // plane column of the tiles' first cell
    const int tx0 = px + P.band.ax0, ty0 = P.row_lo + (int)blockIdx.y * POOL_TILE_H - STEP;
    if (threadIdx.x == 0) {
        mbar_init(s_bar, 1u);
        mbar_expect_tx(s_bar, (uint32_t)((size_t)BW * BH * (20 + 8 * (size_t)signals)));      // what the copies deliver
        const int py = ty0 - P.band.a0;
        tile_load_2d(s_geo, &M.geometry, 4 * px, py, s_bar);
        tile_load_2d(s_inst, &M.instance, px, py, s_bar);
        for (int sgl = 0; sgl < signals; ++sgl) tile_load_2d(s_sig[sgl], &M.signal[sgl], 2 * px, py, s_bar);
        mbar_complete_emulated(s_bar);
    }
    __syncthreads();
    int x, y;
    pool_pixel(x, y, P);
    const bool in_launch = tile_active(P, x, y);
    const size_t idx = in_launch ? render_index(P.band, x, y) : 0;
    // what does not come from the tiles first: the copies run meanwhile
    float2 dg = make_float2(0.0f, 0.0f);
    float dn_var[3] = {0.0f, 0.0f, 0.0f};
    uint2 albedo_bits = make_uint2(0u, 0u);
    if (in_launch) {
        dg = __ldg(&P.planes.depth_gradient[idx]);
#pragma unroll
        for (int sgl = 0; sgl < 3; ++sgl) if (sgl < signals) dn_var[sgl] = __ldg(&P.planes.dn_variance[sgl][idx]);
        if (LEVEL == 3) albedo_bits = __ldg(&P.planes.albedo[idx]);
    }
    mbar_wait(s_bar, 0u);
    if (!in_launch) return;
    const int cx = x - tx0, cy = y - ty0;                   // this pixel's cell of the tiles
    const float4 geometry = s_geo[cy * BW + cx];
    const float depth = geometry.w;
    vec4 result[3];
    result[0] = result[1] = result[2] = v4(0.0f);
    if (!(depth < F32_EPSILON)) {
        const vec2 depth_gradient = v2(dg.x, dg.y);
        const vec3 normal = f4xyz(geometry);
        const float instance = s_inst[cy * BW + cx];
        SignalAcc acc[3];
#pragma unroll
        for (int sgl = 0; sgl < 3; ++sgl) {
            if (sgl >= signals) continue;
            SignalAcc& a = acc[sgl];
            a.lum_denominator = 4.0f * pow025(dn_var[sgl]) + 0.001f;
            const uint2 cb = s_sig[sgl][cy * BW + cx];
            uvec2 cq; cq.x = cb.x; cq.y = cb.y;
            a.irradiance = xyz(unpack_rgba16f(cq));
            a.sum_irradiance = a.irradiance * kernel_at(P, 1, 1);
            a.sum_w = kernel_at(P, 1, 1);
            if (bad3(a.irradiance)) { a.irradiance = v3(0.0f); a.sum_irradiance = v3(0.0f); a.sum_w = 0.0f; }
            a.lum = luminance(a.irradiance);
            a.ff_moment_1 = 0.0f; a.ff_moment_2 = 0.0f; a.ff_count = 0.0f;
        }
        const int OX[8] = {-1, 0, 1, -1, 1, -1, 0, 1};          // tap order of denoise.wgsl:252-268
        const int OY[8] = {-1, -1, -1, 0, 0, 1, 1, 1};
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            const int ox = OX[t], oy = OY[t];
            const int sx = x + ox * STEP, sy = y + oy * STEP;
            const bool valid = !(sx < 0 || sy < 0 || sx >= P.band.RW || sy >= P.band.RH);
            const int cell = (cy + oy * STEP) * BW + (cx + ox * STEP);       // always inside the tile; content is zero outside the plane
            const float4 sample_geometry = s_geo[cell];
            const float sample_instance = s_inst[cell];
            const vec3 sample_normal = f4xyz(sample_geometry);
            const float sample_depth = sample_geometry.w;
            const float w_normal = pow16(fmax_(0.0f, dot(normal, sample_normal)));
            const float w_depth = exp_((-fabsf(depth - sample_depth)) / (fabsf(dot(depth_gradient, v2((float)ox, (float)oy))) + 0.01f));
            const float w_instance = fmax_(0.0f, 1.0f - fabsf(instance - sample_instance));
            const float w_geometry = w_normal * w_depth * w_instance;
            const float k = kernel_at(P, oy + 1, ox + 1);
#pragma unroll
            for (int sgl = 0; sgl < 3; ++sgl) {
                if (sgl >= signals) continue;
                SignalAcc& a = acc[sgl];
                const uint2 bits = s_sig[sgl][cell];
                uvec2 qb; qb.x = bits.x; qb.y = bits.y;
                vec3 irr = xyz(unpack_rgba16f(qb));
                float sample_luminance = luminance(irr);
                float w_luminance = exp_((-fabsf(a.lum - sample_luminance)) / a.lum_denominator);
                float w = clampf(w_geometry * w_luminance, 0.0f, 1.0f) * k;
                if (valid && !bad3(irr)) {
                    a.sum_irradiance = a.sum_irradiance + irr * w;
                    a.sum_w += w;
                    if (sgl != 0) {
                        a.ff_moment_1 += sample_luminance;
                        a.ff_moment_2 += sample_luminance * sample_luminance;
                        a.ff_count += 1.0f;
                    }
                }
            }
        }
        vec4 albedo = v4(1.0f);
        if (LEVEL == 3) { uvec2 ab; ab.x = albedo_bits.x; ab.y = albedo_bits.y; albedo = unpack_rgba16f(ab); }
#pragma unroll
        for (int sgl = 0; sgl < 3; ++sgl) {
            if (sgl >= signals) continue;
            SignalAcc& a = acc[sgl];
            vec3 irradiance = (a.sum_w < 0.0001f) ? v3(0.0f) : a.sum_irradiance / a.sum_w;
            if (sgl != 0) {
                float ff_mean = a.ff_moment_1 / a.ff_count;
                float ff_var = a.ff_moment_2 / a.ff_count - ff_mean * ff_mean;
                if (a.lum > ff_mean + 3.0f * sqrtf(ff_var)) irradiance = ff_mean / a.lum * irradiance;
            }
            vec4 color = v4(irradiance, 1.0f);
            if (LEVEL == 3) color = color * albedo;
            result[sgl] = color;
        }
    }
    if (LEVEL < 3) {
#pragma unroll
        for (int sgl = 0; sgl < 3; ++sgl)
            if (sgl < signals) store16(P.planes.dn_internal[LEVEL + 1][sgl], idx, result[sgl]);
        return;
    }
    vec4 color = v4(0.0f);
#pragma unroll
    for (int sgl = 0; sgl < 3; ++sgl) {
        if (sgl >= signals) continue;
        uvec2 w = pack_rgba16f(result[sgl]);
        if (!FUSE_TONE_MAPPING || keep_denoised) P.planes.dn_render[sgl][idx] = make_uint2(w.x, w.y);
        if (FUSE_TONE_MAPPING) color = color + unpack_rgba16f(w);
    }
    if (FUSE_TONE_MAPPING && (P.tile_images || band_owned(P.band, x, y))) {
        vec3 rgb = reinhard_luminance(vmax(xyz(color), 0.0039f));
        color = v4(rgb, color.w);
        if (!(color.w > 0.0f))
            color = v4(P.in.frame.clear_color[0], P.in.frame.clear_color[1], P.in.frame.clear_color[2], P.in.frame.clear_color[3]);
        store_final(P, x, y, color);
    }
}

// ---------------------------------------------------------------------------------------------- tone mapping
// tone_mapping.wgsl:21-32 stand-alone (denoise off, or nodes run one by one); inputs per post_process.rs:940-954.
__global__ void __launch_bounds__(CTA_THREADS) k_tone_mapping(const __grid_constant__ KParams P) {
    int x, y;
    tile_pixel(x, y, P);
    if (!tile_active(P, x, y)) return;
    const size_t idx = render_index(P.band, x, y);
    const bool dn = P.in.denoise != 0u;
    uint2* const* src = dn ? P.planes.dn_render : P.planes.render;
    vec4 color = load16(src[0], idx);
    color = color + load16(src[1], idx);
    if (P.in.frame.indirect_bounces != 0u) color = color + load16(src[2], idx);
    vec3 rgb = reinhard_luminance(vmax(xyz(color), 0.0039f));
    color = v4(rgb, color.w);
    if (!(color.w > 0.0f))
        color = v4(P.in.frame.clear_color[0], P.in.frame.clear_color[1], P.in.frame.clear_color[2], P.in.frame.clear_color[3]);
    store_final(P, x, y, color);
}

// --------------------------------------------------------------------------------------------- halo copy
// One thread per pixel of the rectangle and per reservoir buffer: 4 x 16-byte loads from the owner's planes (peer memory
// when the owner is another GPU), 4 stores into this tile's ghost ring.
struct HaloArgs {
    ReservoirPlanes dst[10], src[10];
    Band dst_band, src_band;
    int x0, y0, w, h;
};
__global__ void __launch_bounds__(256) k_halo_copy(const __grid_constant__ HaloArgs A) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t n = (size_t)A.w * (size_t)A.h;
    if (i >= n) return;
    const int x = A.x0 + (int)(i % (size_t)A.w), y = A.y0 + (int)(i / (size_t)A.w);
    const size_t si = band_index(A.src_band, x, y), di = band_index(A.dst_band, x, y);
    const int r = (int)blockIdx.y;
#pragma unroll
    for (int q = 0; q < 4; ++q) A.dst[r].q[q][di] = A.src[r].q[q][si];
}

__global__ void __launch_bounds__(256) k_halo_copy_image(uint2* dst, Band db, const uint2* src, Band sb, int scale, int x0, int y0, int w, int h) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)w * (size_t)h) return;
    const int x = x0 + (int)(i % (size_t)w), y = y0 + (int)(i / (size_t)w);     // texel of the scaled image
    const size_t si = (size_t)(y - scale * sb.a0) * (size_t)(scale * sb.AW) + (size_t)(x - scale * sb.ax0);
    const size_t di = (size_t)(y - scale * db.a0) * (size_t)(scale * db.AW) + (size_t)(x - scale * db.ax0);
    dst[di] = src[si];
}

static dim3 grid_for(const KParams& P) {
    int rows = P.row_hi - P.row_lo, cols = P.col_hi - P.col_lo;
    return dim3((unsigned)((cols + TILE_W - 1) / TILE_W), (unsigned)((rows + TILE_H - 1) / TILE_H), 1u);
}

}  // namespace hkd

using namespace hkd;

void hk_launch_demodulation(const KParams& P, int signals, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    k_demodulation<<<grid_for(P), CTA_THREADS, 0, st>>>(P, signals);
}
template <int LEVEL, bool FUSE>
static void launch_denoise_tiled(const KParams& P, const DenoiseMaps& maps, int signals, int keep, cudaStream_t st) {
    const size_t smem = DenoiseTile<LEVEL>::SMEM_BYTES;
    static bool configured[64] = {};     // per instantiation AND per device: the attribute belongs to the function on one device
    int dev = 0;
    cudaGetDevice(&dev);
    if (!configured[dev & 63]) { cudaFuncSetAttribute(kc_denoise<LEVEL, FUSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); configured[dev & 63] = true; }
    const int rows = P.row_hi - P.row_lo, cols = P.col_hi - P.col_lo;
    const dim3 g((unsigned)((cols + POOL_TILE_W - 1) / POOL_TILE_W), (unsigned)((rows + POOL_TILE_H - 1) / POOL_TILE_H), 1u);
    kc_denoise<LEVEL, FUSE><<<g, POOL_THREADS, smem, st>>>(P, maps, signals, keep);
}
// `maps`: the five TMA descriptors of this level's inputs boxed for its tap distance (context.cu), or nullptr / upscale ratio above 1
// for the gather-from-global form.  maps[0] geometry, [1] instance, [2..4] the level's three signal planes.
void hk_launch_denoise_level(const KParams& P, int level, int signals, bool fuse_tone_mapping, bool keep_denoised, const TileMap* maps, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    dim3 g = grid_for(P);
    int keep = keep_denoised ? 1 : 0;
    if (maps && P.ratio1) {
        DenoiseMaps m;
        m.geometry = maps[0]; m.instance = maps[1]; m.signal[0] = maps[2]; m.signal[1] = maps[3]; m.signal[2] = maps[4];
        switch (level) {
            case 0: launch_denoise_tiled<0, false>(P, m, signals, keep, st); break;
            case 1: launch_denoise_tiled<1, false>(P, m, signals, keep, st); break;
            case 2: launch_denoise_tiled<2, false>(P, m, signals, keep, st); break;
            default:
                if (fuse_tone_mapping) launch_denoise_tiled<3, true>(P, m, signals, keep, st);
                else launch_denoise_tiled<3, false>(P, m, signals, keep, st);
        }
        return;
    }
    switch (level) {
        case 0: k_denoise<0, false><<<g, CTA_THREADS, 0, st>>>(P, signals, keep); break;
        case 1: k_denoise<1, false><<<g, CTA_THREADS, 0, st>>>(P, signals, keep); break;
        case 2: k_denoise<2, false><<<g, CTA_THREADS, 0, st>>>(P, signals, keep); break;
        default:
            if (fuse_tone_mapping) k_denoise<3, true><<<g, CTA_THREADS, 0, st>>>(P, signals, keep);
            else k_denoise<3, false><<<g, CTA_THREADS, 0, st>>>(P, signals, keep);
    }
}
void hk_launch_halo_copy(const Planes& dst, const Band& dst_band, const Planes& src, const Band& src_band, int x0, int x1, int y0, int y1,
                         cudaStream_t st) {
    if (x1 <= x0 || y1 <= y0) return;
    HaloArgs a;
    for (int r = 0; r < 10; ++r) { a.dst[r] = dst.reservoir[r]; a.src[r] = src.reservoir[r]; }
    a.dst_band = dst_band; a.src_band = src_band;
    a.x0 = x0; a.y0 = y0; a.w = x1 - x0; a.h = y1 - y0;
    const size_t n = (size_t)a.w * (size_t)a.h;
    k_halo_copy<<<dim3((unsigned)((n + 255) / 256), 10u, 1u), 256, 0, st>>>(a);
}
void hk_launch_halo_copy_image(uint2* dst, const Band& dst_band, const uint2* src, const Band& src_band, int scale, int x0, int x1, int y0, int y1,
                               cudaStream_t st) {
    if (x1 <= x0 || y1 <= y0 || !dst || !src) return;
    const int w = scale * (x1 - x0), h = scale * (y1 - y0);
    const size_t n = (size_t)w * (size_t)h;
    k_halo_copy_image<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dst, dst_band, src, src_band, scale, scale * x0, scale * y0, w, h);
}
void hk_launch_tone_mapping(const KParams& P, cudaStream_t st) {
    if (P.row_hi <= P.row_lo || P.col_hi <= P.col_lo) return;
    k_tone_mapping<<<grid_for(P), CTA_THREADS, 0, st>>>(P);
}

// which flavour of the library this is (context.cu: default of HK_TUNE_WIDE_TRAVERSAL): this unit is one of the two that the product
// build compiles with the tolerance flags (build.py FAST_FLAGS, -DHK_FAST_MATH=1)
int hk_tolerance_build() {
#ifdef HK_FAST_MATH
    return 1;
#else
    return 0;
#endif
}
