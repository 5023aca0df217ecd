// math_probe.cu — the primitives of include/hk_math.h as the device runs them, for tests/test_gpu_device_math.py.
//
// build.py's build_math_probe() compiles this file twice, with the flags of the units that trace rays (libhk_math_probe_exact.so)
// and with those of the tolerance units (libhk_math_probe_fast.so).  The test runs the same inputs through the oracle's build of
// the header (hko_math_batch / hko_math_batch_range / hko_spatial_digest / hko_deferred_digest in oracle/hk_oracle.cpp) and compares
// the bits.  The function numbers are shared with that file and with the test.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "hk_device.cuh"
#include "hk_math.h"
#include "hk_spatial_taps.cuh"

using namespace hk;

enum : int {
    // one 32-bit pattern in, one 32-bit result out
    P_F32_TO_U32 = 0, P_F32_TO_I32, P_F32_TO_F16, P_SNORM8, P_UNORM16, P_FRACT, P_POW5, P_POW16, P_HASH, P_SIN, P_COS, P_POW025,
    P_RANDOM_FLOAT, P_EXP2, P_EXP, P_SATURATE, P_F16_TO_F32, P_UNSNORM8, P_UNORM8, P_UNPACK_UNORM16,
    // two 32-bit patterns in (interleaved), one result out
    P_FMIN = 32, P_FMAX, P_CLAMP_LO, P_CLAMP_HI,
    // several words in, several out (probe_words): lighting functions, and the reservoir record (hk_packed_reservoir: 16 words) and
    // its unpacked state (32 words: radiance, random, visible position, visible normal, visible instance, sample position, sample
    // normal, count, lifetime, w, w_sum, w2_sum, padding)
    P_NORMALIZE3 = 40, P_NORMALIZE2, P_D_GGX, P_V_SMITH, P_ENV_BRDF, P_REINHARD,
    P_RESERVOIR_ROUNDTRIP = 50, P_UNPACK_RESERVOIR, P_PACK_RESERVOIR,
};
__host__ __device__ __forceinline__ void probe_words(int fn, int& in, int& out) {
    in = fn >= P_FMIN ? 2 : 1; out = 1;
    switch (fn) {
        case P_NORMALIZE3: case P_REINHARD: in = 3; out = 3; break;
        case P_NORMALIZE2: in = 2; out = 2; break;
        case P_D_GGX: in = 2; break;
        case P_V_SMITH: in = 3; break;
        case P_ENV_BRDF: in = 5; out = 3; break;
        case P_RESERVOIR_ROUNDTRIP: in = 16; out = 16; break;
        case P_UNPACK_RESERVOIR: in = 16; out = 32; break;
        case P_PACK_RESERVOIR: in = 32; out = 16; break;
        default: break;
    }
}

__device__ __forceinline__ uint32_t probe1(int fn, uint32_t u) {
    const float x = u2f(u);
    switch (fn) {
        case P_F32_TO_U32: return f32_to_u32(x);
        case P_F32_TO_I32: return (uint32_t)f32_to_i32(x);
        case P_F32_TO_F16: return f32_to_f16_bits(x);
        case P_SNORM8: return snorm8(x);
        case P_UNORM16: return pack2x16unorm(x, 0.0f) & 0xFFFFu;
        case P_FRACT: return f2u(fract(x));
        case P_POW5: return f2u(pow5(x));
        case P_POW16: return f2u(pow16(x));
        case P_HASH: return hash_u32(u);
        case P_SIN: { float s, c; sincos_(x, &s, &c); return f2u(s); }
        case P_COS: { float s, c; sincos_(x, &s, &c); return f2u(c); }
        case P_POW025: return f2u(pow025(x));
        case P_RANDOM_FLOAT: return f2u(random_float(u));
        case P_EXP2: return f2u(exp2_(x));
        case P_EXP: return f2u(exp_(x));
        case P_SATURATE: return f2u(saturate(x));
        case P_F16_TO_F32: return f2u(f16_bits_to_f32((uint16_t)u));
        case P_UNSNORM8: return f2u(unsnorm8(u));
        case P_UNORM8: return f2u(unorm8(u));
        case P_UNPACK_UNORM16: return f2u(unpack2x16unorm(u).x);
        default: return 0xDEADBEEFu;
    }
}
__device__ __forceinline__ uint32_t probe2(int fn, uint32_t ua, uint32_t ub) {
    const float a = u2f(ua), b = u2f(ub);
    switch (fn) {
        case P_FMIN: return f2u(fmin_(a, b));
        case P_FMAX: return f2u(fmax_(a, b));
        case P_CLAMP_LO: return f2u(clampf(a, b, 1.0f));
        case P_CLAMP_HI: return f2u(clampf(a, -1.0f, b));
        default: return 0xDEADBEEFu;
    }
}

__device__ __forceinline__ hkd::PackedQuarters quarters(const uint32_t* a) {
    hkd::PackedQuarters p;
    p.q0 = make_uint4(a[0], a[1], a[2], a[3]); p.q1 = make_uint4(a[4], a[5], a[6], a[7]);
    p.q2 = make_uint4(a[8], a[9], a[10], a[11]); p.q3 = make_uint4(a[12], a[13], a[14], a[15]);
    return p;
}
__device__ __forceinline__ void store_quarters(const hkd::PackedQuarters& p, uint32_t* o) {
    const uint4 q[4] = {p.q0, p.q1, p.q2, p.q3};
    for (int k = 0; k < 4; ++k) { o[4 * k] = q[k].x; o[4 * k + 1] = q[k].y; o[4 * k + 2] = q[k].z; o[4 * k + 3] = q[k].w; }
}
__device__ void probe_n(int fn, const uint32_t* a, uint32_t* o) {
    auto f = [&](int k) { return u2f(a[k]); };
    switch (fn) {
        case P_NORMALIZE3: { vec3 r = normalize(v3(f(0), f(1), f(2))); o[0] = f2u(r.x); o[1] = f2u(r.y); o[2] = f2u(r.z); break; }
        case P_NORMALIZE2: { vec2 r = normalize(v2(f(0), f(1))); o[0] = f2u(r.x); o[1] = f2u(r.y); break; }
        case P_D_GGX: o[0] = f2u(D_GGX(f(0), f(1))); break;
        case P_V_SMITH: o[0] = f2u(V_SmithGGXCorrelated(f(0), f(1), f(2))); break;
        case P_ENV_BRDF: { vec3 r = EnvBRDFApprox(v3(f(0), f(1), f(2)), f(3), f(4)); o[0] = f2u(r.x); o[1] = f2u(r.y); o[2] = f2u(r.z); break; }
        case P_REINHARD: { vec3 r = reinhard_luminance(v3(f(0), f(1), f(2))); o[0] = f2u(r.x); o[1] = f2u(r.y); o[2] = f2u(r.z); break; }
        case P_RESERVOIR_ROUNDTRIP: store_quarters(hkd::pack_reservoir(hkd::unpack_reservoir(quarters(a))), o); break;
        case P_UNPACK_RESERVOIR: {
            const hkd::Reservoir r = hkd::unpack_reservoir(quarters(a));
            const float v[32] = {r.s.radiance.x, r.s.radiance.y, r.s.radiance.z, r.s.radiance.w, r.s.random.x, r.s.random.y, r.s.random.z,
                                 r.s.random.w, r.s.visible_position.x, r.s.visible_position.y, r.s.visible_position.z, r.s.visible_position.w,
                                 r.s.visible_normal.x, r.s.visible_normal.y, r.s.visible_normal.z, 0.0f, r.s.sample_position.x,
                                 r.s.sample_position.y, r.s.sample_position.z, r.s.sample_position.w, r.s.sample_normal.x, r.s.sample_normal.y,
                                 r.s.sample_normal.z, r.count, r.lifetime, r.w, r.w_sum, r.w2_sum, 0.0f, 0.0f, 0.0f, 0.0f};
            for (int k = 0; k < 32; ++k) o[k] = f2u(v[k]);
            o[15] = r.s.visible_instance;
            break;
        }
        case P_PACK_RESERVOIR: {
            hkd::Reservoir r;
            r.s.radiance = v4(f(0), f(1), f(2), f(3)); r.s.random = v4(f(4), f(5), f(6), f(7));
            r.s.visible_position = v4(f(8), f(9), f(10), f(11)); r.s.visible_normal = v3(f(12), f(13), f(14));
            r.s.visible_instance = a[15];
            r.s.sample_position = v4(f(16), f(17), f(18), f(19)); r.s.sample_normal = v3(f(20), f(21), f(22));
            r.count = f(23); r.lifetime = f(24); r.w = f(25); r.w_sum = f(26); r.w2_sum = f(27);
            store_quarters(hkd::pack_reservoir(r), o);
            break;
        }
        default: o[0] = 0xDEADBEEFu; break;
    }
}

// `in` == nullptr: input i is the bit pattern first + i (exhaustive ranges)
__global__ void k_probe(int fn, const uint32_t* in, uint32_t first, uint32_t* out, size_t n) {
    int win, wout;
    probe_words(fn, win, wout);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        if (fn >= P_NORMALIZE3) probe_n(fn, in + i * win, out + i * wout);
        else if (fn >= P_FMIN) out[i] = probe2(fn, in[2 * i], in[2 * i + 1]);
        else out[i] = probe1(fn, in ? in[i] : first + (uint32_t)i);
    }
}

// The per-neighbour constants of spatial reuse as context.cu derives them on the host
struct ProbeTable { float phase[17], radius[17]; uint32_t tap_count[17]; float tap_dist[17][6]; };

// The rotation sum4(sample.random) a pixel brings: four f16 values in [0, 1) drawn from a hash of pixel and frame
__host__ __device__ __forceinline__ float probe_rotation(uint32_t pixel, uint32_t frame) {
    vec4 r;
    float* c = &r.x;
    for (uint32_t k = 0; k < 4u; ++k) c[k] = f16_bits_to_f32((uint16_t)(hash_u32(pixel * 4u + k + frame * 0x9E3779B9u) % 0x3C00u));
    return sum4(r);
}

// Per pixel: an FNV-1a digest over the pixel of every neighbour and the pixels of its depth-march taps (upscale ratio 1)
__global__ void k_spatial_digest(const __grid_constant__ ProbeTable T, uint32_t count, int w, int h, uint32_t frame, float random_frame,
                                 float inv_rw, float inv_rh, uint32_t* out) {
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (size_t)w * h) return;
    const int x = (int)(p % (size_t)w), y = (int)(p / (size_t)w);
    const float rotation = probe_rotation((uint32_t)p, frame);
    const vec2 uv = hkd::spatial_pixel_uv(x, y, (float)w, (float)h);
    uint32_t d = 2166136261u;
    for (uint32_t i = 1u; i <= count; ++i) {
        const vec2 offset = hkd::spatial_offset(T.phase[i], T.radius[i], rotation, random_frame);
        int sx, sy;
        hkd::spatial_neighbour_pixel(offset, x, y, sx, sy);
        d = (d ^ (uint32_t)sx) * 16777619u;
        d = (d ^ (uint32_t)sy) * 16777619u;
        const vec2 unit = hkd::spatial_march_unit(offset);
        for (uint32_t j = 1u; j <= T.tap_count[i]; ++j) {
            int tx, ty;
            hkd::spatial_tap_pixel(hkd::spatial_tap_uv(uv, unit, T.tap_dist[i][j - 1u], (float)w, (float)h, inv_rw, inv_rh), w, h, tx, ty);
            d = (d ^ (uint32_t)tx) * 16777619u;
            d = (d ^ (uint32_t)ty) * 16777619u;
        }
    }
    out[p] = d;
}

__host__ __device__ __forceinline__ uint32_t fnv(uint32_t d, uint32_t v) { return (d ^ v) * 16777619u; }

// The velocity a pixel brings to the reprojection: multiples of 2^-16 in [-1/8, 1/8) drawn from a hash of pixel and frame
__host__ __device__ __forceinline__ vec2 probe_velocity(uint32_t pixel, uint32_t frame) {
    const uint32_t h = hash_u32(pixel * 2u + frame * 0x85EBCA6Bu), g = hash_u32(h);
    return v2(mul_rn((float)((int)(h & 0x3FFFu) - 0x2000), 0x1p-16f), mul_rn((float)((int)(g & 0x3FFFu) - 0x2000), 0x1p-16f));
}

// Per render pixel at an upscale ratio above 1, four FNV-1a digests of where the tolerance units look in the G-buffer:
//   [0] light_gbuffer_index (the light passes' and k_spatial's texel of the pixel),
//   [1] denoise_deferred_coords (k_demodulation / k_denoise),
//   [2] previous_pixel, exclusive and inclusive, for velocity 0 and for probe_velocity: the index, or ~0 when rejected,
//   [3] for both tables, each neighbour's render pixel, the texel of each neighbour inside the frame and of each of its depth-march
//       taps, as k_spatial computes them.
__global__ void k_deferred_digest(const __grid_constant__ hkd::KParams P, const __grid_constant__ ProbeTable T16,
                                  const __grid_constant__ ProbeTable T8, uint32_t frame, uint32_t* out) {
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int RW = P.band.RW, RH = P.band.RH;
    if (p >= (size_t)RW * RH) return;
    const int x = (int)(p % (size_t)RW), y = (int)(p / (size_t)RW);
    const vec2 uv = hkd::render_uv(P, x, y);
    uint32_t d[4] = {2166136261u, 2166136261u, 2166136261u, 2166136261u};

    size_t g = hkd::light_gbuffer_index(P, x, y, p);
    d[0] = fnv(fnv(d[0], (uint32_t)(g % (size_t)P.band.AW)), (uint32_t)(g / (size_t)P.band.AW));
    int dx, dy;
    hkd::denoise_deferred_coords(P, uv, x, y, dx, dy);
    d[1] = fnv(fnv(d[1], (uint32_t)dx), (uint32_t)dy);
    const vec2 velocities[2] = {v2(0.0f, 0.0f), probe_velocity((uint32_t)p, frame)};
    for (int v = 0; v < 2; ++v) {
        const vec2 previous_uv = hkd::jittered_deferred_uv(P, uv, 0.25f) - velocities[v];      // as the light passes and k_spatial
        for (int inclusive = 0; inclusive < 2; ++inclusive) {
            size_t pidx;
            d[2] = fnv(d[2], hkd::previous_pixel(P, previous_uv, inclusive != 0, pidx) ? (uint32_t)pidx : 0xFFFFFFFFu);
        }
    }

    const float rotation = probe_rotation((uint32_t)p, frame);
    const vec2 march_uv = hkd::spatial_pixel_uv(x, y, (float)RW, (float)RH);
    for (int t = 0; t < 2; ++t) {
        const ProbeTable& T = t == 0 ? T16 : T8;
        const uint32_t count = t == 0 ? 16u : 8u;
        for (uint32_t i = 1u; i <= count; ++i) {
            const vec2 offset = hkd::spatial_offset(T.phase[i], T.radius[i], rotation, P.random_frame);
            int sx, sy;
            hkd::spatial_neighbour_pixel(offset, x, y, sx, sy);
            d[3] = fnv(fnv(d[3], (uint32_t)sx), (uint32_t)sy);
            if (sx < 0 || sy < 0 || sx >= RW || sy >= RH) continue;
            g = hkd::light_gbuffer_index(P, sx, sy, hkd::render_index(P.band, sx, sy));
            d[3] = fnv(fnv(d[3], (uint32_t)(g % (size_t)P.band.AW)), (uint32_t)(g / (size_t)P.band.AW));
            const vec2 unit = hkd::spatial_march_unit(offset);
            for (uint32_t j = 1u; j <= T.tap_count[i]; ++j) {
                int tx, ty;
                hkd::jittered_deferred_coords(P, hkd::spatial_tap_uv(march_uv, unit, T.tap_dist[i][j - 1u], (float)RW, (float)RH, P.inv_rw,
                                                                     P.inv_rh), tx, ty);
                d[3] = fnv(fnv(d[3], (uint32_t)tx), (uint32_t)ty);
            }
        }
    }
    for (int k = 0; k < 4; ++k) out[4 * p + k] = d[k];
}

// context.cu, "per-neighbour constants of spatial_reuse"
static ProbeTable probe_table(uint32_t count, float range) {
    ProbeTable T = {};
    for (uint32_t i = 1; i <= count; ++i) {
        T.phase[i] = (float)i * GOLDEN_RATIO;
        const float rad = sqrtf((float)i / (float)count) * range;
        T.radius[i] = rad;
        const float tap_interval = fmax_(1.0f, rad / 5.0f);
        const uint32_t tap_count = f32_to_u32(rad / tap_interval);
        T.tap_count[i] = tap_count > 6u ? 6u : tap_count;
        for (uint32_t j = 1; j <= T.tap_count[i]; ++j) T.tap_dist[i][j - 1] = (float)j * tap_interval;
    }
    return T;
}

extern "C" {

// Device pointers; `n` inputs of probe_words(fn) words each, n results of as many words as that gives.  Returns the CUDA error code
// of the launch and its completion (0: success)
int probe_batch(int fn, const uint32_t* in, uint32_t first, uint32_t* out, size_t n) {
    if (n) k_probe<<<4096, 256>>>(fn, in, first, out, n);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

int probe_spatial_digest(uint32_t count, float range, int w, int h, uint32_t frame, uint32_t* out) {
    const ProbeTable T = probe_table(count, range);
    const size_t n = (size_t)w * h;
    k_spatial_digest<<<(unsigned)((n + 255) / 256), 256>>>(T, count, w, h, frame, random_float(frame), 1.0f / (float)w, 1.0f / (float)h, out);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

// A w x h full-frame context at upscale ratio `ratio` in (1, 2], frame `frame`: the KParams fields the pixel mapping reads, derived as
// context.cu's make_params derives them.  `out`: 4 words per render pixel (k_deferred_digest), RW x RH = ceil(size / ratio) pixels
int probe_deferred_digest(int w, int h, float ratio, uint32_t frame, uint32_t* out) {
    hkd::KParams P;
    memset(&P, 0, sizeof(P));
    P.band.W = w; P.band.H = h;
    P.band.ax0 = 0; P.band.ax1 = w; P.band.a0 = 0; P.band.a1 = h;
    P.band.AW = hkd::hk_plane_pitch(w);
    const float scale = 1.0f / ratio;
    P.band.RW = (int)ceilf(scale * (float)w); P.band.RH = (int)ceilf(scale * (float)h); P.band.RS = P.band.RW;
    P.band.cx0 = 0; P.band.cx1 = P.band.RW; P.band.r0 = 0; P.band.r1 = P.band.RH;
    P.in.frame.number = frame; P.in.frame.upscale_ratio = ratio;
    P.ratio1 = 0;
    P.jitter_sign = ((frame & 1u) == 0u) ? -1.0f : 1.0f;
    P.ratio_m1 = ratio - 1.0f;
    P.inv_rw = 1.0f / (float)P.band.RW; P.inv_rh = 1.0f / (float)P.band.RH;
    P.random_frame = random_float(frame);
    const size_t n = (size_t)P.band.RW * P.band.RH;
    k_deferred_digest<<<(unsigned)((n + 255) / 256), 256>>>(P, probe_table(16u, 20.0f), probe_table(8u, 10.0f), frame, out);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

}  // extern "C"
