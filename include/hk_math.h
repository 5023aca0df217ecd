// hk_math.h — arithmetic primitives shared by the CUDA kernels (device) and by the CPU oracle (host).
//
// Only *primitives* live here (vector ops, packing, deterministic transcendental functions, hash).  The
// pass logic (traversal, light selection, BRDF, ReSTIR, denoise) is written twice, independently: once in
// oracle/ following the reference WGSL line by line, once in bevy_hikari_b200/csrc as CUDA kernels.  Sharing
// the primitives is what lets the two be compared bit-for-bit: WGSL leaves FMA contraction and the accuracy
// of sin/cos/exp/pow to the implementation, so "the reference result" is only defined up to those choices;
// this header fixes one choice for both sides (SURVEY.md App. E):
//   * every fused multiply-add is an explicit fmaf(); both sides are compiled with contraction OFF
//     (nvcc -fmad=false, gcc -ffp-contract=off), division and sqrt are IEEE on both sides;
//   * min/max follow IEEE minNum/maxNum (a NaN operand yields the other operand);
//   * sin/cos/exp2/exp are the polynomial routines below, not libm / not the SFU approximations;
//   * pow(x,16) = 4 squarings, pow(x,0.25) = sqrt(sqrt(x)), pow(x,2) = x*x, pow(x,5) = x2*x2*x;
//   * pack/unpack follow the WGSL spec formulas (floor(0.5 + s*clamp(x))) and RNE for f16.
//
// HK_FAST_MATH (device code of the product build's tolerance units only — kernels that trace no rays, see
// bevy_hikari_b200/build.py): exp2_ is the hardware ex2.approx (within 2.06 ulp on [-126, 128): 2.055 measured over every input on
// an H100) instead of the polynomial, and the translation unit is
// compiled with FMA contraction and approximate division / square root.  What ends in an integer stays exact there too:
// sincos_ (the spatial-reuse pass turns its result into integer pixel offsets, where an error of 1e-7 radians flips a neighbour
// now and then) and the snorm8 / unorm16 encodings write every product and sum as mul_rn / add_rn, which nvcc never contracts
// into an FMA whatever -fmad says.  The neighbour and depth-march pixels of spatial reuse at upscale ratio 1 do the same
// (csrc/hk_spatial_taps.cuh).
// tests/test_gpu_device_math.py compares the device build of these primitives, exact and tolerance flavour, with the oracle's.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define HK_HD __host__ __device__ __forceinline__
#include <cuda_fp16.h>
#else
#define HK_HD inline
#if defined(__F16C__)
#include <immintrin.h>
#endif
#endif

namespace hk {

constexpr float PI = 3.141592653589793f;            // bevy_pbr::utils PI
constexpr float TAU = 6.283185307f;                 // light.wgsl:226
constexpr float INV_TAU = 0.159154943f;             // light.wgsl:227
constexpr float F32_EPSILON = 1.1920929E-7f;        // light.wgsl:229
constexpr float F32_MAX = 3.402823466E+38f;         // light.wgsl:230
constexpr uint32_t U32_MAX = 0xFFFFFFFFu;
constexpr uint32_t BVH_LEAF_FLAG = 0x80000000u;     // light.wgsl:232
constexpr float RAY_BIAS = 0.02f;                   // light.wgsl:234
constexpr float DISTANCE_MAX = 65535.0f;            // light.wgsl:235
constexpr uint32_t NOISE_TEXTURE_COUNT = 16u;       // light.wgsl:236
constexpr float GOLDEN_RATIO = 1.618033989f;        // light.wgsl:237
constexpr float MAX_VARIANCE = 10.0f;               // light.wgsl:239
constexpr uint32_t DONT_EXCLUDE = 0xFFFFFFFFu;      // light.wgsl:241
constexpr uint32_t DONT_SAMPLE_EMISSIVE = 0x80000000u;  // light.wgsl:243

// ---------------------------------------------------------------------------------------------- scalars
// The host branches below exist only to mirror what the H100 computes (tests/test_gpu_device_math.py compares them bit for bit).
// The device's arithmetic returns every NaN it produces as 0x7FFFFFFF, whatever the operands; x86 returns 0xFFC00000 or the
// first operand's payload.  canon_nan gives the host the device's encoding where a primitive's result can be a NaN.
HK_HD uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
HK_HD float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
HK_HD float canon_nan(float x) {
#if defined(__CUDA_ARCH__)
    return x;
#else
    return (x != x) ? u2f(0x7FFFFFFFu) : x;
#endif
}
// min.f32 / max.f32: IEEE minNum / maxNum (a NaN operand yields the other operand), -0 below +0, two NaNs give 0x7FFFFFFF
HK_HD float fmin_(float a, float b) {
#if defined(__CUDA_ARCH__)
    return fminf(a, b);
#else
    float m = (a < b) ? a : b;      // minss: returns b when unordered
    if (a == b) m = u2f(f2u(a) | f2u(b));       // min(+0, -0) = -0 in either order
    return (b != b) ? ((a != a) ? u2f(0x7FFFFFFFu) : a) : m;
#endif
}
HK_HD float fmax_(float a, float b) {
#if defined(__CUDA_ARCH__)
    return fmaxf(a, b);
#else
    float m = (a > b) ? a : b;
    if (a == b) m = u2f(f2u(a) & f2u(b));       // max(+0, -0) = +0 in either order
    return (b != b) ? ((a != a) ? u2f(0x7FFFFFFFu) : a) : m;
#endif
}
// a * b and a + b, correctly rounded and never contracted into an FMA, even in a unit compiled with -fmad=true
HK_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
HK_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
// x / y, sqrt(x) and 1 / x correctly rounded even where the unit is compiled with -prec-div=false / -prec-sqrt=false
HK_HD float div_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
HK_HD float sqrt_rn(float a) {
#if defined(__CUDA_ARCH__)
    return __fsqrt_rn(a);
#else
    return sqrtf(a);
#endif
}
HK_HD float rcp_rn(float a) {
#if defined(__CUDA_ARCH__)
    return __frcp_rn(a);
#else
    return 1.0f / a;
#endif
}
HK_HD float clampf(float x, float lo, float hi) { return fmin_(fmax_(x, lo), hi); }
HK_HD float saturate(float x) { return clampf(x, 0.0f, 1.0f); }
HK_HD float fract(float x) { return canon_nan(x - floorf(x)); }
HK_HD float signf(float x) { return (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f); }
HK_HD float mixf(float a, float b, float t) { return fmaf(b, t, a * (1.0f - t)); }
HK_HD float sq(float x) { return x * x; }
HK_HD float pow5(float x) { float x2 = x * x; return canon_nan(x2 * x2 * x); }
HK_HD float pow16(float x) { x = x * x; x = x * x; x = x * x; return canon_nan(x * x); }
HK_HD float pow025(float x) { return canon_nan(sqrtf(sqrtf(x))); }
HK_HD bool is_nan(float v) { return !(v < 0.0f || 0.0f < v || v == 0.0f); }  // utils.wgsl:3-5

// Exact integer -> float for 0 <= v < 2^23 by planting the integer in the mantissa of 2^23 (no I2F on the conversion pipe).
HK_HD float u23_to_float(uint32_t v) { uint32_t b = 0x4B000000u | v; float f; memcpy(&f, &b, 4); return f - 8388608.0f; }

// x / C, correctly rounded, for the three constants the unpack paths divide by (127, 255, 65535) and integer-valued x
// with |x| <= C + 1: q = RN(x * RN(1/C)), one Newton correction with the exact remainder (Markstein).  Three
// instructions instead of the ~12 of a general IEEE division — unpacking reservoirs was ~230 divisions per pixel in the
// spatial pass.  tests/test_math.py checks EVERY possible input against IEEE division, so this is the same function.
template <int C>
HK_HD float div_const(float x) {
    const float y = 1.0f / (float)C;
    float q = x * y;
    float r = fmaf(-q, (float)C, x);
    return fmaf(r, y, q);
}


// WGSL u32(f32): truncate toward zero, clamped to the u32 range (negative / NaN -> 0).
HK_HD uint32_t f32_to_u32(float f) {
#if defined(__CUDA_ARCH__)
    return __float2uint_rz(f);   // cvt.rzi.u32.f32 already saturates and maps NaN to 0: same function, one instruction
#endif
    if (!(f > 0.0f)) return 0u;
    if (f >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)f;
}
// WGSL i32(f32): truncate toward zero, clamped.
HK_HD int32_t f32_to_i32(float f) {
#if defined(__CUDA_ARCH__)
    return __float2int_rz(f);    // cvt.rzi.s32.f32: saturating, NaN -> 0
#endif
    if (f != f) return 0;
    if (f >= 2147483648.0f) return 2147483647;
    if (f <= -2147483648.0f) return (int32_t)0x80000000;
    return (int32_t)f;
}

// ---------------------------------------------------------------------------------- transcendental set
// 2^x, |rel err| < 2 ulp.  Results below 2^-126 flush to 0, above 2^128 to +inf.
HK_HD float exp2_(float x) {
#if defined(HK_FAST_MATH) && defined(__CUDA_ARCH__)
    float y;
    asm("ex2.approx.f32 %0, %1;" : "=f"(y) : "f"(x));     // MUFU.EX2: NaN -> NaN, x < -126 -> subnormal / 0, x >= 128 -> +inf
    return y;
#endif
    if (x != x) return x;
    if (x < -126.0f) return 0.0f;
    if (x >= 128.0f) return u2f(0x7F800000u);
    // round-to-nearest-even of x (|x| <= 128) with the 1.5*2^23 trick: two additions on the FMA pipe instead of
    // FRND + F2I on the quarter-rate conversion pipe; the integer is read straight from the mantissa bits
    float t = x + 12582912.0f;
    float n = t - 12582912.0f;
    float f = x - n;  // [-0.5, 0.5]
    // exp(f ln2), Taylor to degree 7 (Horner, fused)
    float p = 1.5252733804e-5f;
    p = fmaf(p, f, 1.5403530393e-4f);
    p = fmaf(p, f, 1.3333558146e-3f);
    p = fmaf(p, f, 9.6181291076e-3f);
    p = fmaf(p, f, 5.5504108665e-2f);
    p = fmaf(p, f, 2.4022650696e-1f);
    p = fmaf(p, f, 6.9314718056e-1f);
    p = fmaf(p, f, 1.0f);
    int32_t e = (int32_t)f2u(t) - 0x4B400000;
    // p in [0.70, 1.42]; scale by 2^e in two steps so that e = 128 / -126 stay finite-normal where they must
    int32_t e1 = e / 2, e2 = e - e1;
    return p * u2f((uint32_t)(e1 + 127) << 23) * u2f((uint32_t)(e2 + 127) << 23);
}
HK_HD float exp_(float x) { return exp2_(canon_nan(x * 1.4426950408889634f)); }

// sin and cos together; intended range |x| <= ~1e3 (callers pass [0, 2*pi]).
HK_HD void sincos_(float x, float* s_out, float* c_out) {
    float kt = canon_nan(add_rn(mul_rn(x, 0.6366197723675814f), 12582912.0f));   // x * 2/pi, rounded to nearest even (see exp2_)
    float k = add_rn(kt, -12582912.0f);
    float r = fmaf(-k, 1.5707962513e+0f, x);   // Cody-Waite, pi/2 split in three
    r = fmaf(-k, 7.5497894159e-8f, r);
    r = fmaf(-k, 5.3903029534e-15f, r);
    float r2 = mul_rn(r, r);
    float sp = -1.9515295891e-4f;
    sp = fmaf(sp, r2, 8.3321608736e-3f);
    sp = fmaf(sp, r2, -1.6666654611e-1f);
    float s = fmaf(mul_rn(sp, r2), r, r);
    float cp = 2.443315711809948e-5f;
    cp = fmaf(cp, r2, -1.388731625493765e-3f);
    cp = fmaf(cp, r2, 4.166664568298827e-2f);
    float c = fmaf(mul_rn(cp, r2), r2, fmaf(-0.5f, r2, 1.0f));
    int32_t q = ((int32_t)f2u(kt) - 0x4B400000) & 3;
    s = canon_nan(s);
    c = canon_nan(c);
    float sr = (q & 1) ? c : s;
    float cr = (q & 1) ? s : c;
    if (q & 2) sr = -sr;
    if ((q + 1) & 2) cr = -cr;
    *s_out = sr;
    *c_out = cr;
}

// --------------------------------------------------------------------------------------------- vectors
struct vec2 { float x, y; };
struct vec3 { float x, y, z; };
struct vec4 { float x, y, z, w; };
struct uvec2 { uint32_t x, y; };
struct ivec2 { int32_t x, y; };

HK_HD vec2 v2(float x, float y) { vec2 r; r.x = x; r.y = y; return r; }
HK_HD vec3 v3(float x, float y, float z) { vec3 r; r.x = x; r.y = y; r.z = z; return r; }
HK_HD vec3 v3(float s) { return v3(s, s, s); }
HK_HD vec4 v4(float x, float y, float z, float w) { vec4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
HK_HD vec4 v4(vec3 a, float w) { return v4(a.x, a.y, a.z, w); }
HK_HD vec4 v4(float s) { return v4(s, s, s, s); }
HK_HD vec3 xyz(vec4 a) { return v3(a.x, a.y, a.z); }

HK_HD vec2 operator+(vec2 a, vec2 b) { return v2(a.x + b.x, a.y + b.y); }
HK_HD vec2 operator-(vec2 a, vec2 b) { return v2(a.x - b.x, a.y - b.y); }
HK_HD vec2 operator*(vec2 a, vec2 b) { return v2(a.x * b.x, a.y * b.y); }
HK_HD vec2 operator/(vec2 a, vec2 b) { return v2(a.x / b.x, a.y / b.y); }
HK_HD vec2 operator*(vec2 a, float s) { return v2(a.x * s, a.y * s); }
HK_HD vec2 operator*(float s, vec2 a) { return v2(a.x * s, a.y * s); }
HK_HD vec2 operator/(vec2 a, float s) { return v2(a.x / s, a.y / s); }
HK_HD vec2 operator+(vec2 a, float s) { return v2(a.x + s, a.y + s); }
HK_HD vec2 operator-(vec2 a, float s) { return v2(a.x - s, a.y - s); }

HK_HD vec3 operator+(vec3 a, vec3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
HK_HD vec3 operator-(vec3 a, vec3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
HK_HD vec3 operator*(vec3 a, vec3 b) { return v3(a.x * b.x, a.y * b.y, a.z * b.z); }
HK_HD vec3 operator/(vec3 a, vec3 b) { return v3(a.x / b.x, a.y / b.y, a.z / b.z); }
HK_HD vec3 operator*(vec3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
HK_HD vec3 operator*(float s, vec3 a) { return v3(a.x * s, a.y * s, a.z * s); }
HK_HD vec3 operator/(vec3 a, float s) { return v3(a.x / s, a.y / s, a.z / s); }
HK_HD vec3 operator+(vec3 a, float s) { return v3(a.x + s, a.y + s, a.z + s); }
HK_HD vec3 operator-(vec3 a, float s) { return v3(a.x - s, a.y - s, a.z - s); }
HK_HD vec3 operator-(vec3 a) { return v3(-a.x, -a.y, -a.z); }
HK_HD vec3 operator/(float s, vec3 a) { return v3(s / a.x, s / a.y, s / a.z); }

HK_HD vec4 operator+(vec4 a, vec4 b) { return v4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
HK_HD vec4 operator-(vec4 a, vec4 b) { return v4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
HK_HD vec4 operator*(vec4 a, vec4 b) { return v4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
HK_HD vec4 operator*(vec4 a, float s) { return v4(a.x * s, a.y * s, a.z * s, a.w * s); }
HK_HD vec4 operator+(vec4 a, float s) { return v4(a.x + s, a.y + s, a.z + s, a.w + s); }

HK_HD float dot(vec2 a, vec2 b) { return fmaf(a.y, b.y, a.x * b.x); }
HK_HD float dot(vec3 a, vec3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }
HK_HD float dot(vec4 a, vec4 b) { return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x))); }
HK_HD vec3 cross(vec3 a, vec3 b) {
    return v3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x)));
}
HK_HD float length(vec3 a) { return sqrtf(dot(a, a)); }
HK_HD float length(vec2 a) { return sqrtf(dot(a, a)); }
HK_HD vec3 canon_nan(vec3 a) { return v3(canon_nan(a.x), canon_nan(a.y), canon_nan(a.z)); }
// normalize(0) is 0 * inf: a NaN, 0x7FFFFFFF on the device
HK_HD vec3 normalize(vec3 a) { float inv = 1.0f / sqrtf(dot(a, a)); return canon_nan(a * inv); }
HK_HD vec2 normalize(vec2 a) { float inv = 1.0f / sqrtf(dot(a, a)); vec2 r = a * inv; return v2(canon_nan(r.x), canon_nan(r.y)); }
HK_HD vec3 vmin(vec3 a, vec3 b) { return v3(fmin_(a.x, b.x), fmin_(a.y, b.y), fmin_(a.z, b.z)); }
HK_HD vec3 vmax(vec3 a, vec3 b) { return v3(fmax_(a.x, b.x), fmax_(a.y, b.y), fmax_(a.z, b.z)); }
HK_HD vec3 vmax(vec3 a, float s) { return v3(fmax_(a.x, s), fmax_(a.y, s), fmax_(a.z, s)); }
HK_HD vec3 mix(vec3 a, vec3 b, float t) { return v3(mixf(a.x, b.x, t), mixf(a.y, b.y, t), mixf(a.z, b.z, t)); }
HK_HD vec4 fract(vec4 a) { return v4(fract(a.x), fract(a.y), fract(a.z), fract(a.w)); }
HK_HD float sum4(vec4 a) { return dot(a, v4(1.0f)); }  // dot(v, vec4(1.0)), light.wgsl:155

// Column-major 4x4 (glam / WGSL mat4x4<f32>): c[j] is column j.
struct mat4 { vec4 c[4]; };
struct mat3 { vec3 c[3]; };
HK_HD vec4 mul(const mat4& m, vec4 v) {  // m * v
    vec4 r;
    r.x = fmaf(m.c[3].x, v.w, fmaf(m.c[2].x, v.z, fmaf(m.c[1].x, v.y, m.c[0].x * v.x)));
    r.y = fmaf(m.c[3].y, v.w, fmaf(m.c[2].y, v.z, fmaf(m.c[1].y, v.y, m.c[0].y * v.x)));
    r.z = fmaf(m.c[3].z, v.w, fmaf(m.c[2].z, v.z, fmaf(m.c[1].z, v.y, m.c[0].z * v.x)));
    r.w = fmaf(m.c[3].w, v.w, fmaf(m.c[2].w, v.z, fmaf(m.c[1].w, v.y, m.c[0].w * v.x)));
    return r;
}
HK_HD vec4 mul_transposed(const mat4& m, vec4 v) {  // transpose(m) * v : row j of the result = dot(column j, v)
    return v4(dot(m.c[0], v), dot(m.c[1], v), dot(m.c[2], v), dot(m.c[3], v));
}
HK_HD vec3 mul(const mat3& m, vec3 v) {
    vec3 r;
    r.x = fmaf(m.c[2].x, v.z, fmaf(m.c[1].x, v.y, m.c[0].x * v.x));
    r.y = fmaf(m.c[2].y, v.z, fmaf(m.c[1].y, v.y, m.c[0].y * v.x));
    r.z = fmaf(m.c[2].z, v.z, fmaf(m.c[1].z, v.y, m.c[0].z * v.x));
    return r;
}

// utils.wgsl:41-48 — branch-free orthonormal basis; columns (t, b, n).
HK_HD mat3 normal_basis(vec3 n) {
    float s = fmin_(signf(n.z) * 2.0f + 1.0f, 1.0f);
    float u = -1.0f / (s + n.z);
    float v = n.x * n.y * u;
    mat3 m;
    m.c[0] = v3(1.0f + s * n.x * n.x * u, s * v, -s * n.x);
    m.c[1] = v3(v, s + n.y * n.y * u, -n.y);
    m.c[2] = n;
    return m;
}

// utils.wgsl:63-65
HK_HD float luminance(vec3 v) { return dot(v, v3(0.2126f, 0.7152f, 0.0722f)); }

// utils.wgsl:15-28
HK_HD uint32_t hash_u32(uint32_t value) {
    uint32_t state = value;
    state = state ^ 2747636419u;
    state = state * 2654435769u;
    state = state ^ (state >> 16u);
    state = state * 2654435769u;
    state = state ^ (state >> 16u);
    state = state * 2654435769u;
    return state;
}
HK_HD float random_float(uint32_t value) { return (float)hash_u32(value) / 4294967295.0f; }

// --------------------------------------------------------------------------------------------- packing
HK_HD uint16_t f32_to_f16_bits(float f) {
#if defined(__CUDA_ARCH__)
    return __half_as_ushort(__float2half_rn(f));
#else
    if (f != f) return (uint16_t)0x7FFFu;           // cvt.rn.f16.f32 turns every NaN into the canonical 0x7FFF
#if defined(__F16C__)
    return (uint16_t)_cvtss_sh(f, _MM_FROUND_TO_NEAREST_INT | _MM_FROUND_NO_EXC);
#else
    uint32_t x = f2u(f);
    uint32_t sign = (x >> 16) & 0x8000u;
    uint32_t mant = x & 0x007FFFFFu;
    int32_t exp = (int32_t)((x >> 23) & 0xFF);
    if (exp == 255) return (uint16_t)(sign | 0x7C00u);      // +-inf (NaN above)
    int32_t e = exp - 127 + 15;
    if (e >= 31) return (uint16_t)(sign | 0x7C00u);
    if (e <= 0) {
        if (e < -10) return (uint16_t)sign;
        mant |= 0x00800000u;
        uint32_t shift = (uint32_t)(14 - e);
        uint32_t half = mant >> shift;
        uint32_t rem = mant & ((1u << shift) - 1u);
        uint32_t halfway = 1u << (shift - 1);
        if (rem > halfway || (rem == halfway && (half & 1u))) half++;
        return (uint16_t)(sign | half);
    }
    uint32_t half = ((uint32_t)e << 10) | (mant >> 13);
    uint32_t rem = mant & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (half & 1u))) half++;
    return (uint16_t)(sign | half);
#endif
#endif
}
HK_HD float f16_bits_to_f32(uint16_t h) {
#if defined(__CUDA_ARCH__)
    return __half2float(__ushort_as_half(h));
#else
    if ((h & 0x7C00u) == 0x7C00u && (h & 0x3FFu)) return u2f(0x7FFFFFFFu);   // cvt.f32.f16: every NaN becomes the canonical 0x7FFFFFFF
#if defined(__F16C__)
    return _cvtsh_ss(h);
#else
    uint32_t sign = ((uint32_t)h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1Fu;
    uint32_t mant = h & 0x3FFu;
    if (exp == 0) {
        if (mant == 0) return u2f(sign);
        float m = (float)mant * 5.9604644775390625e-8f;  // 2^-24
        return (sign ? -m : m);
    }
    if (exp == 31) return u2f(sign | 0x7F800000u);          // +-inf (NaN above)
    return u2f(sign | ((exp + 112u) << 23) | (mant << 13));
#endif
#endif
}
HK_HD uint32_t pack2x16float(float a, float b) {
    return (uint32_t)f32_to_f16_bits(a) | ((uint32_t)f32_to_f16_bits(b) << 16);
}
HK_HD vec2 unpack2x16float(uint32_t u) {
    return v2(f16_bits_to_f32((uint16_t)(u & 0xFFFFu)), f16_bits_to_f32((uint16_t)(u >> 16)));
}
// WGSL spec: floor(0.5 + 65535 * min(1, max(0, e)))
HK_HD uint32_t pack2x16unorm(float a, float b) {
    uint32_t x = (uint32_t)floorf(add_rn(0.5f, mul_rn(65535.0f, fmin_(1.0f, fmax_(0.0f, a)))));
    uint32_t y = (uint32_t)floorf(add_rn(0.5f, mul_rn(65535.0f, fmin_(1.0f, fmax_(0.0f, b)))));
    return x | (y << 16);
}
HK_HD vec2 unpack2x16unorm(uint32_t u) { return v2(div_const<65535>(u23_to_float(u & 0xFFFFu)), div_const<65535>(u23_to_float(u >> 16))); }
HK_HD float unorm8(uint32_t b) { return div_const<255>(u23_to_float(b & 0xFFu)); }   // Rgba8Unorm texel component
// WGSL spec: floor(0.5 + 127 * min(1, max(-1, e))), two's complement byte
HK_HD uint32_t snorm8(float e) {
    int32_t i = (int32_t)floorf(add_rn(0.5f, mul_rn(127.0f, fmin_(1.0f, fmax_(-1.0f, e)))));
    return (uint32_t)i & 0xFFu;
}
HK_HD uint32_t pack4x8snorm(vec4 v) {
    return snorm8(v.x) | (snorm8(v.y) << 8) | (snorm8(v.z) << 16) | (snorm8(v.w) << 24);
}
HK_HD float unsnorm8(uint32_t b) {   // two's-complement byte -> [-128,127] -> /127, clamped at -1
    float i = u23_to_float((b & 0xFFu) ^ 0x80u) - 128.0f;
    return fmax_(div_const<127>(i), -1.0f);
}
HK_HD vec4 unpack4x8snorm(uint32_t u) {
    return v4(unsnorm8(u), unsnorm8(u >> 8), unsnorm8(u >> 16), unsnorm8(u >> 24));
}
HK_HD uvec2 pack_rgba16f(vec4 v) { uvec2 r; r.x = pack2x16float(v.x, v.y); r.y = pack2x16float(v.z, v.w); return r; }
HK_HD vec4 unpack_rgba16f(uvec2 u) { vec2 a = unpack2x16float(u.x), b = unpack2x16float(u.y); return v4(a.x, a.y, b.x, b.y); }

// ----------------------------------------------------------------------------- bevy_pbr 0.9 lighting
// Restated from the published bevy_pbr 0.9.1 WGSL (pbr_lighting / utils), see SURVEY.md App. D.
HK_HD float perceptualRoughnessToRoughness(float pr) { float c = clampf(pr, 0.089f, 1.0f); return c * c; }
HK_HD float D_GGX(float roughness, float NoH) {
    float oneMinusNoHSquared = 1.0f - NoH * NoH;
    float a = NoH * roughness;
    float k = roughness / (oneMinusNoHSquared + a * a);
    return canon_nan(k * k * (1.0f / PI));
}
HK_HD float V_SmithGGXCorrelated(float roughness, float NoV, float NoL) {
    float a2 = roughness * roughness;
    float lambdaV = NoL * sqrtf((NoV - a2 * NoV) * NoV + a2);
    float lambdaL = NoV * sqrtf((NoL - a2 * NoL) * NoL + a2);
    return canon_nan(0.5f / (lambdaV + lambdaL));
}
HK_HD vec3 F_Schlick_vec(vec3 f0, float f90, float VoH) {
    float p = pow5(1.0f - VoH);
    return f0 + (v3(f90) - f0) * p;
}
HK_HD float F_Schlick(float f0, float f90, float VoH) { return f0 + (f90 - f0) * pow5(1.0f - VoH); }
HK_HD vec3 fresnel(vec3 f0, float LoH) {
    float f90 = saturate(dot(f0, v3(50.0f * 0.33f)));
    return F_Schlick_vec(f0, f90, LoH);
}
HK_HD vec3 specular(vec3 f0, float roughness, float NoV, float NoL, float NoH, float LoH, float specularIntensity) {
    float D = D_GGX(roughness, NoH);
    float V = V_SmithGGXCorrelated(roughness, NoV, NoL);
    vec3 F = fresnel(f0, LoH);
    return (specularIntensity * D * V) * F;
}
HK_HD float Fd_Burley(float roughness, float NoV, float NoL, float LoH) {
    float f90 = 0.5f + 2.0f * roughness * LoH * LoH;
    float lightScatter = F_Schlick(1.0f, f90, NoL);
    float viewScatter = F_Schlick(1.0f, f90, NoV);
    return lightScatter * viewScatter * (1.0f / PI);
}
HK_HD vec3 EnvBRDFApprox(vec3 f0, float perceptual_roughness, float NoV) {
    const vec4 c0 = v4(-1.0f, -0.0275f, -0.572f, 0.022f);
    const vec4 c1 = v4(1.0f, 0.0425f, 1.04f, -0.04f);
    vec4 r = c0 * perceptual_roughness + c1;
    float a004 = fmin_(r.x * r.x, exp2_(-9.28f * NoV)) * r.x + r.y;
    vec2 AB = v2(-1.04f, 1.04f) * a004 + v2(r.z, r.w);
    return canon_nan(f0 * AB.x + AB.y);
}
// bevy_core_pipeline::tonemapping
HK_HD vec3 reinhard_luminance(vec3 color) {
    float l_old = luminance(color);
    float l_new = l_old / (1.0f + l_old);
    return canon_nan(color * (l_new / l_old));
}

// ------------------------------------------------------------------------------------ FSR 1.0 primitives
// The approximations AMD's ffx_a.h builds EASU / RCAS on (src/shaders/fsr/source.zip: ffx_a.h:1843-1845) — integer
// arithmetic on the float's bits, hence exactly defined — and the two constant blocks FSR_Pass.glsl computes in `main`
// (ffx_fsr1.h:156-201 FsrEasuCon, :662-672 FsrRcasCon) with ARcpF1(x) = 1 / x (ffx_a.h:737) as an IEEE division.
HK_HD float fsr_rcp_lo(float a) { return u2f(0x7ef07ebbu - f2u(a)); }                 // APrxLoRcpF1
HK_HD float fsr_rcp_med(float a) { float b = u2f(0x7ef19fffu - f2u(a)); return b * (-b * a + 2.0f); }   // APrxMedRcpF1
HK_HD float fsr_rsq_lo(float a) { return u2f(0x5f347d74u - (f2u(a) >> 1)); }          // APrxLoRsqF1
struct FsrEasuConstants {   // con0 .. con3 as floats (the GLSL passes them around as bit patterns)
    float scale_x, scale_y, offset_x, offset_y;   // con0: output pixel -> input pixel position.  con1 .. con3 only place the
};                                                // four gathers on texel corners (ffx_fsr1.h:175-201): see fsr_easu below
HK_HD FsrEasuConstants fsr_easu_constants(float input_viewport_w, float input_viewport_h, float output_w, float output_h) {
    FsrEasuConstants c;
    c.scale_x = input_viewport_w * (1.0f / output_w);
    c.scale_y = input_viewport_h * (1.0f / output_h);
    c.offset_x = 0.5f * input_viewport_w * (1.0f / output_w) - 0.5f;
    c.offset_y = 0.5f * input_viewport_h * (1.0f / output_h) - 0.5f;
    return c;
}
HK_HD float fsr_rcas_constant(float sharpness) { return exp2_(-sharpness); }           // FsrRcasCon: stops -> linear
constexpr float FSR_RCAS_LIMIT = 0.25f - (1.0f / 16.0f);                               // ffx_fsr1.h:654

}  // namespace hk
