// hk_spatial_taps.cuh — where spatial reuse looks (light.wgsl:1566-1575, 1609-1622): the pixel of neighbour i and the pixels of its
// screen-space depth-march taps.  Both end in an integer pixel, so a rounding difference here is a different neighbour, not a
// small radiance error.  Every product, sum, quotient and square root is written as a correctly rounded operation (hk::mul_rn,
// hk::add_rn, hk::div_rn, hk::rcp_rn, hk::sqrt_rn: __fmul_rn, __fadd_rn, __fdiv_rn, __frcp_rn, __fsqrt_rn on the device), which
// nvcc never contracts or approximates.  So the spatial pass picks the oracle's pixels (oracle/hk_oracle.cpp spatial_neighbour /
// spatial_tap_uv) in the tolerance build (-fmad=true, -prec-div=false, -prec-sqrt=false) as well as in the exact one.  Above upscale
// ratio 1, k_spatial maps the neighbour and each tap to a G-buffer texel with jittered_deferred_coords of hk_device.cuh, written
// the same way, so those texels are the oracle's too.  tests/cuda/math_probe.cu runs these functions for every pixel of a frame, at
// ratio 1 and above it.
#pragma once
#include "hk_math.h"

namespace hkd {

// Offset of neighbour i: radius * (cos, sin)(TAU * fract(phase + rotation + random_frame)), with the table's phase = f32(i) *
// GOLDEN_RATIO and radius = sqrt(f32(i) / f32(COUNT)) * RANGE, rotation = sum4(sample.random), random_frame = random_float(frame)
__device__ __forceinline__ hk::vec2 spatial_offset(float phase, float radius, float rotation, float random_frame) {
    const float t = hk::add_rn(hk::add_rn(phase, rotation), random_frame);
    const float ang = hk::mul_rn(hk::TAU, hk::add_rn(t, -floorf(t)));         // TAU * fract(t)
    float sn, cs;
    hk::sincos_(ang, &sn, &cs);
    return hk::v2(hk::mul_rn(radius, cs), hk::mul_rn(radius, sn));
}
// The neighbour's pixel: i32(offset + coords)
__device__ __forceinline__ void spatial_neighbour_pixel(hk::vec2 offset, int x, int y, int& sx, int& sy) {
    sx = hk::f32_to_i32(hk::add_rn(offset.x, (float)x));
    sy = hk::f32_to_i32(hk::add_rn(offset.y, (float)y));
}
// coords_to_uv (utils.wgsl:37-39): (coords + 0.5) / size, IEEE
__device__ __forceinline__ hk::vec2 spatial_pixel_uv(int x, int y, float rw, float rh) {
    return hk::v2(hk::div_rn(hk::add_rn((float)x, 0.5f), rw), hk::div_rn(hk::add_rn((float)y, 0.5f), rh));
}
// normalize(offset), IEEE: the direction of the march
__device__ __forceinline__ hk::vec2 spatial_march_unit(hk::vec2 offset) {
    const float inv = hk::rcp_rn(hk::sqrt_rn(fmaf(offset.y, offset.y, hk::mul_rn(offset.x, offset.x))));      // = IEEE 1 / sqrt
    return hk::v2(hk::mul_rn(offset.x, inv), hk::mul_rn(offset.y, inv));
}
// uv + tap_dist * unit / size.  With `inv_rw` / `inv_rh` = RN(1 / size) from the host the quotient is x * y, r = fma(-q, C, x),
// fma(r, y, q): the correctly rounded quotient whenever it is a normal number (tools/check_runtime_division.cpp: all 2^32 inputs for
// the benchmark extents); a subnormal quotient is absorbed by the addition to uv >= 0.5 / size
__device__ __forceinline__ hk::vec2 spatial_tap_uv(hk::vec2 uv, hk::vec2 unit, float tap_dist, float rw, float rh, float inv_rw, float inv_rh) {
    const float ox = hk::mul_rn(tap_dist, unit.x), oy = hk::mul_rn(tap_dist, unit.y);
    const float qx = hk::mul_rn(ox, inv_rw), qy = hk::mul_rn(oy, inv_rh);
    return hk::v2(hk::add_rn(uv.x, fmaf(fmaf(-qx, rw, ox), inv_rw, qx)), hk::add_rn(uv.y, fmaf(fmaf(-qy, rh, oy), inv_rh, qy)));
}
// The tap's pixel at upscale ratio 1: i32(tap_uv * size)
__device__ __forceinline__ void spatial_tap_pixel(hk::vec2 tap_uv, int w, int h, int& tx, int& ty) {
    tx = hk::f32_to_i32(hk::mul_rn(tap_uv.x, (float)w));
    ty = hk::f32_to_i32(hk::mul_rn(tap_uv.y, (float)h));
}

}  // namespace hkd
