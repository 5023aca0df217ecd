"""Contraction guard, CPU only: the arithmetic that ends in an integer must stay exact in the tolerance units.

build.py compiles kernels_spatial.cu and kernels_post.cu with -fmad=true -prec-div=false -prec-sqrt=false (FAST_FLAGS).  Under
those flags nvcc fuses a plain a * b + c into one FMA and ptxas may fuse a `mul.f32` / `add.f32` pair that carries no rounding
modifier.  sincos_, snorm8, pack2x16unorm (include/hk_math.h), pack_reservoir (csrc/hk_device.cuh), the spatial-reuse pixel
helpers (csrc/hk_spatial_taps.cuh) and the render pixel -> G-buffer texel mapping above upscale ratio 1 (csrc/hk_device.cuh) feed
f32 -> integer conversions, where one rounding step decides a neighbour, a texel, a stored normal byte or a lifetime, so they
write every product and sum as mul_rn / add_rn (.rn in the PTX: never fused) and every quotient and square root as div_rn /
sqrt_rn / rcp_rn.  This test cross-compiles each of them alone with the tolerance flags and reads the PTX:
  * no f32 mul / add / sub without .rn, no approximate division, square root or reciprocal;
  * exactly as many FMAs as the exact flags give (the explicit fmaf() calls): none was contracted.
tests/test_gpu_device_math.py checks the same functions bit for bit on the H100; this keeps them from regressing between GPU runs."""
import os
import re
import subprocess

import pytest

from bevy_hikari_b200 import build as product_build

# a full-frame context above upscale ratio 1, as context.cu's make_params fills the fields the pixel mapping reads
DEFERRED_PARAMS = ("hkd::KParams P; P.ratio1 = 0; P.band.W = n[0]; P.band.H = n[1]; P.band.RW = n[2]; P.band.RH = n[3]; P.band.RS = n[2]; "
                   "P.band.AW = n[0]; P.band.ax0 = 0; P.band.a0 = 0; P.jitter_sign = i[0]; P.ratio_m1 = i[1]; ")
SNIPPETS = {
    "sincos_": "float s, c; hk::sincos_(i[0], &s, &c); o[0] = s; o[1] = c;",
    "snorm8": "u[0] = hk::snorm8(i[0]);",
    "pack_reservoir": "hkd::Reservoir r = hkd::zero_reservoir(); r.lifetime = i[0]; r.s.visible_normal = hk::v3(i[1], i[2], i[3]); "
                      "r.s.random = hk::v4(i[4], i[5], i[6], i[7]); hkd::PackedQuarters p = hkd::pack_reservoir(r); "
                      "u[0] = p.q3.x; u[1] = p.q0.z; u[2] = p.q0.w;",
    "pack2x16unorm": "u[0] = hk::pack2x16unorm(i[0], i[1]);",
    "spatial_neighbour": "hk::vec2 off = hkd::spatial_offset(i[0], i[1], i[2], i[3]); int sx, sy; "
                         "hkd::spatial_neighbour_pixel(off, n[0], n[1], sx, sy); u[0] = sx; u[1] = sy; o[0] = off.x; o[1] = off.y;",
    "spatial_march_tap": "hk::vec2 uv = hkd::spatial_pixel_uv(n[0], n[1], i[4], i[5]); "
                         "hk::vec2 unit = hkd::spatial_march_unit(hk::v2(i[0], i[1])); int tx, ty; "
                         "hkd::spatial_tap_pixel(hkd::spatial_tap_uv(uv, unit, i[2], i[4], i[5], i[6], i[7]), n[2], n[3], tx, ty); "
                         "u[0] = tx; u[1] = ty;",
    # render pixel -> G-buffer texel above upscale ratio 1 (csrc/hk_device.cuh): k_spatial, k_demodulation, k_denoise
    "light_deferred_coords": DEFERRED_PARAMS + "int dx, dy; hkd::light_deferred_coords(P, hkd::render_uv(P, n[4], n[5]), n[4], n[5], dx, dy); "
                             "u[0] = dx; u[1] = dy;",
    "denoise_deferred_coords": DEFERRED_PARAMS + "int dx, dy; hkd::denoise_deferred_coords(P, hkd::render_uv(P, n[4], n[5]), n[4], n[5], dx, dy); "
                               "u[0] = dx; u[1] = dy;",
    # (the callers' uv - velocity before it is a subtraction of two loaded or correctly rounded values: nothing to contract)
    "previous_pixel": DEFERRED_PARAMS + "hk::vec2 uv = hkd::jittered_deferred_uv(P, hkd::render_uv(P, n[4], n[5]), 0.25f); size_t pidx = 0; "
                      "u[0] = hkd::previous_pixel(P, hk::v2(i[2], i[3]), n[6] != 0, pidx); u[1] = (unsigned)pidx; o[0] = uv.x; o[1] = uv.y;",
    "spatial_deferred_tap": DEFERRED_PARAMS + "hk::vec2 uv = hkd::spatial_pixel_uv(n[4], n[5], (float)n[2], (float)n[3]); "
                            "hk::vec2 unit = hkd::spatial_march_unit(hk::v2(i[2], i[3])); int tx, ty; "
                            "hkd::jittered_deferred_coords(P, hkd::spatial_tap_uv(uv, unit, i[4], (float)n[2], (float)n[3], i[5], i[6]), tx, ty); "
                            "u[0] = tx; u[1] = ty;",
}
SOURCE = """#include "hk_device.cuh"
#include "hk_spatial_taps.cuh"
extern "C" __global__ void probe(const float* i, const int* n, float* o, unsigned* u) { %s }
"""


def ptx(tmp_path, name, body, flavor):
    src = tmp_path / f"{name}.cu"
    out = tmp_path / f"{name}.{flavor}.ptx"
    src.write_text(SOURCE % body)
    flags = [f for f in product_build.probe_flags(flavor) if f != "-lineinfo"]
    r = subprocess.run([product_build.NVCC] + flags + ["-ptx", str(src), "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out.read_text()


@pytest.mark.parametrize("name", sorted(SNIPPETS))
def test_integer_feeding_arithmetic_is_never_contracted_or_approximated(tmp_path, name):
    if not os.path.exists(product_build.NVCC):
        pytest.skip("no nvcc")
    fast, exact = ptx(tmp_path, name, SNIPPETS[name], "fast"), ptx(tmp_path, name, SNIPPETS[name], "exact")
    plain = re.findall(r"^\s*(?:mul|add|sub)\.f32\s.*$", fast, re.M)
    assert not plain, f"{name}: f32 arithmetic without .rn in the tolerance build: {plain[:4]}"
    approx = re.findall(r"^\s*(?:div\.(?:approx|full)|sqrt\.approx|rsqrt|rcp\.approx)\S*\s.*$", fast, re.M)
    assert not approx, f"{name}: approximate division / square root in the tolerance build: {approx[:4]}"
    fma = lambda text: len(re.findall(r"^\s*fma\.rn\.f32\s", text, re.M))
    assert fma(fast) == fma(exact), f"{name}: {fma(fast)} FMAs with the tolerance flags, {fma(exact)} with the exact ones"


# hk_scene_add_meshes and the TLAS build restate bvh 0.7.1 bit for bit against the host mirror: the SAH costs, the bucket of a centre
# and AABB::center (box_center) must round exactly as the host's f32 does, so kernels_scene.cu is compiled with the exact flags
SCENE_BUILDERS = ["kc_build_flat_bvh", "kc_build_blas_top", "kc_build_blas_bottom", "k_mesh_records"]


def test_scene_builders_are_never_contracted_or_approximated(tmp_path):
    assert "csrc/kernels_scene.cu" not in product_build.FAST_TUS, "kernels_scene.cu must not be a tolerance unit"
    if not os.path.exists(product_build.NVCC):
        pytest.skip("no nvcc")
    out = tmp_path / "kernels_scene.ptx"
    flags = [f for f in product_build.probe_flags("exact") if f != "-lineinfo"]      # build.py's flags for a unit outside FAST_TUS
    src = os.path.join(os.path.dirname(product_build.__file__), "csrc", "kernels_scene.cu")
    r = subprocess.run([product_build.NVCC] + flags + ["-ptx", src, "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    text = out.read_text()
    assert not re.search(r"^\s*call", text, re.M), "a device function is called, not inlined: its body must be checked too"
    for name in SCENE_BUILDERS:
        m = re.search(r"^\.visible \.entry _ZN3hkd\d+%s[^\n]*\n(.*?)^\}" % name, text, re.M | re.S)
        assert m, f"{name}: no entry in the PTX"
        body = m.group(1)
        assert re.search(r"^\s*(?:mul|add|sub|div)\.rn\.f32\s", body, re.M), f"{name}: no f32 arithmetic found"
        fma = re.findall(r"^\s*fma\.\S+\s.*$", body, re.M)
        assert not fma, f"{name}: contracted into FMAs: {fma[:4]}"
        plain = re.findall(r"^\s*(?:mul|add|sub)\.f32\s.*$", body, re.M)
        assert not plain, f"{name}: f32 arithmetic without .rn: {plain[:4]}"
        approx = re.findall(r"^\s*(?:div\.(?:approx|full)|sqrt\.approx|rsqrt|rcp\.approx)\S*\s.*$", body, re.M)
        assert not approx, f"{name}: approximate division / square root: {approx[:4]}"
