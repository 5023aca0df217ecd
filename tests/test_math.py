"""Known-answer tests of include/hk_math.h (through the oracle build of the same header): the arithmetic both the CUDA
kernels and the oracle use.  Expected values come from numpy / the WGSL spec formulas, computed independently here."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the oracle's compiler and flags (oracle/Makefile), for the exhaustive host checks below
HOST_CXX = ["/usr/bin/g++", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared", "-std=c++17",
            "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-I", os.path.join(ROOT, "include")]

# Every float in a range through the host build of hk_math.h, checked against float64 libm in C (numpy would take minutes)
ACCURACY_SRC = r"""
#define _GNU_SOURCE 1
#include "hk_math.h"
#include <math.h>
static double ulp_of(double r) { int e; frexp(r, &e); return ldexp(1.0, e - 24 < -149 ? -149 : e - 24); }
extern "C" __attribute__((visibility("default"))) double worst_exp2_ulp(uint32_t lo, uint32_t hi) {
    double worst = 0.0;
#pragma omp parallel for reduction(max : worst) schedule(static)
    for (int64_t b = lo; b <= (int64_t)hi; ++b) {
        const float x = hk::u2f((uint32_t)b);
        const double r = exp2((double)x);
        const double e = fabs((double)hk::exp2_(x) - r) / ulp_of(r);
        worst = e > worst ? e : worst;
    }
    return worst;
}
extern "C" __attribute__((visibility("default"))) double worst_sincos_abs(uint32_t lo, uint32_t hi) {
    double worst = 0.0;
#pragma omp parallel for reduction(max : worst) schedule(static)
    for (int64_t b = lo; b <= (int64_t)hi; ++b) {
        const float x = hk::u2f((uint32_t)b);
        float s, c;
        double rs, rc;
        hk::sincos_(x, &s, &c);
        sincos((double)x, &rs, &rc);
        const double e = fmax(fabs((double)s - rs), fabs((double)c - rc));
        worst = e > worst ? e : worst;
    }
    return worst;
}
"""


def compile_host(tmp_path, name, src, extra=()):
    if not os.path.exists(HOST_CXX[0]):
        pytest.skip("no host C++ compiler")
    cpp, so = tmp_path / (name + ".cpp"), tmp_path / (name + ".so")
    cpp.write_text(src)
    r = subprocess.run(HOST_CXX + list(extra) + ["-o", str(so), str(cpp)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(str(so))


def ulp_diff(a, b):
    a, b = np.float32(a), np.float32(b)
    ia, ib = int(a.view(np.int32)), int(b.view(np.int32))
    return abs(ia - ib)


def test_exp2_is_within_two_ulp_for_every_float_in_its_range(tmp_path):
    """The bound include/hk_math.h states for exp2_, over every float in [-126, 128) against float64"""
    acc = compile_host(tmp_path, "accuracy", ACCURACY_SRC)
    acc.worst_exp2_ulp.restype, acc.worst_exp2_ulp.argtypes = C.c_double, [C.c_uint32, C.c_uint32]
    worst = max(acc.worst_exp2_ulp(0x00000000, 0x42FFFFFF),      # +0 .. the float below 128
                acc.worst_exp2_ulp(0x80000000, 0xC2FC0000))      # -0 .. -126
    assert worst <= 2.0, worst


def test_exp2_and_exp_accuracy():
    lib = oracle.lib()
    for x in np.linspace(-20, 5, 2001).astype(np.float32):
        # WGSL accuracy requirement for exp(x) is 3 + 2|x| ULP; exp_(x) = exp2_(x * log2(e)) stays far inside it
        assert ulp_diff(lib.hko_math_exp(float(x)), np.exp(np.float64(x))) <= 3 + 2 * abs(float(x))
    assert lib.hko_math_exp2(-200.0) == 0.0 and lib.hko_math_exp2(200.0) == float("inf")
    assert lib.hko_math_exp2(0.0) == 1.0 and lib.hko_math_exp2(10.0) == 1024.0


def test_sincos_accuracy_over_the_range_the_path_uses(tmp_path):
    """Every float in [0, 2 pi] (the spatial pass's angles), against float64"""
    acc = compile_host(tmp_path, "accuracy", ACCURACY_SRC)
    acc.worst_sincos_abs.restype, acc.worst_sincos_abs.argtypes = C.c_double, [C.c_uint32, C.c_uint32]
    worst = acc.worst_sincos_abs(0x00000000, int(np.float32(2 * np.pi).view(np.uint32)))
    assert worst < 3e-7, worst
    lib = oracle.lib()
    s, c = C.c_float(), C.c_float()
    lib.hko_math_sincos(0.0, C.byref(s), C.byref(c))
    assert (s.value, c.value) == (0.0, 1.0)


def test_f16_pack_is_ieee_round_to_nearest_even():
    lib = oracle.lib()
    rng = np.random.default_rng(0)
    vals = np.concatenate([rng.normal(0, 100, 2000), rng.normal(0, 1e-5, 500), [0.0, -0.0, 65504.0, 65520.0, 1e9, -1e9, 5.96e-8,
                                                                               2.98e-8, 1.0009765625, 1.00048828125]])
    for v in vals.astype(np.float32):
        with np.errstate(over="ignore"):
            want = int(np.float32(v).astype(np.float16).view(np.uint16))
        got = lib.hko_math_pack2x16float(float(v), 0.0) & 0xFFFF
        assert got == want, (v, hex(got), hex(want))
        back = lib.hko_math_f16_to_f32(got)
        wantf = float(np.uint16(want).view(np.float16).astype(np.float32))
        assert back == wantf or (np.isnan(back) and np.isnan(wantf))


def test_snorm_unorm_pack_follow_the_wgsl_formulas():
    lib = oracle.lib()
    rng = np.random.default_rng(1)
    for v in list(rng.uniform(-1.5, 1.5, 500)) + [0.0, 1.0, -1.0, 0.5, -0.5, 1 / 254.0]:
        v = np.float32(v)
        want = int(np.floor(np.float32(0.5) + np.float32(127.0) * min(np.float32(1), max(np.float32(-1), v)))) & 0xFF
        assert lib.hko_math_pack4x8snorm(float(v), 0, 0, 0) & 0xFF == want
        want = int(np.floor(np.float32(0.5) + np.float32(65535.0) * min(np.float32(1), max(np.float32(0), v))))
        assert lib.hko_math_pack2x16unorm(float(v), 0) & 0xFFFF == want
    # NaN follows IEEE minNum/maxNum: clamps to the lower bound
    assert lib.hko_math_pack4x8snorm(float("nan"), 0, 0, 0) & 0xFF == 0x81


def test_hash_matches_a_python_restatement_of_utils_wgsl():
    def h(v):  # utils.wgsl:15-24
        s = v & 0xFFFFFFFF
        s ^= 2747636419
        s = (s * 2654435769) & 0xFFFFFFFF
        s ^= s >> 16
        s = (s * 2654435769) & 0xFFFFFFFF
        s ^= s >> 16
        s = (s * 2654435769) & 0xFFFFFFFF
        return s
    lib = oracle.lib()
    for v in [0, 1, 2, 3, 64, 12345, 0xFFFFFFFF, 0x80000000]:
        assert lib.hko_math_hash(v) == h(v)


def test_normal_basis_is_orthonormal_with_n_as_third_column():
    lib = oracle.lib()
    rng = np.random.default_rng(2)
    for _ in range(200):
        n = rng.normal(size=3)
        n = (n / np.linalg.norm(n)).astype(np.float32)
        out = np.zeros(9, np.float32)
        lib.hko_math_normal_basis(n.ctypes.data, out.ctypes.data)
        m = out.reshape(3, 3)  # rows = columns t, b, n
        assert np.allclose(m[2], n)
        assert np.allclose(m @ m.T, np.eye(3), atol=2e-6)


def test_reservoir_pack_unpack_is_idempotent_after_one_round_trip():
    """pack(unpack(p)) is not the identity for arbitrary bits (normals get re-normalised) but it is a projection."""
    from bevy_hikari_b200 import layout as L
    lib = oracle.lib()
    rng = np.random.default_rng(3)
    p = np.zeros(64, L.PACKED_RESERVOIR)
    p["visible_position"] = rng.normal(size=(64, 4)).astype(np.float32)
    p["sample_position"][:, :3] = rng.normal(size=(64, 3)).astype(np.float32)
    p["sample_position"][:, 3] = rng.integers(0, 8, 64).astype(np.float32)
    for name in ("radiance", "random", "reservoir"):
        h = np.abs(rng.normal(size=(64, 4))).astype(np.float16)
        p[name] = h.view(np.uint32).reshape(64, 2)
    p["visible_normal"] = rng.integers(0, 2 ** 32, 64, dtype=np.uint64).astype(np.uint32)
    p["sample_normal"] = rng.integers(0, 2 ** 32, 64, dtype=np.uint64).astype(np.uint32)
    once, twice = np.zeros_like(p), np.zeros_like(p)
    for i in range(64):
        lib.hko_pack_reservoir_roundtrip(p[i:i + 1].ctypes.data, once[i:i + 1].ctypes.data)
        lib.hko_pack_reservoir_roundtrip(once[i:i + 1].ctypes.data, twice[i:i + 1].ctypes.data)
    # a normal quantised twice may move by one snorm8 step; everything else is stable
    for name in ("radiance", "random", "visible_position", "sample_position", "reservoir"):
        assert once[name].tobytes() == twice[name].tobytes(), name
    d = (np.ascontiguousarray(once["visible_normal"]).view(np.int8).astype(int) -
         np.ascontiguousarray(twice["visible_normal"]).view(np.int8).astype(int))
    assert np.abs(d).max() <= 1


def test_fast_division_by_constants_is_exactly_ieee_division_for_every_input():
    """unsnorm8 / unorm8 / unorm16 use a 3-instruction correctly-rounded quotient (hk::div_const); exhaustive check."""
    lib = oracle.lib()
    for b in range(256):
        i = b - 256 if b >= 128 else b
        want = max(np.float32(i) / np.float32(127.0), np.float32(-1.0))
        assert np.float32(lib.hko_math_unsnorm8(b)).view(np.uint32) == np.float32(want).view(np.uint32), b
        assert np.float32(lib.hko_math_unorm8(b)).view(np.uint32) == (np.float32(b) / np.float32(255.0)).view(np.uint32), b
    got = np.array([lib.hko_math_unorm16(u) for u in range(65536)], np.float32)
    want = np.arange(65536, dtype=np.float32) / np.float32(65535.0)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_brdf_matches_float64_restatement_of_the_published_formulas():
    """lit() (light.wgsl:796-818) = (Fr + Fd) * radiance * NoL with bevy_pbr 0.9's pbr_lighting functions, which are
    Filament's: D_GGX, V_SmithGGXCorrelated, F_Schlick with f90 = saturate(dot(f0, 50 * 0.33)), Fd_Burley; EnvBRDFApprox is
    Karis' mobile approximation.  Restated here in float64 from the published formulas, independent of include/hk_math.h."""
    lib = oracle.lib()
    rng = np.random.default_rng(3)
    f3 = lambda a: np.ascontiguousarray(a, np.float32)

    def unit(v):
        return v / np.linalg.norm(v)

    worst = 0.0
    for _ in range(400):
        N = unit(rng.normal(size=3))
        V = unit(N + 0.9 * rng.normal(size=3))
        Lv = unit(N + 0.9 * rng.normal(size=3))
        rough = float(np.float32(rng.uniform(0.089, 1.0) ** 2))
        F0 = rng.uniform(0.02, 0.9, 3); diffuse = rng.uniform(0, 1, 3); radiance = rng.uniform(0, 20, 3)
        args = [f3(radiance), f3(diffuse), f3(F0), f3(Lv), f3(N), f3(V)]
        radiance, diffuse, F0, Lv, N, V = [a.astype(np.float64) for a in args]
        out = np.zeros(3, np.float32)
        lib.hko_math_lit(args[0].ctypes.data, args[1].ctypes.data, C.c_float(rough), args[2].ctypes.data, args[3].ctypes.data,
                         args[4].ctypes.data, args[5].ctypes.data, out.ctypes.data)
        H = unit(Lv + V)
        sat = lambda x: min(max(x, 0.0), 1.0)
        NoL, NoH, LoH, NoV = sat(N @ Lv), sat(N @ H), sat(Lv @ H), max(N @ V, 1e-4)
        f90 = 0.5 + 2.0 * rough * LoH * LoH
        fd = (1 + (f90 - 1) * (1 - NoL) ** 5) * (1 + (f90 - 1) * (1 - NoV) ** 5) / np.pi
        a = NoH * rough
        k = rough / (1.0 - NoH * NoH + a * a)
        D = k * k / np.pi
        a2 = rough * rough
        Vis = 0.5 / (NoL * np.sqrt((NoV - a2 * NoV) * NoV + a2) + NoV * np.sqrt((NoL - a2 * NoL) * NoL + a2))
        F = F0 + (sat(F0.sum() * 50.0 * 0.33) - F0) * (1 - LoH) ** 5
        expect = (D * Vis * F + diffuse * fd) * radiance * NoL
        if np.abs(expect).max() > 1e-6:
            worst = max(worst, float(np.abs(out - expect).max() / max(np.abs(expect).max(), 1e-3)))
    assert worst < 2e-4, worst

    worst = 0.0
    for _ in range(400):
        f0 = rng.uniform(0.0, 1.0, 3); pr = float(rng.uniform(0.0, 1.0)); nov = float(rng.uniform(1e-4, 1.0))
        out = np.zeros(3, np.float32)
        f0_32 = f3(f0)
        lib.hko_math_env_brdf_approx(f0_32.ctypes.data, C.c_float(pr), C.c_float(nov), out.ctypes.data)
        pr, nov = float(np.float32(pr)), float(np.float32(nov))
        r = pr * np.array([-1.0, -0.0275, -0.572, 0.022]) + np.array([1.0, 0.0425, 1.04, -0.04])
        a004 = min(r[0] * r[0], 2.0 ** (-9.28 * nov)) * r[0] + r[1]
        ab = np.array([-1.04, 1.04]) * a004 + r[2:]
        expect = f0_32.astype(np.float64) * ab[0] + ab[1]
        worst = max(worst, float(np.abs(out - expect).max()))
    assert worst < 2e-5, worst
    assert lib.hko_math_perceptual_roughness_to_roughness(C.c_float(0.5)) == np.float32(0.25)
    assert lib.hko_math_perceptual_roughness_to_roughness(C.c_float(0.01)) == np.float32(np.float32(0.089) * np.float32(0.089))


F16_SRC = r"""
#include "hk_math.h"
extern "C" __attribute__((visibility("default"))) void to_f16(uint32_t first, uint16_t* out, size_t n) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) out[i] = hk::f32_to_f16_bits(hk::u2f(first + (uint32_t)i));
}
extern "C" __attribute__((visibility("default"))) void from_f16(uint32_t* out) {
    for (uint32_t h = 0; h < 65536u; ++h) out[h] = hk::f2u(hk::f16_bits_to_f32((uint16_t)h));
}
"""


def test_portable_f16_conversion_equals_the_f16c_one_for_every_input(tmp_path):
    """include/hk_math.h has a portable f32 <-> f16 branch for hosts without F16C; it must be the same function as the F16C one
    the oracle is built with: all 2^32 floats to f16 and all 2^16 halves back"""
    f16c = compile_host(tmp_path, "f16c", F16_SRC)
    portable = compile_host(tmp_path, "portable", F16_SRC, ["-mno-f16c"])
    for lib in (f16c, portable):
        lib.to_f16.restype, lib.to_f16.argtypes = None, [C.c_uint32, C.c_void_p, C.c_size_t]
        lib.from_f16.restype, lib.from_f16.argtypes = None, [C.c_void_p]
    a, b = np.empty(65536, np.uint32), np.empty(65536, np.uint32)
    f16c.from_f16(a.ctypes.data)
    portable.from_f16(b.ctypes.data)
    bad = np.flatnonzero(a != b)
    assert bad.size == 0, [(hex(h), hex(a[h]), hex(b[h])) for h in bad[:8]]
    n = 1 << 28
    a, b = np.empty(n, np.uint16), np.empty(n, np.uint16)
    for first in range(0, 1 << 32, n):
        f16c.to_f16(first, a.ctypes.data, n)
        portable.to_f16(first, b.ctypes.data, n)
        bad = np.flatnonzero(a != b)
        assert bad.size == 0, [(hex(first + int(i)), hex(a[i]), hex(b[i])) for i in bad[:8]]
