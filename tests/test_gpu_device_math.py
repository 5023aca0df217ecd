"""The shared arithmetic of include/hk_math.h as the H100 runs it, against the oracle's build of the same header.

The parity suite checks the claim "device == oracle because both compile hk_math.h" through whole images, and the emulator
compiles the kernels for the host, so neither ever runs the `__CUDA_ARCH__` branches of the header on inputs the test frames do
not happen to produce.  tests/cuda/math_probe.cu runs every primitive over an input array on the device, compiled once with the
flags of the units that trace rays ("exact") and once with those of the tolerance units ("fast", build.py FAST_FLAGS);
the oracle's hko_math_batch / hko_math_batch_range / hko_spatial_digest / hko_deferred_digest run the same inputs on the host.
Every comparison is of bits, in chunks of 2^26 values, on the device; a failure names the count and the first differing inputs."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import oracle

pytestmark = pytest.mark.gpu

CHUNK = 1 << 26
FN = dict(f32_to_u32=0, f32_to_i32=1, f32_to_f16_bits=2, snorm8=3, pack2x16unorm_lane=4, fract=5, pow5=6, pow16=7, hash_u32=8,
          sin=9, cos=10, pow025=11, random_float=12, exp2=13, exp=14, saturate=15, f16_bits_to_f32=16, unsnorm8=17, unorm8=18,
          unpack2x16unorm_lane=19, fmin=32, fmax=33, clamp_lo=34, clamp_hi=35, normalize3=40, normalize2=41, D_GGX=42,
          V_SmithGGXCorrelated=43, EnvBRDFApprox=44, reinhard_luminance=45, reservoir_roundtrip=50, unpack_reservoir=51, pack_reservoir=52)
# (words in, words out) per element where that is not (1, 1) / (2, 1): math_probe.cu probe_words
WORDS = dict(normalize3=(3, 3), normalize2=(2, 2), D_GGX=(2, 1), V_SmithGGXCorrelated=(3, 1), EnvBRDFApprox=(5, 3), reinhard_luminance=(3, 3),
             reservoir_roundtrip=(16, 16), unpack_reservoir=(16, 32), pack_reservoir=(32, 16))
# bit-equal in both flavours over all 2^32 inputs: integer encodings, exact polynomials, and what only multiplies / adds under
# mul_rn / add_rn.  sin / cos, snorm8 and the unorm16 lane are the functions the tolerance units once contracted into FMAs.
EXHAUSTIVE_BOTH = ["f32_to_u32", "f32_to_i32", "f32_to_f16_bits", "snorm8", "pack2x16unorm_lane", "fract", "pow5", "pow16", "hash_u32",
                   "sin", "cos", "saturate"]
# bit-equal in the exact flavour; the fast flavour uses approximate sqrt / division (pow025, random_float) or ex2.approx (exp2, exp)
EXHAUSTIVE_EXACT_ONLY = ["pow025", "random_float", "exp2", "exp"]


@pytest.fixture(scope="module")
def probe():
    from tests.conftest import needs_real_gpu
    needs_real_gpu()        # the device branches of the header are the subject: the emulated kernels take the host ones
    import torch
    from bevy_hikari_b200 import build as product_build
    libs = {}
    for flavor, path in product_build.build_math_probe().items():
        lib = C.CDLL(path)
        lib.probe_batch.restype, lib.probe_batch.argtypes = C.c_int, [C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        lib.probe_spatial_digest.restype = C.c_int
        lib.probe_spatial_digest.argtypes = [C.c_uint32, C.c_float, C.c_int, C.c_int, C.c_uint32, C.c_void_p]
        lib.probe_deferred_digest.restype = C.c_int
        lib.probe_deferred_digest.argtypes = [C.c_int, C.c_int, C.c_float, C.c_uint32, C.c_void_p]
        libs[flavor] = lib
    try:    # an OpenMP team of the machine's size under a smaller CPU quota spends its time throttled (oracle.usable_cpus)
        C.CDLL("libgomp.so.1").omp_set_num_threads(oracle.usable_cpus())
    except OSError:
        pass
    torch.cuda.init()
    return torch, libs, oracle.lib()


class Diff:
    """Mismatch count and the first differing inputs of one flavour"""

    def __init__(self):
        self.count, self.first = 0, []

    def add(self, torch, inputs, dev, host, first_index):
        bad = dev != host
        n = int(bad.sum())
        if n and len(self.first) < 8:
            idx = torch.nonzero(bad).flatten()[:8 - len(self.first)].cpu().numpy()
            for i in idx:
                x = int(inputs[i]) if inputs is not None else (first_index + int(i)) & 0xFFFFFFFF
                self.first.append((hex(x) if not isinstance(x, tuple) else x, hex(int(dev[i]) & 0xFFFFFFFF), hex(int(host[i]) & 0xFFFFFFFF)))
        self.count += n

    def __repr__(self):
        return f"{self.count} mismatches, first (input, device, oracle): {self.first}"


def run_range(probe, fn, first, total, flavors=("exact", "fast"), check=None):
    """Bit patterns first .. first + total - 1 through fn on the device (each flavour) and in the oracle.  `check(x, dev)`, if given,
    runs on each fast-flavour chunk (device tensors) instead of the bit comparison."""
    torch, libs, orc = probe
    diffs = {f: Diff() for f in flavors}
    host = torch.empty(min(CHUNK, total), dtype=torch.int32, pin_memory=True)
    dev = torch.empty(min(CHUNK, total), dtype=torch.int32, device="cuda")
    for start in range(0, total, CHUNK):
        n = min(CHUNK, total - start)
        base = (first + start) & 0xFFFFFFFF
        orc.hko_math_batch_range(FN[fn], base, host.data_ptr(), n)
        want = host[:n].to("cuda", non_blocking=True)
        for f in flavors:
            rc = libs[f].probe_batch(FN[fn], None, base, dev.data_ptr(), n)
            assert rc == 0, f"probe_batch({fn}, {f}): CUDA error {rc}"
            if f == "fast" and check is not None:
                check(base, dev[:n])
            else:
                diffs[f].add(torch, None, dev[:n], want, base)
    return diffs


def run_array(probe, fn, inputs, flavors=("exact", "fast"), host_out=None):
    """inputs: uint32 array of WORDS[fn][0] words per element (two for the two-operand functions).  A mismatch is an element with
    any differing output word.  host_out: a list that receives the oracle's outputs (elements x words)."""
    torch, libs, orc = probe
    win, wout = WORDS.get(fn, (2 if FN[fn] >= 32 else 1, 1))
    n = inputs.size // win
    host = np.empty(n * wout, np.uint32)
    orc.hko_math_batch(FN[fn], inputs.ctypes.data, host.ctypes.data, n)
    if host_out is not None:
        host_out.append(host.reshape(n, wout))
    d_in = torch.from_numpy(inputs.view(np.int32)).cuda()
    want = torch.from_numpy(host.view(np.int32)).cuda().view(n, wout)
    dev = torch.empty((n, wout), dtype=torch.int32, device="cuda")
    diffs = {f: Diff() for f in flavors}
    rows = inputs.reshape(n, win)
    for f in flavors:
        assert libs[f].probe_batch(FN[fn], d_in.data_ptr(), 0, dev.data_ptr(), n) == 0
        bad = (dev != want).any(dim=1).cpu().numpy()
        got = dev.cpu().numpy().view(np.uint32) if bad.any() else None
        diffs[f].count = int(bad.sum())
        diffs[f].first = [([hex(int(v)) for v in rows[i]], [hex(int(v)) for v in got[i]], [hex(int(v)) for v in host.reshape(n, wout)[i]])
                          for i in np.flatnonzero(bad)[:4]]
    return diffs


@pytest.mark.parametrize("fn", EXHAUSTIVE_BOTH + EXHAUSTIVE_EXACT_ONLY)
def test_every_bit_pattern_matches_the_oracle(probe, fn):
    """All 2^32 inputs.  Exact flavour: bit-equal for every function.  Fast flavour: bit-equal for everything that ends in an
    integer or only multiplies and adds; the approximate ones are reported (pow025, random_float, exp, whose ex2.approx is not
    bit-exact) or bounded (exp2, below)."""
    fast_asserted = fn in EXHAUSTIVE_BOTH
    d = run_range(probe, fn, 0, 1 << 32, flavors=("exact", "fast") if fn != "exp2" else ("exact",))
    print(fn, {f: repr(v) for f, v in d.items()})
    assert d["exact"].count == 0, f"{fn}, exact flavour: {d['exact']}"
    if fast_asserted:
        assert d["fast"].count == 0, f"{fn}, tolerance flavour: {d['fast']}"


@pytest.mark.parametrize("fn,total", [("f16_bits_to_f32", 1 << 16), ("unsnorm8", 1 << 8), ("unorm8", 1 << 8),
                                      ("unpack2x16unorm_lane", 1 << 16)])
def test_every_small_encoding_decodes_like_the_oracle(probe, fn, total):
    d = run_range(probe, fn, 0, total)
    assert d["exact"].count == 0 and d["fast"].count == 0, (fn, d)


def test_fast_exp2_stays_within_two_ulp_and_saturates_as_documented(probe):
    """hk_math.h: the tolerance units' exp2_ is ex2.approx, within 2.06 ulp on [-126, 128); NaN -> NaN, x >= 128 -> +inf,
    x < -126 -> a subnormal or zero.  Every float input, against float64."""
    torch = probe[0]
    worst = [0.0]
    bad = []

    def check(base, dev):
        bits = torch.arange(base, base + dev.numel(), dtype=torch.int64, device="cuda")
        bits = torch.where(bits >= 1 << 31, bits - (1 << 32), bits).to(torch.int32)       # the u32 patterns as i32
        x = bits.view(torch.float32)
        y = dev.view(torch.float32)
        nan = torch.isnan(x)
        if bool((nan & ~torch.isnan(y)).any()):
            bad.append(("NaN input gave a number", base))
        hi = ~nan & (x >= 128.0)
        if bool((hi & (y != math.inf)).any()):
            bad.append(("x >= 128 not +inf", base))
        lo = ~nan & (x < -126.0)
        if bool((lo & ~((y >= 0.0) & (y < 2.0 ** -126))).any()):
            bad.append(("x < -126 not subnormal / 0", base))
        mid = ~nan & (x >= -126.0) & (x < 128.0)
        if bool(mid.any()):
            ref = torch.exp2(x[mid].double())
            _, e = torch.frexp(ref)
            ulp = torch.ldexp(torch.ones_like(ref), (e - 24).clamp(min=-149))
            err = ((y[mid].double() - ref).abs() / ulp).max().item()
            worst[0] = max(worst[0], err)

    run_range(probe, "exp2", 0, 1 << 32, flavors=("fast",), check=check)
    print("fast exp2_: worst error on [-126, 128) =", round(worst[0], 3), "ulp")
    assert not bad, bad[:8]
    assert worst[0] <= 2.06, worst[0]


def special_floats():
    """±0, ±min / max subnormal, ±1, ±1 ± ulp, ±FLT_MAX, ±inf, quiet NaNs of both signs with two payloads"""
    bits = [0x00000000, 0x00000001, 0x007FFFFF, 0x3F800000, 0x3F7FFFFF, 0x3F800001, 0x7F7FFFFF, 0x7F800000]
    out = bits + [b | 0x80000000 for b in bits] + [0x7FC00000, 0xFFC00000, 0x7FC00001, 0xFFC12345, 0x7FFFFFFF, 0x7FA00000]
    return np.array(out, np.uint32)


@pytest.mark.parametrize("fn", ["fmin", "fmax", "clamp_lo", "clamp_hi"])
def test_min_max_clamp_on_special_pairs_and_random_pairs(probe, fn):
    """Signed zeros and NaN encodings: the host branch of fmin_ / fmax_ exists only to mirror min.f32 / max.f32 (-0 below +0, two
    NaNs give 0x7FFFFFFF)."""
    s = special_floats()
    a, b = np.meshgrid(s, s, indexing="ij")
    rng = np.random.default_rng(20261015)
    rnd = rng.integers(0, 1 << 32, size=2 * (1 << 26), dtype=np.uint64).astype(np.uint32)
    inputs = np.concatenate([np.stack([a.ravel(), b.ravel()], axis=1).ravel(), rnd])
    d = run_array(probe, fn, inputs)
    assert d["exact"].count == 0 and d["fast"].count == 0, (fn, d)


@pytest.mark.parametrize("size", [(131, 67), (1920, 1080), (3840, 2160)])
def test_spatial_neighbour_and_march_tap_pixels_match_the_oracle(probe, size):
    """Every pixel of the frame, both tables (16 neighbours within 20 px, 8 within 10 px), frames 1-8: the digest of each pixel's
    neighbour pixels and depth-march tap pixels (csrc/hk_spatial_taps.cuh) equals the oracle's (spatial_neighbour, spatial_tap_uv),
    in the exact flavour and in the tolerance flavour that the product's k_spatial / kc_spatial are compiled with."""
    torch, libs, orc = probe
    w, h = size
    host = np.empty(w * h, np.uint32)
    dev = torch.empty(w * h, dtype=torch.int32, device="cuda")
    failures = []
    for count, rng_px in ((16, 20.0), (8, 10.0)):
        for frame in range(1, 9):
            orc.hko_spatial_digest(count, rng_px, w, h, frame, host.ctypes.data)
            for f in ("exact", "fast"):
                assert libs[f].probe_spatial_digest(count, rng_px, w, h, frame, dev.data_ptr()) == 0
                bad = np.flatnonzero(dev.cpu().numpy().view(np.uint32) != host)
                if bad.size:
                    failures.append((f, count, frame, int(bad.size), [(int(p % w), int(p // w)) for p in bad[:4]]))
    assert not failures, f"(flavour, neighbours, frame, pixels, first pixels): {failures}"


# 1.3, 1.5, 1.7, 2 and two fixed f32 draws in (1, 2] (numpy default_rng(20261016)).  At 1.5, W / RW is exactly 1.5 for sizes divisible
# by 3: half the columns and rows land exactly on a texel edge in real arithmetic, so their texel is decided by the last bit of the uv
UPSCALE_RATIOS = [1.3, 1.5, 1.7, 2.0, 1.3451449, 1.556715]
DEFERRED_DIGESTS = ["light texel", "denoise texel", "previous pixel", "spatial neighbours and taps"]


def render_size(w, h, ratio):
    """ceil(size / ratio) as context.cu / the oracle compute it in f32"""
    scale = np.float32(1.0) / np.float32(ratio)
    return int(np.ceil(scale * np.float32(w))), int(np.ceil(scale * np.float32(h)))


@pytest.mark.parametrize("size", [(1920, 1080), (3840, 2160), (192, 108), (131, 67), (127, 63), (90, 50)])
def test_render_to_gbuffer_texel_mapping_above_ratio_1_matches_the_oracle(probe, size):
    """Every render pixel at upscale ratios in (1, 2], frames 1-8 (both jitter signs), both flavours: the G-buffer texel the light
    passes and k_spatial read (light_gbuffer_index), the one the denoise passes read (denoise_deferred_coords), the reprojected
    pixel (previous_pixel) for velocity 0 and a drawn velocity, and k_spatial's neighbour pixels with the texels of each neighbour and
    of its depth-march taps (csrc/hk_device.cuh, csrc/hk_spatial_taps.cuh) equal the oracle's (Deferred::jittered_coords / nearest,
    load_previous, spatial_neighbour, spatial_tap_uv) bit for bit.  An off-by-one there reads another texel's normal, depth,
    instance and albedo."""
    torch, libs, orc = probe
    w, h = size
    host = np.empty(w * h * 4, np.uint32)
    dev = torch.empty(w * h * 4, dtype=torch.int32, device="cuda")
    failures, counts = [], {}
    for ratio in UPSCALE_RATIOS:
        rw, rh = render_size(w, h, ratio)
        n = rw * rh * 4
        for frame in range(1, 9):
            orc.hko_deferred_digest(w, h, ratio, frame, host.ctypes.data)
            for f in ("exact", "fast"):
                assert libs[f].probe_deferred_digest(w, h, ratio, frame, dev.data_ptr()) == 0
                bad = (dev[:n].cpu().numpy().view(np.uint32) != host[:n]).reshape(rw * rh, 4)
                px = np.flatnonzero(bad.any(axis=1))
                counts[(f, ratio)] = counts.get((f, ratio), 0) + int(px.size)
                if px.size:
                    which = {DEFERRED_DIGESTS[k]: int(bad[:, k].sum()) for k in range(4) if bad[:, k].any()}
                    failures.append((f, ratio, frame, int(px.size), which, [(int(p % rw), int(p // rw)) for p in px[:4]]))
    print(f"{w}x{h} differing render pixels over frames 1-8 (flavour, ratio):", counts)
    assert not failures, f"(flavour, ratio, frame, pixels, per digest, first render pixels): {failures[:12]}"


def random_words(rng, n, specials):
    """n float bit patterns: a quarter uniform in [-1.5, 1.5], a quarter in [0, 1], a quarter random bits, a quarter specials"""
    out = np.empty(n, np.uint32)
    q = n // 4
    out[:q] = rng.uniform(-1.5, 1.5, q).astype(np.float32).view(np.uint32)
    out[q:2 * q] = rng.uniform(0.0, 1.0, q).astype(np.float32).view(np.uint32)
    out[2 * q:3 * q] = rng.integers(0, 1 << 32, q, dtype=np.uint64).astype(np.uint32)
    out[3 * q:] = rng.choice(specials, n - 3 * q)
    return rng.permutation(out)


@pytest.mark.parametrize("fn", ["normalize3", "normalize2", "D_GGX", "V_SmithGGXCorrelated", "EnvBRDFApprox", "reinhard_luminance"])
def test_vector_and_lighting_functions_match_the_oracle_in_the_exact_flavour(probe, fn):
    """2^24 random arguments (in range, random bits and the special values in every position) plus every special value in every
    argument with the others 0.5: bit-equal in the exact flavour.  The tolerance flavour is held to the product's tolerance contract
    (tests/test_gpu_tolerance.py) rather than to bits."""
    win = WORDS[fn][0]
    rng = np.random.default_rng(20261016 + FN[fn])
    s = special_floats()
    grid = np.full((win * s.size, win), np.float32(0.5).view(np.uint32), np.uint32)
    for k in range(win):
        grid[k * s.size:(k + 1) * s.size, k] = s
    inputs = np.concatenate([grid.ravel(), random_words(rng, win * (1 << 24), s)])
    d = run_array(probe, fn, inputs, flavors=("exact",))
    assert d["exact"].count == 0, (fn, d)


def random_records(n, rng):
    """n packed reservoir records (hk_packed_reservoir, 16 words): f16 / unorm16 / snorm8 fields of random bits, float fields mostly
    in range with +-0, NaN and +-inf mixed in"""
    rec = rng.integers(0, 1 << 32, size=(n, 16), dtype=np.uint64).astype(np.uint32)
    floats = np.r_[4:12]                        # visible_position, sample_position
    vals = rng.normal(0.0, 10.0, size=(n, floats.size)).astype(np.float32).view(np.uint32)
    specials = np.array([0x00000000, 0x80000000, 0x7FC00000, 0xFFC00000, 0x7F800000, 0xFF800000, 0x7FA00001], np.uint32)
    pick = rng.random((n, floats.size)) < 0.1
    vals[pick] = rng.choice(specials, int(pick.sum()))
    rec[:, floats] = vals
    inst = rng.integers(0, 1 << 20, n).astype(np.float32).view(np.uint32)          # sample_position.w = f32(visible_instance)
    rec[:, 11] = np.where(rng.random(n) < 0.9, inst, rec[:, 11])
    return rec


def test_reservoir_round_trip_and_pack_match_the_oracle(probe):
    """pack_reservoir(unpack_reservoir(p)) of 2^22 records: bit-equal to hko_pack_reservoir_roundtrip in the exact flavour (the
    tolerance flavour's unpack re-normalises with approximate square roots).  pack_reservoir alone, fed the oracle's unpacked
    records: bit-equal in both flavours — what the spatial pass stores (normal, lifetime and random bytes) is exact in the product."""
    rng = np.random.default_rng(20261017)
    rec = random_records(1 << 22, rng)
    d = run_array(probe, "reservoir_roundtrip", rec.ravel(), flavors=("exact",))
    assert d["exact"].count == 0, d
    unpacked = []
    d = run_array(probe, "unpack_reservoir", rec.ravel(), flavors=("exact",), host_out=unpacked)
    assert d["exact"].count == 0, d
    d = run_array(probe, "pack_reservoir", np.ascontiguousarray(unpacked[0]).ravel())
    assert d["exact"].count == 0 and d["fast"].count == 0, d
