"""Build the two product libraries in-tree:

  libhikari_host.so   the C++ host mirror up to hikari_make_frame_inputs (scene preparation, settings, frame uniforms):
                      pure CPU, no CUDA dependency — what a CPU-only consumer (the reference arm of bench.py) loads
  libhikari_b200.so   THE PRODUCT: hand-written CUDA for sm_90a + the nodes / HikariPlugin that call it; exports the C ABI of
                      include/hikari_b200.h and, through its dependency on libhikari_host.so ($ORIGIN rpath), every symbol
                      of include/hikari_host.h.  Tolerance build: the translation units that trace no rays (spatial reuse,
                      denoise, tone mapping, upscalers' neighbours in kernels_post.cu / kernels_spatial.cu) are compiled with
                      FMA contraction and approximate division / square root / exp (FAST_FLAGS); everything that walks the BVH
                      or writes an id keeps exact arithmetic.  Contract: ids and temporal reservoirs bit-exact, radiance within
                      1 f16 ulp per pass from identical inputs, < 1e-4 outlier pixels (tests/test_gpu_tolerance.py, and
                      tests/test_gpu_tolerance_upscaled.py at upscale ratios above 1).
  libhikari_b200_exact.so   the same sources with exact arithmetic everywhere: bit-identical to the CPU oracle on every plane
                      (the 0-ulp parity suite runs on it).  Shares every object file with the product except the two above.

nvcc cross-compiles without a GPU.  Flags that matter:
  -gencode arch=compute_90a,code=sm_90a     H100 only, no PTX fallback for other architectures
  -fmad=false / -ffp-contract=off           no implicit FMA contraction: every fused op is an explicit fmaf() in
                                            include/hk_math.h, which is what makes device results comparable bit-for-bit
                                            with the CPU oracle (SURVEY.md App. E)
  -lineinfo                                 ncu source page maps to these files

A stamp (_build/flags.txt) records the full flag list of the objects on disk: a tuning build (HK_NVCC_EXTRA=...) left
behind is rebuilt by the next default build instead of being mistaken for it.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INC = os.path.join(ROOT, "include")
OBJ = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libhikari_b200.so")
EXACT_LIB = os.path.join(HERE, "libhikari_b200_exact.so")
HOST_LIB = os.path.join(HERE, "libhikari_host.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("HK_CXX", "/usr/bin/g++")

CU = ["csrc/context.cu", "csrc/kernels_light.cu", "csrc/kernels_pool.cu", "csrc/kernels_spatial.cu", "csrc/kernels_post.cu", "csrc/kernels_upscale.cu", "csrc/kernels_scene.cu"]
CPP_HOST = ["host/hikari.cpp", "host/hikari_capi.cpp", "host/gltf_ingest.cpp"]                     # -> libhikari_host.so
CPP_PLUGIN = ["host/hikari_plugin.cpp", "host/hikari_plugin_capi.cpp"]     # -> libhikari_b200.so (they call hk_*)
HEADERS = ["csrc/hk_device.cuh", "csrc/hk_pool.cuh", "csrc/hk_wide.cuh", "csrc/wide_build.h", "csrc/hk_tile.cuh", "csrc/hk_spatial_taps.cuh", "csrc/hk_kernels.h", "host/hikari.hpp", "host/hikari_settings_convert.hpp",
           "../include/hk_math.h", "../include/hk_layout.h", "../include/hikari_b200.h", "../include/hikari_host.h"]

NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false",
              "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math", "-I", INC, "-I", os.path.join(HERE, "csrc")]
# translation units without a ray walk or an id decision: tolerance flags in the product build
FAST_TUS = ["csrc/kernels_spatial.cu", "csrc/kernels_post.cu"]
FAST_FLAGS = ["-fmad=true", "-prec-div=false", "-prec-sqrt=false", "-DHK_FAST_MATH=1"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-I", INC, "-I", os.path.join(HERE, "host")]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return r.stdout + r.stderr


def build(force=False, verbose=False, ptxas_info=False, out=None):
    """Builds both libraries; returns the path of libhikari_b200.so.  `out`: write the CUDA library there instead (tuning
    variants, tools/build_variants.py) — its objects go to a scratch directory and the default build is left alone."""
    extra_env = os.environ.get("HK_NVCC_EXTRA", "").split()   # tuning experiments, e.g. -DHK_MINB_INDIRECT=5
    obj_dir = OBJ if out is None else os.path.join(OBJ, "variant_" + os.path.splitext(os.path.basename(out))[0])
    lib = LIB if out is None else out
    os.makedirs(obj_dir, exist_ok=True)
    stamp = os.path.join(obj_dir, "flags.txt")
    wanted = " ".join(NVCC_FLAGS + extra_env + ["|"] + FAST_FLAGS + ["|", os.environ.get("HK_NO_FAST_MATH", "")] + CXX_FLAGS)
    have = open(stamp).read() if os.path.exists(stamp) else None
    if have != wanted:
        force = True
    headers = [os.path.join(HERE, h) for h in HEADERS]
    fast_off = bool(os.environ.get("HK_NO_FAST_MATH"))      # A/B: the product with exact arithmetic everywhere
    jobs, cuda_objs, exact_objs, host_objs = [], [], [], []
    for src in CU:
        s = os.path.join(HERE, src)
        o = os.path.join(obj_dir, os.path.basename(src) + ".o")
        cuda_objs.append(o)
        extra = (["-Xptxas", "-v"] if ptxas_info else []) + extra_env
        fast = src in FAST_TUS and not fast_off
        if force or _newer(o, [s] + headers):
            flags = [f for f in NVCC_FLAGS if not (fast and f == "-fmad=false")] + (FAST_FLAGS if fast else [])
            jobs.append([NVCC] + flags + extra + ["-c", s, "-o", o])
        if out is None:                                      # the exact flavour re-compiles only the tolerance units
            oe = os.path.join(obj_dir, os.path.basename(src) + ".exact.o") if fast else o
            exact_objs.append(oe)
            if fast and (force or _newer(oe, [s] + headers)):
                jobs.append([NVCC] + NVCC_FLAGS + extra_env + ["-c", s, "-o", oe])
    for src in CPP_HOST + CPP_PLUGIN:
        s = os.path.join(HERE, src)
        o = os.path.join(obj_dir, os.path.basename(src) + ".o")
        if src in CPP_HOST:
            host_objs.append(o)
        else:
            cuda_objs.append(o); exact_objs.append(o)
        if force or _newer(o, [s] + headers):
            jobs.append([CXX] + CXX_FLAGS + ["-c", s, "-o", o])
    logs = []
    if jobs:
        with ThreadPoolExecutor(max_workers=len(jobs)) as ex:
            logs = list(ex.map(_run, jobs))
    link = ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static", "-Xcompiler", "-fPIC", "-L", HERE, "-lhikari_host",
            "-Xlinker", "-rpath,$ORIGIN", "-Xlinker", "-rpath," + HERE]
    # (variant builds never re-link the host library: several of them run at once and the default build owns it)
    if (out is None and jobs) or not os.path.exists(HOST_LIB):
        logs.append(_run([CXX, "-shared", "-o", HOST_LIB] + host_objs + ["-lz"]))
    if jobs or not os.path.exists(lib):
        logs.append(_run([NVCC, "-shared", "-o", lib] + cuda_objs + link))
    if out is None and (jobs or not os.path.exists(EXACT_LIB)):
        logs.append(_run([NVCC, "-shared", "-o", EXACT_LIB] + exact_objs + link))
    open(stamp, "w").write(wanted)
    if verbose or ptxas_info:
        print("\n".join(l for l in logs if l.strip()))
    return lib


PROBE_SRC = os.path.join(ROOT, "tests", "cuda", "math_probe.cu")
PROBE_LIBS = {"exact": os.path.join(OBJ, "libhk_math_probe_exact.so"), "fast": os.path.join(OBJ, "libhk_math_probe_fast.so")}


def probe_flags(flavor):
    """nvcc flags of the math probe: those of every unit that traces rays ("exact") or those of FAST_TUS ("fast"), derived from
    NVCC_FLAGS / FAST_FLAGS exactly as build() derives them."""
    fast = flavor == "fast"
    return [f for f in NVCC_FLAGS if not (fast and f == "-fmad=false")] + (FAST_FLAGS if fast else [])


def build_math_probe(force=False):
    """Test infrastructure: tests/cuda/math_probe.cu (the primitives of include/hk_math.h and the spatial-reuse pixel helpers run
    on the device) as two shared libraries, one per flavour; tests/test_gpu_device_math.py compares them with the oracle."""
    os.makedirs(OBJ, exist_ok=True)
    sources = [PROBE_SRC] + [os.path.join(HERE, h) for h in HEADERS]
    jobs = []
    for flavor, lib in PROBE_LIBS.items():
        flags = probe_flags(flavor)
        stamp = lib + ".flags"
        stale = not os.path.exists(stamp) or open(stamp).read() != " ".join(flags)
        if force or stale or _newer(lib, sources):
            jobs.append(([NVCC] + flags + ["-shared", "-cudart", "static", "-o", lib, PROBE_SRC], stamp, flags))
    if jobs:
        with ThreadPoolExecutor(max_workers=len(jobs)) as ex:
            list(ex.map(lambda j: _run(j[0]), jobs))
        for _, stamp, flags in jobs:
            open(stamp, "w").write(" ".join(flags))
    return dict(PROBE_LIBS)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, ptxas_info="--ptxas" in sys.argv))
