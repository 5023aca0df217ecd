#!/usr/bin/env python
"""TEST INFRASTRUCTURE: build tests/emu/_build/libhikari_emu.so — the kernel sources of bevy_hikari_b200/csrc compiled for
the host through tests/emu/cuda_emu.h, behind the same C ABI, so that the kernels' logic can be compared with the oracle
without a GPU (tests/test_emulated_kernels.py; HK_EMULATE_KERNELS=1 pytest -m gpu ... runs any GPU test on the CPU during development).
The only source transformations are
  * `kernel<<<grid, block, 0, stream>>>(args)`  ->  `EMU_LAUNCH(grid, block, kernel(args))`, or `EMU_LAUNCH_COOP(...)` for the
    cooperative kernels (kc_*): shared memory, __syncthreads, ballots and shuffles run for real, threads as fibers (cuda_emu.h)
  * flush_counters' warp reduction (shuffles) -> one atomic add per thread (same totals)."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(ROOT, "bevy_hikari_b200", "csrc")
HOST = os.path.join(ROOT, "bevy_hikari_b200", "host")
ASAN = bool(os.environ.get("HK_EMU_ASAN"))      # AddressSanitizer build: a memcheck for the kernels' indexing (run python with
#                                                  LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0)
ALIGN = bool(os.environ.get("HK_EMU_ALIGN"))    # UBSan alignment build: float4 / uint4 / float2 ... are alignas'd as on the device and cudaMalloc
#                                                  returns 256-byte aligned blocks, so a vector access the GPU would fault on ("misaligned
#                                                  address", sticky) aborts here too — the host's own unaligned moves never notice
GEN, OUT = os.path.join(HERE, "_gen"), os.path.join(HERE, "_build_asan" if ASAN else ("_build_align" if ALIGN else "_build"))
LIB = os.path.join(OUT, "libhikari_emu.so")
CU = ["context.cu", "kernels_light.cu", "kernels_pool.cu", "kernels_spatial.cu", "kernels_post.cu", "kernels_upscale.cu", "kernels_scene.cu"]
CPP = ["hikari.cpp", "hikari_capi.cpp", "gltf_ingest.cpp", "hikari_plugin.cpp", "hikari_plugin_capi.cpp"]
CXX = os.environ.get("HK_CXX", "/usr/bin/g++")
FLAGS = ["-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-std=c++17", "-w",
         "-I" + os.path.join(HERE, "include"), "-I" + SRC, "-I" + HOST, "-I" + os.path.join(ROOT, "include")] + \
        os.environ.get("HK_EMU_EXTRA", "").split()      # e.g. -DHK_WIDE_STACK=32: validate a tuning variant's logic
if ASAN:
    FLAGS = [f for f in FLAGS if f != "-O2"] + ["-O1", "-g1", "-fno-var-tracking-assignments", "-fsanitize=address", "-fno-omit-frame-pointer"]
if ALIGN:
    FLAGS = [f for f in FLAGS if f != "-O2"] + ["-O1", "-g1", "-fsanitize=alignment", "-fno-sanitize-recover=alignment"]

LAUNCH = re.compile(r"([A-Za-z_][A-Za-z_0-9]*(?:<[^<>;]*>)?)<<<([^;]*?)>>>\(([^;]*)\);")
COOPERATIVE = re.compile(r"^kc_")     # kernels with shared memory / barriers / warp collectives: threads of a block run as fibers
FLUSH_OLD = re.compile(r"for \(int o = 16; o > 0; o >>= 1\) \{.*?\n    \}\n    if \(\(threadIdx\.x & 31\) == 0\) \{", re.S)


def transform(text, name):
    def launch(m):
        kernel, cfg, args = m.group(1), m.group(2), m.group(3)
        parts = [p.strip() for p in split_top(cfg)]
        macro = "EMU_LAUNCH_COOP" if COOPERATIVE.match(kernel) else "EMU_LAUNCH"
        return f"{macro}(dim3({parts[0]}), dim3({parts[1]}), {kernel}({args}));"
    out, n = LAUNCH.subn(launch, text)
    if name == "kernels_light.cu":
        out, k = FLUSH_OLD.subn("{", out)
        assert k == 1, "flush_counters pattern changed"
    assert "<<<" not in out, f"unconverted launch in {name}"
    return out, n


def split_top(s):
    parts, depth, cur = [], 0, ""
    for ch in s:
        if ch in "(<[":
            depth += 1
        elif ch in ")>]":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append(cur); cur = ""
        else:
            cur += ch
    parts.append(cur)
    return parts


def newer(target, sources):
    return not os.path.exists(target) or any(os.path.getmtime(s) > os.path.getmtime(target) for s in sources)


def build(force=False):
    os.makedirs(GEN, exist_ok=True); os.makedirs(OUT, exist_ok=True)
    deps = [os.path.join(SRC, f) for f in os.listdir(SRC)] + [os.path.join(HOST, f) for f in os.listdir(HOST)] + \
           [os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))] + \
           [os.path.join(HERE, "cuda_emu.h"), os.path.join(HERE, "emu_runtime.cpp"), os.path.abspath(__file__)]
    # the library on disk must have been built from the current sources AND with the current flags: a tuning-variant or sanitizer
    # build (HK_EMU_EXTRA) left behind must not be mistaken for the default build by the next run
    stamp = os.path.join(OUT, "flags.txt")
    wanted = " ".join(FLAGS)
    have = open(stamp).read() if os.path.exists(stamp) else None
    if not force and not newer(LIB, deps) and have == wanted:
        return LIB
    objs, launches, jobs = [], 0, []
    for f in CU:
        text, n = transform(open(os.path.join(SRC, f)).read(), f)
        launches += n
        g = os.path.join(GEN, f.replace(".cu", ".emu.cpp"))
        open(g, "w").write(text)
        o = os.path.join(OUT, f + ".o")
        jobs.append([CXX] + FLAGS + ["-c", g, "-o", o])
        objs.append(o)
    glue = os.path.join(HERE, "emu_runtime.cpp")
    o = os.path.join(OUT, "emu_globals.o")
    jobs.append([CXX] + FLAGS + ["-I" + HERE, "-c", glue, "-o", o])
    objs.append(o)
    for f in CPP:
        o = os.path.join(OUT, f + ".o")
        jobs.append([CXX] + FLAGS + ["-c", os.path.join(HOST, f), "-o", o])
        objs.append(o)
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as pool:      # one compiler per translation unit (the sanitizer builds of
        for r in pool.map(lambda j: subprocess.run(j).returncode, jobs):           # kernels_light take tens of minutes each otherwise in a row)
            if r != 0:
                raise SystemExit("emulator build failed")
    subprocess.run([CXX, "-shared", "-fopenmp", "-o", LIB] + objs + (["-fsanitize=address"] if ASAN else []) + (["-fsanitize=alignment", "-static-libubsan"] if ALIGN else []) + ["-lz"], check=True)
    open(stamp, "w").write(wanted)
    print(f"emulator: {launches} launch sites converted -> {LIB}")
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
