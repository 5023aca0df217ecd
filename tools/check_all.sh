#!/bin/bash
# Everything that can be checked WITHOUT a GPU, in the order a session should run it after touching kernels or the oracle
# (about 15 minutes on 8 cores).  Exits non-zero at the first failure.
set -e
cd "$(dirname "$0")/.."
echo "== build (nvcc cross-compiles sm_90a; oracle; import)";          python -c "import __graft_entry__ as g; g.build()"
echo "== CPU suite (oracle pins, host logic, ABI, emulated GPU suite in both thread orders, fixed-seed fuzz)"
python -m pytest tests -x -q -m "not gpu"
echo "== generated Rust declarations current";                           python tools/gen_rust_sys.py --check
echo "== AddressSanitizer build of the emulated kernels on the newest device tests"
LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 HK_EMULATE_KERNELS=1 HK_EMU_ASAN=1 \
    python -m pytest tests/test_gpu_zz_fsr.py tests/test_gpu_zz_examples.py tests/test_gpu_upscale.py -m gpu -q -x -p no:cacheprovider
LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 HK_EMULATE_KERNELS=1 HK_EMU_ASAN=1 \
    python -m pytest tests/test_gpu_scene_update_edges.py -m gpu -q -x -p no:cacheprovider -k "non_finite or cache"
echo "== alignment-sanitizer build of the emulated kernels (vector types alignas'd as on the device): the whole device suite"
HK_EMULATE_KERNELS=1 HK_EMU_ALIGN=1 python -m pytest tests -m gpu -q -x -p no:cacheprovider
echo "== a fresh random batch (seeds from the clock)"
SEED=$(( $(date +%s) % 1000000 ))
HK_EMULATE_KERNELS=1 python tools/fuzz_parity.py $SEED 150
HK_EMULATE_KERNELS=1 HK_FUZZ_SOUP=1 python tools/fuzz_parity.py $((SEED + 1000)) 60
HK_EMULATE_KERNELS=1 HK_FUZZ_HALO=1 python tools/fuzz_parity.py $((SEED + 2000)) 40
HK_EMULATE_KERNELS=1 HK_FUZZ_TILES=1 python tools/fuzz_parity.py $((SEED + 3000)) 40
echo "== the WGSL pin between the fixtures (reference shader text executed vs the oracle, fresh seeds)"
python tools/fuzz_wgsl_pin.py $((SEED + 4000)) 40
echo "== static: code size / registers / spills of the light kernels";   python tools/code_size.py | tail -30
echo "all CPU-side checks passed"
