#!/bin/bash
# Round 2, ninth GPU call (1 GPU, benches only): is the instruction cache the lever on the light kernels?  The CTAs-per-SM knob
# (HK_MINB_* variants built by tools/build_variants.py), on the deep scenes where the walk dominates; the new default (primary rays on
# the 4-wide trees) as the baseline.
mkdir -p gpurun_out
O=gpurun_out
T=r2c11
short() { python - "$1" "$2" <<'PY'
import json, sys
try:
    d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
except Exception as e:
    print("  %-12s (no bench line: %s)" % (sys.argv[2], e)); sys.exit(0)
k = d.get("kernel_ms", {})
dn = sum(v for n, v in k.items() if n.startswith("denoise") or n == "demodulation")
print("  %-12s %-14s ms/frame %.3f e2e %.3f | gbuf %.3f direct %.3f emis %.3f emis_spa %.3f indirect %.3f ind_spa %.3f denoise %.3f | Mrays/s %.0f" % (
    sys.argv[2], d["config"]["workload"].split(":")[0], d["ms_per_step"], d["e2e"]["ms_per_step"], k.get("gbuffer", 0), k.get("direct", 0),
    k.get("emissive", 0), k.get("emissive_spatial", 0), k.get("indirect", 0), k.get("indirect_spatial", 0), dn, d["value"]))
PY
}
run() {  # name lib-or-empty config steps warmup
  local libarg=""; [ -n "$2" ] && libarg="--lib $PWD/$2"
  timeout 300 python bench.py $libarg --config $3 --steps $4 --warmup $5 --no-cpu-baseline 2> $O/${T}_$1_$3.err | grep "^{" > $O/${T}_$1_$3.json
  short $O/${T}_$1_$3.json $1
}
for cfg in "cornell_1080p 16 4" "scene_1080p 8 4" "city_4k 6 3"; do
  set -- $cfg
  run default "" $1 $2 $3
  for v in i11 i13 i14 g6 g8 g10 i12e10; do
    [ -f bevy_hikari_b200/variants/$v.so ] && run $v bevy_hikari_b200/variants/$v.so $1 $2 $3
  done
done
ls $O | grep -c ${T}
