#!/bin/bash
# Round 2, call 16 (1 GPU, 8.6 GPU-minutes left):
#   1. the whole device suite on the tree with the reference's SMAA / TAA output extents (Band::OW / OH) and the five upscaler fixtures;
#   2. the default on the three scenes.
mkdir -p gpurun_out
O=gpurun_out
T=r2c16
START=$(date +%s)
LIMIT=${HK_CALL_LIMIT:-250}
left() { echo $(( LIMIT - ( $(date +%s) - START ) )); }
echo "== 1. device suite"
timeout -s INT 120 python -m pytest tests -m gpu -q -p no:cacheprovider > $O/${T}_pytest.txt 2>&1; tail -6 $O/${T}_pytest.txt
short() { python - "$1" "$2" <<'PY'
import json, sys
try:
    d = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
except Exception as e:
    print("  %-10s (no bench line: %s)" % (sys.argv[2], e)); sys.exit(0)
k = d.get("kernel_ms", {})
dn = sum(v for n, v in k.items() if n.startswith("denoise") or n == "demodulation")
print("  %-10s %-14s ms/frame %.3f e2e %.3f | gbuf %.3f direct %.3f emis %.3f emis_spa %.3f indirect %.3f ind_spa %.3f denoise %.3f" % (
    sys.argv[2], d["config"]["workload"].split(":")[0], d["ms_per_step"], d["e2e"]["ms_per_step"], k.get("gbuffer", 0), k.get("direct", 0),
    k.get("emissive", 0), k.get("emissive_spatial", 0), k.get("indirect", 0), k.get("indirect_spatial", 0), dn))
PY
}
run() {  # name lib-or-empty config steps warmup
  local libarg=""; [ -n "$2" ] && libarg="--lib $PWD/$2"
  timeout 60 python bench.py $libarg --config $3 --steps $4 --warmup $5 --no-cpu-baseline 2> $O/${T}_$1_$3.err | grep "^{" > $O/${T}_$1_$3.json
  short $O/${T}_$1_$3.json $1
}
echo "== 2. default ($(left) s left)"
for cfg in "cornell_1080p 16 4" "scene_1080p 8 3" "city_4k 6 3"; do
  set -- $cfg
  [ $(left) -gt 20 ] && run default "" $1 $2 $3
done
echo "== done after $(( $(date +%s) - START )) s"
