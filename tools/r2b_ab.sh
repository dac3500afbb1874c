#!/bin/bash
# NOTE: since the end of round 2 the cluster tile scan is compiled only into the `cluster_scan` variant (python tools/build_variants.py
# cluster_scan; run with GSR_LIB=gaustudio_b200/variants/libgsr_cluster_scan.so): with the default library GSR_SCAN_CLUSTER is ignored.
# One-call A/B of the late round-2 changes (1 x H100): GPU tests first, then bench.py under the knobs
#   GSR_SCAN_CLUSTER (8-CTA cluster scan vs the single-CTA scan), GSR_SPECULATE (exact-mode speculation: drop-in leg),
#   GSR_CARVEOUT (uniform shared-memory carveout), GSR_SKIP_CROWDED (cost of the two empty crowded-tier launches).
mkdir -p gpurun_out
date +%s > gpurun_out/r2b_t0
timeout -k 10 420 python -m pytest tests -m gpu -x -q > gpurun_out/r2b_pytest.txt 2>&1
echo "pytest exit $?" | tee -a gpurun_out/r2b_pytest.txt
tail -3 gpurun_out/r2b_pytest.txt
run() {  # name, env..., -- bench args
  name=$1; shift
  envs=(); while [ "$1" != "--" ]; do envs+=("$1"); shift; done; shift
  s=$(date +%s)
  env "${envs[@]}" timeout -k 10 200 python bench.py --no-cpu-baseline "$@" > gpurun_out/r2b_$name.json 2> gpurun_out/r2b_$name.err
  echo "$name: exit $? in $(( $(date +%s) - s )) s"
}
B="--steps 60 --warmup 5"
run A1 X=1 -- $B
run scan0_1 GSR_SCAN_CLUSTER=0 -- $B
run spec0 GSR_SPECULATE=0 -- $B
run carve100 GSR_CARVEOUT=100 -- $B --dropin 0
run skipcrowded GSR_SKIP_CROWDED=1 -- $B --dropin 0
run A2 X=1 -- $B --dropin 0
run scan0_2 GSR_SCAN_CLUSTER=0 -- $B --dropin 0
run carve50 GSR_CARVEOUT=50 -- $B --dropin 0
run cfg5_A X=1 -- --config cfg5 --steps 20 --warmup 5
run cfg5_scan0 GSR_SCAN_CLUSTER=0 -- --config cfg5 --steps 20 --warmup 5
python - <<'PY'
import json, glob
for f in sorted(glob.glob("gpurun_out/r2b_*.json")):
    try:
        d = json.loads(open(f).read().strip().splitlines()[-1])
        k = d["stages"]["_kernels_ms"]
        dr = d.get("dropin") or {}
        print(f.split("r2b_")[1][:-5].ljust(12), "value %.1f e2e %.1f" % (d["value"], d["e2e"]["value"]),
              "| scan %.4f scatter %.4f sort %.4f fwd %.4f" % (k["tile_scan"], k["scatter"], k["tile_sort"], k["render_fwd"]),
              "| dropin %s e2e %s host %s" % (round(dr.get("value", 0), 1), round((dr.get("e2e") or {}).get("value", 0), 1), dr.get("host_enqueue_ms_per_step")))
    except Exception as e:
        print(f, "ERR", e)
PY
echo "total $(( $(date +%s) - $(cat gpurun_out/r2b_t0) )) s"
