#!/bin/bash
# End-of-round evidence run (1 x H100), most important first: GPU test suite, both bench arms, cfg5, training step, the
# launch list of bench.py, ncu --set full of one steady-state step, then a repeat loop of the binding tests and the same
# suite / benches with the exact-mode speculation off (GSR_SPECULATE=0) for comparison.  (The r2c capture in profiles/
# was taken when the experimental cluster scan was still a run-time default: its `off` leg also had GSR_SCAN_CLUSTER=0.)
# Numbers printed under ncu are never quoted.  usage: final_capture.sh [tag]
TAG=${1:-r2c}
O=gpurun_out
mkdir -p $O
t0=$(date +%s)
lap() { echo "[$(( $(date +%s) - t0 )) s] $*"; }
timeout -k 10 300 python -m pytest tests -m gpu -q > $O/${TAG}_pytest_gpu.txt 2>&1; lap "pytest exit $? : $(tail -1 $O/${TAG}_pytest_gpu.txt)"
timeout -k 10 300 python bench.py --steps 20 --warmup 5 > $O/${TAG}_bench_new.json 2> $O/${TAG}_bench_new.err; lap "bench new $?"
timeout -k 10 300 python bench.py --impl reference --steps 20 --warmup 5 > $O/${TAG}_bench_reference.json 2> $O/${TAG}_bench_reference.err; lap "bench reference $?"
timeout -k 10 200 ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file $O/${TAG}_launches.csv python bench.py --steps 4 --warmup 3 --no-cpu-baseline --dropin 0 > $O/${TAG}_launches.log 2>&1; lap "launch list $?"
timeout -k 10 200 python bench.py --config cfg5 --steps 20 --warmup 5 --no-cpu-baseline > $O/${TAG}_bench_cfg5.json 2> $O/${TAG}_bench_cfg5.err; lap "cfg5 $?"
timeout -k 10 200 python bench.py --train 1 --steps 20 --warmup 6 > $O/${TAG}_train_1gpu.json 2> $O/${TAG}_train_1gpu.err; lap "train $?"
timeout -k 10 200 python bench.py --steps 40 --warmup 5 --no-cpu-baseline > $O/${TAG}_bench_new_40.json 2> $O/${TAG}_bench_new_40.err; lap "bench 40 $?"
# the first twelve binding tests over and over in fresh processes (a one-off mismatch of the sparse fused/un-fused test
# was seen once in the first process of a call: the test now reports which render does not reproduce)
for i in 1 2 3 4 5 6; do
  timeout -k 10 100 python -m pytest tests/test_gpu_api.py -x -q -k "not speculation and not tile_order and not graphed and not pipelined and not concurrent" > $O/${TAG}_loop_$i.txt 2>&1
  echo "loop $i: $(tail -1 $O/${TAG}_loop_$i.txt)"; grep -h "AssertionError: fused" $O/${TAG}_loop_$i.txt | head -2
done; lap "loop"
timeout -k 10 400 ncu --set full --clock-control none --import-source on -k regex:k_ -s 24 -c 12 -f -o $O/${TAG}_prof python tools/profile_one.py cfg3 4 > $O/${TAG}_prof.log 2>&1; lap "ncu full $?"
export GSR_SPECULATE=0
timeout -k 10 300 python -m pytest tests -m gpu -q > $O/${TAG}_off_pytest_gpu.txt 2>&1; lap "pytest (switches off) exit $? : $(tail -1 $O/${TAG}_off_pytest_gpu.txt)"
timeout -k 10 200 python bench.py --steps 20 --warmup 5 --no-cpu-baseline > $O/${TAG}_off_bench_new.json 2> $O/${TAG}_off_bench_new.err; lap "bench new (off) $?"
timeout -k 10 200 python bench.py --config cfg5 --steps 20 --warmup 5 --no-cpu-baseline > $O/${TAG}_off_bench_cfg5.json 2> $O/${TAG}_off_bench_cfg5.err; lap "cfg5 (off) $?"
python - <<PY
import json
for n in ("bench_new", "bench_reference", "bench_cfg5", "train_1gpu", "bench_new_40", "off_bench_new", "off_bench_cfg5"):
    try:
        d = json.loads(open("$O/${TAG}_%s.json" % n).read().strip().splitlines()[-1])
        print(n, round(d["value"], 1), "e2e", round(d["e2e"]["value"], 1), "dropin", round((d.get("dropin") or {}).get("value", 0), 1))
    except Exception as e:
        print(n, "ERR", e)
PY
