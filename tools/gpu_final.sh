#!/bin/bash
# Final evidence of the round in one GPU session (tag r2d): full GPU suite, both bench arms, per-op table, launch
# lists, one --set full capture of the merge tile kernel.
o=gpurun_out; mkdir -p $o; tag=r2d
timeout 300 python bench.py --impl reference --steps 5 --warmup 2 > $o/${tag}_bench_ref.json 2> $o/${tag}_bench_ref.err
timeout 400 python bench.py > $o/${tag}_bench.json 2> $o/${tag}_bench.err; echo "bench rc=$?"
timeout 200 python bench.py --no-resident --no-e2e --no-ops --steps 50 --warmup 5 > $o/${tag}_bench_noresident.json 2>/dev/null
timeout 600 python tools/bench_ops.py --out $o/${tag}_ops.json > $o/${tag}_ops.log 2>&1
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file $o/${tag}_bench_launches.csv \
    python bench.py --steps 2 --warmup 3 --no-e2e --no-ops --no-dense > $o/${tag}_ncu_bench.log 2>&1
timeout 200 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:"mmerge3|mplan2|msample|merge_kernel|mscan|mcompact" -c 60 --csv --log-file $o/${tag}_merge_launches.csv python tools/bench_merge.py --reps 2 > $o/${tag}_ncu_merge.log 2>&1
timeout 300 ncu --set full --import-source on --clock-control none -k regex:mmerge3 -s 1 -c 1 -o $o/${tag}_mmerge3 -f python tools/bench_merge.py --reps 1 > $o/${tag}_ncu_merge2.log 2>&1
timeout 120 python tools/bench_merge.py --dense > $o/${tag}_merge_cases.jsonl 2>/dev/null; cat $o/${tag}_merge_cases.jsonl
timeout 900 python -m pytest tests -m gpu -q --durations=5 > $o/${tag}_tests.log 2>&1; tail -2 $o/${tag}_tests.log
python - <<'PY'
import json
t="gpurun_out/r2d"
d=json.loads(open(t+"_bench.json").read().strip().splitlines()[-1])
r=json.loads(open(t+"_bench_ref.json").read().strip().splitlines()[-1])
n=json.loads(open(t+"_bench_noresident.json").read().strip().splitlines()[-1])
print("value %.4g ms %.4f frac %.3f exact %s | no-resident ms %.4f frac %.3f" % (d["value"], d["ms_per_step"], d["roofline"]["frac"], d["bit_exact"], n["ms_per_step"], n["roofline"]["frac"]))
print("dense", d["dense_variant"]["ms_per_step"], d["dense_variant"]["roofline_frac"])
for k in ("e2e","e2e_cached","e2e_raw_u64"): print(k, round(d[k]["ms_per_step"],3), "%.4g"%d[k]["value"], d[k].get("pcie_GBps"), d[k]["bit_exact"])
print("ref", r["value"], "ratio e2e", d["e2e"]["value"]/r["value"], "ratio value", d["value"]/r["value"])
for o in d["ops"]: print(o["op"], "|", o["ms"], "|", o["frac_of_hbm_peak"], o["check"])
PY
