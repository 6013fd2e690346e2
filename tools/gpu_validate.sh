#!/bin/bash
# final validation on ONE H100: GPU test-suite, smoke, one headline line, per-level profile
O=gpurun_out/final; mkdir -p $O
timeout 500 python -m pytest tests -m gpu -q > $O/gpu_pytest.log 2>&1; echo "pytest rc=$?" >> $O/gpu_pytest.log; tail -3 $O/gpu_pytest.log
timeout 100 python __graft_entry__.py smoke > $O/smoke.log 2>&1; tail -1 $O/smoke.log
timeout 300 python bench.py --steps 20 --warmup 5 > $O/bench_kdd_full.json 2> $O/bench_kdd_full.err
timeout 100 python tools/profile_levels.py --workload kdd_full > $O/levels_kdd_full.txt 2>&1; head -20 $O/levels_kdd_full.txt
python - <<'PY'
import json
d=json.loads(open('gpurun_out/final/bench_kdd_full.json').read().strip().splitlines()[-1]); c=d['cpu_baseline']
print('kdd_full ms/step %.2f value %.1f M/s e2e %.2f ms route %.3f labels_equal %s forest_equal %s' % (d['ms_per_step'], d['value']/1e6, d['e2e']['ms_per_step'], d['kernels']['route_hist_level']['ms_per_step'], c['labels_equal'], c['forest_equal']))
PY
