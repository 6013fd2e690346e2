#!/bin/bash
# measurement suite on ONE H100: tests, one bench line per BASELINE config, ncu launch list + full captures
O=gpurun_out/final; mkdir -p $O
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active --format=csv > $O/smi.txt 2>&1
timeout 900 python -m pytest tests -m gpu -q > $O/gpu_pytest.log 2>&1; echo "pytest rc=$?" >> $O/gpu_pytest.log; tail -3 $O/gpu_pytest.log
timeout 200 python __graft_entry__.py smoke > $O/smoke.log 2>&1; tail -1 $O/smoke.log
timeout 900 python bench.py --steps 20 --warmup 5 > $O/bench_kdd_full.json 2> $O/bench_kdd_full.err
timeout 900 python bench.py --impl reference --steps 3 --warmup 1 > $O/bench_kdd_full_reference.json 2> $O/bench_kdd_full_reference.err
for wl in kdd10 kdd_script cicids_wed cicids_full cicids_script; do
  timeout 600 python bench.py --workload $wl --steps 10 --warmup 3 > $O/bench_$wl.json 2> $O/bench_$wl.err
done
timeout 600 python bench.py --workload cicids_full --trees 100 --depth 16 --steps 3 --warmup 2 --no-sklearn > $O/bench_cicids_full_deep.json 2> $O/bench_cicids_full_deep.err
timeout 600 python bench.py --workload kdd_full --path dense --steps 10 --warmup 3 --no-cpu-baseline --no-e2e > $O/bench_kdd_full_dense_path.json 2> $O/bench_kdd_full_dense_path.err
timeout 900 python bench.py --workload stream --steps 15 --warmup 2 > $O/bench_stream.json 2> $O/bench_stream.err
timeout 300 python tools/bench_encode.py --iters 20 > $O/bench_encode.txt 2>&1
timeout 200 python tools/profile_levels.py --workload kdd_full > $O/levels_kdd_full.txt 2>&1
timeout 200 python tools/timeline.py --workload kdd_full > $O/timeline_kdd_full.txt 2>&1
timeout 200 python tools/timeline.py --workload kdd_script > $O/timeline_kdd_script.txt 2>&1
# launch list of the bench command (serialised, cold-cache: compare shares)
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 1200 --csv --log-file $O/launches_kdd_full.csv python bench.py --steps 2 --warmup 1 --no-cpu-baseline --no-e2e > $O/launches_kdd_full.log 2>&1
# full ncu captures (route_hist_level per workload, misc kernels, encode, csv) are taken separately (tools/summarize_profiles.py)
timeout 300 python tools/bench_csv.py 1000000 > $O/csv_bench.json 2> $O/csv_bench.err
python - <<'PY'
import json,glob
for f in sorted(glob.glob('gpurun_out/final/bench_*.json')):
    try:
        d=json.loads(open(f).read().strip().splitlines()[-1])
        c=d.get('cpu_baseline') or {}
        print(f.split('/')[-1], 'ms/step %.2f'%d['ms_per_step'], 'value %.2f M/s'%(d['value']/1e6), 'e2e', d.get('e2e') and round(d['e2e'].get('ms_per_step',0),2), 'cpu', c.get('value') and round(c['value']), c.get('labels_equal'), c.get('forest_equal'))
    except Exception as e:
        print(f,'ERR',e, open(f.replace('.json','.err')).read()[-500:])
PY
