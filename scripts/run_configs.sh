#!/bin/bash
# scripts/run_configs.sh -- the BASELINE.json configs that are not the driver's default workload, on one GPU:
#   config 4  large_scale_05.yaml geometry, ~50 M-point VoI: per-kernel CUDA-event times + ncu --set full (dram__bytes vs algorithmic bytes)
#   config 5  40 x 360 bins, 262144-point scans, 2 M-point resident map (per-rank share of the frame-sharded job)
#   dense     the seq-05 twin at the size SURVEY 8 estimates for the real sequence
mkdir -p gpurun_out
bash scripts/run_config4.sh
python bench.py --config synthetic40x360 --frames 32 --steps 8 --warmup 3 --lanes 3 --no-offline-pass --no-sweep > gpurun_out/config5_n1.json 2> gpurun_out/config5_n1.err
echo "config5 rc=$?"; tail -2 gpurun_out/config5_n1.err; python -c "
import json; d=json.load(open('gpurun_out/config5_n1.json')); print('config5 N=1 value=%.0f e2e=%.0f ms/step=%.3f parity=%s' % (d['value'], d['e2e']['value'], d['ms_per_step'], d['parity_spot_check']), d['quality_final_map'], {k: v['avg_launch_ms'] for k, v in d['roofline']['by_kernel'].items()})"
python bench.py --config dense --steps 20 --warmup 3 --lanes 3 --no-offline-pass --no-sweep > gpurun_out/bench_dense.json 2> gpurun_out/bench_dense.err
echo "dense rc=$?"; python -c "
import json; d=json.load(open('gpurun_out/bench_dense.json')); print('dense value=%.0f e2e=%.0f ms/step=%.3f parity=%s' % (d['value'], d['e2e']['value'], d['ms_per_step'], d['parity_spot_check']), d['config']['map_points'], d['config']['mean_map_voi_points'], d['config']['mean_query_points'], d['quality_final_map'])"
