#!/bin/bash
# scripts/gpu_session.sh -- one GPU session (gpurun, 1 GPU): parity tests, smoke, both bench arms, launch lists and one
# `ncu --set full` capture per kernel of the node-mode step and of the sequential updater's per-node kernels, phase taps.
mkdir -p gpurun_out
timeout 600 python -m pytest tests -m gpu -x -q 2>&1 | tail -3
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -2
timeout 600 python bench.py > gpurun_out/bench_n1.json 2> gpurun_out/bench_n1.err; tail -c 300 gpurun_out/bench_n1.err
timeout 600 python bench.py --impl reference --steps 3 --warmup 1 > gpurun_out/bench_reference_arm.json 2>> gpurun_out/bench_n1.err
timeout 300 python scripts/k4_profile.py > gpurun_out/k4_phase_profile.txt 2>&1
timeout 300 python scripts/updater_profile.py > gpurun_out/updater_fused_phases.txt 2>&1
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none --kernel-name-base demangled -c 600 --csv --log-file gpurun_out/launches_updater.csv \
    python scripts/updater_profile.py > /dev/null 2>&1
bash scripts/ncu_nodes.sh seq05 20
for k in k_node_fused k4b_voxelize; do
  timeout 300 ncu --set full --clock-control none --import-source on --kernel-name-base demangled -k "regex:$k" -s 2 -c 1 -f -o gpurun_out/prof_updater_$k \
      python scripts/updater_profile.py > gpurun_out/ncu_updater_$k.log 2>&1
  tail -1 gpurun_out/ncu_updater_$k.log
done
