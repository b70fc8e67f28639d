#!/bin/bash
# scripts/run_config4.sh -- BASELINE config 4 on one GPU: large_scale_05.yaml geometry, ~50 M-point VoI per frame:
# per-kernel CUDA-event times, then one `ncu --set full` capture of K1, K2 and R-GPF class C on it (dram__bytes vs algorithmic bytes)
mkdir -p gpurun_out
python scripts/config4_largescale.py 50000000 5 > gpurun_out/config4_largescale.json 2> gpurun_out/config4.err; tail -c 600 gpurun_out/config4_largescale.json; echo
for k in k1_rpod_bin k2_srt_scatter "k4_rgpf<.int.1024"; do
  name=$(echo "$k" | tr -d '<> ,.' )
  timeout 400 ncu --set full --clock-control none --import-source on --kernel-name-base demangled -k "regex:$k" -s 2 -c 1 -f -o gpurun_out/prof_config4_$name \
      python scripts/config4_largescale.py 50000000 1 > gpurun_out/ncu_config4_$name.log 2>&1
  tail -1 gpurun_out/ncu_config4_$name.log
done
