#!/bin/bash
# ncu captures of the bench command (summaries via scripts/summarize_ncu.py):
#   launch list of the bench command, launch list of one training step, --set full of the dominant kernels.
O=gpurun_out
TAG=${1:-rX}
Q="--no-cpu-baseline --no-parity --no-train --no-other-configs"
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file $O/${TAG}_launches.csv python bench.py --steps 2 --warmup 1 $Q > $O/${TAG}_ncu_bench.log 2>&1
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv --log-file $O/${TAG}_train_launches.csv python scripts/train_probe.py darcy241 > $O/${TAG}_train_probe.log 2>&1
for K in k_apply_tc k_dy k_dh k_gemm_tn; do
  timeout 600 ncu --set full --clock-control none --import-source on --profile-from-start off -k regex:$K -c 1 -f -o $O/prof_${TAG}_$K python scripts/train_probe.py darcy241 > $O/${TAG}_ncu_$K.log 2>&1; echo "ncu $K rc=$?"
done
