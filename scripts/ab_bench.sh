#!/bin/bash
# Same-box A/B of library knobs (csrc/options.h) on the bench workload, forward only:
#   scripts/ab_bench.sh TAG "base" "NNCONV_SCATTER_MODE=0" "NNCONV_L2_PERSIST=48 NNCONV_GEMM_B_POLICY=0" ...
# Every variant is one `bench.py --steps 5 --warmup 3` run (no parity / train / CPU legs); one line per variant in
# $AB_OUT/TAG_ab.log (default: a new temporary directory).  Compare variants only inside one run on one GPU.
O=${AB_OUT:-$(mktemp -d)}
mkdir -p "$O"
TAG=$1; shift
Q="--no-cpu-baseline --no-parity --no-train --no-other-configs"
rm -f $O/${TAG}_ab.log
for V in "$@"; do
  if [ "$V" = base ]; then E=""; else E="$V"; fi
  env $E timeout 300 python bench.py --steps 5 --warmup 3 $Q 2>/dev/null | python -c "
import json,sys
d=json.loads(sys.stdin.read()); k=d['kernel_ms_per_step']
print('AB %-50s ms/step %.2f apply %.2f l1 %.2f hidden %.2f clk %s' % ('$V', d['ms_per_step'], k['apply_fused']['ms'], k['edge_layer1']['ms'], k['hidden_gemm']['ms'], d['clocks']['sm_mhz']))" >> $O/${TAG}_ab.log 2>&1
done
cat $O/${TAG}_ab.log
