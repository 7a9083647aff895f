#!/bin/bash
# N-GPU bench under torch.distributed.run on one node with N GPUs:
#   scripts/multi_gpu_bench.sh N TAG [extra bench flags]
# prints value / train / strip of the JSON line.
N=$1; TAG=$2; shift; shift
O=gpurun_out
export NCCL_DEBUG=WARN
timeout 1500 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29541 bench.py --gpus $N --steps 5 --warmup 3 "$@" > $O/${TAG}_bench_n$N.json 2> $O/${TAG}_bench_n$N.err; echo "bench rc=$?"; tail -c 500 $O/${TAG}_bench_n$N.err
python -c "
import json
ls=[l for l in open('$O/${TAG}_bench_n$N.json') if l.startswith('{')]
if not ls: raise SystemExit('no bench line')
d=json.loads(ls[-1])
print('N=$N value', d['value'], 'ms', d['ms_per_step'], 'e2e', d['e2e']['value']); print('train', d['train']); print('strip', d['strip'])"
