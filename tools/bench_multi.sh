#!/bin/bash
# usage: tools/bench_multi.sh <gpus> [out-dir]  -- bench.py under torchrun, one rank per GPU
N=$1
O=${2:-bench_out}
mkdir -p $O
set -x
nvidia-smi -L | wc -l
BENCH_PER_STEP=1 timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29714 bench.py --gpus $N --steps 5 --warmup 3 > $O/g_bench_n$N.json 2> $O/g_bench_n$N.err; echo "rc=$?" >> $O/g_bench_n$N.err
grep "per-step\|rc=\|Error\|error" $O/g_bench_n$N.err | tail -n 12
python - <<PY
import json
try:
    d=json.loads(open('$O/g_bench_n$N.json').read().strip().splitlines()[-1])
    print('N=$N ms/step', round(d['ms_per_step'],2), 'value', round(d['value']/1e9,3), 'kernel ms', round(d['kernel_ms_per_step'],2), 'gap', round(d['host_gap_ms_per_step'],2), 'e2e ms', round(d['e2e']['ms_per_step'],1), 'e2e value', round(d['e2e']['value']/1e9,3))
except Exception as e: print('ERR', e)
PY
