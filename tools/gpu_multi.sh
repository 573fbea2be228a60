#!/bin/bash
# Multi-GPU check: every sharded entry point under NCCL + the headline bench at N GPUs.
#   N=2 bash tools/gpu_multi.sh
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
N=${N:-2}
echo "== multi_gpu_check N=$N"; timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29511 tools/multi_gpu_check.py > gpurun_out/multi_check_n$N.log 2>&1; grep -E "passed|Error|error|assert" gpurun_out/multi_check_n$N.log | tail -6
if [ "${SKIP_HEADLINE:-0}" != "1" ]; then
echo "== bench N=$N"; timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29512 bench.py --gpus $N --steps 5 --warmup 3 > gpurun_out/bench_n$N.log 2>&1; tail -1 gpurun_out/bench_n$N.log
fi
if [ "${BROADCAST:-0}" = "1" ]; then
echo "== bench N=$N, broadcast staging"; SKDIST_B200_STAGE=broadcast timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29513 bench.py --gpus $N --steps 5 --warmup 3 > gpurun_out/bench_n${N}_bcast.log 2>&1; tail -1 gpurun_out/bench_n${N}_bcast.log | cut -c1-900
fi
for cfg in ${CONFIGS:-}; do
echo "== bench --config $cfg N=$N"; timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 2952$cfg bench.py --config $cfg --gpus $N --steps ${CSTEPS:-2} --warmup 1 > gpurun_out/bench_c${cfg}_n$N.log 2>&1; tail -1 gpurun_out/bench_c${cfg}_n$N.log | cut -c1-1200
done
