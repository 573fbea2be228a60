#!/bin/bash
# Validates a tree on an H100: GPU test suite, smoke, bench.
#   bash tools/gpu_check.sh
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
timeout 900 python -m pytest tests -m gpu -q > gpurun_out/pytest_gpu.log 2>&1; tail -4 gpurun_out/pytest_gpu.log
timeout 300 python __graft_entry__.py --smoke 2>&1 | tail -1
timeout 900 python bench.py > gpurun_out/bench.log 2>&1; tail -1 gpurun_out/bench.log | cut -c1-400
