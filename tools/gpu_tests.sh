#!/bin/bash
# Run every -m gpu test file in its own process (a CUDA fault in one file must not poison the others).
# usage (on the GPU box): bash tools/gpu_tests.sh [pytest args]
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,driver_version,memory.total --format=csv > gpurun_out/gpu_info.txt 2>&1
rc=0
for f in tests/test_gpu_*.py; do
  name=$(basename $f .py)
  timeout 900 python -m pytest $f -q -m gpu -s "$@" > gpurun_out/$name.log 2>&1
  r=$?
  echo "== $f exit $r"; tail -n 40 gpurun_out/$name.log
  [ $r -eq 0 ] || rc=1
done
exit $rc
