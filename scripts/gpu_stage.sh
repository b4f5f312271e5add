#!/bin/bash
# Staged GPU validation with early abort (a hung kernel must cost seconds of GPU budget, not the whole call).
#   scripts/gpu_stage.sh <tag>
tag=${1:-run}
mkdir -p gpurun_out
log=gpurun_out/${tag}_stage.log
: > "$log"
run() {  # run <seconds> <label> <cmd...>
  local t=$1 label=$2; shift 2
  echo "===== $label" >> "$log"
  timeout "$t" "$@" >> "$log" 2>&1
  local rc=$?
  echo "----- $label rc=$rc" >> "$log"
  return $rc
}
P="python -m pytest -q -m gpu -rs"
run 200 "attention kernels" $P tests/test_kernels_gpu.py -x -k "attention" || { echo "ABORT: attention kernels" >> "$log"; tail -30 "$log"; exit 1; }
run 240 "gemm kernels" $P tests/test_kernels_gpu.py -k "gemm" || { echo "ABORT: gemm" >> "$log"; tail -30 "$log"; exit 1; }
run 300 "other kernels" $P tests/test_kernels_gpu.py -k "not gemm and not attention"
run 420 "model" $P tests/test_model_gpu.py
run 600 "realwidth" $P tests/test_realwidth_gpu.py -s
run 420 "trainer" $P tests/test_trainer_gpu.py
run 420 "decode" $P tests/test_decode_gpu.py
run 200 "preprocess" $P tests/test_preprocess_gpu.py
grep -E "^=====|^-----|passed|failed|error|\[realwidth\]" "$log" | tail -60
