#!/bin/bash
# Runs the GPU parity suite in separate processes (a hung kernel in one group must not take the others down).
# usage: scripts/gpu_tests.sh [outdir]
OUT=${1:-gpurun_out}
mkdir -p $OUT
nvidia-smi --query-gpu=name,driver_version,memory.total --format=csv > $OUT/gpu.txt 2>&1
run() { # name, timeout, args...
  local name=$1; local to=$2; shift 2
  echo "=== $name" | tee -a $OUT/summary.txt
  timeout -k 10 $to python -m pytest "$@" -q -rP -m gpu -x --no-header -p no:cacheprovider > $OUT/$name.log 2>&1
  echo "exit $?: $(tail -1 $OUT/$name.log)" | tee -a $OUT/summary.txt
}
runall() { # same but without -x
  local name=$1; local to=$2; shift 2
  echo "=== $name" | tee -a $OUT/summary.txt
  timeout -k 10 $to python -m pytest "$@" -q -rP -m gpu --no-header -p no:cacheprovider > $OUT/$name.log 2>&1
  echo "exit $?: $(tail -1 $OUT/$name.log)" | tee -a $OUT/summary.txt
}
: > $OUT/summary.txt
runall kernels 900 tests/test_gpu_kernels.py
runall row_kernels 600 tests/test_gpu_row_kernels.py
runall attention 600 tests/test_gpu_attention.py
runall gemm 900 tests/test_gpu_gemm.py          # about 150 s on an H100, of which about 80 s is its profiling child run (timeout 480 s)
runall gemm_fragment_epilogue 600 tests/test_gpu_gemm_fragment_epilogue.py
runall models 900 tests/test_gpu_models.py
runall aten_rng 600 tests/test_gpu_aten_rng.py
runall full_config 900 tests/test_gpu_full_config.py
runall fused_tail 600 tests/test_gpu_fused_tail.py
runall t5 900 tests/test_gpu_t5.py
runall inpaint 900 tests/test_gpu_inpaint.py
runall edit 900 tests/test_gpu_edit.py
runall maskgit_loss 900 tests/test_gpu_maskgit_loss.py
runall fp8 1200 tests/test_gpu_fp8.py
runall vae_fp8 1200 tests/test_gpu_vae_fp8.py
runall vae_tile_epilogues 900 tests/test_gpu_vae_tile_epilogues.py
runall launch_trace 600 tests/test_gpu_launch_trace.py
runall batch_settings 900 tests/test_gpu_batch_settings.py
runall dim_head128 1200 tests/test_gpu_dim_head128.py
cat $OUT/summary.txt
