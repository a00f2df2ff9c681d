#!/usr/bin/env bash
# Round-2 GPU call #1: re-verify (incl. the new 8B / graph / handle tests), sanitizer, prepared micro-benchmarks,
# bench.py with the 128-token parity block, fresh launch list.   gpurun --timeout 1500 -- 'bash tools/r2_call1.sh'
set -u
mkdir -p gpurun_out
OUT=gpurun_out/r2_call1.log
{
  echo "== nvidia-smi"; nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,memory.total --format=csv,noheader; nproc
  echo "== pytest -m gpu"; timeout 900 python -m pytest tests -m gpu -q -x --durations=8 2>&1 | tail -25
  echo "== micro: helper-fed STRICT chain (tools/micro/chain_pipe.cu)"
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o /tmp/chain_pipe tools/micro/chain_pipe.cu && timeout 20 /tmp/chain_pipe
  echo "== micro: M=8 STRICT chain, warps per SM (tools/micro/chain_mb8.cu)"
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o /tmp/chain_mb8 tools/micro/chain_mb8.cu && timeout 30 /tmp/chain_mb8
  echo "== kernels alone + graph decode, both modes"; timeout 200 python tools/kbench.py fast,strict 2>&1 | tail -4
  echo "== bench.py"; timeout 500 python bench.py > gpurun_out/r2_bench_n1.json 2> gpurun_out/r2_bench_n1.err; echo "rc=$?"; tail -c 3000 gpurun_out/r2_bench_n1.json; tail -5 gpurun_out/r2_bench_n1.err
} > "$OUT" 2>&1
bash tools/sanitize.sh >> "$OUT" 2>&1
tail -60 "$OUT"
