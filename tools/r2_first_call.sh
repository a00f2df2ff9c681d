#!/usr/bin/env bash
# One gpurun call that opens round 2: re-verify, run the prepared micro-benchmarks, refresh the evidence.
#   /usr/local/graft/bin/gpurun --timeout 900 -- 'bash tools/r2_first_call.sh'
# Everything lands in gpurun_out/ (merged back by gpurun); each step is bounded by its own timeout.
set -u
mkdir -p gpurun_out
OUT=gpurun_out/r2_first_call.log
{
  echo "== pytest -m gpu"; timeout 300 python -m pytest tests -m gpu -q -x 2>&1 | tail -5
  echo "== micro: helper-fed STRICT chain (tools/micro/chain_pipe.cu)"
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o /tmp/chain_pipe tools/micro/chain_pipe.cu && timeout 20 /tmp/chain_pipe
  echo "== micro: M=8 STRICT chain, warps per SM (tools/micro/chain_mb8.cu)"
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o /tmp/chain_mb8 tools/micro/chain_mb8.cu && timeout 30 /tmp/chain_mb8
  echo "== kernels alone + graph decode, both modes"; timeout 200 python tools/kbench.py fast,strict 2>&1 | tail -4
  echo "== RMSNorm-scale A/B"; for a in chain seg; do LNB_RMS_ALGO=$a timeout 90 python tools/kbench.py strict 2>&1 | tail -1; done
  echo "== batched decode"; timeout 120 python tools/batch_bench.py fast 8 32 2>&1 | tail -1; timeout 120 python tools/batch_bench.py strict 8 8 2>&1 | tail -1
  echo "== bench.py"; timeout 400 python bench.py 2>&1 | tail -1
} > "$OUT" 2>&1
# launch list of the STRICT decode with the current kernels (ncu serialises: compare shares only)
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 700 --csv --log-file gpurun_out/r2_launches_strict.csv \
  python tools/prof_decode.py strict > gpurun_out/r2_prof_strict.log 2>&1
python tools/ncu_summarize.py gpurun_out/r2_launches_strict.csv > gpurun_out/r2_launches_strict.txt 2>&1 || true
tail -40 "$OUT"
