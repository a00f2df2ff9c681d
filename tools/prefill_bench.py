"""Config 3 of BASELINE.json: prefill of S=2048 tokens on one H100 (tensor-core GEMM path, LNB_ACC_FAST).
Prints prompt-processing tokens/s and the tensor-core throughput of the projections.
Usage: python tools/prefill_bench.py [S] [reps]"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import lnb_b200 as L

S = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
args = dict(L.synth.LLAMA31_8B)
m = L.model.LoadSyntheticModel(args)
ctx = L.model.InferenceContext(m.Transformer, L.model.InferenceArgs(S + 1), max_rows=S, acc_mode=L._capi.LNB_ACC_FAST)
rng = np.random.default_rng(0)
toks = rng.integers(0, 128000, size=S).astype(np.int32)
times = []
for r in range(reps + 1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    nxt, _ = m.Transformer.forward_argmax(ctx, toks, 0)      # synchronous: H2D tokens, forward, D2H token
    times.append(time.perf_counter() - t0)
best = min(times[1:])
lin_flops = 2 * 6_979_321_856 * S          # all projections incl. LM head for ONE row (last row only)
lin_flops -= 2 * 128256 * 4096 * (S - 1)   # the generate loop only needs the last row of the head
print(f"prefill S={S}: {best * 1e3:.2f} ms -> {S / best:.0f} tokens/s; projections {lin_flops / best / 1e12:.1f} TFLOP/s "
      f"(incl. SDPA + elementwise time); next token {nxt}; launches {ctx.launch_count()}")
ctx.close(); m.Free()
