"""What the packed copies of w1|w3 and the LM head (csrc/wpack.cuh) buy the STRICT decode engine on the synthetic 8B model:
the packed-unit share and bytes per pass of each packed matrix, the extra HBM the copies hold, and the time and bandwidth of
every projection phase alone (lnb_session_bench_kernel: bytes are what the phase reads, packed units included) next to the
STRICT decode rate.  Run it in the parent tree for the before column (it then skips the packing report), and
tools/engine_prof.py strict for the per-section cycles.  Usage: python tools/wpack_bench.py"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import lnb_b200 as L

args = dict(L.synth.LLAMA31_8B)
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip(), flush=True)
m = L.model.LoadSyntheticModel(args)
lib = L._capi.lib
if hasattr(lib, "lnb_model_wpack_read"):
    extra = 0
    for layer, nm in [(0, "w1|w3 layer 0"), (args["n_layers"] - 1, f"w1|w3 layer {args['n_layers'] - 1}"), (-1, "LM head")]:
        info = np.zeros(5, np.int64)
        if L._capi.check(lib.lnb_model_wpack_read(m.Transformer.h, layer, None, None, None, info.ctypes.data_as(L._capi.i64p))) != 1:
            print("no packed copy:", lib.lnb_last_error().decode())
            break
        kt, n_units, packed, rb, N = (int(v) for v in info)
        bf = N * args["dim"] * 2
        print(f"{nm:>16s}: kt {kt}, {packed}/{n_units} units packed ({100.0 * packed / n_units:.2f} %), "
              f"{rb / 1e6:.1f} MB per pass against {bf / 1e6:.1f} MB bf16 ({100.0 * (rb / bf - 1):+.1f} %)", flush=True)
    ffn2 = 2 * args["ffn_dim"] * args["dim"]
    extra = (args["n_layers"] * ffn2 + args["vocab_size"] * args["dim"]) * 12 // 8
    print(f"packed copies: {extra / 1e9:.2f} GB of HBM beside the bf16 weights", flush=True)

ctx = L.model.InferenceContext(m.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_STRICT)
first, _ = m.Transformer.forward_argmax(ctx, np.array(L.synth.PROMPT_8, np.int32), 0)
ctx.decode_run(first, 8, 16)
rates = []
for _ in range(3):
    _, ms, _ = ctx.decode_run(first, 8, 127)
    rates.append(127e3 / ms)
print(f"STRICT decode: {' '.join(f'{r:.1f}' for r in rates)} tokens/s", flush=True)
for k, nm in {0: "wq|wk|wv", 1: "wo", 2: "w1|w3", 3: "w2", 4: "LM head"}.items():
    ms_k, nb, _ = ctx.bench_kernel(k, reps=5)
    print(f"  {nm:>9s}: {ms_k * 1e3:7.2f} us per phase, {nb / 1e6:8.1f} MB read, {nb / ms_k / 1e6:7.1f} GB/s", flush=True)
ctx.close()
m.Free()
