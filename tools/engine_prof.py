"""Where the persistent decode engine spends its time (LNB_ENGINE_PROF=1): cycles of consumer thread 0 per section, mean
and max over the CTAs, for a full decode run and for every projection phase alone.  Usage: python tools/engine_prof.py [fast,strict]"""
import os
import sys

os.environ["LNB_ENGINE_PROF"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import lnb_b200 as L

modes = (sys.argv[1] if len(sys.argv) > 1 else "fast,strict").split(",")
MHZ = 1965.0
m = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B))
names = {0: "wqkv", 1: "wo", 2: "w13", 3: "w2", 4: "lm_head"}


def show(tag, prof, n):
    parts = []
    for k, (mean, mx) in prof.items():
        if mx > 0 and k != "scan_count":
            parts.append(f"{k} {mean / n / MHZ:6.2f}/{mx / n / MHZ:6.2f}")
    print(f"  {tag:>10s} us per unit (mean/max over CTAs): " + " | ".join(parts), flush=True)


for mode in modes:
    acc = L._capi.LNB_ACC_FAST if mode == "fast" else L._capi.LNB_ACC_STRICT
    ctx = L.model.InferenceContext(m.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=acc)
    first, _ = m.Transformer.forward_argmax(ctx, np.array(L.synth.PROMPT_8, np.int32), 0)
    ctx.decode_run(first, 8, 16)
    ctx.engine_profile()
    toks, ms, _ = ctx.decode_run(first, 8, 64)
    print(f"[{mode}] decode {ms / 64:.4f} ms/token = {64e3 / ms:.1f} tok/s", flush=True)
    show("step", ctx.engine_profile(), 64)
    for k, nm in names.items():
        ms_k, nb, nl = ctx.bench_kernel(k, reps=3)
        prof = ctx.engine_profile()
        print(f"[{mode}] {nm}: {ms_k * 1e3:7.2f} us per phase, {nb / ms_k / 1e6:7.1f} GB/s", flush=True)
        show(nm, prof, nl * 4 / 3)      # the warm-up sweep is counted too
    ctx.close()
m.Free()
