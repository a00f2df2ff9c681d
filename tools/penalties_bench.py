"""Cost of the penalties and logit bias (csrc/penalty.cuh, DESIGN.md §9e) on the 8B synthetic model.

(a) The job alone: lnb_op_penalize_f32 on 1 and 8 rows of 128 256 logits, histories of T = 32 768 and 131 072 positions,
    window 64, 4 096 and the whole history (rp 1.2, fp 0.3, pp 0.2, 8 biased tokens); the device time of the two penalty
    kernels from torch.profiler (CUDA activities): mean over the launches of a window, median over --reps windows.
(b) Single-sequence decode: lnb_decode_run of 127 steps after the 8-token prompt (graph replays), sampled-only against
    sampled and penalized, STRICT and FAST; both run the kernel chain.  Device time (CUDA events).
(c) FAST lnb_forward_batch with 8 sequences at position 64: sampled-only against sampled and penalized; host clock around
    the synchronised calls.

Every timing is the median of --reps runs after one warm-up run.  Prints the card name and power limit, read in the same
run, then one JSON line per measurement.
Usage: python tools/penalties_bench.py [--legs op,decode,batch] [--reps 5] [--launches 50]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.continuous_bench import card  # noqa: E402

V = 128256
BIAS = {i * 997: -1.5 for i in range(1, 9)}


def op_leg(L, reps, launches, emit):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    for T in (32768, 131072):
        for n in (1, 8):
            x = np.ascontiguousarray(rng.normal(0.0, 3.0, (n, V)), np.float32)
            h = np.ascontiguousarray(rng.integers(0, V, size=(n, T)), np.int32)
            pn = np.full(n, T, np.int32)
            out = np.empty_like(x)
            for window in (64, 4096, 0):
                p = L.model.PenaltyArgs(1.2, 0.3, 0.2, Window=window, CountPrompt=True, LogitBias=BIAS).c(0)
                par = (L._capi.PenaltiesC * n)(*([p] * n))

                def call():
                    L._capi.check(L._capi.lib.lnb_op_penalize_f32(L._capi.ptr(x, L._capi.f32p), n, V, par, L._capi.ptr(h, L._capi.i32p), T,
                                                                  L._capi.ptr(pn, L._capi.i32p), L._capi.ptr(out, L._capi.f32p)))
                call()
                torch.cuda.synchronize()
                means = []
                for _ in range(reps):
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(launches):
                            call()
                        torch.cuda.synchronize()
                    us = sum(e.device_time_total for e in prof.events() if "penalty_count" in e.name or "penalty_apply" in e.name)
                    means.append(us / launches)
                emit(dict(leg="op", rows=n, T=T, window=window or T, launches=launches, us_per_job=statistics.median(means)))


def decode_time(L, gm, acc, pen, reps, steps=127):
    import numpy as np
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=acc)
    try:
        ctx.set_sampling(0, L.model.SamplingArgs(0.8, 40, 0.95, 7))
        if pen is not None:
            ctx.set_penalties(0, pen, 8)
        prompt = np.array(L.synth.PROMPT_8, np.int32)
        first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        ms = []
        for r in range(reps + 1):
            toks, t, graphed = ctx.decode_run(first, 8, steps, use_graph=True)
            if r:
                ms.append(t / steps)
        return statistics.median(ms), graphed
    finally:
        ctx.close()


def decode_leg(L, gm, reps, emit):
    pen = L.model.PenaltyArgs(1.2, 0.3, 0.2, Window=64, LogitBias=BIAS)
    for mode, acc in (("strict", L._capi.LNB_ACC_STRICT), ("fast", L._capi.LNB_ACC_FAST)):
        s, _ = decode_time(L, gm, acc, None, reps)
        p, graphed = decode_time(L, gm, acc, pen, reps)
        emit(dict(leg="decode", mode=mode, sampled_ms_per_step=s, penalized_ms_per_step=p, penalty_cost_ms=p - s, graph=graphed))


def batch_leg(L, gm, reps, emit, steps=32):
    import numpy as np
    pen = L.model.PenaltyArgs(1.2, 0.3, 0.2, Window=64, LogitBias=BIAS)
    res = {}
    for name, p in (("sampled", None), ("penalized", pen)):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST, n_seq=8)
        try:
            for i in range(8):
                ctx.set_sampling(i, L.model.SamplingArgs(0.8, 40, 0.95, 7 + i))
                if p is not None:
                    ctx.set_penalties(i, p, 8)
                ctx.set_active_sequence(i)
                gm.Transformer.forward_argmax(ctx, np.array(L.synth.PROMPT_8, np.int32), 0)
            toks = [int(t) for t in L.synth.PROMPT_8]
            ms = []
            for r in range(reps + 1):
                t0 = time.perf_counter()
                for k in range(steps):
                    ctx.forward_batch(toks, [64 + k] * 8)
                if r:
                    ms.append((time.perf_counter() - t0) * 1e3 / steps)
            res[name] = statistics.median(ms)
        finally:
            ctx.close()
    emit(dict(leg="batch8", mode="fast", sampled_ms_per_step=res["sampled"], penalized_ms_per_step=res["penalized"],
              penalty_cost_ms=res["penalized"] - res["sampled"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="op,decode,batch")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import lnb_b200 as L
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    lines = []

    def emit(d):
        d = dict(d, card=name, power_limit=power)
        lines.append(d)
        print(json.dumps(d), flush=True)
    legs = a.legs.split(",")
    if "op" in legs:
        op_leg(L, a.reps, a.launches, emit)
    if "decode" in legs or "batch" in legs:
        gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
        try:
            if "decode" in legs:
                decode_leg(L, gm, a.reps, emit)
            if "batch" in legs:
                batch_leg(L, gm, a.reps, emit)
        finally:
            gm.Free()
    if a.out:
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
