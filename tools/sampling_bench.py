"""Cost of seeded sampling (csrc/sample.cuh) on the 8B synthetic model.

(a) The sampler kernel alone: lnb_op_sample_f32 on 1 and 8 rows of 128 256 logits, K 40 / P 0.95 and K 0 / P 1; the
    device time of the two sampler kernels from torch.profiler (CUDA activities): mean over --launches launches per
    window, median over --reps windows.
(b) Single-sequence decode: lnb_decode_run of 127 steps after the 8-token prompt, greedy against sampled, both on the
    kernel chain (LNB_ENGINE=0 for both arms), STRICT and FAST: the difference is the sampler.  Device time (CUDA events).
(c) Leaving the engine: STRICT greedy on the persistent decode engine against STRICT sampled (kernel chain).
(d) Batch of 8: FAST lnb_forward_batch steps, greedy against sampled; host clock around synchronised calls.

Every timing is the median of --reps runs after one warm-up run.  Prints the card name and power limit, read in the same
run, then one JSON line per measurement.
Usage: python tools/sampling_bench.py [--legs op,decode,engine,batch] [--reps 5] [--launches 200]
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

SAMPLED = (0.8, 40, 0.95, 2024)


def op_leg(L, reps, launches, emit):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    V = 128256
    rng = np.random.default_rng(0)
    rows = rng.normal(0.0, 3.0, (8, V)).astype(np.float32)
    for name, (K, P) in (("k40_p0.95", (40, 0.95)), ("full_vocab", (0, 1.0))):
        for n in (1, 8):
            p = (L._capi.SamplingC * n)(*[L._capi.SamplingC(0.8, K, P, 7 + i) for i in range(n)])
            pn = np.arange(1, n + 1, dtype=np.int32)
            out = np.empty(n, np.int32)
            x = np.ascontiguousarray(rows[:n])

            def call():
                L._capi.check(L._capi.lib.lnb_op_sample_f32(L._capi.ptr(x, L._capi.f32p), n, V, p, L._capi.ptr(pn, L._capi.i32p),
                                                            L._capi.ptr(out, L._capi.i32p)))
            call()
            torch.cuda.synchronize()
            means = []
            for _ in range(reps):   # one profiler window per rep: the mean over its launches of both sampler kernels' time
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(launches):
                        call()
                    torch.cuda.synchronize()
                us = sum(e.device_time_total for e in prof.events() if "sample_" in e.name and "kernel" in e.name
                         and "set_params" not in e.name)
                means.append(us / launches)
            emit(dict(leg="op", case=name, rows=n, launches=launches, us_per_launch=statistics.median(means)))


def decode_time(L, gm, acc, sampled, reps, steps=127):
    import numpy as np
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=acc)
    try:
        if sampled:
            ctx.set_sampling(0, L.model.SamplingArgs(*SAMPLED))
        prompt = np.array(L.synth.PROMPT_8, np.int32)
        first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        ms = []
        for r in range(reps + 1):
            _, t, graphed = ctx.decode_run(first, 8, steps, use_graph=True)
            if r:
                ms.append(t / steps)
        return statistics.median(ms), graphed, ctx.uses_engine()
    finally:
        ctx.close()


def decode_leg(L, gm, reps, emit):
    saved = os.environ.get("LNB_ENGINE")
    os.environ["LNB_ENGINE"] = "0"
    try:
        for mode, acc in (("strict", L._capi.LNB_ACC_STRICT), ("fast", L._capi.LNB_ACC_FAST)):
            g, _, _ = decode_time(L, gm, acc, False, reps)
            s, graphed, _ = decode_time(L, gm, acc, True, reps)
            emit(dict(leg="decode_chain", mode=mode, greedy_ms_per_step=g, sampled_ms_per_step=s, sampler_ms=s - g,
                      sampler_share=(s - g) / g, graph=graphed))
    finally:
        if saved is None:
            os.environ.pop("LNB_ENGINE", None)
        else:
            os.environ["LNB_ENGINE"] = saved


def engine_leg(L, gm, reps, emit):
    g, _, eng = decode_time(L, gm, L._capi.LNB_ACC_STRICT, False, reps)
    s, graphed, _ = decode_time(L, gm, L._capi.LNB_ACC_STRICT, True, reps)
    emit(dict(leg="leave_engine", mode="strict", greedy_engine=eng, greedy_ms_per_step=g, sampled_chain_ms_per_step=s,
              ratio=s / g, graph=graphed))


def batch_leg(L, gm, reps, emit, steps=32):
    import numpy as np
    res = {}
    for sampled in (False, True):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(256), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST, n_seq=8)
        try:
            if sampled:
                for k in range(8):
                    ctx.set_sampling(k, L.model.SamplingArgs(SAMPLED[0], SAMPLED[1], SAMPLED[2], SAMPLED[3] + k))
            prompt = np.array(L.synth.PROMPT_8, np.int32)
            toks = []
            for k in range(8):
                ctx.set_active_sequence(k)
                toks.append(gm.Transformer.forward_argmax(ctx, prompt, 0)[0])
            ms = []
            for r in range(reps + 1):
                cur, pos = list(toks), [8] * 8
                t0 = time.perf_counter()
                for _ in range(steps):
                    nxt, _ = ctx.forward_batch(cur, pos)
                    cur = [int(t) for t in nxt]
                    pos = [p + 1 for p in pos]
                if r:
                    ms.append((time.perf_counter() - t0) * 1e3 / steps)
            res[sampled] = statistics.median(ms)
        finally:
            ctx.close()
    emit(dict(leg="batch8", mode="fast", greedy_ms_per_step=res[False], sampled_ms_per_step=res[True],
              sampler_ms=res[True] - res[False], sampler_share=(res[True] - res[False]) / res[False]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="op,decode,engine,batch")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200)
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
    if any(x in legs for x in ("decode", "engine", "batch")):
        gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
        try:
            if "decode" in legs:
                decode_leg(L, gm, a.reps, emit)
            if "engine" in legs:
                engine_leg(L, gm, a.reps, emit)
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
