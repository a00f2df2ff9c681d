"""Cost of token log-probabilities (csrc/logprob.cuh, DESIGN.md §9d) on the 8B synthetic model.

(a) The kernels alone: lnb_op_logprobs_f32 on 1, 8 and 2048 rows of 128 256 logits, top_n 0 and 20; the device time of
    the two logprob kernels from torch.profiler (CUDA activities): mean over the launches of a window, median over --reps
    windows.
(b) Single-sequence decode: lnb_decode_run of 127 steps after the 8-token prompt (graph replays), without and with
    logprobs (top_n 5), STRICT and FAST.  Without logprobs STRICT runs the persistent engine and FAST the kernel chain (the
    defaults); with logprobs both run the kernel chain.  Device time (CUDA events).
(c) Scoring 2048 tokens: lnb_score (2049 tokens, one forward of 2048 rows with the LM head over all rows, then the logprob
    job over 2048 rows) against a plain S = 2048 prefill (lnb_forward, last-row LM head), FAST and STRICT; host clock
    around the synchronised calls.

Every timing is the median of --reps runs after one warm-up run.  Prints the card name and power limit, read in the same
run, then one JSON line per measurement.
Usage: python tools/logprobs_bench.py [--legs op,decode,score] [--reps 5] [--launches 50]
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


def op_leg(L, reps, launches, emit):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    rows = rng.normal(0.0, 3.0, (2048, V)).astype(np.float32)
    for n in (1, 8, 2048):
        x = np.ascontiguousarray(rows[:n])
        t = np.ascontiguousarray(rng.integers(0, V, size=n), np.int32)
        k = launches if n < 2048 else max(2, launches // 10)   # each call also copies the rows to the device
        for top_n in (0, 20):
            out = (L._capi.LogprobC * n)()

            def call():
                L._capi.check(L._capi.lib.lnb_op_logprobs_f32(L._capi.ptr(x, L._capi.f32p), n, V, L._capi.ptr(t, L._capi.i32p), top_n, out))
            call()
            torch.cuda.synchronize()
            means = []
            for _ in range(reps):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(k):
                        call()
                    torch.cuda.synchronize()
                us = sum(e.device_time_total for e in prof.events() if "logprob_" in e.name
                         and "set_top_n" not in e.name)
                means.append(us / k)
            us = statistics.median(means)
            emit(dict(leg="op", rows=n, top_n=top_n, launches=k, us_per_job=us,
                      gb_per_s=2 * n * V * 4 / (us * 1e-6) / 1e9))   # two passes over the rows


def decode_time(L, gm, acc, top_n, reps, steps=127):
    import numpy as np
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=acc)
    try:
        if top_n is not None:
            ctx.set_logprobs(0, top_n)
        prompt = np.array(L.synth.PROMPT_8, np.int32)
        first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        ms = []
        for r in range(reps + 1):
            toks, t, graphed = ctx.decode_run(first, 8, steps, use_graph=True)
            if r:
                ms.append(t / steps)
        return statistics.median(ms), graphed, ctx.uses_engine(), [int(x) for x in toks]
    finally:
        ctx.close()


def decode_leg(L, gm, reps, emit):
    for mode, acc in (("strict", L._capi.LNB_ACC_STRICT), ("fast", L._capi.LNB_ACC_FAST)):
        g, _, eng, tg = decode_time(L, gm, acc, None, reps)
        s, graphed, _, ts = decode_time(L, gm, acc, 5, reps)
        emit(dict(leg="decode", mode=mode, plain_ms_per_step=g, plain_engine=eng, logprobs_ms_per_step=s,
                  logprobs_cost_ms=s - g, ratio=s / g, graph=graphed, same_tokens=tg == ts))


def score_leg(L, gm, reps, emit):
    import numpy as np
    rng = np.random.default_rng(1)
    toks = rng.integers(0, V, size=2049).astype(np.int32)
    for mode, acc in (("fast", L._capi.LNB_ACC_FAST), ("strict", L._capi.LNB_ACC_STRICT)):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(2064), max_rows=2048, acc_mode=acc)
        try:
            ctx.set_logprobs(0, 20)
            res = {}
            for name, call in (("prefill", lambda: gm.Transformer.forward_argmax(ctx, toks[:-1], 0)),
                               ("score", lambda: L._capi.check(L._capi.lib.lnb_score(ctx.h, L._capi.ptr(toks, L._capi.i32p), 2049, 0)))):
                ms = []
                for r in range(reps + 1):
                    t0 = time.perf_counter()
                    call()
                    if r:
                        ms.append((time.perf_counter() - t0) * 1e3)
                res[name] = statistics.median(ms)
            emit(dict(leg="score2048", mode=mode, prefill_ms=res["prefill"], score_ms=res["score"],
                      extra_ms=res["score"] - res["prefill"], extra_share=(res["score"] - res["prefill"]) / res["prefill"]))
        finally:
            ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="op,decode,score")
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
    if "decode" in legs or "score" in legs:
        gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
        try:
            if "decode" in legs:
                decode_leg(L, gm, a.reps, emit)
            if "score" in legs:
                score_leg(L, gm, a.reps, emit)
        finally:
            gm.Free()
    if a.out:
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
