"""Cost of regex-constrained generation (csrc/grammar.cuh, DESIGN.md §9g) on the 8B synthetic model.

(a) Mask build: lnb_grammar_create at V = 128 256 (the synthetic tokenizer's vocabulary) for grammars of about 10, 500 and
    4 000 states; the mask kernel's device time (CUDA events, lnb_grammar_info).
(b) The jobs alone: FAST lnb_forward_batch over 1 and 8 constrained sequences; the device time of grammar_apply_kernel
    and grammar_record_kernel from torch.profiler (CUDA activities), mean over the calls of a window.
(c) Single-sequence decode: lnb_decode_run of 127 steps after the 8-token prompt (graph replays), greedy without a
    grammar (STRICT: the decode engine; FAST: its engine or chain) against greedy with one (the kernel chain), STRICT and
    FAST.  Device time (CUDA events).
(d) FAST lnb_forward_batch with 8 sequences at position 64: without and with a grammar on every sequence; host clock
    around the synchronised calls.

Every timing is the median of --reps runs after one warm-up run.  Prints the card name and power limit, read in the same
run, then one JSON line per measurement.
Usage: python tools/grammar_bench.py [--legs build,job,decode,batch] [--reps 3]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.continuous_bench import card  # noqa: E402

V = 128256
BUILD = [("dates", r"\d{4}-\d{2}-\d{2}"), ("suffix8", r"(a|b)*a(a|b){8}"), ("suffix11", r"(a|b)*a(a|b){11}")]
TEXT = r"[a-z ,]{1,400}\."


def build_leg(L, gm, vocab, reps, emit):
    for name, pattern in BUILD:
        ns, info = [], None
        for _ in range(reps + 1):
            g = L.model.Grammar(gm, pattern, vocab)
            info = g.info()
            ns.append(info["build_ns"])
            g.close()
        emit(dict(leg="build", grammar=name, states=info["states"], stuck=info["stuck"], device_bytes=info["bytes"],
                  build_ms=statistics.median(ns[1:]) / 1e6))


def job_leg(L, gm, g, reps, emit, calls=32):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    for n in (1, 8):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST, n_seq=8)
        try:
            for i in range(n):
                ctx.set_grammar(i, g, 64)
            toks = [int(t) for t in L.synth.PROMPT_8][:n]
            ctx.forward_batch(toks, [64] * n)
            torch.cuda.synchronize()
            apply_us, record_us = [], []
            for _ in range(reps):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for k in range(calls):
                        ctx.forward_batch(toks, [64] * n)
                    torch.cuda.synchronize()
                apply_us.append(sum(e.device_time_total for e in prof.events() if "grammar_apply" in e.name) / calls)
                record_us.append(sum(e.device_time_total for e in prof.events() if "grammar_record" in e.name) / calls)
            emit(dict(leg="job", rows=n, apply_us=statistics.median(apply_us), record_us=statistics.median(record_us)))
        finally:
            ctx.close()


def decode_time(L, gm, acc, g, reps, steps=127):
    import numpy as np
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=acc)
    try:
        if g is not None:
            ctx.set_grammar(0, g, 8)
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


def decode_leg(L, gm, g, reps, emit):
    for mode, acc in (("strict", L._capi.LNB_ACC_STRICT), ("fast", L._capi.LNB_ACC_FAST)):
        s, _ = decode_time(L, gm, acc, None, reps)
        c, graphed = decode_time(L, gm, acc, g, reps)
        emit(dict(leg="decode", mode=mode, plain_ms_per_step=s, constrained_ms_per_step=c, grammar_cost_ms=c - s, graph=graphed))


def batch_leg(L, gm, g, reps, emit, steps=32):
    import numpy as np
    res = {}
    for name, gg in (("plain", None), ("constrained", g)):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST, n_seq=8)
        try:
            for i in range(8):
                if gg is not None:
                    ctx.set_grammar(i, gg, 64)
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
    emit(dict(leg="batch8", mode="fast", plain_ms_per_step=res["plain"], constrained_ms_per_step=res["constrained"],
              grammar_cost_ms=res["constrained"] - res["plain"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="build,job,decode,batch")
    ap.add_argument("--reps", type=int, default=3)
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
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "tokenizer.model")
        L._capi.check(L._capi.lib.lnb_vocab_write_synthetic(path.encode(), V - 256))
        vocab = L.vocabulary.Load(path)
        gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
        try:
            if "build" in legs:
                build_leg(L, gm, vocab, a.reps, emit)
            g = L.model.Grammar(gm, TEXT, vocab)
            if "job" in legs:
                job_leg(L, gm, g, a.reps, emit)
            if "decode" in legs:
                decode_leg(L, gm, g, a.reps, emit)
            if "batch" in legs:
                batch_leg(L, gm, g, a.reps, emit)
            g.close()
        finally:
            gm.Free()
    if a.out:
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
