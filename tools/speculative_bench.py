"""Speculative decoding (lnb_forward_speculative) on the 8B synthetic model at the BASELINE decode workload: the 8-token
prompt, SequenceLength 136 (inside the engines' 145-position limit), one sequence, STRICT and FAST.

(a) ms per verify call of 1..8 rows (one segment: the last token + 0..7 drafts at position 8), next to the plain S = 1
    step (forward_argmax of one token).  Host clock around synchronised calls (every call ends in a stream sync); median of
    --reps windows of --calls calls after a warm-up window.
(b) tokens/s of whole generations (127 tokens after the prompt) through a host loop that verifies k drafts per call, for
    three drafters: perfect (the next k tokens of the plain stream: the upper bound), wrong (tokens the model never
    predicts: the cost of a miss) and prompt lookup (inference.prompt_lookup_drafts: acceptance as it comes out), plus the
    same loop with k = 0 (one-row calls = plain steps).  Prefill excluded; median of --reps runs after one warm-up run.
    Every arm's stream is checked against the plain stream; the prompt-lookup arm also reports its acceptance histogram.
    The synthetic weights have no natural repetition, so prompt-lookup acceptance here says little about real checkpoints.

Prints the card name, power limit and SM clocks (read in the same run), then one JSON line per measurement.
Usage: python tools/speculative_bench.py [--modes strict,fast] [--reps 3] [--calls 20] [--ks 1,3,7] [--out FILE]
"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEQ_LEN = 136


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception:
        import torch
        return dict(card=torch.cuda.get_device_name(0), power_limit="unknown", sm_clock="unknown", sm_clock_max="unknown")


def call_costs(L, gm, acc, reps, calls, emit, mode):
    import numpy as np
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(SEQ_LEN), max_rows=8, acc_mode=acc)
    try:
        prompt = np.array(L.synth.PROMPT_8, np.int32)
        first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        one = np.array([first], np.int32)

        def window(fn):
            t0 = time.perf_counter()
            for _ in range(calls):
                fn()
            return (time.perf_counter() - t0) * 1e3 / calls

        # arm 0 = the plain step, arm r = a verify call of r rows; the arms alternate inside every repetition so that a
        # power-capped card's clock drift falls on all of them alike
        fns = {0: lambda: gm.Transformer.forward_argmax(ctx, one, 8)}
        launches = {}
        for rows in range(1, 9):
            seg = [(0, 8, [first] + [(first + 1 + j) % 128000 for j in range(rows - 1)])]
            fns[rows] = (lambda s: lambda: ctx.forward_speculative(s))(seg)
            l0 = ctx.launch_count()
            fns[rows]()
            launches[rows] = ctx.launch_count() - l0
        for fn in fns.values():
            window(fn)                                   # warm-up: module loads, phase lists, buffers
        ms = {r: [] for r in fns}
        for _ in range(reps):
            for r, fn in fns.items():
                ms[r].append(window(fn))
        plain = statistics.median(ms[0])
        emit(dict(leg="call", mode=mode, rows=0, what="plain S=1 step", ms=plain))
        for rows in range(1, 9):
            m = statistics.median(ms[rows])
            # break-even: emitted tokens per call at which the call pays for itself against plain steps
            emit(dict(leg="call", mode=mode, rows=rows, ms=m, launches=launches[rows], break_even_tokens=m / plain))
    finally:
        ctx.close()


def generate(L, gm, ctx, prompt, k, drafter, plain):
    """one generation after the prompt with k drafts per call; returns (stream, seconds, accepted-draft counts per call)"""
    import numpy as np
    first, _ = gm.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0)
    hist = list(prompt) + [first]
    out, accs = [first], []
    t0 = time.perf_counter()
    while len(hist) < SEQ_LEN:
        pos = len(hist) - 1
        kk = min(k, SEQ_LEN - 2 - pos)
        d = drafter(hist, kk, plain, pos - len(prompt)) if kk > 0 else []
        nxt, na, _ = ctx.forward_speculative([(0, pos, [hist[-1]] + d)])
        a = int(na[0])
        accs.append(a)
        for j in range(a + 1):
            hist.append(int(nxt[j]))
            out.append(int(nxt[j]))
            if len(hist) == SEQ_LEN:
                break
    return out, time.perf_counter() - t0, accs


def arms(L, gm, acc, reps, ks, emit, mode):
    import numpy as np
    V = gm.Transformer.args.VocabSize
    prompt = [int(t) for t in L.synth.PROMPT_8]
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(SEQ_LEN), max_rows=8, acc_mode=acc)
    try:
        plain, _, _ = generate(L, gm, ctx, prompt, 0, None, None)
        assert len(plain) == SEQ_LEN - len(prompt)
        drafters = {
            "perfect": lambda h, k, p, i: p[i + 1:i + 1 + k],
            "wrong": lambda h, k, p, i: [(p[i + 1 + j] + 1) % V if i + 1 + j < len(p) else 0 for j in range(k)],
            "prompt_lookup": lambda h, k, p, i: L.inference.prompt_lookup_drafts(h, k),
        }
        runs = [("plain", 0)] + [(name, k) for name in drafters for k in ks]
        for name, k in runs:
            times, hist = [], collections.Counter()
            for r in range(reps + 1):
                out, sec, accs = generate(L, gm, ctx, prompt, k, drafters.get(name), plain)
                assert out == plain, f"{mode} {name} k={k}: the stream differs from the plain stream"
                if r:
                    times.append(sec)
                    hist.update(accs)
            sec = statistics.median(times)
            n_tok = len(plain) - 1                       # tokens after the prefill's
            calls = sum(hist.values()) / reps
            emit(dict(leg="tokens_per_s", mode=mode, drafter=name, k=k, tokens_per_s=n_tok / sec, calls=calls,
                      tokens_per_call=n_tok / calls, accept_hist={int(a): c // reps for a, c in sorted(hist.items())},
                      stream_equals_plain=True))
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="strict,fast")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--ks", default="1,3,7")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import lnb_b200 as L
    info = card()
    print(f"card: {info['card']}, power limit {info['power_limit']}, SM clock {info['sm_clock']} (max {info['sm_clock_max']})", flush=True)
    lines = []

    def emit(d):
        d = dict(d, **info)
        lines.append(d)
        print(json.dumps(d), flush=True)
    ks = [int(k) for k in a.ks.split(",")]
    gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
    try:
        for mode in a.modes.split(","):
            acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
            call_costs(L, gm, acc, a.reps, a.calls, emit, mode)
            arms(L, gm, acc, a.reps, ks, emit, mode)
    finally:
        gm.Free()
    info_end = card()
    print(f"SM clock at the end: {info_end['sm_clock']}", flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
