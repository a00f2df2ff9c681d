"""Tree speculative decoding (lnb_forward_speculative_tree) against chain speculation and plain decoding on the 8B synthetic
model, one sequence, STRICT and FAST.

Workloads: prompts built deterministically to hold repeated n-grams with divergent continuations (a few "phrases" that
share their opening tokens and then part ways, interleaved by a seeded generator), plus one prompt of distinct tokens with
no repeat at all (where a tree cannot help).  127 tokens are generated after each prompt.  Arms: the plain loop, and
GenerateTokens with SpeculativeArgs(7, Branches=B) for B = 1 (chains), 2 and 4.  The arms alternate inside every
repetition; median of --reps runs after one warm-up run; prefill excluded (step_times after the first entry).  Every arm's
stream is checked against the plain stream.

Reports, per (mode, prompt, arm): accepted tokens per call (emitted tokens / verify calls) and ms per emitted token, plus the
card name, power limit and SM clocks read in the same run.  One JSON line per measurement.
Usage: python tools/spec_tree_bench.py [--modes strict,fast] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEN = 127


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=20).stdout.strip()
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)


def prompts(vocab):
    """name -> token list.  "divergent": 4 phrases of 6 tokens, phrases 0/1 and 2/3 sharing their first 3 tokens, laid out
    24 times in a seeded order (so every 3-gram opening has two continuations, the most recent one right only part of the
    time).  "norepeat": 96 distinct tokens."""
    import numpy as np
    rng = np.random.default_rng(2026)
    base = [int(t) for t in rng.choice(vocab, size=18, replace=False)]
    phrases = [base[0:3] + base[3:6], base[0:3] + base[6:9], base[9:12] + base[12:15], base[9:12] + base[15:18]]
    order = rng.integers(0, 4, size=16)
    div = [t for k in order for t in phrases[int(k)]]
    return {"divergent": div, "norepeat": [int(t) for t in rng.choice(vocab, size=96, replace=False)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="strict,fast")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import lnb_b200 as L
    info = card()
    print(json.dumps(info), flush=True)
    gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)

    class NoStop:
        StopTokenIds = (10**9,)
        PadId = gm.Vocabulary.PadId
    gm.Vocabulary = NoStop
    lines = []
    arms = [("plain", None)] + [(f"branches{b}", L.inference.SpeculativeArgs(7, Branches=b)) for b in (1, 2, 4)]
    for mode in a.modes.split(","):
        acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
        for pname, prompt in prompts(L.synth.LLAMA31_8B["vocab_size"]).items():
            seq = len(prompt) + GEN + 1
            eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=acc, max_rows=len(prompt))
            res = {name: [] for name, _ in arms}
            ref = None
            for rep in range(a.reps + 1):
                for name, spec in arms:
                    times, stats = [], []
                    toks = [t for _, t in eng.GenerateTokens(prompt, step_times=times, speculative=spec, spec_stats=stats)]
                    if ref is None:
                        ref = toks
                    assert toks == ref, (mode, pname, name)
                    calls = len(times) - 1
                    emitted = len(toks) - 1
                    if rep:
                        res[name].append((sum(times[1:]) * 1e3 / emitted, emitted / calls))
            for name, _ in arms:
                ms = statistics.median(x for x, _ in res[name])
                per_call = statistics.median(y for _, y in res[name])
                row = dict(mode=mode, prompt=pname, arm=name, ms_per_token=round(ms, 3), tokens_per_call=round(per_call, 3),
                           generated=GEN, reps=a.reps, **info)
                print(json.dumps(row), flush=True)
                lines.append(row)
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    gm.Free()


if __name__ == "__main__":
    main()
