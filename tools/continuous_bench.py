"""Ragged forwards and continuous batching on the 8B synthetic model, STRICT and FAST.

(a) Admission: 8 prompts of 8, 128 and 512 tokens -- serial lnb_session_set_active_sequence + lnb_forward prefills against
    ONE lnb_forward_ragged call.  ms per admission of all 8 prompts, host clock around synchronised calls (every call
    returns after its stream synchronise), median of --reps runs after one warm-up run.
(b) Mixed workload: --prompts prompts with lengths spread over 8..512 at SequenceLength --seq-len, so generation lengths
    differ too.  GenerateTokensContinuous(slots=8) against GenerateTokensBatch in waves of 8.  Every prompt is submitted at
    t = 0: time to first token of a prompt is the host time from the start of the run to the yield of its first token.
    Aggregate tokens/s = generated tokens / wall time of the run.  In STRICT both arms must produce the same tokens.
    --sweep runs the continuous arm again, FAST only, with other step_tokens values.

Prints the card name and power limit, read in the same run, then one JSON line per measurement.
Usage: python tools/continuous_bench.py [--modes strict,fast] [--legs admission,mixed] [--seq-len 1024] [--prompts 32]
       [--step-tokens N] [--sweep 32,128,256] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def admission(L, gm, mode, plen, reps, emit):
    import numpy as np
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(plen)
    prompts = [rng.integers(0, 128000, size=plen).astype(np.int32) for _ in range(8)]
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(plen + 16), max_rows=8 * plen, acc_mode=acc, n_seq=8)
    try:
        def serial():
            out = []
            for b, p in enumerate(prompts):
                ctx.set_active_sequence(b)
                out.append(gm.Transformer.forward_argmax(ctx, p, 0)[0])
            return out

        def ragged():
            return list(ctx.forward_ragged([(b, 0, p) for b, p in enumerate(prompts)])[0])

        res = {}
        for name, fn in (("serial", serial), ("ragged", ragged)):
            toks = fn()   # warm-up
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            res[name] = (sorted(ts)[len(ts) // 2], toks)
        same = [int(t) for t in res["serial"][1]] == [int(t) for t in res["ragged"][1]]
        emit(dict(leg="admission", mode=mode, prompt_len=plen, prompts=8, serial_ms=round(res["serial"][0], 2),
                  ragged_ms=round(res["ragged"][0], 2), speedup=round(res["serial"][0] / res["ragged"][0], 2), same_tokens=same))
    finally:
        ctx.close()


def run_arm(gen, n):
    t0 = time.perf_counter()
    first = [None] * n
    toks = [[] for _ in range(n)]
    for i, _, tok in gen:
        if first[i] is None:
            first[i] = time.perf_counter() - t0
        toks[i].append(int(tok))
    wall = time.perf_counter() - t0
    return wall, first, toks


def mixed(L, gm, mode, seq_len, n_prompts, step_tokens, emit, only_continuous=False):
    import numpy as np
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(32)
    lens = np.linspace(8, 512, n_prompts).astype(int)
    rng.shuffle(lens)
    prompts = [rng.integers(0, 128000, size=int(n)).astype(np.int32).tolist() for n in lens]
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq_len), acc_mode=acc, max_rows=512)

    def stats(arm, wall, first, toks, extra):
        total = sum(len(t) for t in toks)
        ttft = np.array(first) * 1e3
        emit(dict(leg="mixed", mode=mode, arm=arm, prompts=n_prompts, seq_len=seq_len, tokens=total, wall_s=round(wall, 2),
                  tokens_per_s=round(total / wall, 1), ttft_mean_ms=round(float(ttft.mean()), 1),
                  ttft_p90_ms=round(float(np.percentile(ttft, 90)), 1), **extra))

    # warm-up: one short continuous run (builds the batch engine, allocates the ragged buffers)
    list(eng.GenerateTokensContinuous(prompts[:2], slots=8, step_tokens=step_tokens))
    wall, first, toks_c = run_arm(eng.GenerateTokensContinuous(prompts, slots=8, step_tokens=step_tokens), n_prompts)
    stats("continuous", wall, first, toks_c, dict(slots=8, step_tokens=step_tokens))
    if only_continuous:
        return
    def waves():
        for w in range(0, n_prompts, 8):
            for i, st, tok in eng.GenerateTokensBatch(prompts[w:w + 8]):
                yield w + i, st, tok
    wall, first, toks_w = run_arm(waves(), n_prompts)
    stats("waves_of_8", wall, first, toks_w, dict(same_tokens_as_continuous=toks_w == toks_c))
    if mode == "strict" and toks_w != toks_c:
        raise SystemExit("STRICT: continuous batching and waves of 8 generated different tokens")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="strict,fast")
    ap.add_argument("--legs", default="admission,mixed")
    ap.add_argument("--seq-len", type=int, default=1024)
    ap.add_argument("--prompts", type=int, default=32)
    ap.add_argument("--step-tokens", type=int, default=None, help="default: inference.DEFAULT_STEP_TOKENS")
    ap.add_argument("--sweep", default="", help="extra FAST step_tokens values for the continuous arm")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    a = ap.parse_args()
    import lnb_b200 as L

    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    lines = []

    def emit(d):
        d = dict(d, card=name, power_limit=power)
        lines.append(d)
        print(json.dumps(d), flush=True)

    step_tokens = a.step_tokens or L.inference.DEFAULT_STEP_TOKENS
    gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
    try:
        for mode in a.modes.split(","):
            if "admission" in a.legs:
                for plen in (8, 128, 512):
                    admission(L, gm, mode, plen, a.reps, emit)
            if "mixed" in a.legs:
                mixed(L, gm, mode, a.seq_len, a.prompts, step_tokens, emit)
        for st in [int(x) for x in a.sweep.split(",") if x]:
            mixed(L, gm, "fast", a.seq_len, a.prompts, st, emit, only_continuous=True)
    finally:
        gm.Free()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
