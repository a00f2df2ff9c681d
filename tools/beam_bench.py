"""Cost of forking and permuting sequences (csrc/seqcopy.cuh) and of a beam-search step (DESIGN.md §9f) on the 8B synthetic
model.

(a) The copy alone: lnb_session_copy_sequences at the 8B cache layout (32 layers, K and V, 2 KB rows), B = 4 and 8 sequences
    in one worst-case permutation (every beam takes another's rows), ranges of 128 and 2048 positions.  Time of --launches
    calls ended by one synchronise, and the effective GB/s (bytes read + written, from the shapes); beside it a
    device-to-device cudaMemcpyAsync (torch copy_) of the same bytes.
(b) The beam step: ms per step of GenerateBeams (B = 2, 4, 8; 8-token prompt, 128 generated tokens, no stop ids, so every
    step runs) against lnb_forward_batch of B sequences at the same positions, STRICT and FAST; and the split of a step:
    the batch forward with logprobs on, the B record reads, the copy.

Every timing is the median of --reps runs after one warm-up run.  Prints the card name and power limit, read in the same
run, then one JSON line per measurement.
Usage: python tools/beam_bench.py [--legs copy,step] [--reps 3] [--launches 50]
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


def copy_leg(L, gm, reps, launches, emit):
    import torch
    a = gm.Transformer.args
    row = a.N_KVHeads * a.HeadDim * 2
    for B in (4, 8):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(4096), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST, n_seq=B)
        try:
            src = [(i + 1) % B for i in range(B)]   # a B-cycle: every sequence is a source and a destination
            for n_pos in (128, 2048):
                moved = 2 * a.N_Layers * B * n_pos * row   # bytes copied; read + written is twice that
                ctx.copy_sequences(src, list(range(B)), 0, n_pos)
                L._capi.check(L._capi.lib.lnb_session_sync(ctx.h))
                ts = []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    for _ in range(launches):
                        ctx.copy_sequences(src, list(range(B)), 0, n_pos)
                    L._capi.check(L._capi.lib.lnb_session_sync(ctx.h))
                    ts.append((time.perf_counter() - t0) / launches)
                t = statistics.median(ts)
                x = torch.empty(moved, dtype=torch.uint8, device="cuda")
                y = torch.empty_like(x)
                y.copy_(x)
                torch.cuda.synchronize()
                tm = []
                for _ in range(reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(launches):
                        y.copy_(x)
                    e1.record()
                    torch.cuda.synchronize()
                    tm.append(e0.elapsed_time(e1) / 1e3 / launches)
                m = statistics.median(tm)
                del x, y
                emit(dict(leg="copy", B=B, positions=n_pos, mb_moved=moved / 1e6, us=t * 1e6, gbps=2 * moved / t / 1e9,
                          memcpy_us=m * 1e6, memcpy_gbps=2 * moved / m / 1e9))
        finally:
            ctx.close()


def step_leg(L, gm, reps, emit):
    import numpy as np
    prompt = list(L.synth.PROMPT_8)
    n_gen = 128
    seq_len = len(prompt) + n_gen
    gm.Vocabulary = L.model.Vocabulary(StopTokenIds=())
    for mode, acc in (("strict", L._capi.LNB_ACC_STRICT), ("fast", L._capi.LNB_ACC_FAST)):
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq_len), acc_mode=acc)
        for B in (2, 4, 8):
            beams = L.inference.BeamSearchArgs(B, 1.0, False)
            eng.GenerateBeams(prompt, beams)   # warm-up
            per = []
            for _ in range(reps):
                st = []
                eng.GenerateBeams(prompt, beams, step_times=st)
                per.append(statistics.median(st[1:]) * 1e3)   # the steps after the prefill, ms
            # the parts of a step at the same shapes: batch forward (logprobs on / off), B record reads, the copy
            ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq_len), max_rows=8, acc_mode=acc, n_seq=B)
            try:
                first, _ = gm.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0)
                ctx.copy_sequences([0] * (B - 1), list(range(1, B)), 0, len(prompt))
                toks = [first] * B

                def timed(fn, n=32):
                    fn(0)
                    L._capi.check(L._capi.lib.lnb_session_sync(ctx.h))
                    out = []
                    for _ in range(reps):
                        t0 = time.perf_counter()
                        for k in range(n):
                            fn(k)
                        L._capi.check(L._capi.lib.lnb_session_sync(ctx.h))
                        out.append((time.perf_counter() - t0) / n)
                    return statistics.median(out) * 1e3
                pos = len(prompt) + n_gen // 2
                plain = timed(lambda k: ctx.forward_batch(toks, [pos] * B))
                for b in range(B):
                    ctx.set_logprobs(b, 2 * B)
                with_lp = timed(lambda k: ctx.forward_batch(toks, [pos] * B))
                reads = timed(lambda k: [ctx.read_logprobs(b, pos + 1, 1) for b in range(B)])
                src = [(i + 1) % B for i in range(B)]
                copy = timed(lambda k: ctx.copy_sequences(src, list(range(B)), len(prompt), len(prompt) + n_gen // 2))
            finally:
                ctx.close()
            emit(dict(leg="step", mode=mode, B=B, beam_step_ms=statistics.median(per), batch_step_ms=plain,
                      batch_step_logprobs_ms=with_lp, record_reads_ms=reads, copy_64_rows_ms=copy))
    gm.Vocabulary = L.model.Vocabulary()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="copy,step")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()
    import lnb_b200 as L
    name, power = card()
    print(json.dumps(dict(card=name, power_limit=power)), flush=True)

    def emit(d):
        print(json.dumps(d), flush=True)
    gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
    try:
        legs = args.legs.split(",")
        if "copy" in legs:
            copy_leg(L, gm, args.reps, args.launches, emit)
        if "step" in legs:
            step_leg(L, gm, args.reps, emit)
    finally:
        gm.Free()


if __name__ == "__main__":
    main()
