"""bf16 against MXFP8 KV caches on the 8B synthetic model (DESIGN.md §9j), one H100, card name and power limit read in the
same run.  Every comparison alternates the two formats, median of 3:
  - single-sequence lnb_decode_run tokens/s (graph, greedy) at T = 4 096, 32 768 and 131 048, FAST and STRICT, with bf16
    and (--weights) MXFP8 weights.  Decode is timed at position T over the zero-filled caches: a step's work (keys read,
    chains run) depends on T, not on the cache contents (tools/long_context_bench.py);
  - FAST 8-sequence batched steps at SequenceLength 8 192 (positions 8 000);
  - the 2 048-token FAST prefill (bf16: tensor-core attention; MXFP8: the streamed kernels);
  - the largest n_seq of 131 072 positions each format can create next to the weights.
Usage: python tools/kv_cache_bench.py [--weights bf16,mxfp8] [--steps 16] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.long_context_bench import card  # noqa: E402

FMTS = ("bf16", "mxfp8")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--weights", default="bf16,mxfp8")
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--ts", default="4096,32768,131048")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import lnb_b200 as L
    C = L._capi

    name, power = card()
    lines = []

    def emit(d):
        d = dict(d, card=name, power_limit=power)
        print(json.dumps(d), flush=True)
        lines.append(d)

    args = dict(L.synth.LLAMA31_8B, max_seq_len=131072)
    for wf in a.weights.split(","):
        gm = L.model.LoadSyntheticModel(args, weight_format=wf)
        tf = gm.Transformer
        for T in [int(t) for t in a.ts.split(",")]:
            for mode in ("fast", "strict"):
                acc = C.LNB_ACC_FAST if mode == "fast" else C.LNB_ACC_STRICT
                steps = a.steps if mode == "fast" or T < 100000 else max(4, a.steps // 4)
                ctxs = {f: L.model.InferenceContext(tf, L.model.InferenceArgs(T + steps + 8), acc_mode=acc, max_rows=8, kv_format=f)
                        for f in FMTS}
                ms = {f: [] for f in FMTS}
                toks = {}
                for f in FMTS:
                    ctxs[f].decode_run(1, T, steps, use_graph=True)          # warm-up (captures the graph)
                for _ in range(3):
                    for f in FMTS:
                        t, m, _ = ctxs[f].decode_run(1, T, steps, use_graph=True)
                        ms[f].append(m / steps)
                        toks[f] = t.tolist()
                for f in FMTS:
                    med = statistics.median(ms[f])
                    emit(dict(workload="decode_run", weights=wf, kv=f, acc=mode, T=T, ms_per_token=round(med, 4),
                              tokens_per_s=round(1000.0 / med, 2), runs_ms=[round(x, 4) for x in ms[f]],
                              cache_bytes=ctxs[f].kv_info()[1], decode_path="kernel chain" if f == "mxfp8" or not ctxs[f].uses_engine() else "engine"))
                    ctxs[f].close()
        if wf != "bf16":
            gm.Free()
            continue
        # FAST batched steps, 8 sequences at SequenceLength 8192
        ctxs = {f: L.model.InferenceContext(tf, L.model.InferenceArgs(8192), acc_mode=C.LNB_ACC_FAST, n_seq=8, max_rows=8, kv_format=f)
                for f in FMTS}
        ms = {f: [] for f in FMTS}
        toks8 = np.arange(1, 9, dtype=np.int32)
        for f in FMTS:
            ctxs[f].forward_batch(toks8, np.full(8, 7990, np.int32))
        for _ in range(3):
            for f in FMTS:
                C.check(C.lib.lnb_session_sync(ctxs[f].h))
                t0 = time.perf_counter()
                for i in range(a.steps):
                    ctxs[f].forward_batch(toks8, np.full(8, 8000 + i, np.int32))
                C.check(C.lib.lnb_session_sync(ctxs[f].h))
                ms[f].append((time.perf_counter() - t0) * 1000.0 / a.steps)
        for f in FMTS:
            med = statistics.median(ms[f])
            emit(dict(workload="batch8_step", weights="bf16", kv=f, acc="fast", seq_len=8192, pos=8000, ms_per_step=round(med, 4),
                      tokens_per_s=round(8000.0 / med, 1), runs_ms=[round(x, 4) for x in ms[f]]))
            ctxs[f].close()
        # the 2048-token FAST prefill
        ctxs = {f: L.model.InferenceContext(tf, L.model.InferenceArgs(2048), acc_mode=C.LNB_ACC_FAST, max_rows=2048, kv_format=f)
                for f in FMTS}
        prompt = L.ml.Tensor(np.random.default_rng(1).integers(0, args["vocab_size"], 2048).astype(np.int32), L.ml.DT_INT32)
        ms = {f: [] for f in FMTS}
        for f in FMTS:
            tf.forward_argmax(ctxs[f], prompt.RawData, 0)
        for _ in range(3):
            for f in FMTS:
                C.check(C.lib.lnb_session_sync(ctxs[f].h))
                t0 = time.perf_counter()
                tf.forward_argmax(ctxs[f], prompt.RawData, 0)
                C.check(C.lib.lnb_session_sync(ctxs[f].h))
                ms[f].append((time.perf_counter() - t0) * 1000.0)
        for f in FMTS:
            emit(dict(workload="prefill_2048", weights="bf16", kv=f, acc="fast", ms=round(statistics.median(ms[f]), 3),
                      runs_ms=[round(x, 3) for x in ms[f]]))
            ctxs[f].close()
        # capacity: the largest n_seq of 131072 positions each format creates next to the bf16 weights
        for f in FMTS:
            best = 0
            for n in range(8, 0, -1):
                try:
                    c = L.model.InferenceContext(tf, L.model.InferenceArgs(131072), acc_mode=C.LNB_ACC_FAST, n_seq=n,
                                                 max_rows=max(8, n), kv_format=f)
                    c.close()
                    best = n
                    break
                except C.LnbError:
                    continue
            emit(dict(workload="capacity", weights="bf16", kv=f, seq_len=131072, max_n_seq=best,
                      free_bytes_after_weights=torch.cuda.mem_get_info()[0]))
        gm.Free()
    if a.out:
        with open(a.out, "w") as fh:
            for d in lines:
                fh.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
