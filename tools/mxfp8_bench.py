"""MXFP8 (and MXFP4) against bf16 weights (DESIGN.md §9h, §9i) on the synthetic 8B model, all held on one GPU.

The models of --formats (default bf16,mxfp8; the first is the reference) are built from the same synthetic weights, and
every measurement alternates them, --rounds times each:
  decode      lnb_decode_run of 127 steps after the 8-token prompt, FAST and STRICT, device time (CUDA events); each
              model on its default route (bf16 STRICT: the decode engine; MXFP8, MXFP4: the kernel chain)
  batch8      FAST lnb_forward_batch over 8 sequences, 64 steps, host clock around the synchronised calls
  prefill     one FAST forward of S = 2048 tokens at position 0 (tensor-core route), host clock
  kernels     every projection alone (lnb_session_bench_kernel, FAST kernel chain): ms per launch and GB/s of the bytes the
              weight format streams
  error       each model against the reference over 128 teacher-forced tokens (the 8-token prompt and the bf16 model's
              120 greedy tokens, one FAST forward): logits max-abs difference and argmax agreement.  Reported, not asserted.
              Synthetic weights say nothing about the quantization error of a trained checkpoint.
Prints the card name and power limit, read in the same run, then one JSON line per measurement.  With two formats the
ratio and overlap keys compare the second with the first; with more, ratio_median_<fmt> compares each with the first and
overlap_<a>_<b> says whether two formats' samples overlap.
Usage: python tools/mxfp8_bench.py [--rounds 3] [--formats bf16,mxfp8,mxfp4] [--legs decode,batch8,prefill,kernels,error]
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

KINDS = ["wqkv", "wo", "w1|w3", "w2", "output"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--legs", default="decode,batch8,prefill,kernels,error")
    ap.add_argument("--formats", default="bf16,mxfp8")
    a = ap.parse_args()
    fmts = a.formats.split(",")
    ref = fmts[0]
    legs = set(a.legs.split(","))
    import numpy as np
    import torch
    import lnb_b200 as L

    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    emit = lambda d: print(json.dumps(d), flush=True)   # noqa: E731
    models = {}
    for fmt in fmts:
        t0 = time.perf_counter()
        models[fmt] = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), weight_format=fmt)
        emit(dict(leg="load", weights=fmt, s=round(time.perf_counter() - t0, 1), **models[fmt].Transformer.weight_info()))
    prompt = np.array(L.synth.PROMPT_8, np.int32)
    FAST, STRICT = L._capi.LNB_ACC_FAST, L._capi.LNB_ACC_STRICT

    def ctx_of(fmt, seq, acc, **kw):
        return L.model.InferenceContext(models[fmt].Transformer, L.model.InferenceArgs(seq), acc_mode=acc, **kw)

    def alternate(measure):
        vals = {fmt: [] for fmt in fmts}
        for _ in range(a.rounds):
            for fmt in fmts:
                vals[fmt].append(measure(fmt))
        return vals

    def report(leg, unit, vals, **extra):
        out = dict(leg=leg, unit=unit, **extra)
        for fmt, v in vals.items():
            out[fmt] = [round(x, 2) for x in v]
            out[fmt + "_median"] = round(statistics.median(v), 2)
        overlap = lambda x, y: not (min(vals[y]) > max(vals[x]) or max(vals[y]) < min(vals[x]))   # noqa: E731
        if len(fmts) == 2:
            out["ratio_median"] = round(out[fmts[1] + "_median"] / out[ref + "_median"], 3)
            out["overlap"] = overlap(ref, fmts[1])
        else:
            for i, x in enumerate(fmts):
                if i:
                    out["ratio_median_" + x] = round(out[x + "_median"] / out[ref + "_median"], 3)
                for y in fmts[i + 1:]:
                    out[f"overlap_{x}_{y}"] = overlap(x, y)
        emit(out)

    if "decode" in legs:
        for mode, acc in (("fast", FAST), ("strict", STRICT)):
            ctxs = {fmt: ctx_of(fmt, 136, acc) for fmt in models}

            def decode(fmt):
                ctx = ctxs[fmt]
                first, _ = models[fmt].Transformer.forward_argmax(ctx, prompt, 0)
                toks, ms, _ = ctx.decode_run(first, len(prompt), 127, use_graph=True)
                return 127 / (ms / 1e3)
            for fmt in models:
                decode(fmt)   # warm-up: graph capture
            report("decode", "tokens/s", alternate(decode), mode=mode,
                   route={fmt: ("engine" if ctxs[fmt].uses_engine() else "kernel chain") for fmt in models})
            for c in ctxs.values():
                c.close()

    if "batch8" in legs:
        ctxs = {fmt: ctx_of(fmt, 200, FAST, n_seq=8) for fmt in models}

        def batch8(fmt, steps=64):
            ctx, tf = ctxs[fmt], models[fmt].Transformer
            last = []
            for b in range(8):
                ctx.set_active_sequence(b)
                last.append(tf.forward_argmax(ctx, np.array(L.synth.batch_prompt(b), np.int32), 0)[0])
            pos = [len(L.synth.batch_prompt(b)) for b in range(8)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(steps):
                nxt, _ = ctx.forward_batch(last, [p + j for p in pos])
                last = list(nxt)
            return 8 * steps / (time.perf_counter() - t0)
        for fmt in models:
            batch8(fmt, 4)
        report("batch8", "tokens/s (aggregate)", alternate(batch8), mode="fast")
        for c in ctxs.values():
            c.close()

    if "prefill" in legs:
        S = 2048
        toks = np.random.default_rng(0).integers(0, 128000, S).astype(np.int32)
        ctxs = {fmt: ctx_of(fmt, S + 1, FAST, max_rows=S) for fmt in models}

        def prefill(fmt):
            t0 = time.perf_counter()
            models[fmt].Transformer.forward_argmax(ctxs[fmt], toks, 0)
            return (time.perf_counter() - t0) * 1e3
        for fmt in models:
            prefill(fmt)
        report("prefill", "ms (S = 2048)", alternate(prefill), mode="fast")
        for c in ctxs.values():
            c.close()

    if "kernels" in legs:
        ctxs = {}
        for fmt in models:
            os.environ["LNB_ENGINE"] = "0"
            ctxs[fmt] = ctx_of(fmt, 136, FAST)
            ctxs[fmt].uses_engine()
            os.environ.pop("LNB_ENGINE")
        for kind, kname in enumerate(KINDS):
            res = {}

            def kern(fmt):
                ms, nb, _ = ctxs[fmt].bench_kernel(kind, 3)
                res[fmt] = nb
                return ms * 1e3
            vals = alternate(kern)
            report("kernel", "us per launch", vals, projection=kname, mode="fast",
                   gbps={fmt: round(res[fmt] / (statistics.median(vals[fmt]) * 1e-6) / 1e9, 1) for fmt in models},
                   bytes={fmt: res[fmt] for fmt in models})
        for c in ctxs.values():
            c.close()

    if "error" in legs:
        n = 128
        c = ctx_of(ref, n + 8, FAST)
        first, _ = models[ref].Transformer.forward_argmax(c, prompt, 0)
        gen, _, _ = c.decode_run(first, len(prompt), n - len(prompt) - 1, use_graph=False)
        c.close()
        seq = np.concatenate([prompt, [first], gen]).astype(np.int32)[:n]
        lg = {}
        for fmt in models:
            c = ctx_of(fmt, n + 1, FAST, max_rows=n)
            lg[fmt] = models[fmt].Transformer.forward_argmax(c, seq, 0, want_logits="all")[1]
            c.close()
        for fmt in fmts[1:]:
            d = np.abs(lg[ref] - lg[fmt])
            emit(dict(leg="error", **({} if len(fmts) == 2 else {"weights": fmt}), tokens=n, logits_max_abs=float(d.max()),
                      logits_mean_abs=float(d.mean()), argmax_agreement=float((lg[ref].argmax(1) == lg[fmt].argmax(1)).mean()),
                      **{ref + "_logits_max_abs": float(np.abs(lg[ref]).max())}))

    for m in models.values():
        m.Free()


if __name__ == "__main__":
    main()
