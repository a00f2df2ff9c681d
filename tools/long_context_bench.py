"""Long-context decode on the 8B synthetic model (max_seq_len 131072): single-sequence decode at context T in STRICT and
FAST, and batched decode at SequenceLength 2048 / 8192 (n = 8) and 32768 (n = 3).

Caches are filled by chunked prefill of seeded random ids.  Single sequences are timed with device-resident lnb_decode_run
(CUDA events around the run, after a warm-up run at the same positions); batches with host-driven lnb_forward_batch steps,
as bench.py --config batch8 does (wall clock around the loop, after warm-up steps).  One session per mode is prefilled
step by step to 32K, 64K and 128K and measured at each length; the 16K leg uses its own session, whose SequenceLength
still fits the shared-memory kernels, for contrast.

Bytes per step are counted as 15 009 857 536 (weights) + 131 072 * T per sequence (K and V of every layer), and the
achieved GB/s is that count over the whole step time -- a whole-step figure, not the attention kernel's bandwidth.

Usage: python tools/long_context_bench.py [--budget S] [--legs single,batch] [--modes strict,fast] [--out FILE]
Each leg stops prefilling when its time budget (seconds) runs out (STRICT prefill to 128K takes far longer than FAST) and says
so: `cache_filled_to` is then below T and the cache rows above it keep their zero fill.  Decode is still timed at position T,
because the work of a decode step (keys read, chains run) depends on T and not on the cache contents.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WEIGHT_BYTES = 15_009_857_536
KV_BYTES_PER_POS = 131_072
HBM_PEAK = 3.35e12   # H100 SXM data sheet
FULL = 131072


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget", type=float, default=300.0, help="seconds of prefill per leg")
    ap.add_argument("--legs", default="single,batch")
    ap.add_argument("--modes", default="strict,fast")
    ap.add_argument("--steps", type=int, default=16, help="timed decode steps per workload")
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    a = ap.parse_args()
    import numpy as np
    import lnb_b200 as L

    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    args = dict(L.synth.LLAMA31_8B, max_seq_len=FULL)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    tf = gm.Transformer
    rng = np.random.default_rng(2024)
    ids = rng.integers(0, args["vocab_size"], size=FULL).astype(np.int32)
    rows = []

    def emit(**kw):
        kw.update(card=name, power_limit=power)
        rows.append(kw)
        print(json.dumps(kw), flush=True)

    def prefill(ctx, start, end, chunk, deadline):
        """chunked prefill of ids[start:end]; returns (seconds, reached position, greedy id of the last row)"""
        t0 = time.perf_counter()
        pos, nxt = start, None
        while pos < end:
            if time.perf_counter() > deadline:
                break
            n = min(chunk, end - pos)
            nxt, _ = tf.forward_argmax(ctx, ids[pos:pos + n], pos)
            pos += n
        return time.perf_counter() - t0, pos, nxt

    modes = [m for m in a.modes.split(",") if m]
    acc = {"strict": L._capi.LNB_ACC_STRICT, "fast": L._capi.LNB_ACC_FAST}
    chunk = {"strict": 2048, "fast": 8192}

    if "single" in a.legs:
        for mode in modes:
            legs = [(16384, 16384 + 64), (32768, FULL), (65536, FULL), (131072 - a.steps - 8, FULL)]
            ctx, ctx_len, reached, t_pre = None, 0, 0, 0.0
            for T, seq in legs:
                if ctx is None or seq != ctx_len:
                    if ctx is not None:
                        ctx.close()
                    ctx = L.model.InferenceContext(tf, L.model.InferenceArgs(seq), max_rows=chunk[mode], acc_mode=acc[mode])
                    ctx.allow_chunked_prefill(True)
                    ctx_len, reached, t_pre = seq, 0, 0.0
                deadline = time.perf_counter() + a.budget
                dt, reached, nxt = prefill(ctx, reached, T, chunk[mode], deadline)
                t_pre += dt
                first = int(nxt) if nxt is not None else 0
                ctx.decode_run(first, T, 4, use_graph=True)                  # warm-up at the same positions
                toks, ms, graphed = ctx.decode_run(first, T, a.steps, use_graph=True)
                ms_tok = ms / a.steps
                b = WEIGHT_BYTES + KV_BYTES_PER_POS * T
                emit(workload=f"single {mode} T={T}", kernel="sdpa_kernel (shared memory)" if seq <= 17024 else "streamed (sdpa_stream.cuh)",
                     cache_filled_to=reached, prefill_budget_ran_out=reached < T,
                     tokens_per_s=round(1e3 / ms_tok, 2), ms_per_token=round(ms_tok, 3), prefill_s_cumulative=round(t_pre, 2),
                     bytes_per_step=b, whole_step_GBps=round(b / (ms_tok * 1e-3) / 1e9, 1),
                     whole_step_frac_of_3_35TBps=round(b / (ms_tok * 1e-3) / HBM_PEAK, 4), graph=graphed,
                     timing="CUDA events around lnb_decode_run")
            if ctx is not None:
                ctx.close()

    if "batch" in a.legs:
        for mode in modes:
            for n, seq in ((8, 2048), (8, 8192), (3, 32768)):
                ctx = L.model.InferenceContext(tf, L.model.InferenceArgs(seq), max_rows=chunk[mode], acc_mode=acc[mode], n_seq=n)
                ctx.allow_chunked_prefill(True)
                T = seq - a.steps - 8
                deadline = time.perf_counter() + a.budget
                cur, t_pre, filled = [], 0.0, []
                for i in range(n):
                    ctx.set_active_sequence(i)
                    dt, reached, nxt = prefill(ctx, 0, T, chunk[mode], deadline)
                    t_pre += dt
                    cur.append(int(nxt) if nxt is not None else 0)
                    filled.append(reached)
                for _ in range(4):                                      # warm-up at the same positions
                    ctx.forward_batch(cur, [T] * n)
                pos = [T] * n
                t0 = time.perf_counter()
                c = list(cur)
                for _ in range(a.steps):
                    nxt, _ = ctx.forward_batch(c, pos)
                    c = [int(t) for t in nxt]
                    pos = [p + 1 for p in pos]
                dt = time.perf_counter() - t0
                ms_step = 1e3 * dt / a.steps
                b = WEIGHT_BYTES + n * KV_BYTES_PER_POS * T
                emit(workload=f"batch {mode} n={n} SequenceLength={seq} T={T}", cache_filled_to=filled,
                     prefill_budget_ran_out=min(filled) < T, tokens_per_s=round(n * a.steps / dt, 2),
                     ms_per_step=round(ms_step, 3), ms_per_token=round(ms_step / n, 3), prefill_s=round(t_pre, 2),
                     bytes_per_step=b, whole_step_GBps=round(b / (ms_step * 1e-3) / 1e9, 1),
                     whole_step_frac_of_3_35TBps=round(b / (ms_step * 1e-3) / HBM_PEAK, 4),
                     timing="wall clock around host-driven lnb_forward_batch steps")
                ctx.close()
    gm.Free()
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
