"""Workload for compute-sanitizer (SURVEY.md section 5 "race detection"): every kernel family of the decode and prefill
paths once, on the TINY miniature, checked against the oracle so that the run is also a correctness run.
  compute-sanitizer --tool memcheck  python tools/sanitize_run.py
  compute-sanitizer --tool racecheck python tools/sanitize_run.py
(tools/sanitize.sh runs both under compute-sanitizer)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import lnb_b200 as L
from tests.helpers import host_tensors, oracle_model

# LNB_ENGINE=1: every S=1 step through the persistent decode engine (both modes); LNB_ENGINE=0: the kernel chain
which = os.environ.get("LNB_ENGINE", "default")
args = dict(L.synth.TINY)
tensors = host_tensors(args, 7)
om = oracle_model(args, tensors)
gm = L.model.LoadModelFromTensors(args, tensors)
prompt = np.array([1, 50, 999, 7, 300, 12, 64, 2], np.int32)
ok = True
for mode, acc in (("strict", L._capi.LNB_ACC_STRICT), ("fast", L._capi.LNB_ACC_FAST)):
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(48), max_rows=40, acc_mode=acc, n_seq=2)
    osess = om.new_session(48)
    exp = osess.forward(prompt, 0, all_rows=True)
    got = gm.Transformer.Forward(ctx, L.ml.Tensor(prompt, L.ml.DT_INT32), 0).RawData           # short-prompt path (GEMV, M=8)
    good = np.array_equal(got, exp) if mode == "strict" else float(np.abs(got - exp).max()) <= 1e-2
    first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
    eager, _, _ = ctx.decode_run(first, 8, 6, use_graph=False)                                  # decode chain, PDL, eager
    graph, _, g = ctx.decode_run(first, 8, 6, use_graph=True)                                   # the same as CUDA-graph replays
    good = good and list(eager) == list(graph)
    ctx.set_active_sequence(1)
    long_prompt = np.arange(3, 43, dtype=np.int32)                                              # S=40: tensor-core prefill in FAST, 8-row blocks in STRICT
    lo = osess.forward(long_prompt[:1], 0)                                                      # (oracle session reused only for shapes)
    nxt, lg = gm.Transformer.forward_argmax(ctx, long_prompt, 0, want_logits="last")
    o2 = om.new_session(48)
    e2 = o2.forward(long_prompt, 0, all_rows=False)
    good = good and (np.array_equal(lg, e2) if mode == "strict" else float(np.abs(lg - e2).max()) <= 2e-2)
    nb, _ = ctx.forward_batch([5, 6], [8, 40])                                                  # batched decode step, 2 sequences
    print(f"[sanitize_run] LNB_ENGINE={which} {mode}: parity {'ok' if good else 'MISMATCH'}; graph={g}; launches so far {ctx.launch_count()}", flush=True)
    ok = ok and good
    ctx.close(); osess.close(); o2.close()
# prompt attention on the tensor cores (head_dim 128 only, so the TINY model never reaches it): op-level call, FAST, S = 70
from oracle import oracle as O
from tests.helpers import rand_bf16
rng = np.random.default_rng(3)
q = rand_bf16(rng, (70, 8, 128)); ck = rand_bf16(rng, (70, 2, 128)); cv = rand_bf16(rng, (70, 2, 128))
out = np.empty((70, 8 * 128), np.uint16)
c = L._capi
c.check(c.lib.lnb_op_attention_bf16(c.ptr(q, c.u16p), c.ptr(ck, c.u16p), c.ptr(cv, c.u16p), c.ptr(out, c.u16p), 70, 70, 8, 2, 128, 1, c.LNB_ACC_FAST))
d = np.abs(O.bf16_to_f32(out).astype(np.float64) - O.bf16_to_f32(O.attention(q, ck, cv, 70, 1)).astype(np.float64))
print(f"[sanitize_run] prompt attention on the tensor cores (default kernel) S=70: max-abs vs oracle {d.max():.2e}", flush=True)
ok = ok and d.max() <= 2.0 ** -7
# op-level entry points (generic kernels)
x = np.arange(6, dtype=np.float32).reshape(2, 3)
t = L.ml.Tensor.from_f32(x)
L.ml.LinearTransformation(t, L.ml.Tensor.from_f32(np.ones((4, 3), np.float32)))
L.ml.Silu(t)
gm.Free(); om.close()
print("[sanitize_run] done", "OK" if ok else "FAILED", flush=True)
sys.exit(0 if ok else 1)
