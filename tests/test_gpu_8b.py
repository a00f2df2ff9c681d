"""GPU parity at the BASELINE size: the synthetic Llama-3.1-8B checkpoint (random-init weights of the 8B architecture,
the same bits in HBM and in the oracle's host copy) through the model-level C-ABI, teacher-forced against the CPU
oracle; and the op-level linear at the two largest projection shapes of the model.  The oracle costs about 0.1 s per
S=1 step on the host cores of a GPU machine, so a dozen positions fit a test run; bench.py compares all 128 generated tokens.

STRICT must reproduce the oracle bit for bit (north_star: logits within 1e-2, greedy ids identical -- met with 0.0).
FAST is a documented reorder of the long fp32 sums: every logit stays within a few bf16 ulps, and the test pins the
measured distance so that a real bug (wrong stream order, missing truncation) cannot hide behind "reorder noise"."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import host_tensors, oracle_model, rand_bf16

pytestmark = pytest.mark.gpu

N_STEPS = 10          # S=1 decode positions after the 8-token prompt


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module")
def big(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    args = dict(L.synth.LLAMA31_8B)
    tensors = host_tensors(args, L.synth.SEED)            # 16 GB on the host: the oracle's generator
    om = oracle_model(args, tensors)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)   # the device generator (same bits, test_gpu_model pins that)
    prompt = np.array(L.synth.PROMPT_8, np.int32)
    sess = om.new_session(136)
    ref = [sess.forward(prompt, 0, all_rows=True)]        # [8, V]: every prompt row, like the reference's Forward
    toks = [O.argmax_f32(ref[0][-1])]
    for i in range(N_STEPS):
        ref.append(sess.forward(np.array([toks[-1]], np.int32), 8 + i, all_rows=False))
        toks.append(O.argmax_f32(ref[-1][0]))
    caches = [tuple(c.copy() for c in sess.cache(l)) for l in (0, 31)]
    sess.close()
    yield args, om, gm, prompt, ref, toks, caches
    gm.Free()
    om.close()


def _teacher_forced(L, gm, acc, prompt, toks, all_rows_prefill=True):
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=acc)
    out = []
    nxt, lg = gm.Transformer.forward_argmax(ctx, prompt, 0, want_logits="all" if all_rows_prefill else "last")
    out.append((nxt, lg))
    for i in range(N_STEPS):
        nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([toks[i]], np.int32), 8 + i, want_logits="last")
        out.append((nxt, lg))
    return ctx, out


def test_8b_strict_logits_bit_exact_teacher_forced(L, big):
    args, om, gm, prompt, ref, toks, caches = big
    ctx, got = _teacher_forced(L, gm, L._capi.LNB_ACC_STRICT, prompt, toks)
    try:
        for i, ((nxt, lg), exp) in enumerate(zip(got, ref)):
            assert np.array_equal(lg, exp), f"call {i}: max-abs {np.abs(lg - exp).max()}"
            assert nxt == toks[i]
        for (ok, ov), layer in zip(caches, (0, 31)):       # KV cache rows written so far, first and last layer
            n = 8 + N_STEPS
            assert np.array_equal(ctx.CacheK(layer).RawData[:n], ok[:n])
            assert np.array_equal(ctx.CacheV(layer).RawData[:n], ov[:n])
    finally:
        ctx.close()


def test_8b_strict_device_loop_equals_oracle_tokens(L, big):
    """the timed path of bench.py (`value`): prefill + device-resident graph decode, greedy ids = the oracle's"""
    args, om, gm, prompt, ref, toks, _ = big
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_STRICT)
    try:
        first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        out, _, graphed = ctx.decode_run(first, 8, N_STEPS, use_graph=True)
        assert [first] + [int(t) for t in out] == toks
        out2, _, _ = ctx.decode_run(first, 8, N_STEPS, use_graph=False)
        assert list(out2) == list(out)
    finally:
        ctx.close()


def test_8b_fast_stays_within_the_documented_distance(L, big):
    """LNB_ACC_FAST against the reference order on the 8B model: |logit| < 2 here, one bf16 ulp is 2^-7 = 0.0078 there, and
    the reorder decorrelates every tensor at the 1-ulp level after a few layers (DESIGN.md section 3): the bound pinned
    here is 0.05 absolute on every logit (measured 0.0254 = 3.25 ulps at |logit| in [1, 2)) and greedy agreement wherever
    the oracle's winner leads by more than that."""
    args, om, gm, prompt, ref, toks, _ = big
    ctx, got = _teacher_forced(L, gm, L._capi.LNB_ACC_FAST, prompt, toks, all_rows_prefill=False)
    try:
        worst = 0.0
        for i, ((nxt, lg), exp) in enumerate(zip(got, ref)):
            e = exp[-1:]
            worst = max(worst, float(np.abs(lg - e).max()))
            top2 = np.sort(e[0])[-2:]
            if top2[1] - top2[0] > 0.1:                    # a clear winner must stay the winner
                assert nxt == toks[i]
        assert worst <= 0.05, worst
    finally:
        ctx.close()


@pytest.mark.parametrize("N,K", [(28672, 4096), (128256, 4096), (4096, 14336)])
def test_full_size_linear_strict_bit_exact(L, N, K):
    """lnb_op_linear_bf16 at the model's largest shapes: w1|w3 stacked (28672 x 4096), the LM head (128256 x 4096) and
    w2 (4096 x 14336) -- ml.LinearTransformation (operations_lineartransform.go:37-70), one activation row"""
    rng = np.random.default_rng(N)
    x = rand_bf16(rng, (1, K), 1.0)
    w = rand_bf16(rng, (N, K), 1.0 / np.sqrt(K))
    exp = O.linear_bf16(x, w)
    got = L.ml.LinearTransformation(L.ml.Tensor(x, L.ml.DT_BF16), L.ml.Tensor(w, L.ml.DT_BF16)).RawData
    assert np.array_equal(got, exp)
    L.ml.ACC_MODE = L._capi.LNB_ACC_FAST
    try:
        fast = L.ml.LinearTransformation(L.ml.Tensor(x, L.ml.DT_BF16), L.ml.Tensor(w, L.ml.DT_BF16)).RawData
    finally:
        L.ml.ACC_MODE = L._capi.LNB_ACC_STRICT
    # a single op: at most one bf16 ulp from the reference order (absolute floor for outputs that cancel to ~0)
    e, f = O.bf16_to_f32(exp).astype(np.float64), O.bf16_to_f32(fast).astype(np.float64)
    ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(e), 1e-30))) - 7)
    assert (np.abs(f - e) <= np.maximum(ulp, 1e-5)).all()


# largest |logit| distance of any row: measured 0.0273 (median row 0.0230) on an H100 SXM (80 GB), pinned at 0.05
PREFILL_136_MAX_ABS = 0.05


def test_8b_fast_tensor_core_prefill_all_rows(L, big):
    """a FAST prefill of 136 synthetic tokens (max_rows 136, every row's logits) runs the tensor-core path at the real shapes:
    sdpa_tc_kernel with 32 heads over 8 KV heads, gemm_tc_kernel at K = 14336 (w2), and the TC_EPI_F32TRUNC LM head at
    N = 128256 for rows 0..134.  Every row is compared with the oracle's all-rows forward (13 s of CPU on the GPU machine's
    host; the whole test took 14 s)."""
    import time
    args, om, gm, _, _, _, _ = big
    S = 136
    toks = np.random.default_rng(136).integers(0, args["vocab_size"], size=S).astype(np.int32)
    t0 = time.perf_counter()
    sess = om.new_session(S)
    try:
        exp = sess.forward(toks, 0, all_rows=True)
    finally:
        sess.close()
    t_oracle = time.perf_counter() - t0
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(S), max_rows=S, acc_mode=L._capi.LNB_ACC_FAST)
    try:
        nxt, got = gm.Transformer.forward_argmax(ctx, toks, 0, want_logits="all")
    finally:
        ctx.close()
    per_row = np.abs(got - exp).max(1)
    print(f"8B prefill S={S}: oracle {t_oracle:.1f} s, max-abs per row: max {per_row.max():.4f}, median {np.median(per_row):.4f}")
    assert nxt == int(np.argmax(got[-1]))
    assert per_row.max() <= PREFILL_136_MAX_ABS, (int(per_row.argmax()), float(per_row.max()))


# ---- the engines at the 8B shapes, against the kernel chain (pinned to the oracle above) ---------------------------------
ENGINE_SEQ = 145      # the longest SequenceLength the engines accept at head_dim 128 with 4 query heads per KV head


def _engine_context(L, gm, acc, engine, max_rows=8, n_seq=1):
    import os
    old = os.environ.get("LNB_ENGINE")
    os.environ["LNB_ENGINE"] = "1" if engine else "0"       # read at the session's first decode
    try:
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(ENGINE_SEQ), max_rows=max_rows, acc_mode=acc,
                                       n_seq=n_seq)
        gm.Transformer.forward_argmax(ctx, np.array([1], np.int32), 0)
    finally:
        if old is None:
            os.environ.pop("LNB_ENGINE", None)
        else:
            os.environ["LNB_ENGINE"] = old
    return ctx


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_8b_batch_engine_equals_the_batched_chain(L, big, mode, monkeypatch):
    """8 sequences with prompts of 8 .. 136 tokens, batched steps until the longest reaches position 144: every step's logits
    and tokens, and the caches of layers 0 and 31, of the batch engine equal those of the batched kernel chain"""
    monkeypatch.delenv("LNB_BATCH_TC", raising=False)
    args, om, gm = big[:3]
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(8)
    lens = (136, 8, 40, 100, 17, 64, 9, 121)
    prompts = [rng.integers(0, args["vocab_size"], size=k).astype(np.int32) for k in lens]
    ce = _engine_context(L, gm, acc, True, max_rows=136, n_seq=8)
    cc = _engine_context(L, gm, acc, False, max_rows=136, n_seq=8)
    try:
        cur, pos = [], []
        for i, p in enumerate(prompts):
            got = []
            for ctx in (ce, cc):
                ctx.set_active_sequence(i)
                got.append(gm.Transformer.forward_argmax(ctx, p, 0))
            assert got[0][0] == got[1][0]
            cur.append(got[0][0]); pos.append(len(p))
        while max(pos) < ENGINE_SEQ:
            l0 = ce.launch_count()
            te, le = ce.forward_batch(cur, pos, want_logits=True)
            assert ce.launch_count() - l0 == 1, "the batch engine did not run"
            tc, lc = cc.forward_batch(cur, pos, want_logits=True)
            assert np.array_equal(le, lc), f"positions {pos}"
            assert list(te) == list(tc)
            cur = [int(t) for t in te]; pos = [p + 1 for p in pos]
        for i in range(8):
            ce.set_active_sequence(i); cc.set_active_sequence(i)
            for layer in (0, 31):
                assert np.array_equal(ce.CacheK(layer).RawData[:pos[i]], cc.CacheK(layer).RawData[:pos[i]]), (i, layer)
                assert np.array_equal(ce.CacheV(layer).RawData[:pos[i]], cc.CacheV(layer).RawData[:pos[i]]), (i, layer)
    finally:
        ce.close(); cc.close()


def test_8b_fast_decode_engine_equals_the_fast_chain(L, big):
    """LNB_ENGINE=1 in FAST: ten host-driven steps up to position 144 equal the FAST kernel chain's, logits and tokens"""
    args, om, gm = big[:3]
    acc = L._capi.LNB_ACC_FAST
    prompt = np.random.default_rng(135).integers(0, args["vocab_size"], size=135).astype(np.int32)
    ce = _engine_context(L, gm, acc, True, max_rows=135)
    cc = _engine_context(L, gm, acc, False, max_rows=135)
    try:
        assert ce.uses_engine() and not cc.uses_engine()
        te, _ = gm.Transformer.forward_argmax(ce, prompt, 0)
        tc, _ = gm.Transformer.forward_argmax(cc, prompt, 0)
        assert te == tc
        for p in range(135, ENGINE_SEQ):
            x = np.array([te], np.int32)
            te, le = gm.Transformer.forward_argmax(ce, x, p, want_logits="last")
            tc, lc = gm.Transformer.forward_argmax(cc, x, p, want_logits="last")
            assert np.array_equal(le, lc), f"position {p}"
            assert te == tc
        for layer in (0, 31):
            assert np.array_equal(ce.CacheK(layer).RawData[:ENGINE_SEQ], cc.CacheK(layer).RawData[:ENGINE_SEQ])
    finally:
        ce.close(); cc.close()
