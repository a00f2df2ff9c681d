"""LNB_ACC_FAST bit for bit against the oracle's statement of its summation order (oracle/lnb_oracle.h, orc_order): on every
route that sums on the FMA pipe -- the GEMV projections, the in-CTA and standalone RMSNorm, sdpa_kernel, sdpa_decode_kernel and
the streamed kernels -- the GPU must give exactly the bits of the oracle run in that order (O.ORDER_FAST with the shared-memory
attention kernels, O.ORDER_FAST_STREAM where rows stream).  Every assertion is an equality; there are no tolerances.
Tensor-core routes (FAST prompts of >= 32 rows) accumulate in the hardware's order and cannot be restated: where one runs
first, its caches are copied into the oracle session and the decode steps that follow are compared."""
import os
import time

import numpy as np
import pytest

from oracle import oracle as O
from tests.engine_shapes import wide_args
from tests.helpers import bf, f32, host_tensors, oracle_model, rand_bf16
from tests.test_gpu_long_context import OP_CASES, SHAPES, _attention
from tests.test_gpu_ops import _adversarial_rows

pytestmark = pytest.mark.gpu

SEED = 1234
TREE, STREAM = O.ORDER_FAST, O.ORDER_FAST_STREAM

_WALL = {}


@pytest.fixture(autouse=True)
def _wall_time(request):
    t0 = time.perf_counter()
    yield
    _WALL[request.node.name] = time.perf_counter() - t0


def teardown_module(module):
    print("\nwall time per test (s): " + ", ".join(f"{k} {v:.1f}" for k, v in _WALL.items()) +
          f"\nwall time, all tests: {sum(_WALL.values()):.1f} s, without 8B: "
          f"{sum(v for k, v in _WALL.items() if '8b' not in k):.1f} s")


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _load(L, args):
    tensors = host_tensors(args, SEED)
    return args, oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)


@pytest.fixture(scope="module")
def models(L):
    """TINY (head_dim 32), TINY128 (head_dim 128) and `wide` (32 heads of 64, FFN sized from the SM count so w2's K leaves a
    short last k-tile), loaded once"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = {"tiny": _load(L, dict(L.synth.TINY)), "tiny128": _load(L, dict(L.synth.TINY128)), "wide": _load(L, wide_args(sms))}
    yield out
    for _, om, gm in out.values():
        gm.Free()
        om.close()


def _eq(got, exp, what):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    assert np.array_equal(got, exp), f"{what}: {(got != exp).sum()} of {got.size} differ"


def _ctx(L, gm, seq, max_rows=8, n_seq=1, engine=None):
    """a FAST session; engine True / False sets LNB_ENGINE while the engines are probed (None: the default)"""
    old = os.environ.get("LNB_ENGINE")
    if engine is not None:
        os.environ["LNB_ENGINE"] = "1" if engine else "0"
    try:
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=max_rows, acc_mode=L._capi.LNB_ACC_FAST,
                                       n_seq=n_seq)
        gm.Transformer.forward_argmax(ctx, np.array([1], np.int32), 0)     # probe now (overwritten by every test's prefill)
    finally:
        if old is None:
            os.environ.pop("LNB_ENGINE", None)
        else:
            os.environ["LNB_ENGINE"] = old
    return ctx


def _inject(ctx, osess, n_layers, rows):
    """the session's K/V cache rows [0, rows) of every layer into the oracle session (tensor-core prefill: not restatable)"""
    for layer in range(n_layers):
        ok, ov = osess.cache(layer)
        ok[:rows] = ctx.CacheK(layer).RawData[:rows]
        ov[:rows] = ctx.CacheV(layer).RawData[:rows]


def _caches_eq(ctx, osess, layers, rows, what):
    for layer in layers:
        ok, ov = osess.cache(layer)
        _eq(ctx.CacheK(layer).RawData[:rows], ok[:rows], f"{what}: K cache, layer {layer}")
        _eq(ctx.CacheV(layer).RawData[:rows], ov[:rows], f"{what}: V cache, layer {layer}")


# ---- 1. op level -----------------------------------------------------------------------------------------------------------

# the cases lnb_op_attention_bf16 sends to sdpa_kernel: S = 1; masked S > 1 at head_dim 32 (masked at head_dim 128 goes to
# sdpa_prefill_kernel); unmasked S > 1 at head_dim 128.  (nh, nkv): n_rep 4 and 8.
SDPA_CASES = [(S, T, causal, hd, nh, nkv) for hd in (32, 128) for nh, nkv in ((32, 8), (16, 2))
              for S, T, causal in ((1, 1, 0), (1, 130, 0), (1, 1500, 0), (2, 2, 1), (5, 5, 1), (2, 40, 0), (5, 300, 0))
              if not (causal and hd == 128)]


@pytest.mark.parametrize("S,T,causal,hd,nh,nkv", SDPA_CASES)
def test_op_attention_sdpa_kernel_equals_the_tree_statement(L, S, T, causal, hd, nh, nkv):
    rng = np.random.default_rng(S * 1009 + T * 7 + hd + nh)
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (T, nkv, hd)), rand_bf16(rng, (T, nkv, hd))
    got = _attention(L, q, ck, cv, S, T, causal, L._capi.LNB_ACC_FAST)
    _eq(got, O.attention_order(q, ck, cv, T, causal, T - S if causal else 0, O.ATTN_TREE), "every head")


@pytest.mark.parametrize("shape,T,S", OP_CASES)
def test_op_attention_streamed_equals_the_stream_statement(L, shape, T, S):
    """the streamed lengths of test_gpu_long_context, up to the 131 072-token window, every query head"""
    nh, nkv, hd = SHAPES[shape]
    rng = np.random.default_rng(T * 13 + S + hd)
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (T, nkv, hd)), rand_bf16(rng, (T, nkv, hd))
    got = _attention(L, q, ck, cv, S, T, 2, L._capi.LNB_ACC_FAST)
    _eq(got, O.attention_order(q, ck, cv, T, 1, T - S, O.ATTN_STREAM), "every head")


@pytest.mark.parametrize("D", [256, 1024, 4096])
def test_op_rmsnorm_equals_the_256_part_statement(L, D):
    rng = np.random.default_rng(D)
    x = _adversarial_rows(rng, 14, D)
    x[-1] = 0
    w = bf(1 + 0.1 * rng.standard_normal(D))
    out = np.empty_like(x)
    c = L._capi
    c.check(c.lib.lnb_op_rmsnorm_bf16(c.ptr(x, c.u16p), c.ptr(w, c.u16p), c.ptr(out, c.u16p), x.shape[0], D, 1e-5, c.LNB_ACC_FAST))
    r = O.rms_scale_order(x, 1e-5, 256)
    exp = bf(f32(bf(f32(x) * r[:, None])) * f32(w)[None, :])
    _eq(out, exp.reshape(x.shape), "rmsnorm")


@pytest.mark.parametrize("N,K", [(128256, 4096), (4096, 14336)])
def test_op_linear_8b_shapes_equal_the_ks8_statement(L, N, K):
    """the 8B LM head and w2, one activation row (the GEMV)"""
    rng = np.random.default_rng(N + K)
    x = rand_bf16(rng, (1, K))
    w = rand_bf16(rng, (N, K), 1.0 / np.sqrt(K))
    L.ml.ACC_MODE = L._capi.LNB_ACC_FAST
    try:
        got = L.ml.LinearTransformation(L.ml.Tensor(x, L.ml.DT_BF16), L.ml.Tensor(w, L.ml.DT_BF16)).RawData
    finally:
        L.ml.ACC_MODE = L._capi.LNB_ACC_STRICT
    _eq(got, O.linear_order_bf16(x, w, 8), "linear")


# ---- 2. prompts below the tensor-core cut (sdpa_kernel at every head_dim) ------------------------------------------------

@pytest.mark.parametrize("name", ["tiny", "tiny128", "wide"])
@pytest.mark.parametrize("start", [0, 1, 64])
@pytest.mark.parametrize("S", [1, 2, 8, 9, 31])
def test_prompt_below_the_tensor_core_cut(L, models, name, start, S):
    """S rows at position `start` (the prefix fed in chunks of at most 31 rows, so nothing runs on the tensor cores): all-row
    logits, the residual stream after every layer, and the caches of the first and last layer"""
    args, om, gm = models[name]
    nl = args["n_layers"]
    seq = 96
    toks = np.random.default_rng(S * 100 + start).integers(0, args["vocab_size"], size=start + S).astype(np.int32)
    pieces = [(p, min(31, start - p)) for p in range(0, start, 31)] + [(start, S)]

    def feed(ctx, osess):
        out = None
        for p, n in pieces:
            if p == 0:
                exp = osess.forward(toks[:n], 0, all_rows=True, order=TREE)
            else:
                exp = osess.forward_chunk(toks[p:p + n], p, all_rows=True, order=TREE)
            _, got = gm.Transformer.forward_argmax(ctx, toks[p:p + n], p, want_logits="all")
            out = (got, exp)
        return out

    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=31, acc_mode=L._capi.LNB_ACC_FAST)
    osess = om.new_session(seq)
    try:
        ctx.allow_chunked_prefill(True)
        got, exp = feed(ctx, osess)
        _eq(got, exp, "logits")
        _caches_eq(ctx, osess, (0, nl - 1), start + S, "caches")
    finally:
        ctx.close(); osess.close()
    if start:
        return
    osess = om.new_session(seq)
    try:
        _, tr = osess.forward(toks[:S], 0, all_rows=True, trace=True, order=TREE)
        for n in range(1, nl + 1):
            ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=31, acc_mode=L._capi.LNB_ACC_FAST)
            try:
                ctx.set_layer_limit(n)
                gm.Transformer.forward_argmax(ctx, toks[:S], 0)
                _eq(ctx.residual(S), tr[n], f"residual after layer {n}")
            finally:
                ctx.close()
    finally:
        osess.close()


# ---- 3. decode --------------------------------------------------------------------------------------------------------------

def _prefill(L, gm, ctx, osess, prompt, order=TREE):
    nxt, lg = gm.Transformer.forward_argmax(ctx, prompt, 0, want_logits="last")
    exp = osess.forward(prompt, 0, all_rows=False, order=order)
    _eq(lg, exp, "prefill logits")
    assert nxt == O.argmax_f32(exp[0])
    return nxt


@pytest.mark.parametrize("name", ["tiny", "tiny128", "wide"])
@pytest.mark.parametrize("engine", [False, True])
def test_host_driven_decode_equals_the_statement(L, models, name, engine):
    """host-driven steps on the FAST kernel chain (engine False) and on the decode engine (LNB_ENGINE=1): logits, greedy ids
    and both caches"""
    args, om, gm = models[name]
    seq = 40
    prompt = np.random.default_rng(21).integers(0, args["vocab_size"], size=8).astype(np.int32)
    ctx = _ctx(L, gm, seq, engine=engine)
    osess = om.new_session(seq)
    try:
        assert ctx.uses_engine() == engine
        tok = _prefill(L, gm, ctx, osess, prompt)
        for pos in range(8, 24):
            nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), pos, want_logits="last")
            exp = osess.forward(np.array([tok], np.int32), pos, order=TREE)
            _eq(lg, exp, f"position {pos}")
            assert nxt == O.argmax_f32(exp[0]), pos
            tok = nxt
        _caches_eq(ctx, osess, (0, args["n_layers"] - 1), 24, "caches")
    finally:
        ctx.close(); osess.close()


@pytest.mark.parametrize("name", ["tiny", "tiny128"])
@pytest.mark.parametrize("use_graph", [False, True])
def test_device_resident_decode_equals_the_statement(L, models, name, use_graph):
    args, om, gm = models[name]
    seq = 40
    prompt = np.random.default_rng(22).integers(0, args["vocab_size"], size=8).astype(np.int32)
    ctx = _ctx(L, gm, seq)
    osess = om.new_session(seq)
    try:
        first = _prefill(L, gm, ctx, osess, prompt)
        want, tok = [], first
        for pos in range(8, 8 + 16):
            tok = O.argmax_f32(osess.forward(np.array([tok], np.int32), pos, order=TREE)[0])
            want.append(tok)
        toks, _, graphed = ctx.decode_run(first, 8, 16, use_graph=use_graph)
        assert graphed == use_graph
        assert list(toks) == want
    finally:
        ctx.close(); osess.close()


@pytest.mark.parametrize("name", ["tiny", "tiny128", "wide"])
@pytest.mark.parametrize("n", [3, 8])
def test_batched_decode_equals_the_statement(L, models, name, n):
    """lnb_forward_batch with n sequences at mixed positions (the batch engine's FMA form where it runs): every row's logits
    and greedy id, and every sequence's caches"""
    args, om, gm = models[name]
    seq = 48
    rng = np.random.default_rng(n * 5 + len(name))
    lens = [1 + (7 * i) % 20 for i in range(n)]
    prompts = [rng.integers(0, args["vocab_size"], size=k).astype(np.int32) for k in lens]
    ctx = _ctx(L, gm, seq, max_rows=31, n_seq=n)
    osess = [om.new_session(seq) for _ in range(n)]
    try:
        cur, pos = [], []
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            cur.append(_prefill(L, gm, ctx, osess[i], p)); pos.append(len(p))
        for step in range(6):
            nxt, lg = ctx.forward_batch(cur, pos, want_logits=True)
            for i in range(n):
                exp = osess[i].forward(np.array([cur[i]], np.int32), pos[i], order=TREE)
                _eq(lg[i], exp[0], f"sequence {i} step {step}")
                assert nxt[i] == O.argmax_f32(exp[0])
            cur = [int(t) for t in nxt]; pos = [p + 1 for p in pos]
        for i in range(n):
            ctx.set_active_sequence(i)
            _caches_eq(ctx, osess[i], (0, args["n_layers"] - 1), pos[i], f"sequence {i}")
    finally:
        ctx.close()
        for o in osess:
            o.close()


@pytest.mark.parametrize("name", ["tiny", "tiny128"])
def test_speculative_call_equals_the_statement(L, models, name):
    """one speculative call whose draft is right twice, then wrong: every row's logits are the statement's rows of that chunk"""
    args, om, gm = models[name]
    seq = 40
    prompt = np.random.default_rng(23).integers(0, args["vocab_size"], size=8).astype(np.int32)
    ctx = _ctx(L, gm, seq)
    osess, plain = om.new_session(seq), om.new_session(seq)
    try:
        t0 = _prefill(L, gm, ctx, osess, prompt)
        plain.forward(prompt, 0, all_rows=False, order=TREE)
        greedy, tok = [], t0
        for pos in range(8, 12):
            tok = O.argmax_f32(plain.forward(np.array([tok], np.int32), pos, order=TREE)[0])
            greedy.append(tok)
        drafts = [greedy[0], greedy[1], (greedy[2] + 1) % args["vocab_size"], greedy[3]]
        rows = np.array([t0] + drafts, np.int32)
        nxt, acc, lg = ctx.forward_speculative([(0, 8, rows)], want_logits=True)
        exp = osess.forward_chunk(rows, 8, all_rows=True, order=TREE)
        _eq(lg, exp, "speculative rows")
        assert [int(t) for t in nxt] == [O.argmax_f32(e) for e in exp]
        assert int(acc[0]) == 2
        _caches_eq(ctx, osess, (0, args["n_layers"] - 1), 8 + len(rows), "caches")
    finally:
        ctx.close(); osess.close(); plain.close()


@pytest.mark.parametrize("name", ["tiny", "tiny128"])
def test_ragged_calls_below_32_rows_equal_the_stream_statement(L, models, name):
    """ragged calls of fewer than 32 rows (GEMV chain, streamed attention): prompts, a prompt chunk and decode rows of three
    sequences; each segment's last-row logits and greedy id, and the caches"""
    args, om, gm = models[name]
    seq = 48
    rng = np.random.default_rng(24)
    t = lambda k: rng.integers(0, args["vocab_size"], size=k).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=31, acc_mode=L._capi.LNB_ACC_FAST, n_seq=3)
    osess = [om.new_session(seq) for _ in range(3)]
    pos = [0, 0, 0]
    try:
        calls = [[(0, t(7)), (1, t(5))], [(0, None), (1, t(3)), (2, t(9))], [(0, None), (1, None), (2, t(2))]]
        last = {}
        for call in calls:
            segs = [(s, pos[s], np.array([last[s]], np.int32) if tk is None else tk) for s, tk in call]
            assert sum(len(tk) for _, _, tk in segs) < 32
            nxt, lg = ctx.forward_ragged(segs, want_logits=True)
            for i, (s, p, tk) in enumerate(segs):
                if p == 0:
                    exp = osess[s].forward(tk, 0, all_rows=False, order=STREAM)
                elif len(tk) > 1:
                    exp = osess[s].forward_chunk(tk, p, all_rows=False, order=STREAM)
                else:
                    exp = osess[s].forward(tk, p, order=STREAM)
                _eq(lg[i], exp[0], f"segment {i} (sequence {s} at {p})")
                assert nxt[i] == O.argmax_f32(exp[0])
                pos[s] += len(tk); last[s] = int(nxt[i])
        for s in range(3):
            ctx.set_active_sequence(s)
            _caches_eq(ctx, osess[s], (0, args["n_layers"] - 1), pos[s], f"sequence {s}")
    finally:
        ctx.close()
        for o in osess:
            o.close()


# ---- 4. decode after a tensor-core prefill ------------------------------------------------------------------------------

def test_decode_after_tensor_core_prefill_tiny128(L, models):
    """a FAST prefill of 40 rows (gemm_tc / sdpa_tc: hardware order), its caches copied into the oracle session, then 16
    greedy steps on the kernel chain: logits and ids of every step"""
    args, om, gm = models["tiny128"]
    S, seq = 40, 64
    prompt = np.random.default_rng(25).integers(0, args["vocab_size"], size=S).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=S, acc_mode=L._capi.LNB_ACC_FAST)
    osess = om.new_session(seq)
    try:
        tok, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        _inject(ctx, osess, args["n_layers"], S)
        for pos in range(S, S + 16):
            nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), pos, want_logits="last")
            exp = osess.forward(np.array([tok], np.int32), pos, order=TREE)
            _eq(lg, exp, f"position {pos}")
            assert nxt == O.argmax_f32(exp[0])
            tok = nxt
        _caches_eq(ctx, osess, (0, args["n_layers"] - 1), S + 16, "caches")
    finally:
        ctx.close(); osess.close()


# ---- 5. the 8B model ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def big8b(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    args = dict(L.synth.LLAMA31_8B)
    om = oracle_model(args, host_tensors(args, L.synth.SEED))
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    yield args, om, gm
    gm.Free()
    om.close()


def test_8b_teacher_forced_prompt_and_decode_equal_the_statement(L, big8b):
    """8 prompt rows (every row's logits: the 128 256-row LM head) and 4 decode steps, K = 14 336 in w2"""
    args, om, gm = big8b
    prompt = np.array(L.synth.PROMPT_8, np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST)
    osess = om.new_session(136)
    try:
        nxt, lg = gm.Transformer.forward_argmax(ctx, prompt, 0, want_logits="all")
        exp = osess.forward(prompt, 0, all_rows=True, order=TREE)
        _eq(lg, exp, "prompt logits")
        tok = O.argmax_f32(exp[-1])
        assert nxt == tok
        for pos in range(8, 12):
            nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), pos, want_logits="last")
            exp = osess.forward(np.array([tok], np.int32), pos, order=TREE)
            _eq(lg, exp, f"position {pos}")
            tok = O.argmax_f32(exp[0])
            assert nxt == tok
        _caches_eq(ctx, osess, (0, 31), 12, "caches")
    finally:
        ctx.close(); osess.close()


def test_8b_decode_after_tensor_core_prefill_equals_the_statement(L, big8b):
    args, om, gm = big8b
    S = 135
    prompt = np.random.default_rng(135).integers(0, args["vocab_size"], size=S).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(144), max_rows=S, acc_mode=L._capi.LNB_ACC_FAST)
    osess = om.new_session(144)
    try:
        tok, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        _inject(ctx, osess, args["n_layers"], S)
        for pos in range(S, S + 4):
            nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), pos, want_logits="last")
            exp = osess.forward(np.array([tok], np.int32), pos, order=TREE)
            _eq(lg, exp, f"position {pos}")
            assert nxt == O.argmax_f32(exp[0])
            tok = nxt
    finally:
        ctx.close(); osess.close()
