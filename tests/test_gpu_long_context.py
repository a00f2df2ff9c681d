"""Streamed decode / prompt attention (csrc/sdpa_stream.cuh): every row that the shared-memory attention kernels cannot
hold -- sessions whose SequenceLength exceeds sdpa_kernel's fit, batched steps beyond sdpa_decode_kernel's fit, and
lnb_op_attention_bf16 beyond the old T limit.  STRICT must reproduce the oracle bit for bit at every length; FAST stays
inside order-free bounds (op level) or pinned ulps (model level).  Inside today's limits nothing changes: the launch
counts of those sessions are pinned to the values measured before the streamed kernel existed."""
import os
import subprocess
import tempfile
import time

import numpy as np
import pytest

from oracle import oracle as O
from tests import precise as P
from tests.helpers import bf16_ulp_diff, f32, host_tensors, oracle_model, rand_bf16

pytestmark = pytest.mark.gpu

SEED = 1234
SS_CH, SS_KT, SS_VT = 1024, 128, 256   # chunk and tile sizes of sdpa_stream.cuh

_WALL = {}


@pytest.fixture(autouse=True)
def _wall_time(request):
    t0 = time.perf_counter()
    yield
    _WALL[request.node.name] = time.perf_counter() - t0


def teardown_module(module):
    print("\nwall time per test (s): " + ", ".join(f"{k} {v:.1f}" for k, v in _WALL.items()))


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _old_cap(hd):
    """largest T sdpa_kernel held in shared memory (T * 12 + hd * 4 <= 200 KB)"""
    return (200 * 1024 - hd * 4) // 12


def _attention(L, q, ck, cv, S, T, causal, acc):
    nh, hd = q.shape[1], q.shape[2]
    nkv = ck.shape[1]
    out = np.empty((S, nh * hd), np.uint16)
    c = L._capi
    c.check(c.lib.lnb_op_attention_bf16(c.ptr(q, c.u16p), c.ptr(ck, c.u16p), c.ptr(cv, c.u16p), c.ptr(out, c.u16p),
                                        S, T, nh, nkv, hd, causal, acc))
    return out


# ---- 1. op level: 8B head shapes (32 / 8 / 128) and TINY's (8 / 2 / 32) ------------------------------------------------

SHAPES = {"8b": (32, 8, 128), "tiny": (8, 2, 32)}


def _lengths(hd):
    # just above the old cap; one below, at and one above 17 chunks (17408), 32 chunks (32768: also every tile size); the
    # full 128K window
    return [_old_cap(hd) + 1, 17 * SS_CH - 1, 17 * SS_CH, 17 * SS_CH + 1, 32767, 32768, 32769, 131072]


OP_CASES = [(shape, T, S) for shape in SHAPES for T in _lengths(SHAPES[shape][2]) for S in (1, 4)]


def _kv_pairs(nh, nkv):
    """one query head per KV head, covering every slot of the GQA group"""
    rep = nh // nkv
    return [(h * rep + h % rep, h) for h in range(nkv)]


@pytest.mark.parametrize("shape,T,S", OP_CASES)
def test_op_strict_bit_exact_beyond_the_old_limit(L, shape, T, S):
    nh, nkv, hd = SHAPES[shape]
    rng = np.random.default_rng(T * 7 + S + hd)
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (T, nkv, hd)), rand_bf16(rng, (T, nkv, hd))
    got = _attention(L, q, ck, cv, S, T, 2, L._capi.LNB_ACC_STRICT)
    exp = O.attention(q, ck, cv, T, 1, q_pos0=T - S)
    assert np.array_equal(got, exp), f"{(got != exp).sum()} of {got.size} differ"


@pytest.mark.parametrize("shape,T,S", OP_CASES)
def test_op_fast_within_order_free_bounds_beyond_the_old_limit(L, shape, T, S):
    nh, nkv, hd = SHAPES[shape]
    rng = np.random.default_rng(T * 11 + S + hd)
    q, ck = P.exact_score_qk(rng, S, T, nh, nkv, hd)
    cv = rand_bf16(rng, (T, nkv, hd))
    got = _attention(L, q, ck, cv, S, T, 2, L._capi.LNB_ACC_FAST).reshape(S, nh, hd)
    for H, h in _kv_pairs(nh, nkv):
        lo, hi = P.attention_bounds(q[:, H:H + 1], ck[:, h:h + 1], cv[:, h:h + 1], T, T - S)
        g = got[:, H]
        assert P.within(g, lo, hi).all(), (H, P.outside_report(g, lo, hi))


def _long_probe(T, nh, nkv, S, hd):
    """mask probe for any T: only the keys at positions >= T - S - 1 are nonzero; key t is 16 at dimension t % m and at
    m + (t // m) % m (m = hd / 2), row qpos asks for both coordinates of qpos and of qpos + 1, so the diagonal and the first
    future key score 512 / t(sqrt(hd)) and every other key at most half of that.  v row t carries the bits of t as +-2 in
    dimensions 0..7, so the output names the keys a row attends to."""
    m = hd // 2
    pos0 = T - S

    def onehot(t):
        e = np.zeros(hd, np.float32)
        e[t % m] = 16
        e[m + (t // m) % m] = 16
        return e
    k1 = np.zeros((T, hd), np.float32)
    for t in range(max(0, pos0 - 1), T):
        k1[t] = onehot(t)
    q1 = np.stack([np.maximum(onehot(p), onehot(p + 1)) for p in range(pos0, pos0 + S)])
    v1 = np.zeros((T, hd), np.float32)
    for j in range(8):
        v1[:, j] = 4 * ((np.arange(T) >> j) & 1) - 2
    bf = lambda a: O.bf16_bits(np.ascontiguousarray(a, np.float32))
    q = bf(np.repeat(q1[:, None, :], nh, 1)).reshape(S, nh, hd)
    k = bf(np.repeat(k1[:, None, :], nkv, 1)).reshape(T, nkv, hd)
    v = bf(np.repeat(v1[:, None, :], nkv, 1)).reshape(T, nkv, hd)
    return q, k, v


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("shape,T", [("8b", 17025), ("8b", 32769), ("tiny", 17057), ("tiny", 32768)])
def test_op_mask_probes_beyond_the_old_limit(L, shape, T, mode):
    """a leaked first future key, or a lost diagonal key, moves every affected row by at least 0.25"""
    nh, nkv, hd = SHAPES[shape]
    S = 4
    pos0 = T - S
    q, k, v = _long_probe(T, nh, nkv, S, hd)
    assert P.exact_score_inputs(q, k)
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    got = f32(_attention(L, q, k, v, S, T, 2, acc)).reshape(S, nh, hd)[:, :, :8].astype(np.float64)
    vis = P.visible_keys(S, T, pos0)
    rows = np.arange(S)
    vf = f32(v).reshape(T, nkv, hd)[:, :1, :8].astype(np.float64)

    def out(visible):
        p = P.attention_probs(q[:, :1], k[:, :1], T, visible)
        return np.einsum("sht,thd->shd", p, vf)[:, 0]
    ok = out(vis)
    leak = vis.copy()
    fut = rows[pos0 + rows + 1 < T]
    leak[fut, pos0 + fut + 1] = True
    assert (np.abs(out(leak) - ok).max(1)[fut] >= 0.25).all()
    nodiag = vis.copy()
    nodiag[rows, pos0 + rows] = False
    assert (np.abs(out(nodiag) - ok).max(1) >= 0.25).all()
    err = np.abs(got - ok[:, None, :]).max((1, 2))
    assert (err < 0.125).all(), f"rows {np.nonzero(err >= 0.125)[0]} attend to the wrong keys (max err {err.max()})"


def test_op_fast_tiled_prompt_kernel_has_no_hidden_length_limit(L):
    """FAST prompts of >= 32 rows keep the tensor-core prompt kernel beyond the old limit: 64 rows over 20 000 keys stay inside
    the order-free bounds"""
    nh, nkv, hd, S, T = 8, 2, 128, 64, 20000
    rng = np.random.default_rng(5)
    q, ck = P.exact_score_qk(rng, S, T, nh, nkv, hd)
    cv = rand_bf16(rng, (T, nkv, hd))
    got = _attention(L, q, ck, cv, S, T, 2, L._capi.LNB_ACC_FAST).reshape(S, nh, hd)
    for H, h in _kv_pairs(nh, nkv):
        lo, hi = P.attention_bounds(q[:, H:H + 1], ck[:, h:h + 1], cv[:, h:h + 1], T, T - S)
        assert P.within(got[:, H], lo, hi).all(), (H, P.outside_report(got[:, H], lo, hi))


# ---- 2. a long TINY session: SequenceLength 20 000 (the old cap for head_dim 32 was 17 056) --------------------------------

LONG_T = 20000
LONG_PROMPT = 17060          # chunked prefill just past the old cap
LONG_CHUNK = 2048
LONG_STEPS = 16
# FAST distance from the oracle of the tensor-core prefill chunks, bf16 ulps of the element (floor 2^-6 of the largest
# magnitude), pinned at about 1.5x the largest measured on an H100 SXM (80 GB): last-row logits 75.4.  The decode steps that
# follow are compared bit for bit with the oracle run in FAST's streamed order on the caches the prefill left.
LONG_FAST_ULPS = dict(prefill=112)


def _ulps(got, exp):
    g, e = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    floor = 2.0 ** -6 * max(np.abs(e).max(), 2.0 ** -100)
    return np.abs(g - e) / 2.0 ** (np.floor(np.log2(np.maximum(np.abs(e), floor))) - 7)


@pytest.fixture(scope="module")
def tiny_long(L):
    """TINY with max_seq_len 20 000 and the oracle's chunked prefill to 17 060 tokens plus 16 greedy decode steps"""
    args = dict(L.synth.TINY, max_seq_len=LONG_T)
    tensors = host_tensors(args, SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    prompt = np.random.default_rng(2024).integers(0, args["vocab_size"], size=LONG_PROMPT).astype(np.int32)
    osess = om.new_session(LONG_T)
    ref = {"prefill": [], "decode": [], "ids": []}
    pos = 0
    while pos < LONG_PROMPT:
        n = min(LONG_CHUNK, LONG_PROMPT - pos)
        lg = osess.forward(prompt[:n], 0, all_rows=False) if pos == 0 else osess.forward_chunk(prompt[pos:pos + n], pos, all_rows=False)
        ref["prefill"].append(lg)
        pos += n
    tok = O.argmax_f32(ref["prefill"][-1][0])
    for i in range(LONG_STEPS):
        ref["ids"].append(int(tok))
        lg = osess.forward(np.array([tok], np.int32), LONG_PROMPT + i)
        ref["decode"].append(lg)
        tok = O.argmax_f32(lg[0])
    ref["ids"].append(int(tok))
    end = LONG_PROMPT + LONG_STEPS
    ref["cache"] = {l: tuple(np.array(c[:end]) for c in osess.cache(l)) for l in (0, args["n_layers"] - 1)}
    osess.close()
    yield args, om, gm, prompt, ref
    gm.Free()
    om.close()


def _run_long(L, gm, prompt, acc):
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(0), max_rows=LONG_CHUNK, acc_mode=acc)
    ctx.allow_chunked_prefill(True)
    pre, dec, ids = [], [], []
    pos = 0
    while pos < LONG_PROMPT:
        n = min(LONG_CHUNK, LONG_PROMPT - pos)
        nxt, lg = gm.Transformer.forward_argmax(ctx, prompt[pos:pos + n], pos, want_logits="last")
        pre.append(lg)
        pos += n
    for i in range(LONG_STEPS):
        ids.append(nxt)
        nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([nxt], np.int32), LONG_PROMPT + i, want_logits="last")
        dec.append(lg)
    ids.append(nxt)
    return ctx, pre, dec, ids


def test_long_session_strict_bit_exact(L, tiny_long):
    args, _, gm, prompt, ref = tiny_long
    assert args["max_seq_len"] > _old_cap(args["head_dim"])
    ctx, pre, dec, ids = _run_long(L, gm, prompt, L._capi.LNB_ACC_STRICT)
    try:
        assert ctx.SequenceLength == LONG_T
        for i, (g, e) in enumerate(zip(pre, ref["prefill"])):
            assert np.array_equal(g, e), f"prefill chunk {i}"
        for i, (g, e) in enumerate(zip(dec, ref["decode"])):
            assert np.array_equal(g, e), f"decode step {i}"
        assert ids == ref["ids"]
        end = LONG_PROMPT + LONG_STEPS
        for layer, (ok, ov) in ref["cache"].items():
            assert np.array_equal(ctx.CacheK(layer).RawData[:end], ok), f"K cache, layer {layer}"
            assert np.array_equal(ctx.CacheV(layer).RawData[:end], ov), f"V cache, layer {layer}"
    finally:
        ctx.close()


def test_long_session_fast_within_pinned_ulps(L, tiny_long):
    """the chunked tensor-core prefill within LONG_FAST_ULPS of the oracle; then its caches are copied into an oracle session
    and the 16 greedy decode steps (streamed attention) must be that session's FAST streamed order bit for bit"""
    args, om, gm, prompt, ref = tiny_long
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(0), max_rows=LONG_CHUNK, acc_mode=L._capi.LNB_ACC_FAST)
    osess = om.new_session(LONG_T)
    try:
        ctx.allow_chunked_prefill(True)
        pre, pos = [], 0
        while pos < LONG_PROMPT:
            n = min(LONG_CHUNK, LONG_PROMPT - pos)
            nxt, lg = gm.Transformer.forward_argmax(ctx, prompt[pos:pos + n], pos, want_logits="last")
            pre.append(lg)
            pos += n
        m = max(_ulps(g, e).max() for g, e in zip(pre, ref["prefill"]))
        print(f"long TINY FAST: prefill {m:.2f}")
        assert m <= LONG_FAST_ULPS["prefill"], m
        for layer in range(args["n_layers"]):
            ok, ov = osess.cache(layer)
            ok[:LONG_PROMPT] = ctx.CacheK(layer).RawData[:LONG_PROMPT]
            ov[:LONG_PROMPT] = ctx.CacheV(layer).RawData[:LONG_PROMPT]
        for i in range(LONG_STEPS):
            tok = np.array([nxt], np.int32)
            exp = osess.forward(tok, LONG_PROMPT + i, order=O.ORDER_FAST_STREAM)
            nxt, lg = gm.Transformer.forward_argmax(ctx, tok, LONG_PROMPT + i, want_logits="last")
            assert np.array_equal(lg, exp), f"decode step {i}"
            assert nxt == O.argmax_f32(exp[0])
        end = LONG_PROMPT + LONG_STEPS
        for layer in (0, args["n_layers"] - 1):
            ok, ov = osess.cache(layer)
            assert np.array_equal(ctx.CacheK(layer).RawData[:end], ok[:end]), f"K cache, layer {layer}"
            assert np.array_equal(ctx.CacheV(layer).RawData[:end], ov[:end]), f"V cache, layer {layer}"
    finally:
        ctx.close(); osess.close()


def test_long_session_streams_from_position_zero(L, tiny_long):
    """routing is per session: a short prompt and decode steps from position 1 upward in the long session run the streamed
    kernel (three launches per layer instead of one) and give the oracle's bits"""
    args, om, gm, _, _ = tiny_long
    nl = args["n_layers"]
    prompt = np.array([5, 900, 17], np.int32)
    strict, fast = L._capi.LNB_ACC_STRICT, L._capi.LNB_ACC_FAST
    lng = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(0), max_rows=8, acc_mode=strict)
    osess = om.new_session(64)
    try:
        nxt, lg = gm.Transformer.forward_argmax(lng, prompt, 0, want_logits="last")
        assert np.array_equal(lg, osess.forward(prompt, 0, all_rows=False))
        for pos in range(3, 8):
            e = osess.forward(np.array([nxt], np.int32), pos)
            nxt, lg = gm.Transformer.forward_argmax(lng, np.array([nxt], np.int32), pos, want_logits="last")
            assert np.array_equal(lg, e), pos
        one = np.array([7], np.int32)
        counts = []
        for seq in (LONG_T, 136):
            ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=8, acc_mode=fast)
            try:
                gm.Transformer.forward_argmax(ctx, one, 0)
                n0 = ctx.launch_count()
                gm.Transformer.forward_argmax(ctx, one, 1)
                counts.append(ctx.launch_count() - n0)
            finally:
                ctx.close()
        assert counts[0] - counts[1] == 2 * nl, counts
    finally:
        lng.close(); osess.close()


# ---- 3. batched decode beyond sdpa_decode_kernel's fit: TINY128 at SequenceLength 1024 (old batched limit 351) --------------

@pytest.fixture(scope="module")
def t128(L):
    args = dict(L.synth.TINY128, max_seq_len=1024)
    tensors = host_tensors(args, SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    yield args, tensors, om, gm
    gm.Free()
    om.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_batched_decode_beyond_the_shared_memory_fit(L, t128, mode):
    """sequences prefilled to different lengths (some past 351) and stepped together; STRICT: every sequence bit-identical to
    its own oracle context, logits, greedy ids and caches; FAST: the prefill (the tensor-core path from 32 rows on) leaves
    caches that are copied into each sequence's oracle session, and every batched step (streamed attention) must be the
    oracle's FAST streamed order bit for bit"""
    args, _, om, gm = t128
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(99)
    lens = (3, 352, 351, 700, 40)
    prompts = [rng.integers(0, args["vocab_size"], size=k).astype(np.int32) for k in lens]
    nseq = len(prompts)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(0), max_rows=704, acc_mode=acc, n_seq=nseq)
    osess = [om.new_session(1024) for _ in range(nseq)]
    try:
        assert ctx.SequenceLength == 1024
        cur, pos = [], []
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            nxt, lg = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
            if mode == "strict":
                exp = osess[i].forward(p, 0, all_rows=False)
                assert np.array_equal(lg, exp)
                cur.append(int(np.argmax(exp[0])))
            else:
                for layer in range(args["n_layers"]):
                    ok, ov = osess[i].cache(layer)
                    ok[:len(p)] = ctx.CacheK(layer).RawData[:len(p)]
                    ov[:len(p)] = ctx.CacheV(layer).RawData[:len(p)]
                cur.append(int(nxt))
            pos.append(len(p))
        order = None if mode == "strict" else O.ORDER_FAST_STREAM
        for step in range(4):
            nxt, lg = ctx.forward_batch(cur, pos, want_logits=True)
            for i in range(nseq):
                exp = osess[i].forward(np.array([cur[i]], np.int32), pos[i], order=order)
                assert np.array_equal(lg[i], exp[0]), f"sequence {i} step {step}"
                assert nxt[i] == O.argmax_f32(exp[0])
                cur[i] = int(np.argmax(exp[0])); pos[i] += 1
        for i in range(nseq):
            ctx.set_active_sequence(i)
            for layer in range(args["n_layers"]):
                ok, ov = osess[i].cache(layer)
                assert np.array_equal(ctx.CacheK(layer).RawData[:pos[i]], ok[:pos[i]])
                assert np.array_equal(ctx.CacheV(layer).RawData[:pos[i]], ov[:pos[i]])
    finally:
        ctx.close()
        for o in osess:
            o.close()


def test_generate_tokens_batch_with_the_default_sequence_length(L, t128):
    """GenerateTokensBatch with SequenceLength left at its default (MaxSequenceLength 1024) equals per-prompt generation"""
    args, _, _, gm = t128
    prompts = [[1, 50, 999, 7, 300, 12, 64, 2], [5, 6, 7], [1000]]
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(), acc_mode=L._capi.LNB_ACC_STRICT)
    got = [[] for _ in prompts]
    for i, _, tok in eng.GenerateTokensBatch(prompts):
        got[i].append(tok)
    for i, p in enumerate(prompts):
        one = [t for _, t in eng.GenerateTokens(p)]
        assert got[i] == one, i
        assert len(one) >= 1


def test_cli_batched_generation_past_the_old_fit(L):
    """host/lnb_generate at SequenceLength 2048 with batch=3 on a checkpoint directory (max_seq_len 2048); for head_dim 32 the
    old batched limit was 1061.  A prefix of every stream equals the oracle's."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    args = dict(L.synth.TINY)
    om = oracle_model(args, host_tensors(args, 7))
    base = [1, 50, 999, 7, 300, 12, 64, 2]
    try:
        with tempfile.TemporaryDirectory() as d:
            subprocess.check_call([exe, "--write-synthetic", d, "tiny"])
            out = subprocess.run([exe, "2048", "strict", d, "batch=3"], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr
        for b in range(3):
            prompt = [base[0]] + [(t + 977 * b) % 1000 for t in base[1:]]
            line = [l for l in out.stdout.splitlines() if l.startswith(f"tokens[{b}]:")][0]
            got = [int(t) for t in line.split()[1:]]
            exp = list(om.generate(prompt, 64, stop_ids=(10**9,)))
            assert len(got) > len(exp) and got[:len(exp)] == exp, b
    finally:
        om.close()


# ---- 4. the 8B model at the full 131 072-token window -------------------------------------------------------------------

FULL = 131072


@pytest.fixture(scope="module")
def big_long(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 60 * 2 ** 30:
        pytest.skip("needs about 60 GB of free device memory")
    args = dict(L.synth.LLAMA31_8B, max_seq_len=FULL)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    yield args, gm
    gm.Free()


def test_8b_fast_full_window_prefill_and_decode(L, big_long):
    args, gm = big_long
    n_prompt, chunk = 100_352, 8192
    prompt = np.random.default_rng(3).integers(0, args["vocab_size"], size=n_prompt).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(FULL), max_rows=chunk, acc_mode=L._capi.LNB_ACC_FAST)
    try:
        ctx.allow_chunked_prefill(True)
        pos = 0
        while pos < n_prompt:
            n = min(chunk, n_prompt - pos)
            nxt, lg = gm.Transformer.forward_argmax(ctx, prompt[pos:pos + n], pos, want_logits="last")
            pos += n
        assert np.isfinite(lg).all()
        first = nxt
        runs = []
        for _ in range(2):                       # the same steps twice over the same cache rows: the same bits
            tok, ids, lgs = first, [], []
            for i in range(4):
                tok, lg = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), n_prompt + i, want_logits="last")
                assert np.isfinite(lg).all()
                ids.append(tok); lgs.append(lg)
            runs.append((ids, lgs))
        assert runs[0][0] == runs[1][0]
        assert all(np.array_equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
        toks, _, _ = ctx.decode_run(first, n_prompt, 4, use_graph=True)   # device-resident decode: the same greedy ids
        assert list(toks) == runs[0][0]
    finally:
        ctx.close()


def test_8b_strict_full_window_session(L, big_long):
    args, gm = big_long
    prompt = np.array(L.synth.PROMPT_8, np.int32)
    ids = []
    for _ in range(2):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(FULL), max_rows=8, acc_mode=L._capi.LNB_ACC_STRICT)
        try:
            nxt, lg = gm.Transformer.forward_argmax(ctx, prompt, 0, want_logits="last")
            out = [nxt]
            for i in range(4):
                nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([nxt], np.int32), len(prompt) + i, want_logits="last")
                assert np.isfinite(lg).all()
                out.append(nxt)
            ids.append(out)
        finally:
            ctx.close()
    assert ids[0] == ids[1]


def test_8b_batch_session_too_large_is_enomem(L, big_long):
    args, gm = big_long
    with pytest.raises(L._capi.LnbError) as e:
        L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(FULL), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST, n_seq=8)
    LNB_ENOMEM = -5   # include/lnb.h
    assert e.value.code == LNB_ENOMEM and "bytes" in str(e.value), str(e.value)
    print(f"8 x {FULL} positions: {e.value}")
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_FAST)
    try:
        nxt, lg = gm.Transformer.forward_argmax(ctx, np.array(L.synth.PROMPT_8, np.int32), 0, want_logits="last")
        assert np.isfinite(lg).all() and 0 <= nxt < args["vocab_size"]
    finally:
        ctx.close()


# ---- 5. no change inside today's limits ----------------------------------------------------------------------------------

# Launches of one step, measured on an H100 at the commit before the streamed kernel existed (TINY128, two layers).
# STRICT single-sequence decode runs the persistent engine (set_state + one launch); the rest is the kernel chain.
PINNED_LAUNCHES = {
    ("single136", "strict", "decode"): 2,
    ("single136", "fast", "decode"): 13,
    ("single136", "strict", "prompt"): 18,
    ("single136", "fast", "prompt"): 13,
    ("batch300", "strict", "batch"): 19,
    ("batch300", "fast", "batch"): 14,
}


def launch_counts(L, gm, om=None):
    """{key: launches of one step}; with the oracle, STRICT logits of every step are checked bit for bit"""
    out = {}
    prompt = np.array([1, 50, 999, 7, 300, 12, 64, 2], np.int32)
    for mode in ("strict", "fast"):
        acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=acc)
        osess = om.new_session(136) if om is not None else None
        try:
            n0 = ctx.launch_count()
            nxt, lg = gm.Transformer.forward_argmax(ctx, prompt, 0, want_logits="last")
            out[("single136", mode, "prompt")] = ctx.launch_count() - n0
            if osess is not None and mode == "strict":
                assert np.array_equal(lg, osess.forward(prompt, 0, all_rows=False))
            n0 = ctx.launch_count()
            tok = np.array([nxt], np.int32)
            nxt, lg = gm.Transformer.forward_argmax(ctx, tok, len(prompt), want_logits="last")
            out[("single136", mode, "decode")] = ctx.launch_count() - n0
            if osess is not None and mode == "strict":
                assert np.array_equal(lg, osess.forward(tok, len(prompt)))
        finally:
            ctx.close()
            if osess is not None:
                osess.close()
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(300), max_rows=8, acc_mode=acc, n_seq=3)
        osess = [om.new_session(300) for _ in range(3)] if om is not None else None
        try:
            cur = []
            for i in range(3):
                ctx.set_active_sequence(i)
                nxt, _ = gm.Transformer.forward_argmax(ctx, prompt[:3 + i], 0)
                if osess is not None:
                    osess[i].forward(prompt[:3 + i], 0, all_rows=False)
                cur.append(nxt)
            pos = [3, 4, 5]
            n0 = ctx.launch_count()
            _, lg = ctx.forward_batch(cur, pos, want_logits=True)
            out[("batch300", mode, "batch")] = ctx.launch_count() - n0
            if osess is not None and mode == "strict":
                for i in range(3):
                    assert np.array_equal(lg[i], osess[i].forward(np.array([cur[i]], np.int32), pos[i])[0]), i
        finally:
            ctx.close()
            if osess is not None:
                for o in osess:
                    o.close()
    return out


def test_launch_counts_and_bits_inside_todays_limits(L):
    args = dict(L.synth.TINY128)
    tensors = host_tensors(args, SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    try:
        got = launch_counts(L, gm, om)
    finally:
        gm.Free()
        om.close()
    print("launch counts: " + ", ".join(f"{'/'.join(k)} {v}" for k, v in sorted(got.items())))
    assert got == PINNED_LAUNCHES
