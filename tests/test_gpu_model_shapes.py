"""The forward at the model shapes of tests/model_shapes.py: GQA ratios 1, 2, 3, 8 and 16, head dims 48, 64, 96, 128 and
256, widths off the 128-wide tiles, unscaled RoPE and a single layer.  First the library must take the route the host
restatement names for each shape (decode engine or its refusal reason, batch engine, streamed kernels, tensor-core prompt
path), so the comparisons after it are never vacuous; then STRICT is bit for bit against the oracle on every route, FAST is
bit for bit against the oracle's FAST summation order wherever it sums on the FMA pipe, and the tensor-core routes keep
tiny128's pinned bounds.  Calls the restatement says a shape cannot serve must fail with LNB_EINVAL, enqueue nothing and
leave the session usable."""
import json
import os
import time

import numpy as np
import pytest

from oracle import oracle as O
from tests import model_shapes as M
from tests.helpers import f32, host_tensors, oracle_model
from tests.test_gpu_model import TC_ULPS, _tc_launches, _ulps

pytestmark = pytest.mark.gpu

SEED = 4321
NAMES = list(M.CATALOGUE)
SERVED = [n for n in NAMES if M.traits(n)["batched"] != "refused"]       # every call kind
CHAIN_ONLY = [n for n in NAMES if n not in SERVED]                         # hd256, rep16
STREAMED = [n for n in NAMES if M.traits(n)["streamed_batched"]]
TC = [n for n in NAMES if M.traits(n)["prompt_tc"]]
REF, TREE, STREAM = None, O.ORDER_FAST, O.ORDER_FAST_STREAM
SEQ = 64

_WALL = {}


@pytest.fixture(autouse=True)
def _wall_time(request):
    t0 = time.perf_counter()
    yield
    _WALL[request.node.name] = time.perf_counter() - t0


def teardown_module(module):
    print("\nwall time per test (s): " + ", ".join(f"{k} {v:.1f}" for k, v in _WALL.items()) +
          f"\nwall time, all tests: {sum(_WALL.values()):.1f} s")


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module")
def models(L):
    """name -> (args, host tensors, oracle model, GPU model), loaded on first use"""
    cache = {}

    def get(name):
        if name not in cache:
            args = dict(M.CATALOGUE[name])
            tensors = host_tensors(args, SEED)
            cache[name] = (args, tensors, oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors))
        return cache[name]
    yield get
    for _, _, om, gm in cache.values():
        gm.Free()
        om.close()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _eq(got, exp, what):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    assert np.array_equal(got, exp), f"{what}: {(got != exp).sum()} of {got.size} differ"


def _caches_eq(ctx, osess, n_layers, rows, what):
    for layer in range(n_layers):
        ok, ov = osess.cache(layer)
        _eq(ctx.CacheK(layer).RawData[:rows], ok[:rows], f"{what}: K cache, layer {layer}")
        _eq(ctx.CacheV(layer).RawData[:rows], ov[:rows], f"{what}: V cache, layer {layer}")


def _ctx(L, gm, seq, mode, max_rows=8, n_seq=1):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)


def _toks(args, seed, n):
    return np.random.default_rng(seed).integers(0, args["vocab_size"], size=n).astype(np.int32)


def _one(t):
    return np.array([t], np.int32)


def _engine_env(monkeypatch, engine=None, batch=None):
    for var, val in (("LNB_ENGINE", engine), ("LNB_BATCH_ENGINE", batch)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)
    monkeypatch.delenv("LNB_BATCH_TC", raising=False)
    monkeypatch.delenv("LNB_SDPA_TC", raising=False)


# ---- 1. route evidence ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_routes_are_the_restatements(L, models, sms, name, monkeypatch):
    """the decode engine or its refusal reason (STRICT, FAST with LNB_ENGINE=1, LNB_ENGINE=0), one batch-engine launch per
    batched step where the batch engine runs, two more launches per layer for a batched step past sdpa_decode_kernel's fit
    (the streamed kernels), the tensor-core prompt path's launch count and sdpa_tc_kernel's own bits"""
    args, _, _, gm = models(name)
    nl = args["n_layers"]
    for mode, env in (("strict", None), ("fast", "1"), ("strict", "0"), ("fast", None)):
        _engine_env(monkeypatch, engine=env)
        ctx = _ctx(L, gm, SEQ, mode)
        try:
            want = M.uses_engine(args, SEQ, mode == "strict", sms, env)
            assert ctx.uses_engine() == want, (mode, env)
            if not want:
                why = M.engine_refusal(args, SEQ, mode == "strict", sms, env) or "single-GPU FAST: the kernel chain is the default"
                assert L._capi.lib.lnb_last_error().decode() == why, (mode, env)
        finally:
            ctx.close()
    if name in SERVED:
        for mode in ("strict", "fast"):
            _engine_env(monkeypatch)
            ctx = _ctx(L, gm, SEQ, mode, n_seq=3)
            try:
                ctx.forward_batch([1, 2, 3], [0, 0, 0])
                l0 = ctx.launch_count()
                ctx.forward_batch([4, 5, 6], [1, 1, 1])
                n = ctx.launch_count() - l0
                assert (n == 1) == M.batch_engine(args, SEQ, mode == "strict", sms), (mode, n)
            finally:
                ctx.close()
    if name in STREAMED:
        _engine_env(monkeypatch, batch="0")
        fit = M.sdpa_decode_fit(args)
        counts = []
        for seq in (fit, fit + 1):
            assert M.engine_refusal(args, seq, True, sms) is not None      # past the engines' attention limit, or stories
            ctx = _ctx(L, gm, seq, "strict", n_seq=3)
            try:
                ctx.forward_batch([1, 2, 3], [0, 0, 0])
                l0 = ctx.launch_count()
                ctx.forward_batch([4, 5, 6], [1, 1, 1])
                counts.append(ctx.launch_count() - l0)
            finally:
                ctx.close()
        assert counts[1] - counts[0] == 2 * nl, counts
    if name in TC:
        _engine_env(monkeypatch)
        toks = _toks(args, 5, 40)
        ctx = _ctx(L, gm, SEQ, "fast", max_rows=40)
        try:
            l0 = ctx.launch_count()
            _, a = gm.Transformer.forward_argmax(ctx, toks, 0, want_logits="all")
            assert ctx.launch_count() - l0 == _tc_launches(nl, 40, True)
            monkeypatch.setenv("LNB_SDPA_TC", "0")
            _, b = gm.Transformer.forward_argmax(ctx, toks, 0, want_logits="all")
            # sdpa_tc_kernel and sdpa_prefill_kernel sum in different orders: different bits where head_dim 128 selects them
            assert np.array_equal(a, b) == (M.traits(name)["prompt_attention"] != "sdpa_tc")
        finally:
            ctx.close()


# ---- 2. STRICT, bit for bit -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("engine", [None, "0"])
def test_strict_prefill_and_host_driven_decode(L, models, sms, name, engine, monkeypatch):
    """prefills of 1, 7 and 40 rows (every row's logits and every layer's caches), then six host-driven S = 1 steps on the
    default route (the decode engine where it runs) or the kernel chain (LNB_ENGINE=0)"""
    _engine_env(monkeypatch, engine=engine)
    args, _, om, gm = models(name)
    nl = args["n_layers"]
    for S in (1, 7, 40):
        toks = _toks(args, S, S)
        ctx, osess = _ctx(L, gm, SEQ, "strict", max_rows=40), om.new_session(SEQ)
        try:
            assert ctx.uses_engine() == M.uses_engine(args, SEQ, True, sms, engine)
            nxt, lg = gm.Transformer.forward_argmax(ctx, toks, 0, want_logits="all")
            exp = osess.forward(toks, 0, all_rows=True)
            _eq(lg, exp, f"prefill S={S}")
            assert nxt == O.argmax_f32(exp[-1])
            _caches_eq(ctx, osess, nl, S, f"prefill S={S}")
            if S != 7:
                continue
            tok = nxt
            for pos in range(7, 13):
                nxt, lg = gm.Transformer.forward_argmax(ctx, _one(tok), pos, want_logits="last")
                exp = osess.forward(_one(tok), pos)
                _eq(lg, exp, f"step at {pos}")
                assert nxt == O.argmax_f32(exp[0])
                tok = nxt
            _caches_eq(ctx, osess, nl, 13, "after the steps")
        finally:
            ctx.close(); osess.close()


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("use_graph", [False, True])
def test_strict_device_resident_decode(L, models, name, use_graph, monkeypatch):
    _engine_env(monkeypatch)
    args, _, om, gm = models(name)
    prompt = _toks(args, 11, 7)
    ctx, osess = _ctx(L, gm, SEQ, "strict"), om.new_session(SEQ)
    try:
        first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        tok = O.argmax_f32(osess.forward(prompt, 0, all_rows=False)[0])
        assert first == tok
        want = []
        for pos in range(7, 7 + 12):
            tok = O.argmax_f32(osess.forward(_one(tok), pos)[0])
            want.append(tok)
        toks, _, graphed = ctx.decode_run(first, 7, 12, use_graph=use_graph)
        assert list(toks) == want
        _caches_eq(ctx, osess, args["n_layers"], 7 + 12, "caches")
    finally:
        ctx.close(); osess.close()


def _batched(L, args, om, gm, mode, seq, order, n_steps, seed, engine, prefill_order=None):
    """3 sequences prefilled to different lengths, then n_steps batched steps: every row's logits and greedy id, every
    sequence's caches (STRICT, or FAST with the prompts in `prefill_order` and the batched rows in `order`).  engine: the
    batch engine runs each step as its one launch (else the kernel chain)"""
    lens = [3, 7, 1]
    prompts = [_toks(args, seed + i, k) for i, k in enumerate(lens)]
    ctx = _ctx(L, gm, seq, mode, n_seq=3)
    osess = [om.new_session(seq) for _ in range(3)]
    try:
        cur, pos = [], []
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            nxt, lg = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
            exp = osess[i].forward(p, 0, all_rows=False, order=prefill_order or order)
            _eq(lg, exp, f"prefill of sequence {i}")
            cur.append(nxt); pos.append(len(p))
        for step in range(n_steps):
            l0 = ctx.launch_count()
            nxt, lg = ctx.forward_batch(cur, pos, want_logits=True)
            assert (ctx.launch_count() - l0 == 1) == engine, (step, ctx.launch_count() - l0)
            for i in range(3):
                exp = osess[i].forward(_one(cur[i]), pos[i], order=order)
                _eq(lg[i], exp[0], f"sequence {i} step {step}")
                assert nxt[i] == O.argmax_f32(exp[0])
            cur = [int(t) for t in nxt]; pos = [p + 1 for p in pos]
        for i in range(3):
            ctx.set_active_sequence(i)
            _caches_eq(ctx, osess[i], args["n_layers"], pos[i], f"sequence {i}")
    finally:
        ctx.close()
        for o in osess:
            o.close()


@pytest.mark.parametrize("name", SERVED)
@pytest.mark.parametrize("batch", [None, "0"])
def test_strict_batched_decode(L, models, sms, name, batch, monkeypatch):
    """lnb_forward_batch of 3 sequences on the batch engine (where it runs) and on the kernel chain (LNB_BATCH_ENGINE=0)"""
    _engine_env(monkeypatch, batch=batch)
    args, _, om, gm = models(name)
    _batched(L, args, om, gm, "strict", SEQ, REF, 6, 100, M.batch_engine(args, SEQ, True, sms, batch_env=batch))


@pytest.mark.parametrize("name", STREAMED)
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_batched_decode_just_past_the_decode_kernel_fit(L, models, name, mode, monkeypatch):
    """a SequenceLength one past sdpa_decode_kernel's fit: batched rows run the streamed kernels at this shape's n_rep (the
    engines' attention limit is shorter still); STRICT bit for bit, FAST in the streamed order"""
    _engine_env(monkeypatch)
    args, _, om, gm = models(name)
    seq = M.sdpa_decode_fit(args) + 1
    assert M.attention_kernel(args, seq, "batched", 3) == "stream" and M.engine_refusal(args, seq, mode == "strict") is not None
    # the prompts run sdpa_kernel (the session does not stream every row): the FAST tree order
    _batched(L, args, om, gm, mode, seq, REF if mode == "strict" else STREAM, 3, 200, False, REF if mode == "strict" else TREE)


@pytest.mark.parametrize("name", SERVED)
def test_strict_ragged_speculative_and_chunked(L, models, sms, name, monkeypatch):
    """a ragged call of prompts, a prompt chunk and a decode row (the streamed kernels); a 4-row speculative call (the batch
    engine where it runs, else sdpa_decode_kernel on the chain); a prompt prefilled in chunks of 7, 20 and 13"""
    _engine_env(monkeypatch)
    args, _, om, gm = models(name)
    nl = args["n_layers"]
    # ragged
    ctx = _ctx(L, gm, SEQ, "strict", max_rows=31, n_seq=3)
    osess = [om.new_session(SEQ) for _ in range(3)]
    try:
        calls = [[(0, _toks(args, 1, 7)), (1, _toks(args, 2, 5))], [(0, None), (1, _toks(args, 3, 3)), (2, _toks(args, 4, 9))]]
        pos, last = [0, 0, 0], {}
        for call in calls:
            segs = [(s, pos[s], _one(last[s]) if tk is None else tk) for s, tk in call]
            nxt, lg = ctx.forward_ragged(segs, want_logits=True)
            for i, (s, p, tk) in enumerate(segs):
                if p == 0:
                    exp = osess[s].forward(tk, 0, all_rows=False)
                elif len(tk) > 1:
                    exp = osess[s].forward_chunk(tk, p, all_rows=False)
                else:
                    exp = osess[s].forward(tk, p)
                _eq(lg[i], exp[0], f"ragged segment {i} (sequence {s} at {p})")
                assert nxt[i] == O.argmax_f32(exp[0])
                pos[s] += len(tk); last[s] = int(nxt[i])
        for s in range(3):
            ctx.set_active_sequence(s)
            _caches_eq(ctx, osess[s], nl, pos[s], f"ragged, sequence {s}")
    finally:
        ctx.close()
        for o in osess:
            o.close()
    # speculative: a draft right twice, then wrong
    prompt = _toks(args, 23, 8)
    ctx, osess, plain = _ctx(L, gm, SEQ, "strict"), om.new_session(SEQ), om.new_session(SEQ)
    try:
        t0, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        osess.forward(prompt, 0, all_rows=False)
        greedy, tok = [], O.argmax_f32(plain.forward(prompt, 0, all_rows=False)[0])
        assert tok == t0
        for p in range(8, 11):
            tok = O.argmax_f32(plain.forward(_one(tok), p)[0])
            greedy.append(tok)
        rows = np.array([t0, greedy[0], greedy[1], (greedy[2] + 1) % args["vocab_size"]], np.int32)
        l0 = ctx.launch_count()
        nxt, acc, lg = ctx.forward_speculative([(0, 8, rows)], want_logits=True)
        assert (ctx.launch_count() - l0 == 1) == M.batch_engine(args, SEQ, True, sms)
        exp = osess.forward_chunk(rows, 8, all_rows=True)
        _eq(lg, exp, "speculative rows")
        assert [int(t) for t in nxt] == [O.argmax_f32(e) for e in exp] and int(acc[0]) == 2
        _caches_eq(ctx, osess, nl, 12, "speculative")
    finally:
        ctx.close(); osess.close(); plain.close()
    # chunked prefill
    prompt = _toks(args, 40, 40)
    ctx, osess = _ctx(L, gm, SEQ, "strict", max_rows=20), om.new_session(SEQ)
    try:
        ctx.allow_chunked_prefill(True)
        p = 0
        for size in (7, 20, 13):
            _, lg = gm.Transformer.forward_argmax(ctx, prompt[p:p + size], p, want_logits="all")
            exp = osess.forward(prompt[:size], 0, all_rows=True) if p == 0 else osess.forward_chunk(prompt[p:p + size], p)
            _eq(lg, exp, f"chunk at {p}")
            p += size
        _caches_eq(ctx, osess, nl, 40, "chunked")
    finally:
        ctx.close(); osess.close()


@pytest.mark.parametrize("name", CHAIN_ONLY)
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_refused_calls_enqueue_nothing_and_leave_the_session_usable(L, models, name, mode, monkeypatch):
    """head_dim 256 / n_rep 16: batched, ragged and speculative calls fail with LNB_EINVAL before any launch, a session
    past sdpa_kernel's SequenceLength is refused, and the session's next S = 1 step has the oracle's bits (STRICT) / FAST
    order bits"""
    _engine_env(monkeypatch)
    args, _, om, gm = models(name)
    order = REF if mode == "strict" else TREE
    last = (M.SMEM_200K - args["head_dim"] * 4) // 12
    with pytest.raises(L._capi.LnbError, match="streamed attention kernel") as e:
        _ctx(L, gm, last + 1, mode)
    assert e.value.code == -1
    ctx, osess = _ctx(L, gm, SEQ, mode, max_rows=8, n_seq=3), om.new_session(SEQ)
    try:
        prompt = _toks(args, 9, 5)
        tok, lg = gm.Transformer.forward_argmax(ctx, prompt, 0, want_logits="last")
        _eq(lg, osess.forward(prompt, 0, all_rows=False, order=order), "prefill")
        calls = [lambda: ctx.forward_batch([1, 2], [0, 0]),
                 lambda: ctx.forward_ragged([(1, 0, _toks(args, 1, 3)), (2, 0, _toks(args, 2, 2))]),
                 lambda: ctx.forward_speculative([(0, 5, np.array([tok, 7, 8], np.int32))])]
        for i, call in enumerate(calls):
            l0 = ctx.launch_count()
            with pytest.raises(L._capi.LnbError) as e:
                call()
            assert e.value.code == -1, (i, str(e.value))
            assert "n_rep <= 8" in str(e.value), (i, str(e.value))
            assert ctx.launch_count() == l0, f"call {i} enqueued work"
        for pos in range(5, 8):
            nxt, lg = gm.Transformer.forward_argmax(ctx, _one(tok), pos, want_logits="last")
            exp = osess.forward(_one(tok), pos, order=order)
            _eq(lg, exp, f"step at {pos}")
            tok = nxt
        _caches_eq(ctx, osess, args["n_layers"], 8, "caches")
    finally:
        ctx.close(); osess.close()


# ---- 3. FAST on the FMA pipe, bit for bit against the oracle's FAST order ---------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_fast_fma_routes_equal_the_fast_order(L, models, sms, name, monkeypatch):
    """a 9-row prompt (and a 40-row one where the shape keeps prompts off the tensor cores), S = 1 steps on the kernel chain
    and with LNB_ENGINE=1, then (where served) batched steps and a speculative call"""
    args, _, om, gm = models(name)
    nl = args["n_layers"]
    for engine in (None, "1"):
        _engine_env(monkeypatch, engine=engine)
        ctx, osess = _ctx(L, gm, SEQ, "fast", max_rows=40), om.new_session(SEQ)
        try:
            assert ctx.uses_engine() == M.uses_engine(args, SEQ, False, sms, engine)
            S = 9 if engine is None or M.traits(name)["prompt_tc"] else 40
            prompt = _toks(args, 70 + S, S)
            tok, lg = gm.Transformer.forward_argmax(ctx, prompt, 0, want_logits="all")
            _eq(lg, osess.forward(prompt, 0, all_rows=True, order=TREE), f"prompt of {S}")
            for pos in range(S, S + 6):
                nxt, lg = gm.Transformer.forward_argmax(ctx, _one(tok), pos, want_logits="last")
                exp = osess.forward(_one(tok), pos, order=TREE)
                _eq(lg, exp, f"step at {pos}")
                assert nxt == O.argmax_f32(exp[0])
                tok = nxt
            _caches_eq(ctx, osess, nl, S + 6, "caches")
        finally:
            ctx.close(); osess.close()
    if name not in SERVED:
        return
    _engine_env(monkeypatch)
    _batched(L, args, om, gm, "fast", SEQ, TREE, 4, 300, M.batch_engine(args, SEQ, False, sms))
    prompt = _toks(args, 24, 8)
    ctx, osess = _ctx(L, gm, SEQ, "fast"), om.new_session(SEQ)
    try:
        t0, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        assert t0 == O.argmax_f32(osess.forward(prompt, 0, all_rows=False, order=TREE)[0])
        rows = np.array([t0, 5, 6, 7], np.int32)
        nxt, _, lg = ctx.forward_speculative([(0, 8, rows)], want_logits=True)
        exp = osess.forward_chunk(rows, 8, all_rows=True, order=TREE)
        _eq(lg, exp, "speculative rows")
        _caches_eq(ctx, osess, nl, 12, "speculative")
    finally:
        ctx.close(); osess.close()


# ---- 4. FAST on the tensor cores: tiny128's pinned bounds -------------------------------------------------------------------

@pytest.mark.parametrize("name", TC)
def test_fast_tensor_core_prompt(L, models, name, monkeypatch):
    """a 40-row FAST prompt on the tensor cores within TC_ULPS of the oracle (logits, caches, decode steps on its caches);
    rows do not depend on later rows; 40 + 33 rows in chunks equal the 73-row one-shot prefill bit for bit"""
    _engine_env(monkeypatch)
    args, _, om, gm = models(name)
    nl = args["n_layers"]
    toks = _toks(args, 41, 77)
    ctx, osess = _ctx(L, gm, 80, "fast", max_rows=40), om.new_session(80)
    try:
        exp = osess.forward(toks[:40], 0, all_rows=True)
        _, got = gm.Transformer.forward_argmax(ctx, toks[:40], 0, want_logits="all")
        m = dict(logits=_ulps(got, exp).max(), cache=0.0, decode=0.0)
        for layer in range(nl):
            ok, ov = osess.cache(layer)
            m["cache"] = max(m["cache"], _ulps(f32(ctx.CacheK(layer).RawData[:40]), f32(ok[:40])).max(),
                             _ulps(f32(ctx.CacheV(layer).RawData[:40]), f32(ov[:40])).max())
        for pos in range(40, 44):
            e = osess.forward(toks[pos:pos + 1], pos)
            g = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[pos:pos + 1], L.ml.DT_INT32), pos).RawData
            m["decode"] = max(m["decode"], _ulps(g, e).max())
        print(f"{name} S=40: " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(m.items())))
        for k, v in m.items():
            assert v <= TC_ULPS[k], (k, v)
    finally:
        ctx.close(); osess.close()
    a, b = _ctx(L, gm, 80, "fast", max_rows=33), _ctx(L, gm, 80, "fast", max_rows=73)
    chk = _ctx(L, gm, 80, "fast", max_rows=40)
    try:
        _, la = gm.Transformer.forward_argmax(a, toks[:33], 0, want_logits="all")
        _, lb = gm.Transformer.forward_argmax(b, toks[:73], 0, want_logits="all")
        for layer in range(nl):
            _eq(a.CacheK(layer).RawData[:33], b.CacheK(layer).RawData[:33], f"K cache, layer {layer}")
            _eq(a.CacheV(layer).RawData[:33], b.CacheV(layer).RawData[:33], f"V cache, layer {layer}")
        _eq(a.residual(33), b.residual(73)[:33], "residual")
        _eq(la[:32], lb[:32], "logits")
        chk.allow_chunked_prefill(True)
        _, l1 = gm.Transformer.forward_argmax(chk, toks[:40], 0, want_logits="all")
        _, l2 = gm.Transformer.forward_argmax(chk, toks[40:73], 40, want_logits="all")
        _eq(l1[:-1], lb[:39], "first chunk")
        _eq(l2, lb[40:73], "second chunk")
        for layer in range(nl):
            _eq(chk.CacheK(layer).RawData[:73], b.CacheK(layer).RawData[:73], f"chunked K cache, layer {layer}")
            _eq(chk.CacheV(layer).RawData[:73], b.CacheV(layer).RawData[:73], f"chunked V cache, layer {layer}")
    finally:
        a.close(); b.close(); chk.close()


@pytest.mark.parametrize("name", [n for n in SERVED if M.batch_engine(M.CATALOGUE[n], SEQ, False)])
def test_batch_engine_tensor_core_form(L, models, name, monkeypatch):
    """LNB_BATCH_TC=1: three sequences' batched steps within 1e-2 of the oracle"""
    _engine_env(monkeypatch)
    monkeypatch.setenv("LNB_BATCH_TC", "1")
    args, _, om, gm = models(name)
    ctx = _ctx(L, gm, SEQ, "fast", n_seq=3)
    osess = [om.new_session(SEQ) for _ in range(3)]
    try:
        cur, pos = [], []
        for i, k in enumerate((3, 7, 1)):
            p = _toks(args, 400 + i, k)
            ctx.set_active_sequence(i)
            gm.Transformer.forward_argmax(ctx, p, 0)
            cur.append(O.argmax_f32(osess[i].forward(p, 0, all_rows=False)[0])); pos.append(k)
        for step in range(4):
            l0 = ctx.launch_count()
            _, lg = ctx.forward_batch(cur, pos, want_logits=True)
            assert ctx.launch_count() - l0 == 1
            for i in range(3):
                exp = osess[i].forward(_one(cur[i]), pos[i])
                assert np.abs(lg[i] - exp[0]).max() <= 1e-2, (i, step)
                cur[i] = O.argmax_f32(exp[0]); pos[i] += 1
    finally:
        ctx.close()
        for o in osess:
            o.close()


# ---- 5. params.json round trip ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_params_json_round_trip(L, models, name, tmp_path):
    """params.json + consolidated.00.pth of the shape, LoadModel'ed: one STRICT forward with the bits of the model loaded
    from the same tensors, and of the oracle"""
    import torch
    args, tensors, om, gm = models(name)
    (tmp_path / "params.json").write_text(json.dumps(M.params_json(args)))
    torch.save({k: torch.from_numpy(v.view(np.int16)).view(torch.bfloat16) for k, v in tensors.items()},
               str(tmp_path / "consolidated.00.pth"))
    lm = L.model.LoadModel(str(tmp_path), max_seq_len=args["max_seq_len"])
    try:
        d = lm.Transformer.args
        assert (d.Dim, d.N_Heads, d.N_KVHeads, d.HeadDim, d.FFNDim, d.VocabSize) == \
            (args["dim"], args["n_heads"], args["n_kv_heads"], args["head_dim"], args["ffn_dim"], args["vocab_size"])
        toks = _toks(args, 50, 6)
        outs = []
        for m in (lm, gm):
            ctx = _ctx(L, m, SEQ, "strict")
            try:
                outs.append(m.Transformer.forward_argmax(ctx, toks, 0, want_logits="all")[1])
            finally:
                ctx.close()
        _eq(outs[0], outs[1], "LoadModel vs LoadModelFromTensors")
        osess = om.new_session(SEQ)
        try:
            _eq(outs[0], osess.forward(toks, 0, all_rows=True), "LoadModel vs the oracle")
        finally:
            osess.close()
    finally:
        lm.Free()
        os.remove(tmp_path / "consolidated.00.pth")
