"""The token pipeline after the LM head -- penalties, grammar mask, sampler or greedy slot, logprob records -- at real
vocabulary sizes, where each job splits a row into many 4096-logit CTAs and the last one is partial.  TINY widths with
32 000 (Llama 2) and 128 256 (Llama 3) tokens keep the CPU oracle cheap.  The ops against their C statements on the row
classes of tests/vocab_rows.py, both sampler kernels in one launch; STRICT streams of one sequence with every control on
every path, and of eight sequences with eight different controls in one call, against the oracle's statement; FAST calls
against the statement applied to the rows they returned; beams; and an MXFP8 prompt whose LM head runs in 125 full row
slices and a partial one."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import vocab_rows as VR
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 4321
SEQ_LEN = 32
PATTERN = r"[a-z ]{1,5}"   # one byte per token here: five letters reach the state whose mask is the stop set alone
PROMPT = [1, 50, 999, 7, 300, 12, 64, 2]
PROMPTS = [PROMPT, [5, 6, 5, 6, 5], [900, 3, 4, 17, 22, 3, 4], [8], [77, 31, 400], [1, 50, 999, 7], [300, 12], [64, 2, 9]]
TOP_N = 20


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _ptr(L, a, t):
    return L._capi.ptr(a, t)


# ---- the ops ------------------------------------------------------------------------------------------------------------
def _sample_op(L, rows, params, pos):
    rows = np.ascontiguousarray(rows, np.float32)
    n, V = rows.shape
    p = (L._capi.SamplingC * n)(*[L._capi.SamplingC(float(t), int(k), float(q), int(s) & (2**64 - 1)) for t, k, q, s in params])
    pn = np.ascontiguousarray(pos, np.int32)
    out = np.empty(n, np.int32)
    L._capi.check(L._capi.lib.lnb_op_sample_f32(_ptr(L, rows, L._capi.f32p), n, V, p, _ptr(L, pn, L._capi.i32p),
                                                _ptr(L, out, L._capi.i32p)))
    return out


@pytest.mark.parametrize("V", VR.VOCABS)
def test_sample_op_mixes_both_kernels_bit_exact(L, V):
    rng = np.random.default_rng(V)
    chunks = VR.interleaved(VR.cases(rng, V))
    hit = set()
    for chunk in chunks:
        got = _sample_op(L, np.stack([c[1] for c in chunk]), [c[2] for c in chunk], [c[3] for c in chunk])
        for g, (name, row, (T, K, P, s), pn) in zip(got, chunk):
            assert g == SR.sample_row(row, T, K, P, s, pn), (V, name, T, K, P, s, pn, g)
            hit.add("split" if VR.split_k(T, K, V) else ("full" if T > 0 else "greedy"))
    assert hit == {"split", "full", "greedy"}
    # the split kernel's counters are reset by the last CTA: the same launch again gives the same tokens
    chunk = chunks[0]
    a = _sample_op(L, np.stack([c[1] for c in chunk]), [c[2] for c in chunk], [c[3] for c in chunk])
    assert list(a) == [SR.sample_row(c[1], *c[2], c[3]) for c in chunk]


def _penalize_op(L, rows, params, hist, pos_next):
    rows = np.ascontiguousarray(rows, np.float32)
    n, V = rows.shape
    h = np.ascontiguousarray(hist, np.int32)
    pn = np.ascontiguousarray(pos_next, np.int32)
    par = (L._capi.PenaltiesC * n)(*[L._capi.PenaltiesC.from_buffer_copy(bytes(p)) for p in params])
    out = np.empty_like(rows)
    L._capi.check(L._capi.lib.lnb_op_penalize_f32(_ptr(L, rows, L._capi.f32p), n, V, par, _ptr(L, h, L._capi.i32p), h.shape[1],
                                                  _ptr(L, pn, L._capi.i32p), _ptr(L, out, L._capi.f32p)))
    return out


def _edge_tokens(V):
    return [t for t in (0, 4095, 4096, 8191, 8192, V - 2, V - 1) if t < V]


@pytest.mark.parametrize("V", [32000, 128256])
def test_penalize_op_biases_at_slice_edges(L, V):
    rng = np.random.default_rng(V + 5)
    n, T = 8, 512
    rows = rng.normal(0, 3, (n, V)).astype(np.float32)
    edges = _edge_tokens(V)
    hist = rng.choice(edges + list(rng.integers(0, V, 8)), size=(n, T)).astype(np.int32)   # the edge tokens are counted too
    params = []
    for r in range(n):
        vals = [float(rng.uniform(-6, 6)) if (r + j) % 3 else -np.inf for j in range(len(edges))]
        params.append(SR.penalties([1.0, 1.3, 0.7][r % 3], 0.3 * (r % 2), 0.2, [0, 64][r % 2], r, dict(zip(edges, vals))))
    params[3] = SR.penalties(bias={V - 1: -np.inf, 4096: -np.inf, 4095: 5.0})   # a bias only: counts off, biases alone
    rows[5, 4090:4100] = np.float32(7.0)                                          # ties straddling the edge the biases sit on
    pn = [T, T - 1, 17, T, 0, T, 300, T]
    got = _penalize_op(L, rows, params, hist, pn)
    exp = SR.penalize_rows(rows, params, hist, pn)
    for r in range(n):
        bad = np.flatnonzero(got[r].view(np.uint32) != exp[r].view(np.uint32))
        assert bad.size == 0, (V, r, bad[:8], got[r][bad[:8]], exp[r][bad[:8]])
        assert np.isneginf(got[r][[t for t, b in zip(params[r].bias_token, params[r].bias[:params[r].n_bias]) if b == -np.inf]]).all()


# ---- models with a real vocabulary ----------------------------------------------------------------------------------------
class Model:
    def __init__(self, L, V, tmp):
        self.V = V
        self.args = dict(L.synth.TINY, vocab_size=V)
        tensors = host_tensors(self.args, SEED)
        self.om, self.gm = oracle_model(self.args, tensors), L.model.LoadModelFromTensors(self.args, tensors)
        path = os.path.join(tmp, f"tokenizer_{V}.model")
        L._capi.check(L._capi.lib.lnb_vocab_write_synthetic(path.encode(), V - 256))
        self.vocab = L.vocabulary.Load(path)
        self.gm.Vocabulary = self.vocab          # stop tokens = the grammar's Z, in the last slice
        self.tok = L.model.vocabulary_token_bytes(self.vocab, V)
        self.stop = list(self.vocab.StopTokenIds)
        trans, accept = L.model.regex_dfa(PATTERN)
        self.tables = SR.GrammarTables(trans, accept, self.tok, self.stop)
        self.masks, _ = SR.grammar_masks(self.tables)
        self.grammar = L.model.Grammar(self.gm, PATTERN, self.vocab)

    def allowed(self, q):
        bits = self.masks[q if q >= 0 else self.tables.Q]
        i = np.arange(self.V)
        return ((bits[i >> 5] >> (i & 31).astype(np.uint32)) & 1).astype(bool)

    def close(self):
        self.grammar.close()
        self.gm.Free()
        self.om.close()


@pytest.fixture(scope="module", params=[32000, 128256])
def model(L, request, tmp_path_factory):
    m = Model(L, request.param, str(tmp_path_factory.mktemp("vocab")))
    assert all(VR.slices_of([t], m.V) == {VR.slices(m.V) - 1} for t in m.stop)
    yield m
    m.close()


def _pen(L, V):
    bias = {4095: 1.5, 4096: -np.inf, 8191: 2.0, V - 1: -np.inf, ord("e"): 2.5, ord("x"): -np.inf}
    return L.model.PenaltyArgs(1.3, 0.4, 0.2, LogitBias=bias)


def _opens(pen, prompt_len):
    return None if pen is None else SR.Penalties.from_buffer_copy(bytes(pen.c(prompt_len)))


def _want(m, prompt, samp, pen, grammar, seq_len, seed_off=0):
    T, K, P, seed = (samp.Temperature, samp.TopK, samp.TopP, samp.Seed) if samp else (0.0, 0, 1.0, 0)
    op = _opens(pen, len(prompt))
    if grammar:
        return list(SR.generate_constrained(m.om, prompt, seq_len, T, K, P, seed + seed_off, op, m.tables, len(prompt),
                                            stop_ids=m.stop))
    return list(SR.generate_processed(m.om, prompt, seq_len, T, K, P, seed + seed_off, op, stop_ids=m.stop))


def _oracle_records(m, prompt, stream, top_n):
    """the statement's records on the oracle's raw logits, teacher-forced along the stream"""
    sess = m.om.new_session(SEQ_LEN)
    rows = [sess.forward(np.asarray(prompt, np.int32), 0, all_rows=False)[0]]
    for i, t in enumerate(stream[:-1]):
        rows.append(sess.forward(np.array([t], np.int32), len(prompt) + i, all_rows=False)[0])
    sess.close()
    return SR.logprob_rows(np.stack(rows), stream, top_n)


def _read(L, ctx, seq, pos0, n):
    out = np.zeros(n, SR.LOGPROB_DTYPE)
    L._capi.check(L._capi.lib.lnb_session_logprobs_read(ctx.h, seq, pos0, n, out.ctypes.data))
    return out


def _same(a, b, what=""):
    for f in ("token", "rank", "n_top", "top_token"):
        assert np.array_equal(a[f], b[f]), (what, f, a[f], b[f])
    for f in ("logprob", "top_logprob"):
        assert np.array_equal(a[f].view(np.uint64), b[f].view(np.uint64)), (what, f, a[f], b[f])


def _as_records(recs):
    """model.TokenLogprob list -> LOGPROB_DTYPE"""
    out = np.zeros(len(recs), SR.LOGPROB_DTYPE)
    for i, r in enumerate(recs):
        out[i]["token"], out[i]["rank"], out[i]["logprob"], out[i]["n_top"] = r.Token, r.Rank, r.Logprob, len(r.Top)
        for j, (t, x) in enumerate(r.Top):
            out[i]["top_token"][j], out[i]["top_logprob"][j] = t, x
    return out


_OPEN = []   # the sessions _ctx opened: closed after each test, so that a failed one leaves the module's grammar free


@pytest.fixture(autouse=True)
def _close_sessions():
    yield
    while _OPEN:
        _OPEN.pop().close()


def _ctx(L, m, mode="strict", n_seq=1, max_rows=8, seq_len=SEQ_LEN):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    ctx = L.model.InferenceContext(m.gm.Transformer, L.model.InferenceArgs(seq_len), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)
    _OPEN.append(ctx)
    return ctx


def _forward_device(L, ctx, toks, pos):
    t = np.ascontiguousarray(toks, np.int32)
    nxt, gen = C.c_int32(-1), C.c_int64(0)
    L._capi.check(L._capi.lib.lnb_forward_device(ctx.h, _ptr(L, t, L._capi.i32p), t.shape[0], pos, 1, C.byref(nxt), C.byref(gen)))
    return nxt.value


def _states(m, prompt, stream):
    return [int(q) for q in SR.grammar_history(m.tables, list(prompt) + list(stream), len(prompt))[len(prompt):len(prompt) + len(stream)]]


# ---- STRICT: one sequence with every control, on every path ---------------------------------------------------------------
SAMPLERS = {"split": (0.8, 40, 1.0, 21), "full": (0.9, 0, 0.9, 23)}


@pytest.mark.parametrize("sampler", ["split", "full"])
def test_strict_stream_with_every_control_on_every_path(L, model, sampler):
    m = model
    samp = L.model.SamplingArgs(*SAMPLERS[sampler])
    assert bool(VR.split_k(samp.Temperature, samp.TopK, m.V)) == (sampler == "split")
    pen = _pen(L, m.V)
    want = _want(m, PROMPT, samp, pen, True, SEQ_LEN)
    n = len(want)
    # the stream's masks span slice 0 and the last, partial slice, and it reaches the state that allows the stop set alone
    states = _states(m, PROMPT, want)
    spans = [VR.slices_of(np.flatnonzero(m.allowed(q)), m.V) for q in states]
    assert any(len(s) >= 2 and VR.slices(m.V) - 1 in s for s in spans), spans
    assert any(set(np.flatnonzero(m.allowed(q))) == set(m.stop) for q in states), states
    assert want[-1] in m.stop and n >= 3
    records = _oracle_records(m, PROMPT, want, TOP_N)

    def setup(ctx):
        ctx.set_sampling(0, samp)
        ctx.set_penalties(0, pen, len(PROMPT))
        ctx.set_grammar(0, m.grammar, len(PROMPT))
        ctx.set_logprobs(0, TOP_N)

    for device in (False, True):     # lnb_forward (host loop) and lnb_forward_device
        ctx = _ctx(L, m)
        setup(ctx)
        fwd = (lambda t, p: _forward_device(L, ctx, t, p)) if device else (lambda t, p: m.gm.Transformer.forward_argmax(ctx, t, p)[0])
        got = [fwd(np.array(PROMPT, np.int32), 0)]
        for i in range(n - 1):
            got.append(fwd(np.array([got[-1]], np.int32), len(PROMPT) + i))
        assert got == want, ("device" if device else "host", got, want)
        _same(_read(L, ctx, 0, len(PROMPT), n), records, ("device" if device else "host"))
        ctx.close()
    for use_graph in (False, True):  # lnb_decode_run, and the captured graph replayed from the same state
        ctx = _ctx(L, m)
        setup(ctx)
        first, _ = m.gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        for rep in range(2 if use_graph else 1):
            toks, _, graphed = ctx.decode_run(first, len(PROMPT), n - 1, use_graph=use_graph)
            assert [first] + list(toks) == want and graphed == use_graph, (use_graph, rep)
            _same(_read(L, ctx, 0, len(PROMPT), n), records, ("decode_run", use_graph, rep))
        ctx.close()
    eng = L.inference.InferenceEngine(m.gm, L.model.InferenceArgs(SEQ_LEN), acc_mode=L._capi.LNB_ACC_STRICT, max_rows=8)
    kw = dict(sampling=samp, penalties=pen, grammar=m.grammar, logprobs=TOP_N)
    for extra in (dict(prefill_chunk=3), dict(speculative=L.inference.SpeculativeArgs(4))):
        out = []
        assert [t for _, t in eng.GenerateTokens(PROMPT, logprobs_out=out, **kw, **extra)] == want, extra
        _same(_as_records(out), records, extra)


# ---- STRICT and FAST: eight sequences with eight different controls in one call ---------------------------------------------
KINDS = ["greedy", "split", "top_p", "pen_greedy", "pen_sampled", "grammar_greedy", "grammar_pen_sampled", "logprobs"]


def _controls(L, m):
    """per sequence (kind, sampling, penalties, grammar, logprobs top_n); the sampled ones straddle the split kernel's edge"""
    e = VR.k_edge(m.V)
    S, pen = L.model.SamplingArgs, _pen(L, m.V)
    ctl = [("greedy", None, None, False, None),
           ("split", S(0.8, 40, 1.0, 31), None, False, 5),
           ("top_p", S(0.9, 0, 0.9, 32), None, False, None),
           ("pen_greedy", None, pen, False, None),
           ("pen_sampled", S(0.7, e + 1, 0.95, 34), pen, False, None),
           ("grammar_greedy", None, None, True, None),
           ("grammar_pen_sampled", S(0.9, e, 1.0, 36), pen, True, TOP_N),
           ("logprobs", None, None, False, TOP_N)]
    kernels = {k: ("split" if s and VR.split_k(s.Temperature, s.TopK, m.V) else "full" if s else "greedy") for k, s, _, _, _ in ctl}
    assert kernels["split"] == kernels["grammar_pen_sampled"] == "split" and kernels["top_p"] == kernels["pen_sampled"] == "full"
    assert [c[0] for c in ctl] == KINDS
    return ctl


def _apply(ctx, m, ctl):
    for k, (_, samp, pen, gram, lp) in enumerate(ctl):
        ctx.set_sampling(k, samp)
        ctx.set_penalties(k, pen, len(PROMPTS[k]))
        ctx.set_grammar(k, m.grammar if gram else None, len(PROMPTS[k]))
        ctx.set_logprobs(k, lp)


def _prefill(ctx, want_logits=False):
    """one ragged call over the eight prompts: (first tokens, their logits or None)"""
    nxt, lg = ctx.forward_ragged([(k, 0, p) for k, p in enumerate(PROMPTS)], want_logits=want_logits)
    return [int(t) for t in nxt], lg


N_GEN = 10   # tokens each sequence emits in the mixed calls


def _mixed_wants(m, ctl):
    return [_want(m, PROMPTS[k], s, p, g, len(PROMPTS[k]) + N_GEN) for k, (_, s, p, g, _) in enumerate(ctl)]


def _check_mixed(L, m, ctx, ctl, got, wants, what):
    for k, (kind, _, _, _, lp) in enumerate(ctl):
        w = wants[k]
        assert got[k][:len(w)] == w, (what, kind, got[k], w)
        if lp is not None:
            _same(_read(L, ctx, k, len(PROMPTS[k]), len(w)), _oracle_records(m, PROMPTS[k], w, lp), (what, kind))


@pytest.mark.parametrize("route", ["batch_engine", "batch_chain", "ragged"])
def test_strict_mixed_call_equals_each_sequences_statement(L, model, route, monkeypatch):
    m = model
    if route == "batch_chain":
        monkeypatch.setenv("LNB_BATCH_ENGINE", "0")
    ctl = _controls(L, m)
    wants = _mixed_wants(m, ctl)
    assert any(w[-1] in m.stop for w in wants)
    ctx = _ctx(L, m, n_seq=8, max_rows=48)
    _apply(ctx, m, ctl)
    first, _ = _prefill(ctx)
    got = [[t] for t in first]
    pos = [len(p) for p in PROMPTS]
    for _ in range(N_GEN - 1):
        toks = [g[-1] for g in got]
        if route == "ragged":
            nxt, _ = ctx.forward_ragged([(k, pos[k], [toks[k]]) for k in range(8)])
        else:
            nxt, _ = ctx.forward_batch(toks, pos)
        for k in range(8):
            got[k].append(int(nxt[k]))
        pos = [p + 1 for p in pos]
    _check_mixed(L, m, ctx, ctl, got, wants, route)
    ctx.close()


@pytest.mark.parametrize("drafts", ["perfect", "wrong"])
def test_strict_mixed_speculative_calls(L, model, drafts):
    """each call verifies four of the sequences with one draft each (the eight-row budget), alternating halves"""
    m = model
    ctl = _controls(L, m)
    wants = _mixed_wants(m, ctl)
    ctx = _ctx(L, m, n_seq=8, max_rows=48)
    _apply(ctx, m, ctl)
    first, _ = _prefill(ctx)
    got = [[t] for t in first]
    for half in [0, 1] * N_GEN:
        segs, plan = [], []
        for k in range(4 * half, 4 * half + 4):
            pos = len(PROMPTS[k]) + len(got[k]) - 1
            if len(got[k]) >= N_GEN:
                continue
            d = wants[k][len(got[k])] if len(got[k]) < len(wants[k]) else 5
            if drafts == "wrong":
                d = (d + 1) % m.V
            segs.append((k, pos, [got[k][-1], d]))
            plan.append(k)
        if not segs:
            continue
        nxt, acc, _ = ctx.forward_speculative(segs)
        for j, k in enumerate(plan):
            a = int(acc[j])
            if len(got[k]) + 1 < len(wants[k]):
                assert a == (1 if drafts == "perfect" else 0), (k, a)
            got[k] += [int(t) for t in nxt[2 * j:2 * j + a + 1]]
    _check_mixed(L, m, ctx, ctl, got, wants, ("speculative", drafts))
    ctx.close()


def test_strict_continuous_mixes_grammar_penalties_sampling_and_logprobs(L, model):
    """GenerateTokensContinuous takes one sampler and one penalty setting for every prompt and a grammar per prompt: the
    prompts alternate constrained and free, sampled on the split kernel, penalized, with records"""
    m = model
    samp, pen = L.model.SamplingArgs(0.8, 40, 1.0, 41), _pen(L, m.V)
    grams = [m.grammar if i % 2 else None for i in range(len(PROMPTS))]
    eng = L.inference.InferenceEngine(m.gm, L.model.InferenceArgs(20), acc_mode=L._capi.LNB_ACC_STRICT, max_rows=8)
    lps = []
    out = list(eng.GenerateTokensContinuous(PROMPTS, slots=3, step_tokens=8, sampling=samp, penalties=pen, grammar=grams,
                                            logprobs=3, logprobs_out=lps))
    for i, p in enumerate(PROMPTS):
        w = _want(m, p, samp, pen, grams[i] is not None, 20, seed_off=i)
        assert [t for s, _, t in out if s == i] == w, i
        _same(_as_records(lps[i]), _oracle_records(m, p, w, 3), ("continuous", i))


@pytest.mark.parametrize("route", ["batch", "ragged"])
def test_fast_mixed_call_equals_the_statement_on_its_rows(L, model, route):
    m = model
    ctl = _controls(L, m)
    ctx = _ctx(L, m, "fast", n_seq=8, max_rows=48)
    _apply(ctx, m, ctl)
    hist = [list(p) for p in PROMPTS]
    first, lg = _prefill(ctx, want_logits=True)
    masked_multi_slice = z_only = False
    for step in range(N_GEN):
        if step:
            toks, pos = [h[-1] for h in hist], [len(h) - 1 for h in hist]
            if route == "ragged":
                first, lg = ctx.forward_ragged([(k, pos[k], [toks[k]]) for k in range(8)], want_logits=True)
            else:
                first, lg = ctx.forward_batch(toks, pos, want_logits=True)
        for k, (kind, samp, pen, gram, lp) in enumerate(ctl):
            pn = len(hist[k])
            row = lg[k]
            if pen is not None:
                h = np.array(hist[k], np.int32)[None]
                row = SR.penalize_rows(row[None], [_opens(pen, len(PROMPTS[k]))], h, [pn])[0]
            if gram:
                q = int(SR.grammar_history(m.tables, hist[k], len(PROMPTS[k]))[-1])
                ok = m.allowed(q)
                row = np.where(ok, row, np.float32(-np.inf)).astype(np.float32)
                fin = np.flatnonzero(np.isfinite(row))
                masked_multi_slice |= len(VR.slices_of(fin, m.V)) >= 2 and VR.slices(m.V) - 1 in VR.slices_of(fin, m.V)
                z_only |= set(np.flatnonzero(ok)) == set(m.stop)
            T, K, P, seed = (samp.Temperature, samp.TopK, samp.TopP, samp.Seed) if samp else (0.0, 0, 1.0, 0)
            tok = int(first[k])
            assert tok == SR.sample_row(row, T, K, P, seed, pn), (route, step, kind)
            if lp is not None:
                _same(_read(L, ctx, k, pn, 1), SR.logprob_rows(lg[k][None], [tok], lp), (route, step, kind))
            hist[k].append(tok)
    assert masked_multi_slice and z_only
    ctx.close()


# ---- beams --------------------------------------------------------------------------------------------------------------
def test_strict_beams_rank_the_multi_slice_top_2b(L, tmp_path):
    V, B, seq_len = 32000, 4, 20
    args = dict(L.synth.TINY, vocab_size=V)
    tensors = host_tensors(args, SEED)
    om, gm = oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)
    try:
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq_len), acc_mode=L._capi.LNB_ACC_STRICT)
        for alpha in (0.0, 1.0):
            for early in (False, True):
                got = eng.GenerateBeams(PROMPT, L.inference.BeamSearchArgs(B, alpha, early, NumReturn=B))
                exp, _ = SR.beam_search(om, PROMPT, seq_len, B, alpha, early, stop_ids=(-1,))
                assert len(got) == len(exp) >= 1, (alpha, early)
                for g, e in zip(got, exp):
                    assert g.Tokens == e["tokens"] and g.State == e["state"], (alpha, early)
                    assert g.Logprobs == e["logprobs"] and g.Score == e["s"] and g.NormalizedScore == e["h"], (alpha, early)
    finally:
        gm.Free()
        om.close()


# ---- MXFP8: the LM head in 1024-row slices and a 256-row tail ---------------------------------------------------------------
def test_mxfp8_all_rows_logits_and_scores_at_128256(L):
    from tests.test_gpu_mxfp8 import Pair
    V, S = 128256, 40
    p = Pair(L, dict(L.synth.TINY, vocab_size=V))
    try:
        a = p.args
        ffn, q, kv, d = a["ffn_dim"], a["n_heads"] * a["head_dim"], a["n_kv_heads"] * a["head_dim"], a["dim"]
        slice_rows = max((q + 2 * kv) * d, d * q, 2 * ffn * d, d * ffn, 128 * d) // d // 128 * 128
        assert (slice_rows, V // slice_rows, V % slice_rows) == (1024, 125, 256)
        toks = np.random.default_rng(9).integers(0, V, S + 1).astype(np.int32)
        toks[:4] = [V - 1, 4095, 4096, V - 257]
        out = []
        for m in (p.mx, p.dw):
            ctx = L.model.InferenceContext(m.Transformer, L.model.InferenceArgs(64), max_rows=48, acc_mode=L._capi.LNB_ACC_FAST)
            try:
                # the S rows lnb_score evaluates for S + 1 tokens: all but the last on the tensor cores, in row slices
                _, lg = m.Transformer.forward_argmax(ctx, toks[:-1], 0, want_logits="all")
                ctx.set_logprobs(0, TOP_N)
                m.Transformer.score(ctx, toks, 0)
                out.append((lg, _read(L, ctx, 0, 1, S)))
            finally:
                ctx.close()
        (lm, rm), (ld, rd) = out
        assert lm.shape == (S, V) and np.isfinite(lm).all()
        bad = np.flatnonzero((lm.view(np.uint32) != ld.view(np.uint32)).any(axis=0))
        assert bad.size == 0, ("columns differ", bad[:8], bad[-8:])
        _same(rm, rd, "score")
        _same(rm, SR.logprob_rows(lm, toks[1:], TOP_N), "score vs its logits")
    finally:
        p.close()
