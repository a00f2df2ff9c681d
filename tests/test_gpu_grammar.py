"""Regex-constrained generation on the device (csrc/grammar.cuh, DESIGN.md §9g) against its C statement
(orc_grammar_masks and orc_generate_constrained, oracle_sampling/lnb_sample_ref.c): the mask tables bit for bit, STRICT
constrained streams equal to the statement on every path (greedy and sampled, with and without penalties), FAST streams
equal to the statement's mask and sampler on the rows the same calls return, every stream a viable prefix of the
language, sessions without a grammar unchanged, decode-graph re-capture, validation, and the 8B model."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 4321
PROMPT = [1, 50, 999, 7, 300, 12, 64, 2]
PROMPTS = [PROMPT, [5, 6, 5, 6, 5], [900, 3, 4, 17, 22, 3, 4], [8]]
SEQ_LEN = 32
SAMP = (0.9, 0, 1.0, 5)   # temperature, top_k, top_p, seed
PATTERNS = [r"(yes|no|maybe)", r"[0-9]{4}-[0-9]{2}-[0-9]{2}", r"[a-z]+( [a-z]+)*\.", r"(ab|c[de])*f?[\w\s]{0,30}"]


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _vocab(L, tmp, V):
    path = os.path.join(tmp, f"tokenizer_{V}.model")
    L._capi.check(L._capi.lib.lnb_vocab_write_synthetic(path.encode(), V - 256))
    return L.vocabulary.Load(path)


@pytest.fixture(scope="module", params=["TINY", "TINY128"])
def model(L, request, tmp_path_factory):
    args = dict(getattr(L.synth, request.param))
    tensors = host_tensors(args, SEED)
    om, gm = oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)
    vocab = _vocab(L, str(tmp_path_factory.mktemp("vocab")), args["vocab_size"])
    gm.Vocabulary = vocab   # the generate loops stop at its stop tokens, which are the grammars' Z
    tok = L.model.vocabulary_token_bytes(vocab, args["vocab_size"])
    yield args, om, gm, vocab, tok
    gm.Free()
    om.close()


def _tables(L, pattern, tok, stop):
    trans, accept = L.model.regex_dfa(pattern)
    return SR.GrammarTables(trans, accept, tok, stop)


def _samp(L, sampled):
    return L.model.SamplingArgs(*SAMP) if sampled else None


def _ctx(L, gm, mode="strict", seq_len=SEQ_LEN, max_rows=8, n_seq=1):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq_len), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)


def _engine(L, gm, mode="strict", seq_len=SEQ_LEN, max_rows=8):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq_len), acc_mode=acc, max_rows=max_rows)


def _oracle(om, prompt, tables, stop, sampled, pen=None, seq_len=SEQ_LEN, seed_off=0):
    T, K, P, seed = SAMP if sampled else (0.0, 0, 1.0, 0)
    return list(SR.generate_constrained(om, prompt, seq_len, T, K, P, seed + seed_off, pen, tables, len(prompt), stop_ids=stop))


def _check_viable(pattern, tables, tok, stream, stop):
    """the bytes of the stream are a viable prefix of the language at every step (a walk of the trimmed DFA that never
    falls off it), and a full match when a stop token ends them"""
    q, data = 0, b""
    for i, t in enumerate(stream):
        if t in stop:
            assert tables.accept[q], (pattern, data)
            assert re.fullmatch(pattern, data.decode("utf-8"), re.ASCII), (pattern, data)
            assert all(u in stop for u in stream[i:]), stream
            return True
        for b in tok[t]:
            q = int(tables.trans[q, b])
            assert q >= 0, (pattern, data, t)
        data += tok[t]
    return False


# ---- the mask tables --------------------------------------------------------------------------------------------------
def test_masks_equal_the_statement(L, model):
    args, _, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    for pattern in PATTERNS + [r"\d+(\.\d+)?", "[^a]*é"]:
        g = L.model.Grammar(gm, pattern, vocab)
        exp, stuck = SR.grammar_masks(_tables(L, pattern, tok, stop))
        for q in range(g.NumStates):
            assert (g.read_mask(q) == exp[q]).all(), (pattern, q)
        assert (g.read_mask(-1) == exp[g.NumStates]).all()
        info = g.info()
        assert info["stuck"] == stuck and info["states"] == exp.shape[0] - 1 and info["build_ns"] > 0
        g.close()


def test_masks_at_128256_tokens_and_over_1000_states(L, tmp_path):
    args = dict(L.synth.TINY, vocab_size=128256)
    tr = L.model.LlamaTransformer(L.model.ModelArgs.from_c_dict(args))
    vocab = _vocab(L, str(tmp_path), 128256)
    tok = L.model.vocabulary_token_bytes(vocab, 128256)
    pattern = r"(a|b)*a(a|b){10}( [0-9a-f]{1,4})*"
    g = L.model.Grammar(tr, pattern, vocab)
    assert g.NumStates > 1000
    exp, stuck = SR.grammar_masks(_tables(L, pattern, tok, list(vocab.StopTokenIds)))
    for q in list(range(g.NumStates)) + [-1]:
        assert (g.read_mask(q) == exp[q if q >= 0 else g.NumStates]).all(), q
    assert g.info()["stuck"] == stuck
    g.close()
    tr.close()


# ---- STRICT streams on every path ---------------------------------------------------------------------------------------
def _forward_device(L, ctx, toks, pos):
    t = np.ascontiguousarray(toks, np.int32)
    nxt, gen = C.c_int32(-1), C.c_int64(0)
    L._capi.check(L._capi.lib.lnb_forward_device(ctx.h, L._capi.ptr(t, L._capi.i32p), t.shape[0], pos, 1, C.byref(nxt), C.byref(gen)))
    return nxt.value


def _host_loop(L, gm, ctx, prompt, steps, device=False):
    fwd = (lambda t, p: _forward_device(L, ctx, t, p)) if device else (lambda t, p: gm.Transformer.forward_argmax(ctx, t, p)[0])
    out = [fwd(np.array(prompt, np.int32), 0)]
    for i in range(steps - 1):
        out.append(fwd(np.array([out[-1]], np.int32), len(prompt) + i))
    return out


@pytest.mark.parametrize("penalized", [False, True])
@pytest.mark.parametrize("sampled", [False, True])
def test_strict_streams_equal_the_statement_on_every_path(L, model, sampled, penalized):
    _, om, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    pen = L.model.PenaltyArgs(1.3, 0.4, 0.2) if penalized else None
    opens = None if pen is None else SR.Penalties.from_buffer_copy(bytes(pen.c(len(PROMPT))))
    pattern = PATTERNS[3] if sampled else PATTERNS[2]
    g = L.model.Grammar(gm, pattern, vocab)
    tables = _tables(L, pattern, tok, stop)
    want = _oracle(om, PROMPT, tables, stop, sampled, opens)
    _check_viable(pattern, tables, tok, want, stop)
    n = len(want)
    eng = _engine(L, gm)
    kw = dict(sampling=_samp(L, sampled), penalties=pen, grammar=g)
    assert [t for _, t in eng.GenerateTokens(PROMPT, **kw)] == want
    assert [t for _, t in eng.GenerateTokens(PROMPT, prefill_chunk=3, **kw)] == want
    for device in (False, True):
        ctx = _ctx(L, gm)
        ctx.set_sampling(0, _samp(L, sampled))
        ctx.set_penalties(0, pen, len(PROMPT))
        ctx.set_grammar(0, g, len(PROMPT))
        assert _host_loop(L, gm, ctx, PROMPT, n, device) == want, device
        ctx.close()
    for use_graph in (False, True):
        ctx = _ctx(L, gm)
        ctx.set_sampling(0, _samp(L, sampled))
        ctx.set_penalties(0, pen, len(PROMPT))
        ctx.set_grammar(0, g, len(PROMPT))
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        if n > 1:
            toks, _, graphed = ctx.decode_run(first, len(PROMPT), n - 1, use_graph=use_graph)
            assert [first] + list(toks) == want and graphed == use_graph
        ctx.close()
    assert [t for _, t in eng.GenerateTokens(PROMPT, speculative=L.inference.SpeculativeArgs(4), **kw)] == want
    # batches beside an unconstrained and a differently-constrained neighbour
    g2 = L.model.Grammar(gm, PATTERNS[0], vocab)
    t2 = _tables(L, PATTERNS[0], tok, stop)
    grams, tabs = [g, None, g2, g], [tables, None, t2, tables]
    wants = []
    for i, p in enumerate(PROMPTS):
        op = None if pen is None else SR.Penalties.from_buffer_copy(bytes(pen.c(len(p))))
        if tabs[i] is None:
            T, K, P, seed = SAMP if sampled else (0.0, 0, 1.0, 0)
            wants.append(list(SR.generate_processed(om, p, SEQ_LEN, T, K, P, seed + i, op, stop_ids=stop)))
        else:
            wants.append(_oracle(om, p, tabs[i], stop, sampled, op, seed_off=i))
    for spec in (None, L.inference.SpeculativeArgs(3)):
        out = list(eng.GenerateTokensBatch(PROMPTS, sampling=_samp(L, sampled), penalties=pen, grammar=grams, speculative=spec))
        for i in range(len(PROMPTS)):
            assert [t for s, _, t in out if s == i] == wants[i], ("batch", spec, i)
    out = list(eng.GenerateTokensContinuous(PROMPTS, slots=2, step_tokens=4, sampling=_samp(L, sampled), penalties=pen,
                                            grammar=grams))
    for i in range(len(PROMPTS)):
        assert [t for s, _, t in out if s == i] == wants[i], ("continuous", i)
    g2.close()
    g.close()


def test_finite_language_always_ends_in_a_stop_token(L, model):
    _, om, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    g = L.model.Grammar(gm, PATTERNS[0], vocab)
    tables = _tables(L, PATTERNS[0], tok, stop)
    eng = _engine(L, gm)
    for sampled in (False, True):
        for p in PROMPTS:
            got = [t for _, t in eng.GenerateTokens(p, sampling=_samp(L, sampled), grammar=g)]
            assert _check_viable(PATTERNS[0], tables, tok, got, stop), got
    g.close()


@pytest.mark.parametrize("sampled", [False, True])
def test_speculative_calls_with_perfect_wrong_and_out_of_grammar_drafts(L, model, sampled):
    _, om, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    pattern = PATTERNS[3]
    g = L.model.Grammar(gm, pattern, vocab)
    tables = _tables(L, pattern, tok, stop)
    want = _oracle(om, PROMPT, tables, stop, sampled)
    p0 = len(PROMPT)
    outside = next(t for t in range(len(tok)) if tok[t] and tok[t][0] == ord("!"))   # never a viable continuation
    for kind in ("perfect", "wrong", "outside"):
        ctx = _ctx(L, gm)
        ctx.set_sampling(0, _samp(L, sampled))
        ctx.set_grammar(0, g, p0)
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        assert first == want[0]
        got, pos = [first], p0
        while len(got) < len(want):
            k = min(5, len(want) - len(got), SEQ_LEN - 2 - pos)
            drafts = list(want[len(got):len(got) + k])
            if kind == "wrong" and drafts:
                drafts[-1] = (drafts[-1] + 1) % len(tok)
            elif kind == "outside" and drafts:
                drafts[len(drafts) // 2] = outside
            nxt, acc, _ = ctx.forward_speculative([(0, pos, [got[-1]] + drafts)])
            a = int(acc[0])
            assert a == {"perfect": len(drafts), "wrong": max(len(drafts) - 1, 0), "outside": len(drafts) // 2}[kind], kind
            got += [int(t) for t in nxt[:a + 1]]
            pos += a + 1
        assert got[:len(want)] == want, kind
        ctx.close()
    g.close()


# ---- FAST streams ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sampled", [False, True])
def test_fast_streams_equal_the_statement_mask_on_their_rows(L, model, sampled):
    _, _, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    pattern = PATTERNS[2]
    g = L.model.Grammar(gm, pattern, vocab)
    tables = _tables(L, pattern, tok, stop)
    masks, _ = SR.grammar_masks(tables)
    T, K, P, seed = SAMP if sampled else (0.0, 0, 1.0, 0)
    ctx = _ctx(L, gm, "fast")
    ctx.set_sampling(0, _samp(L, sampled))
    ctx.set_grammar(0, g, len(PROMPT))
    toks, pos = np.array(PROMPT, np.int32), 0
    stream = []
    for _ in range(16):
        nxt, logits = gm.Transformer.forward_argmax(ctx, toks, pos, want_logits="last")
        hist = SR.grammar_history(tables, PROMPT + stream, len(PROMPT))
        q = int(hist[-1])
        bits = masks[q if q >= 0 else tables.Q]
        allowed = (bits[np.arange(len(tok)) >> 5] >> (np.arange(len(tok)) & 31).astype(np.uint32)) & 1
        row = np.where(allowed.astype(bool), logits[0], np.float32(-np.inf)).astype(np.float32)
        assert nxt == SR.sample_row(row, T, K, P, seed, len(PROMPT) + len(stream))
        pos += toks.shape[0]
        stream.append(nxt)
        toks = np.array([nxt], np.int32)
    _check_viable(pattern, tables, tok, stream, stop)
    ctx.close()
    g.close()


# ---- no grammar, graphs, validation -------------------------------------------------------------------------------------
def test_sessions_without_a_grammar_are_unchanged(L, model):
    _, _, gm, vocab, _ = model
    g = L.model.Grammar(gm, PATTERNS[1], vocab)
    runs = []
    for toggled in (False, True):
        ctx = _ctx(L, gm)
        if toggled:
            ctx.set_grammar(0, g, 3)
            ctx.set_grammar(0, None)
        c0 = ctx.launch_count()
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        toks, _, _ = ctx.decode_run(first, len(PROMPT), 12, use_graph=True)
        runs.append(([first] + list(toks), ctx.launch_count() - c0))
        ctx.close()
    assert runs[0] == runs[1]
    g.close()


def _graph_instantiations(fn):
    """fn() under torch.profiler (CUDA activities): the number of cudaGraphInstantiate calls the trace shows"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "cudaGraphInstantiate" in e.name)


def test_toggling_recaptures_the_graph_and_switching_does_not(L, model):
    _, om, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    pa, pb = PATTERNS[2], PATTERNS[3]
    ga, gb = L.model.Grammar(gm, pa, vocab), L.model.Grammar(gm, pb, vocab)
    n = 6
    ctx = _ctx(L, gm)
    c0 = ctx.launch_count()
    first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
    ctx.decode_run(first, len(PROMPT), n, use_graph=True)
    plain = (ctx.launch_count() - c0)
    res = {}

    def run(g, pattern):
        # the grammar from the prompt's end on: the first token comes from a constrained row, so the whole stream is the
        # statement's
        ctx.set_grammar(0, g, len(PROMPT))
        c = ctx.launch_count()
        f, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        toks, _, graphed = ctx.decode_run(f, len(PROMPT), n, use_graph=True)
        want = _oracle(om, PROMPT, _tables(L, pattern, tok, stop), stop, False, seq_len=len(PROMPT) + n + 1)
        assert graphed and [f] + list(toks)[:len(want) - 1] == want, pattern
        res[pattern] = ctx.launch_count() - c
    inst_toggle = _graph_instantiations(lambda: run(ga, pa))   # off -> on: a new capture
    inst_switch = _graph_instantiations(lambda: run(gb, pb))   # another grammar: the same graph reads the new slot
    assert res[pa] == res[pb] > plain
    assert inst_switch == 0, inst_switch
    assert inst_toggle >= 1 or inst_toggle == inst_switch == 0   # (when the trace shows runtime calls at all)
    ctx.set_grammar(0, None)
    c1 = ctx.launch_count()
    f, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
    toks, _, _ = ctx.decode_run(f, len(PROMPT), n, use_graph=True)
    assert ctx.launch_count() - c1 < res[pa] and f == first   # back on the decode engine, without the grammar job
    ctx.close()
    ga.close()
    gb.close()


def test_switching_to_a_smaller_grammar_behind_fed_positions(L, model):
    """decode under a large grammar, then switch the sequence to a small one with an earlier first_pos: the states the
    large grammar recorded are never read (the rows past first_pos see ⊥, only stop tokens) until the caller feeds the
    positions from first_pos again, after which the stream is the statement's for the small grammar"""
    _, om, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    big_p, small_p = r"(a|b|c|d| )*a(a|b|c|d| ){7}", PATTERNS[1]
    big, small = L.model.Grammar(gm, big_p, vocab), L.model.Grammar(gm, small_p, vocab)
    assert big.NumStates > 100 > small.NumStates
    p0 = len(PROMPT)
    ctx = _ctx(L, gm)
    ctx.allow_chunked_prefill(True)
    ctx.set_grammar(0, big, p0)
    first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
    toks, _, _ = ctx.decode_run(first, p0, 12, use_graph=True)
    fed = PROMPT + [first] + list(toks)[:-1]          # positions 0 .. p0 + 11
    ctx.set_grammar(0, small, p0 - 3)
    nxt, _ = gm.Transformer.forward_argmax(ctx, np.array([fed[-1]], np.int32), len(fed) - 1)
    assert nxt in stop, nxt                          # g[len(fed)] is ⊥ after the switch
    for fp, chunk in ((p0 - 3, 4), (p0 + 2, 3)):     # feed again from first_pos (multi-row record walks), then generate
        ctx.set_grammar(0, small, fp)
        pos, out = fp, None
        while pos < len(fed):
            c = fed[pos:pos + chunk]
            out, _ = gm.Transformer.forward_argmax(ctx, np.array(c, np.int32), pos)
            pos += len(c)
        want = list(SR.generate_constrained(om, fed, len(fed) + 1, 0.0, 0, 1.0, 0, None, _tables(L, small_p, tok, stop), fp,
                                            stop_ids=stop))
        assert out == want[0], (fp, out, want)
    ctx.close()
    big.close()
    small.close()


@pytest.mark.parametrize("sampled", [False, True])
def test_first_pos_inside_the_prompt(L, model, sampled):
    """the grammar starts inside the prompt, so the prefill's rows past first_pos walk the state serially in one thread
    (one-shot and chunked prefill, lnb_forward and lnb_decode_run), equal to the statement"""
    _, om, gm, vocab, tok = model
    stop = list(vocab.StopTokenIds)
    pattern = PATTERNS[3]
    prompt = [1, 50, 999] + list(b"abcd ce")          # bytes of the synthetic tokens 0..255: inside the language
    fp = 3
    g = L.model.Grammar(gm, pattern, vocab)
    tables = _tables(L, pattern, tok, stop)
    T, K, P, seed = SAMP if sampled else (0.0, 0, 1.0, 0)
    want = list(SR.generate_constrained(om, prompt, SEQ_LEN, T, K, P, seed, None, tables, fp, stop_ids=stop))
    hist = SR.grammar_history(tables, prompt, fp)
    assert hist[-1] >= 0                             # the prompt's tail is inside the grammar: a real walk
    for chunk in (len(prompt), 3):
        ctx = _ctx(L, gm, max_rows=16)
        ctx.allow_chunked_prefill(True)
        ctx.set_sampling(0, _samp(L, sampled))
        ctx.set_grammar(0, g, fp)
        pos = 0
        while pos < len(prompt):
            c = prompt[pos:pos + chunk]
            first, _ = gm.Transformer.forward_argmax(ctx, np.array(c, np.int32), pos)
            pos += len(c)
        got = [first]
        if len(want) > 1:
            toks, _, _ = ctx.decode_run(first, len(prompt), len(want) - 1, use_graph=True)
            got += list(toks)
        assert got == want, chunk
        ctx.close()
    g.close()


def test_cli_regex_prints_what_the_python_mirror_generates(L, tmp_path):
    """host/lnb_generate <seq_len> strict <dir> regex=PATTERN (single and batch=3) runs the C++ mirror's model::Grammar on
    the directory's tokenizer; its tokens equal the Python mirror's GenerateTokens / GenerateTokensBatch with grammar="""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    d = str(tmp_path)
    subprocess.run([exe, "--write-synthetic", d, "tiny"], check=True, capture_output=True, timeout=120)
    gm = L.model.LoadModel(d)
    try:
        prompt = [1, 50, 999, 7, 300, 12, 64, 2]
        eng = _engine(L, gm, seq_len=32)
        for pattern in (PATTERNS[2], PATTERNS[0]):
            g = L.model.Grammar(gm, pattern, gm.Vocabulary)
            out = subprocess.run([exe, "32", "strict", d, f"regex={pattern}"], capture_output=True, text=True, timeout=120)
            assert out.returncode == 0, out.stderr
            line = next(ln for ln in out.stdout.splitlines() if ln.startswith("tokens:"))
            assert [int(t) for t in line.split()[1:]] == [t for _, t in eng.GenerateTokens(prompt, grammar=g)], pattern
            out = subprocess.run([exe, "32", "strict", d, "batch=3", f"regex={pattern}"], capture_output=True, text=True, timeout=120)
            assert out.returncode == 0, out.stderr
            prompts = [[prompt[0]] + [(t + 977 * b) % 1000 for t in prompt[1:]] for b in range(3)]
            res = list(eng.GenerateTokensBatch(prompts, grammar=g))
            for b in range(3):
                line = next(ln for ln in out.stdout.splitlines() if ln.startswith(f"tokens[{b}]:"))
                assert [int(t) for t in line.split()[1:]] == [t for s, _, t in res if s == b], (pattern, b)
            g.close()
    finally:
        gm.Free()


def test_validation(L, model):
    args, _, gm, vocab, tok = model
    g = L.model.Grammar(gm, PATTERNS[0], vocab)
    ctx = _ctx(L, gm, n_seq=2)
    E = L._capi.LnbError
    lib = L._capi.lib
    for seq, fp in ((-1, 0), (2, 0), (0, -1), (0, SEQ_LEN + 1)):
        with pytest.raises(E) as ei:
            ctx.set_grammar(seq, g, fp)
        assert ei.value.code == -1
    ctx.set_grammar(1, g, SEQ_LEN)   # first_pos = seq_len is legal
    other = L.model.LlamaTransformer(L.model.ModelArgs.from_c_dict(args))
    g_other = L.model.Grammar(other, PATTERNS[0], vocab)
    with pytest.raises(E):
        ctx.set_grammar(0, g_other, 0)
    with pytest.raises(E) as ei:   # still in use by sequence 1
        g.close()
    assert ei.value.code == -4
    ctx.set_grammar(1, None)
    with pytest.raises(E):
        L.model.Grammar(gm, "a(", vocab)
    with pytest.raises(E):
        L.model.Grammar(gm, "a", token_bytes=tok, stop_ids=[])
    with pytest.raises(E):
        L.model.Grammar(gm, "a", token_bytes=tok, stop_ids=[len(tok)])
    with pytest.raises(L.ml.MlError):
        next(_engine(L, gm).GenerateTokens(PROMPT, use_reference_api=True, grammar=g))
    with pytest.raises(L.ml.MlError):
        _engine(L, gm).GenerateBeams(PROMPT, L.inference.BeamSearchArgs(2), grammar=g)
    # a session left as it was: an unconstrained stream
    first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
    assert lib.lnb_grammar_destroy(None) == 0
    ctx.close()
    g.close()
    g_other.close()
    other.close()


# ---- the 8B model -------------------------------------------------------------------------------------------------------
def test_8b_decode_run_and_batch(L, tmp_path):
    args = dict(L.synth.LLAMA31_8B)
    tensors = host_tensors(args, SEED)
    om, gm = oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)
    try:
        vocab = _vocab(L, str(tmp_path), args["vocab_size"])
        tok = L.model.vocabulary_token_bytes(vocab, args["vocab_size"])
        stop = list(vocab.StopTokenIds)
        pattern = r"[a-z ]{1,40}\."
        g = L.model.Grammar(gm, pattern, vocab)
        tables = _tables(L, pattern, tok, stop)
        prompt = L.synth.PROMPT_8
        want = _oracle(om, prompt, tables, stop, False, seq_len=len(prompt) + 16)
        ctx = _ctx(L, gm, seq_len=len(prompt) + 16)
        ctx.set_grammar(0, g, len(prompt))
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0)
        toks, _, _ = ctx.decode_run(first, len(prompt), len(want) - 1, use_graph=True)
        assert [first] + list(toks) == want
        ctx.close()
        gm.Vocabulary = vocab
        eng = _engine(L, gm, seq_len=len(prompt) + 16)
        prompts = [prompt, prompt[:5], prompt[2:], prompt[:3]]
        out = list(eng.GenerateTokensBatch(prompts, grammar=g))
        for i, p in enumerate(prompts):
            assert [t for s, _, t in out if s == i] == _oracle(om, p, tables, stop, False, seq_len=len(prompt) + 16), i
        g.close()
    finally:
        gm.Free()
        om.close()
