"""Forking and permuting sequences on the device (csrc/seqcopy.cuh) and beam search on top of it (DESIGN.md §9f): the copy
bit for bit against a snapshot of every cache, record and history row, one launch per call, validation; a fork followed by
batched decoding equal to sessions that prefilled every sequence; STRICT beam search equal to its C statement
(orc_beam_search) and to an lnb_score re-score of every hypothesis; FAST determinism; and the 8B cache layout."""
import math

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 4321
PROMPT = [1, 50, 999, 7, 300, 12, 64, 2]
SEQ_LEN = 20


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module", params=["TINY", "TINY128"])
def model(L, request):
    args = dict(getattr(L.synth, request.param))
    tensors = host_tensors(args, SEED)
    om, gm = oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)
    yield args, om, gm
    gm.Free()
    om.close()


def _acc(L, mode):
    return L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST


def _ctx(L, gm, mode="strict", seq_len=SEQ_LEN, max_rows=8, n_seq=1):
    return L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq_len), max_rows=max_rows, acc_mode=_acc(L, mode), n_seq=n_seq)


def _caches(ctx, n_layers):
    """[seq][layer] (K, V) bits of every sequence"""
    out = []
    for q in range(ctx.n_seq):
        ctx.set_active_sequence(q)
        out.append([(ctx.CacheK(l).RawData.copy(), ctx.CacheV(l).RawData.copy()) for l in range(n_layers)])
    ctx.set_active_sequence(0)
    return out


def _records(ctx, seq_len):
    return [[(r.Token, r.Rank, r.Logprob, tuple(r.Top)) for r in ctx.read_logprobs(q, 1, seq_len)] for q in range(ctx.n_seq)]


# swap 0<->1, 3-cycle 2<-3<-4<-2, fork 5 -> 6, 7 and the no-op pair 5 -> 5
PERM_SRC = [1, 0, 3, 4, 2, 5, 5, 5]
PERM_DST = [0, 1, 2, 3, 4, 5, 6, 7]


def _filled_session(L, gm, mode, seq_len, max_rows=8):
    """8 sequences with distinct contents at every position, logprob records on"""
    ctx = _ctx(L, gm, mode, seq_len=seq_len, max_rows=max_rows, n_seq=8)
    ctx.allow_chunked_prefill(True)
    V = gm.Transformer.args.VocabSize
    rng = np.random.default_rng(7)
    for q in range(8):
        ctx.set_logprobs(q, 3)
        ctx.set_active_sequence(q)
        toks = rng.integers(0, V, seq_len - 1).astype(np.int32)
        for p0 in range(0, seq_len - 1, max_rows):
            gm.Transformer.forward_argmax(ctx, toks[p0:p0 + max_rows], p0)
    ctx.set_active_sequence(0)
    return ctx


def _check_permuted(before, after, pos0, pos1):
    for q, layers in enumerate(after):
        src = PERM_SRC[PERM_DST.index(q)] if q in PERM_DST else q
        for l, (k, v) in enumerate(layers):
            for got, which in ((k, 0), (v, 1)):
                exp = before[q][l][which].copy()
                exp[pos0:pos1] = before[src][l][which][pos0:pos1]
                assert np.array_equal(got, exp), (q, l, which, pos0, pos1)


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_copy_permutes_caches_and_records(L, model, mode):
    args, _, gm = model
    seq_len = 24
    ctx = _filled_session(L, gm, mode, seq_len)
    try:
        for pos0, pos1 in [(0, seq_len), (3, 9), (seq_len - 1, seq_len), (0, 1)]:
            before, rb = _caches(ctx, args["n_layers"]), _records(ctx, seq_len)
            n0 = ctx.launch_count()
            ctx.copy_sequences(PERM_SRC, PERM_DST, pos0, pos1)
            assert ctx.launch_count() == n0 + 1
            _check_permuted(before, _caches(ctx, args["n_layers"]), pos0, pos1)
            ra = _records(ctx, seq_len)
            for q in range(8):
                src = PERM_SRC[PERM_DST.index(q)]
                for p in range(1, seq_len + 1):   # record p sits at index p - 1
                    exp = rb[src][p - 1] if pos0 <= p < pos1 else rb[q][p - 1]
                    assert ra[q][p - 1] == exp, (q, p, pos0, pos1)
    finally:
        ctx.close()


def test_copy_long_context_and_subset(L):
    """TINY128 at seq_len 512, past the shared-memory attention fit; a copy of a subset of the sequences"""
    args = dict(L.synth.TINY128)
    gm = L.model.LoadModelFromTensors(args, host_tensors(args, SEED))
    ctx = _filled_session(L, gm, "fast", 512, max_rows=64)
    try:
        before = _caches(ctx, args["n_layers"])
        ctx.copy_sequences([2, 1], [1, 2], 100, 512)   # a swap only: sequences 0, 3..7 untouched
        after = _caches(ctx, args["n_layers"])
        for q in range(8):
            src = {1: 2, 2: 1}.get(q, q)
            for l in range(args["n_layers"]):
                for w in range(2):
                    exp = before[q][l][w].copy()
                    exp[100:512] = before[src][l][w][100:512]
                    assert np.array_equal(after[q][l][w], exp)
    finally:
        ctx.close()
        gm.Free()


def test_copy_validation(L, model):
    args, _, gm = model
    ctx = _filled_session(L, gm, "strict", 16)
    try:
        before = _caches(ctx, args["n_layers"])
        n0 = ctx.launch_count()
        bad = [([0], [1, 2], 0, 4),            # shapes differ (host side)
               ([], [], 0, 4),                  # n < 1
               ([0] * 9, list(range(9)), 0, 4),  # n > n_seq, dst out of range
               ([0, 1], [2, 2], 0, 4),          # dst repeated
               ([8], [0], 0, 4), ([-1], [0], 0, 4), ([0], [8], 0, 4), ([0], [-1], 0, 4),
               ([0], [1], 4, 4), ([0], [1], 5, 4), ([0], [1], -1, 4), ([0], [1], 0, 17)]
        for src, dst, p0, p1 in bad:
            with pytest.raises((L._capi.LnbError, L.ml.MlError)) as e:
                ctx.copy_sequences(src, dst, p0, p1)
            if isinstance(e.value, L._capi.LnbError):
                assert e.value.code == -1, (src, dst, p0, p1)   # LNB_EINVAL
        assert ctx.launch_count() == n0
        after = _caches(ctx, args["n_layers"])
        assert all(np.array_equal(a, b) for x, y in zip(before, after) for p, r in zip(x, y) for a, b in zip(p, r))
    finally:
        ctx.close()


def test_forked_penalized_prompt_decodes_the_statement_stream(L, model):
    args, om, gm = model
    pen = L.model.PenaltyArgs(1.3, 0.4, 0.2, CountPrompt=True)
    exp = list(SR.generate_processed(om, PROMPT, SEQ_LEN, 0.0, 0, 1.0, 0, SR.Penalties.from_buffer_copy(bytes(pen.c(len(PROMPT)))),
                                     stop_ids=L.synth.STOP_IDS))
    ctx = _ctx(L, gm, "strict", n_seq=2)
    try:
        ctx.set_penalties(0, pen, len(PROMPT))
        ctx.set_penalties(1, pen, len(PROMPT))   # before the fork: enabling clears the history the copy brings
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        ctx.copy_sequences([0], [1], 0, len(PROMPT))
        ctx.set_active_sequence(1)
        got, tok = [first], first
        for p in range(len(PROMPT), SEQ_LEN - 1):
            tok, _ = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), p)
            got.append(tok)
        assert got == exp[:len(got)]
    finally:
        ctx.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_fork_then_decode_equals_own_prefills(L, model, mode):
    args, om, gm = model
    steps = 5
    a = _ctx(L, gm, mode, n_seq=8)
    b = _ctx(L, gm, mode, n_seq=8)
    try:
        first, _ = gm.Transformer.forward_argmax(a, np.array(PROMPT, np.int32), 0)
        a.copy_sequences([0] * 7, list(range(1, 8)), 0, len(PROMPT))
        for q in range(8):
            b.set_active_sequence(q)
            f, _ = gm.Transformer.forward_argmax(b, np.array(PROMPT, np.int32), 0)
            assert f == first
        cur = [(first + 3 * q) % args["vocab_size"] for q in range(8)]   # the sequences diverge from the first fed token
        fed = [[c] for c in cur]
        for k in range(steps):
            pos = [len(PROMPT) + k] * 8
            ta, la = a.forward_batch(cur, pos, want_logits=True)
            tb, lb = b.forward_batch(cur, pos, want_logits=True)
            assert np.array_equal(ta, tb) and np.array_equal(la.view(np.uint32), lb.view(np.uint32)), k
            if mode == "strict" and k == steps - 1:
                for q in (0, 5):
                    s = om.new_session(SEQ_LEN)
                    s.forward(np.array(PROMPT, np.int32), 0)
                    for j, t in enumerate(fed[q]):
                        lo = s.forward(np.array([t], np.int32), len(PROMPT) + j)
                    s.close()
                    assert np.array_equal(lo.reshape(-1).view(np.uint32), la[q].view(np.uint32))
            cur = [int(t) for t in ta]
            for q in range(8):
                fed[q].append(cur[q])
        ca, cb = _caches(a, args["n_layers"]), _caches(b, args["n_layers"])
        assert all(np.array_equal(x, y) for p, r in zip(ca, cb) for u, w in zip(p, r) for x, y in zip(u, w))
    finally:
        a.close()
        b.close()


# ---- beam search -----------------------------------------------------------------------------------------------------------
def _engine(L, gm, mode="strict", seq_len=SEQ_LEN, stop=None):
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq_len), acc_mode=_acc(L, mode))
    if stop is not None:
        gm.Vocabulary = L.model.Vocabulary(StopTokenIds=tuple(stop))
    return eng


def _beams(L, gm, B, alpha, early, mode="strict", seq_len=SEQ_LEN, stop=(), prompt=PROMPT, copies=None):
    eng = _engine(L, gm, mode, seq_len, stop)
    if copies is not None:
        orig = L.model.InferenceContext.copy_sequences

        def rec(self, src, dst, p0, p1):
            copies.append((list(src), list(dst), p0, p1))
            return orig(self, src, dst, p0, p1)
        L.model.InferenceContext.copy_sequences = rec
    try:
        return eng.GenerateBeams(prompt, L.inference.BeamSearchArgs(B, alpha, early, NumReturn=B))
    finally:
        if copies is not None:
            L.model.InferenceContext.copy_sequences = orig
        gm.Vocabulary = L.model.Vocabulary()


def _rescore(L, gm, prompt, toks, mode="strict", seq_len=SEQ_LEN):
    """the sequential f64 sum of lnb_score's logprobs of toks after prompt, and the list of them"""
    ctx = _ctx(L, gm, mode, seq_len=seq_len, max_rows=64)
    try:
        ctx.set_logprobs(0, 0)
        recs = gm.Transformer.score(ctx, list(prompt) + list(toks), 0)
    finally:
        ctx.close()
    lps = [r.Logprob for r in recs[len(prompt) - 1:]]
    s = 0.0
    for x in lps:
        s += x
    return s, lps


def _stop_from_free_run(L, gm, B):
    """stop ids that the unconstrained search emits mid-way"""
    free = _beams(L, gm, B, 1.0, False)
    return sorted({h.Tokens[3] for h in free[:2]} | {free[-1].Tokens[6]})


@pytest.mark.parametrize("B", [1, 2, 3, 4, 8])
def test_strict_beams_equal_the_statement(L, model, B):
    args, om, gm = model
    stop = _stop_from_free_run(L, gm, B)
    finished_mid = False
    for alpha in (0.0, 1.0, 1.5):
        for early in (False, True):
            for st in ((), stop):
                got = _beams(L, gm, B, alpha, early, stop=st)
                exp, _ = SR.beam_search(om, PROMPT, SEQ_LEN, B, alpha, early, stop_ids=st or (-1,))
                assert len(got) == len(exp) >= 1, (alpha, early, st)
                for g, e in zip(got, exp):
                    assert g.Tokens == e["tokens"] and g.State == e["state"], (alpha, early, st)
                    assert g.Logprobs == e["logprobs"] and g.Score == e["s"]
                    assert g.NormalizedScore == e["h"] or (math.isnan(g.NormalizedScore) and math.isnan(e["h"]))
                    finished_mid |= g.State == L.inference.GSFinishedByReachingEOS and len(g.Tokens) < SEQ_LEN - len(PROMPT)
                if alpha == 1.0 and not early:
                    for g in got:
                        s, lps = _rescore(L, gm, PROMPT, g.Tokens)
                        assert g.Logprobs == lps and g.Score == s
    assert finished_mid or B == 1


def test_strict_beams_reorder_and_reach_seq_len(L, model):
    _, om, gm = model
    seen_cycle = False
    for prompt in (PROMPT, [5, 6, 5, 6, 5], [900, 3, 4, 17, 22, 3, 4]):
        copies = []
        got = _beams(L, gm, 4, 1.0, False, prompt=prompt, copies=copies)
        assert copies and copies[0][2:] == (0, len(prompt)) and set(copies[0][0]) == {0}
        for src, dst, p0, p1 in copies[1:]:
            assert p0 == len(prompt) and all(s != d for s, d in zip(src, dst))
            seen_cycle |= bool(set(src) & set(dst))
        assert all(h.State == L.inference.GSFinishedByReachingSeqLen for h in got)   # no stop ids: every hypothesis is full
        exp, moves = SR.beam_search(om, prompt, SEQ_LEN, 4, 1.0, False, stop_ids=(-1,))
        assert moves == len(copies)
        assert [h.Tokens for h in got] == [e["tokens"] for e in exp]
    assert seen_cycle, "no reorder moved a beam that was also a parent (a swap or a cycle)"


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_b1_early_is_the_greedy_stream(L, model, mode):
    _, _, gm = model
    free = _beams(L, gm, 2, 1.0, False, mode=mode)
    for stop in ((), (free[0].Tokens[4],)):
        got = _beams(L, gm, 1, 1.0, True, mode=mode, stop=stop)
        eng = _engine(L, gm, mode, stop=stop)
        try:
            greedy = [t for _, t in eng.GenerateTokens(PROMPT)]
        finally:
            gm.Vocabulary = L.model.Vocabulary()
        assert len(got) == 1 and got[0].Tokens == greedy


def test_fast_beams_are_deterministic_and_near_strict(L, model):
    _, _, gm = model
    for B in (2, 4):
        a = _beams(L, gm, B, 1.0, False, mode="fast")
        b = _beams(L, gm, B, 1.0, False, mode="fast")
        assert [(h.Tokens, h.Score, h.Logprobs) for h in a] == [(h.Tokens, h.Score, h.Logprobs) for h in b]
        for h in a:
            s, _ = _rescore(L, gm, PROMPT, h.Tokens, mode="strict")
            assert abs(h.Score - s) <= 0.02 * len(h.Tokens), (h.Score, s)


def test_8b_copy_and_strict_beams(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    args = dict(L.synth.LLAMA31_8B)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    try:
        ctx = _ctx(L, gm, "fast", seq_len=4096, max_rows=512, n_seq=4)
        try:
            ctx.allow_chunked_prefill(True)
            rng = np.random.default_rng(3)
            for q in range(4):
                ctx.set_active_sequence(q)
                toks = rng.integers(0, args["vocab_size"], 4095).astype(np.int32)
                for p0 in range(0, 4095, 512):
                    gm.Transformer.forward_argmax(ctx, toks[p0:p0 + 512], p0)
            layers = (0, 31)

            def snap():
                out = []
                for q in range(4):
                    ctx.set_active_sequence(q)
                    out.append([(ctx.CacheK(l).RawData.copy(), ctx.CacheV(l).RawData.copy()) for l in layers])
                return out
            before = snap()
            ctx.copy_sequences([1, 2, 0, 0], [0, 1, 2, 3], 0, 4096)   # a 3-cycle and a fork
            after = snap()
            for q, src in enumerate([1, 2, 0, 0]):
                for i in range(len(layers)):
                    for w in range(2):
                        assert np.array_equal(after[q][i][w], before[src][i][w]), (q, layers[i], w)
        finally:
            ctx.close()
        prompt = list(L.synth.PROMPT_8)
        seq_len = len(prompt) + 8
        got = _beams(L, gm, 4, 1.0, False, seq_len=seq_len, prompt=prompt)
        assert len(got) == 4
        for h in got:
            s, lps = _rescore(L, gm, prompt, h.Tokens, seq_len=seq_len)
            assert h.Logprobs == lps and h.Score == s
    finally:
        gm.Free()


def test_cli_and_cpp_mirror_print_what_the_python_mirror_finds(L):
    """host/lnb_generate beams=B len_pen= early_stop= runs the C++ mirror's inference::GenerateBeams; STRICT, its hypotheses
    (state, s and h printed with %.17g, so exact, and tokens) equal GenerateBeams of the Python mirror on the same model"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    args = dict(L.synth.TINY)
    gm = L.model.LoadModelFromTensors(args, host_tensors(args, 7))     # lnb_generate's tiny model (seed 7)
    base = [1, 50, 999, 7, 300, 12, 64, 2]
    try:
        for B, alpha, early in ((4, 1.0, False), (4, 0.0, True), (3, 1.5, False), (1, 1.0, True), (8, 1.0, False)):
            flags = [f"beams={B}", f"len_pen={alpha!r}", f"early_stop={int(early)}"]
            out = subprocess.run([exe, "24", "strict", "tiny"] + flags, capture_output=True, text=True, timeout=120)
            assert out.returncode == 0, out.stderr
            lines = [ln for ln in out.stdout.splitlines() if ln.startswith("beam[")]
            eng = _engine(L, gm, "strict", 24, stop=(10**9,))   # the CLI's tiny model stops on no token
            try:
                got = eng.GenerateBeams(base, L.inference.BeamSearchArgs(B, alpha, early, NumReturn=B))
            finally:
                gm.Vocabulary = L.model.Vocabulary()
            assert len(lines) == len(got) == B, (flags, out.stdout)
            for i, (ln, h) in enumerate(zip(lines, got)):
                head, toks = ln.split("|")
                f = head.split()
                assert f[0] == f"beam[{i}]:" and int(f[2]) == h.State
                assert float(f[4]) == h.Score and float(f[6]) == h.NormalizedScore, (flags, i)
                assert [int(t) for t in toks.split()] == h.Tokens, (flags, i)
    finally:
        gm.Free()
