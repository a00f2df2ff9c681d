"""Speculative decoding without a GPU: the prompt-lookup drafter against a brute-force restatement, the host loop's draft
clamping, stop handling and row budget against a fake context that records its calls, and the C-ABI entry's binding."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _drafts_brute(h, max_draft, nmax, nmin):
    """the definition, literally: for n = nmax .. nmin, the largest j with j + n < L and h[j:j+n] == h[L-n:]"""
    L = len(h)
    if max_draft <= 0:
        return []
    for n in range(nmax, nmin - 1, -1):
        best = None
        for j in range(L):
            if j + n < L and L - n >= 0 and list(h[j:j + n]) == list(h[L - n:]):
                best = j
        if best is not None:
            return [int(t) for t in h[best + n:min(best + n + max_draft, L)]]
    return []


@pytest.mark.parametrize("seed", range(6))
def test_drafter_equals_brute_force(L, seed):
    rng = np.random.default_rng(seed)
    for _ in range(300):
        L_ = int(rng.integers(0, 40))
        alphabet = int(rng.integers(1, 6)) if seed % 2 else int(rng.integers(2, 1000))   # repetitive / random histories
        h = [int(t) for t in rng.integers(0, alphabet, size=L_)]
        md, nmax = int(rng.integers(0, 9)), int(rng.integers(1, 5))
        nmin = int(rng.integers(1, nmax + 1))
        assert L.inference.prompt_lookup_drafts(h, md, nmax, nmin) == _drafts_brute(h, md, nmax, nmin), (h, md, nmax, nmin)


def test_drafter_edge_cases(L):
    d = L.inference.prompt_lookup_drafts
    assert d([], 4) == [] and d([5], 4) == []                # L < n + 1 for every n
    assert d([5, 5], 4) == [5]                               # n = 1: j = 0 (j + 1 < 2), drafts h[1:2]
    assert d([1, 2, 3, 9, 1, 2, 3], 8) == [9, 1, 2, 3]       # trigram at j = 0, clamped at L
    assert d([1, 2, 3, 9, 1, 2, 3], 2) == [9, 1]             # MaxDraft
    assert d([1, 2, 3, 9, 1, 2, 3], 0) == []
    assert d([7, 1, 2, 8, 1, 2], 4, 3, 3) == []              # no trigram, NgramMin 3
    assert d([7, 1, 2, 8, 1, 2], 4, 3, 2) == [8, 1, 2]       # bigram
    assert d([4, 1, 4, 2, 4], 4, 1, 1) == [2, 4]             # the LARGEST j wins (j = 2, not 0)


class FakeSpecContext:
    """'model': the token at position p of sequence i is tok(i, p); stop id at positions of `stop_at`.  forward_speculative
    checks the call like the C-ABI and returns what the model predicts for every row and the acceptance counts."""

    def __init__(self, seq_len, max_rows, tok):
        self.SequenceLength, self.max_rows, self.tok = seq_len, max_rows, tok
        self.calls = []

    def forward_speculative(self, segs):
        rows = sum(len(t) for _, _, t in segs)
        assert rows <= min(8, self.max_rows)
        assert len({s for s, _, _ in segs}) == len(segs)
        out, acc = [], []
        for s, p, t in segs:
            assert p + len(t) - 1 < self.SequenceLength - 1, "a row past the last position the plain loop feeds"
            nxt = [self.tok(s, p + 1 + j) for j in range(len(t))]
            a = 0
            while a < len(t) - 1 and nxt[a] == t[a + 1]:
                a += 1
            out += nxt
            acc.append(a)
        self.calls.append([(s, p, list(t)) for s, p, t in segs])
        return np.array(out, np.int32), np.array(acc, np.int32), None


def _engine(L, stop_id=999):
    class M:
        Vocabulary = L.model.Vocabulary(StopTokenIds=(stop_id,))
    return L.inference.InferenceEngine(M, L.model.InferenceArgs(0))


def _plain(i, start, seq_len, tok, stop_id=999):
    out = []
    for pos in range(start, seq_len):
        out.append(tok(i, pos))
        if out[-1] == stop_id:
            break
    return out


@pytest.mark.parametrize("max_draft", [0, 1, 3, 7, 12])
def test_speculative_loop_emits_the_plain_streams(L, max_draft):
    """three sequences: a periodic one (the drafter fires and is right), one that stops on the stop id mid-acceptance, one
    of random tokens; every stream equals the plain one, every live sequence has a row, drafts go out in sequence order"""
    rng = np.random.default_rng(max_draft)
    rnd = rng.integers(0, 900, size=200)
    seq_len = 60

    def tok(i, p):
        if i == 0:
            return 10 + p % 4
        if i == 1:
            return 999 if p == 37 else 20 + p % 3
        return int(rnd[p])

    prompts = [[10, 11, 12, 13, 10], [20, 21, 22, 20, 21, 22, 20], [int(t) for t in rnd[:6]]]
    eng = _engine(L)
    ctx = FakeSpecContext(seq_len, 8, tok)
    hists = [p + [tok(i, len(p))] for i, p in enumerate(prompts)]    # the prefill emitted the first token
    stats, times = [], []
    out = list(eng._generate_speculative(ctx, hists, [0, 1, 2], L.inference.SpeculativeArgs(max_draft), times, stats))
    streams = {i: [] for i in range(3)}
    last = {}
    for i, state, t in out:
        assert last.get(i, L.inference.GSInProgress) == L.inference.GSInProgress
        streams[i].append(t)
        last[i] = state
    for i, p in enumerate(prompts):
        assert [hists[i][len(p)]] + streams[i] == _plain(i, len(p), seq_len, tok), i
    assert last[1] == L.inference.GSFinishedByReachingEOS
    assert last[0] == last[2] == L.inference.GSFinishedByReachingSeqLen
    assert len(stats) == len(times) == len(ctx.calls)
    pos = {i: len(p) for i, p in enumerate(prompts)}     # position of the token each sequence feeds next
    done = set()
    for call, (rows, accepted) in zip(ctx.calls, stats):
        assert {s for s, _, _ in call} == {0, 1, 2} - done, "every unfinished sequence gets its row"
        assert [s for s, _, _ in call] == sorted(s for s, _, _ in call)
        assert rows == sum(len(t) for _, _, t in call) <= 8
        left, acc_sum = 8 - len(call), 0
        for s, p, t in call:               # drafts in sequence order: each takes what the drafter offers of the rest
            assert p == pos[s] and t[0] == hists[s][p]
            want = L.inference.prompt_lookup_drafts(hists[s][:p + 1], min(max_draft, left, seq_len - 2 - p))
            assert t[1:] == want
            left -= len(want)
            a = 0
            while a < len(t) - 1 and tok(s, p + 1 + a) == t[a + 1]:
                a += 1
            acc_sum += a
            for j in range(a + 1):
                if tok(s, p + 1 + j) == 999 or p + 2 + j == seq_len:
                    done.add(s)
                    break
            pos[s] = p + a + 1
        assert accepted == acc_sum
    assert done == {0, 1, 2}
    if max_draft >= 3:
        assert sum(a for _, a in stats) > 0, "the periodic sequence must accept drafts"


def test_speculative_loop_clamps_at_sequence_length(L):
    """a sequence two positions before the end gets no draft; the last emitted token is at SequenceLength - 1"""
    eng = _engine(L)
    ctx = FakeSpecContext(12, 8, lambda i, p: 5)
    hists = [[5] * 10]                       # token at position 9 is fed next; 10 and 11 remain
    out = list(eng._generate_speculative(ctx, hists, [0], L.inference.SpeculativeArgs(6)))
    assert [t for _, _, t in out] == [5, 5]
    assert out[-1][1] == L.inference.GSFinishedByReachingSeqLen
    assert ctx.calls == [[(0, 9, [5, 5])]]   # one draft: the row at position 10 predicts position 11


def test_speculative_loop_row_budget(L):
    """8 live sequences leave no room for drafts; max_rows 4 caps a single sequence at 3 drafts; too many sequences is an error"""
    eng = _engine(L)
    ctx = FakeSpecContext(30, 8, lambda i, p: 7)
    hists = [[7] * 5 for _ in range(8)]
    gen = eng._generate_speculative(ctx, hists, list(range(8)), L.inference.SpeculativeArgs(4))
    next(gen)
    assert all(len(t) == 1 for _, _, t in ctx.calls[0])
    ctx = FakeSpecContext(30, 4, lambda i, p: 1 + p % 5)
    list(eng._generate_speculative(ctx, [[1 + p % 5 for p in range(15)]], [0], L.inference.SpeculativeArgs(8)))
    assert max(len(t) for c in ctx.calls for _, _, t in c) == 4
    ctx = FakeSpecContext(30, 2, lambda i, p: 7)
    with pytest.raises(L.ml.MlError):
        list(eng._generate_speculative(ctx, [[7] * 5] * 3, [0, 1, 2], L.inference.SpeculativeArgs(2)))


def test_speculative_argument_errors(L):
    class M:
        Vocabulary = L.model.Vocabulary()
    eng = L.inference.InferenceEngine(M, L.model.InferenceArgs(16))
    with pytest.raises(L.ml.MlError):
        list(eng.GenerateTokens([1], use_reference_api=True, speculative=L.inference.SpeculativeArgs(4)))
    for bad in (L.inference.SpeculativeArgs(-1), L.inference.SpeculativeArgs(4, 2, 3), L.inference.SpeculativeArgs(4, 3, 0)):
        with pytest.raises(L.ml.MlError):
            list(eng.GenerateTokens([1], speculative=bad))
        with pytest.raises(L.ml.MlError):
            list(eng.GenerateTokensBatch([[1], [2]], speculative=bad))


def test_forward_speculative_symbol_is_declared_and_bound(L):
    import os
    import re
    c = L._capi
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "lnb.h")).read()
    assert re.search(r"int lnb_forward_speculative\(lnb_session\* s, int n_segs, const int32_t\* seq, const int32_t\* start_pos, "
                     r"const int32_t\* n_draft,\s+const int32_t\* tokens, float\* logits, int32_t\* next_out, int32_t\* n_accepted\);", hdr)
    assert "lnb_forward_speculative" in c.SIGNATURES
    seq = np.zeros(1, np.int32)
    assert c.lib.lnb_forward_speculative(None, 1, c.ptr(seq, c.i32p), c.ptr(seq, c.i32p), c.ptr(seq, c.i32p), c.ptr(seq, c.i32p),
                                         None, None, None) == -1
    assert b"NULL" in c.lib.lnb_last_error()
