"""Beam search without a GPU (DESIGN.md §9f): the selection and pool rules of the Python loop and of the C statement against
a brute-force restatement of the contract, and the whole search -- Python loop on a recording fake context, C statement on
the same fake model -- including the fork, every reorder's pairs and ranges, and the order of the calls."""
import math

import numpy as np
import pytest


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module")
def SR():
    from oracle_sampling import sample_ref
    return sample_ref


NAN, INF = float("nan"), float("inf")


def _before(a, b) -> bool:
    """candidate a is walked before b: score descending with -inf after every finite score and NaN last, then beam, then rank"""
    sa, sb = a[0], b[0]
    if math.isnan(sa) != math.isnan(sb):
        return math.isnan(sb)
    if not math.isnan(sa) and sa != sb:
        return sa > sb
    return (a[1], a[2]) < (b[1], b[2])


def _select_brute(cands, B, stop):
    """§9f step 3 literally: the walk index of each candidate is the number of candidates walked before it"""
    idx = {id(c): sum(_before(d, c) for d in cands) for c in cands}
    walk = sorted(cands, key=lambda c: idx[id(c)])
    new, fin = [], []
    for i, c in enumerate(walk):
        if len(new) == B:
            break
        if c[3] in stop:
            if i < B:
                fin.append(c)
        else:
            new.append(c)
    return new, fin


def _select_broken(cands, B, stop):
    """NaN sorted first: a rule the restatement must reject"""
    walk = sorted(cands, key=lambda c: ((0, 0.0) if math.isnan(c[0]) else (1, -c[0]), c[1], c[2]))
    new, fin = [], []
    for i, c in enumerate(walk):
        if len(new) == B:
            break
        if c[3] not in stop:
            new.append(c)
        elif i < B:
            fin.append(c)
    return new, fin


def _tables(seed, n_tables=200):
    rng = np.random.default_rng(seed)
    for _ in range(n_tables):
        B = int(rng.integers(1, 9))
        n_beams = int(rng.integers(1, B + 1))
        width = int(rng.integers(1, 2 * B + 1))
        pool = [-0.5, -1.0, -1.0, -2.25, -INF, INF, NAN, 0.0] if seed % 2 else None
        cands = []
        for b in range(n_beams):
            for j in range(width):
                sc = float(rng.choice(pool)) if pool is not None else float(-rng.exponential(2.0))
                cands.append((sc, b, j, int(rng.integers(0, 6 if seed % 2 else 50))))
        rng.shuffle(cands)
        stop = {int(t) for t in rng.integers(0, 6, size=int(rng.integers(0, 3)))}
        yield [tuple(c) for c in cands], B, stop


def _same(a, b):
    """equal candidate lists (NaN scores equal)"""
    return len(a) == len(b) and all((x[1:4] == y[1:4]) and (x[0] == y[0] or (math.isnan(x[0]) and math.isnan(y[0]))) for x, y in zip(a, b))


@pytest.mark.parametrize("seed", range(4))
def test_selection_equals_restatement(L, SR, seed):
    broken_differs = False
    for cands, B, stop in _tables(seed):
        exp_new, exp_fin = _select_brute(cands, B, stop)
        new, fin = L.inference.beam_select(cands, B, stop)
        assert _same([c[:4] for c in new], exp_new) and _same([c[:4] for c in fin], exp_fin), (cands, B, stop)
        cnew, cfin = SR.beam_select(cands, B, stop)
        assert _same(cnew, exp_new) and _same(cfin, exp_fin), (cands, B, stop)
        bn, bf = _select_broken(cands, B, stop)
        broken_differs |= not (_same(bn, exp_new) and _same(bf, exp_fin))
    if seed % 2:   # the tables with NaN scores tell the broken rule apart
        assert broken_differs


def test_selection_stop_rule(L, SR):
    # stop tokens at walk index < B finish, at index >= B are skipped; the walk ends once B new beams exist
    cands = [(-1.0, 0, 0, 9), (-1.5, 0, 1, 3), (-2.0, 0, 2, 9), (-3.0, 0, 3, 4), (-4.0, 0, 4, 5)]
    for sel in (L.inference.beam_select, SR.beam_select):
        new, fin = sel(cands, 2, {9})
        assert [c[3] for c in new] == [3, 4] and [c[3] for c in fin] == [9]   # index 2 >= B: skipped
        new, fin = sel(cands, 3, {9})
        assert [c[3] for c in new] == [3, 4, 5] and [c[3] for c in fin] == [9, 9]


def _pool_brute(hs, B):
    """keep the best B by h (NaN lowest), ties won by the earlier insertion; best first"""
    kept = []
    for i, h in enumerate(hs):
        kept.append(i)
        if len(kept) > B:
            key = lambda j: ((1, 0.0) if math.isnan(hs[j]) else (0, -hs[j]), j)   # noqa: E731
            kept.remove(max(kept, key=key))
    return sorted(kept, key=lambda j: ((1, 0.0) if math.isnan(hs[j]) else (0, -hs[j]), j))


@pytest.mark.parametrize("seed", range(3))
def test_pool_equals_restatement(L, SR, seed):
    rng = np.random.default_rng(100 + seed)
    vals = [-1.0, -2.0, -2.0, -0.5, -INF, NAN, -3.0]
    for _ in range(300):
        B = int(rng.integers(1, 9))
        hs = [float(rng.choice(vals)) if seed else float(-rng.exponential()) for _ in range(int(rng.integers(0, 20)))]
        exp = _pool_brute(hs, B)
        pool = L.inference.BeamPool(B)
        for i, h in enumerate(hs):
            pool.add(L.inference.BeamHypothesis([i], h, h, [], 1))
        assert [x.Tokens[0] for x in pool.result()] == exp, (hs, B)
        assert SR.beam_pool_run(hs, B) == exp, (hs, B)


def test_normalized_score_uses_pow(L):
    for s, n, a in [(-3.5, 7, 1.5), (-1.0, 3, 0.0), (-2.0, 1, 1.0), (-INF, 4, 1.0)]:
        assert L.inference.beam_normalized(s, n, a) == s / math.pow(n, a)


# ---- the whole search on a fake model -------------------------------------------------------------------------------------
class FakeModel:
    """next-token tables as a function of the whole history: top 2B (token, logprob) pairs, logprobs non-increasing, with
    ties and -inf tails; vocabulary V"""

    def __init__(self, seed, B, V=10):
        self.seed, self.B, self.V = seed, B, V

    def top(self, hist):
        rng = np.random.default_rng([self.seed] + [int(t) + 1 for t in hist])
        n = min(2 * self.B, self.V)
        toks = rng.permutation(self.V)[:n]
        lps = -np.sort(rng.choice([0.25, 0.5, 0.5, 1.0, 1.5, 2.0, 3.0], size=n))
        if rng.random() < 0.2:
            lps[-1] = -INF
        return [(int(t), float(x)) for t, x in zip(toks, lps)]


class FakeBeamContext:
    """n_seq 'caches' of token ids; records computed from the cache rows that precede them, so a missing or wrong reorder
    changes what later steps see.  Every call is recorded."""

    def __init__(self, model, seq_len, n_seq):
        self.model, self.SequenceLength, self.max_rows, self.n_seq = model, seq_len, 8, n_seq
        self.cache = [[-1] * seq_len for _ in range(n_seq)]
        self.rec = [dict() for _ in range(n_seq)]
        self.calls = []
        self.lp = {}

    def set_logprobs(self, seq, top_n):
        self.lp[seq] = top_n

    def prefill(self, tokens):
        self.calls.append(("forward", 0, len(tokens)))
        for p, t in enumerate(tokens):
            self.cache[0][p] = int(t)
        self.rec[0][len(tokens)] = self.model.top(self.cache[0][:len(tokens)])

    def forward_batch(self, tokens, positions):
        self.calls.append(("forward", len(tokens), list(positions)))
        for b, (t, p) in enumerate(zip(tokens, positions)):
            assert all(x >= 0 for x in self.cache[b][:p]), "a row before the fed position was never filled"
            self.cache[b][p] = int(t)
            self.rec[b][p + 1] = self.model.top(self.cache[b][:p + 1])
        return np.zeros(len(tokens), np.int32), None

    def read_logprobs(self, seq, pos0, n):
        self.calls.append(("records", seq, pos0))
        assert n == 1 and self.lp.get(seq) == 2 * self.model.B
        top = self.rec[seq][pos0]
        return [type("R", (), dict(Token=top[0][0], Logprob=top[0][1], Rank=1, Top=top))()]

    def copy_sequences(self, src, dst, pos0, pos1):
        self.calls.append(("copy", list(src), list(dst), pos0, pos1))
        assert len(set(dst)) == len(dst) and 0 <= pos0 < pos1 <= self.SequenceLength
        snap = [list(self.cache[s][pos0:pos1]) for s in src]
        for d, rows in zip(dst, snap):
            self.cache[d][pos0:pos1] = rows


def _engine(L, stop):
    class T:
        @staticmethod
        def forward_argmax(ctx, tokens, start):
            assert start == 0
            ctx.prefill(list(tokens))
            return 0, None

    class M:
        Vocabulary = L.model.Vocabulary(StopTokenIds=tuple(stop))
        Transformer = T
    return L.inference.InferenceEngine(M, L.model.InferenceArgs(0))


def _c_search(SR, model, prompt, seq_len, stop, B, alpha, early):
    caches = [[-1] * seq_len for _ in range(B)]
    caches[0][:len(prompt)] = list(prompt)

    def step(k, last):
        if k == 0:
            return [model.top(caches[0][:len(prompt)])]
        out = []
        for b, t in enumerate(last):
            p = len(prompt) + k - 1
            caches[b][p] = t
            out.append(model.top(caches[b][:p + 1]))
        return out

    def reorder(src, dst, pos0, pos1):
        snap = [list(caches[s][pos0:pos1]) for s in src]
        for d, rows in zip(dst, snap):
            caches[d][pos0:pos1] = rows
    return SR.beam_search_io(step, reorder, len(prompt), seq_len, stop, B, alpha, early)


CASES = [(B, alpha, early, seed) for B in (1, 2, 3, 4, 8) for alpha in (0.0, 1.0, 1.5) for early in (False, True)
         for seed in range(2)]


@pytest.mark.parametrize("B,alpha,early,seed", CASES)
def test_search_python_equals_c_statement(L, SR, B, alpha, early, seed):
    model = FakeModel(seed * 31 + B, B)
    prompt = [3, 7, 2][:1 + seed % 3] if seed else [5, 1, 4, 1, 5]
    seq_len = len(prompt) + 6 + B
    stop = (0, 1)
    eng = _engine(L, stop)
    ctx = FakeBeamContext(model, seq_len, B)
    got = eng._generate_beams(ctx, prompt, L.inference.BeamSearchArgs(B, alpha, early))
    exp = _c_search(SR, model, prompt, seq_len, stop, B, alpha, early)
    assert len(got) == len(exp) >= 1
    for g, e in zip(got, exp):
        assert g.Tokens == e["tokens"] and g.Logprobs == e["logprobs"] and g.State == e["state"]
        assert g.Score == e["s"] and (g.NormalizedScore == e["h"] or (math.isnan(g.NormalizedScore) and math.isnan(e["h"])))
    # independent of both loops: every hypothesis's logprobs are the model's for its own history, s their sequential sum
    for g in got:
        s = 0.0
        for i, t in enumerate(g.Tokens):
            lp = dict(model.top(prompt + g.Tokens[:i]))[t]
            assert g.Logprobs[i] == lp
            s += lp
        assert g.Score == s
        assert g.State in (L.inference.GSFinishedByReachingEOS, L.inference.GSFinishedByReachingSeqLen)
        assert (g.Tokens[-1] in stop) == (g.State == L.inference.GSFinishedByReachingEOS)
    _check_calls(ctx.calls, len(prompt), B)


def _check_calls(calls, Lp, B):
    """forward -> records -> (copy) per step; the fork copies [0, L) from beam 0; step k's reorder copies [L, L + k)"""
    assert calls[0] == ("forward", 0, Lp)
    k, i = 0, 0
    while i < len(calls):
        assert calls[i][0] == "forward"
        n = 1 if k == 0 else B
        if k:
            assert calls[i] == ("forward", B, [Lp + k - 1] * B)
        recs = calls[i + 1:i + 1 + n]
        assert [c[:2] for c in recs] == [("records", b) for b in range(n)] and all(c[2] == Lp + k for c in recs)
        i += 1 + n
        if i < len(calls) and calls[i][0] == "copy":
            _, src, dst, p0, p1 = calls[i]
            assert all(s != d for s, d in zip(src, dst)) and dst == sorted(dst)
            assert (p0, p1) == ((0, Lp) if k == 0 else (Lp, Lp + k))
            if k == 0:
                assert src == [0] * len(dst)
            i += 1
        k += 1


def test_no_copy_when_every_parent_is_itself(L):
    """a model whose every beam's best continuation stays ahead of the others keeps p_i = i: no copy after the fork"""
    B = 3

    class Dominant:
        def __init__(self):
            self.B = B

        def top(self, hist):
            # after the prompt: tokens 10.. at -1, -2, ..; later every beam has one good continuation and 2B - 1 poor ones,
            # so beam b's rank 0 is the b-th candidate of the walk and becomes new beam b
            if len(hist) == 4:
                return [(10 + j, -1.0 * (j + 1)) for j in range(2 * B)]
            return [(20, -0.001)] + [(21 + j, -1000.0 - j) for j in range(2 * B - 1)]

    ctx = FakeBeamContext(Dominant(), 12, B)
    eng = _engine(L, (0,))
    got = eng._generate_beams(ctx, [1, 2, 3, 4], L.inference.BeamSearchArgs(B, 1.0, False))
    copies = [c for c in ctx.calls if c[0] == "copy"]
    assert copies == [("copy", [0, 0], [1, 2], 0, 4)]
    assert [h.State for h in got] == [L.inference.GSFinishedByReachingSeqLen] * B


def test_b1_early_is_greedy(L):
    """B = 1 with EarlyStopping: the rank-0 token every step, ending at the first stop token (or SequenceLength)"""
    model = FakeModel(7, 1)
    prompt = [2, 2]
    for stop in ((0,), (0, 1, 2, 3), ()):
        ctx = FakeBeamContext(model, 14, 1)
        got = _engine(L, stop)._generate_beams(ctx, prompt, L.inference.BeamSearchArgs(1, 1.0, True))
        greedy, hist = [], list(prompt)
        while True:
            t = model.top(hist)[0][0]
            greedy.append(t)
            hist.append(t)
            if t in stop or len(hist) == 14:
                break
        assert len(got) == 1 and got[0].Tokens == greedy
        assert not [c for c in ctx.calls if c[0] == "copy"]


def test_generate_beams_rejects_combinations_and_bad_args(L):
    eng = _engine(L, (0,))
    for bad in (L.inference.BeamSearchArgs(0), L.inference.BeamSearchArgs(9), L.inference.BeamSearchArgs(2, INF),
                L.inference.BeamSearchArgs(2, NAN), L.inference.BeamSearchArgs(2, NumReturn=3), L.inference.BeamSearchArgs(2, NumReturn=0)):
        with pytest.raises(L.ml.MlError):
            eng.GenerateBeams([1, 2], bad)
    for kw in (dict(sampling=L.model.SamplingArgs(0.7)), dict(penalties=L.model.PenaltyArgs(1.2)),
               dict(speculative=L.inference.SpeculativeArgs(2))):
        with pytest.raises(L.ml.MlError):
            eng.GenerateBeams([1, 2], L.inference.BeamSearchArgs(2), **kw)


def test_copy_sequences_is_bound(L):
    assert "lnb_session_copy_sequences" in L._capi.SIGNATURES
    assert hasattr(L.model.InferenceContext, "copy_sequences")


def test_pool_statement_rejects_sizes_outside_1_8(SR):
    for B in (0, 9):
        with pytest.raises(ValueError):
            SR.beam_pool_run([-1.0, -2.0], B)
