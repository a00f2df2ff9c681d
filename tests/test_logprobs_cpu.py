"""Token log-probabilities without a GPU (DESIGN.md §9d): the sequential C statement (orc_logprob_row in
oracle_sampling/lnb_sample_ref.c) against an independent restatement in Python integers, the contract against an exact
log-softmax within its stated bound, and the host loops' record bookkeeping against fake contexts."""
import math

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR


def _ord(x) -> int:
    u = int(np.float32(x).view(np.uint32))
    return (~u & 0xFFFFFFFF) if u & 0x80000000 else (u | 0x80000000)


def _finish(l, m, S) -> float:
    """(f64(l) - f64(m)) - log(f64(S) 2^-40); log(0) is -inf as in C"""
    d = float(l) - float(m)
    x = math.ldexp(float(S), -40)
    return d - (math.log(x) if x > 0 else -math.inf)


def _restate(row, target: int, top_n: int) -> dict:
    row = np.asarray(row, np.float32)
    V = row.shape[0]
    order = sorted(range(V), key=lambda i: (-_ord(row[i]), i))
    m = row[order[0]]
    with np.errstate(invalid="ignore", over="ignore"):
        z = row - m                                    # f32 - f32: one rounded f32 operation
    assert z.dtype == np.float32
    keep = z >= np.float32(-28.0)
    e = SR.exp_det(np.where(keep, z, 0).astype(np.float64))
    W = np.where(keep, np.floor(e * 2.0 ** 40), 0).astype(np.uint64)
    S = sum(int(w) for w in W)
    n_top = min(top_n, V)
    return dict(token=target, rank=order.index(target) + 1, logprob=_finish(row[target], m, S), n_top=n_top,
                top_token=order[:n_top], top_logprob=[_finish(row[i], m, S) for i in order[:n_top]])


def _bits(x: float) -> int:
    return int(np.float64(x).view(np.uint64))


def _check_rows(rows, targets, top_n):
    got = SR.logprob_rows(rows, targets, top_n)
    for r, (row, t) in enumerate(zip(rows, targets)):
        want = _restate(row, int(t), top_n)
        g = got[r]
        assert int(g["token"]) == want["token"] and int(g["rank"]) == want["rank"] and int(g["n_top"]) == want["n_top"], r
        assert _bits(g["logprob"]) == _bits(want["logprob"]), (r, g["logprob"], want["logprob"])
        n = want["n_top"]
        assert list(g["top_token"][:n]) == want["top_token"], r
        assert [_bits(x) for x in g["top_logprob"][:n]] == [_bits(x) for x in want["top_logprob"]], r
        assert not g["top_token"][n:].any() and not g["top_logprob"][n:].any()


@pytest.mark.parametrize("V", [64, 4097, 128256])
@pytest.mark.parametrize("top_n", [0, 1, 20])
def test_statement_equals_restatement_on_random_rows(V, top_n):
    rng = np.random.default_rng(V * 31 + top_n)
    n = 3 if V > 5000 else 8
    rows = (rng.standard_normal((n, V)) * rng.choice([0.5, 3.0, 12.0], size=(n, 1))).astype(np.float32)
    targets = rng.integers(0, V, size=n)
    targets[0] = int(np.argmax(rows[0]))               # the greedy token: rank 1
    _check_rows(rows, targets, top_n)


def test_statement_on_ties():
    rng = np.random.default_rng(5)
    V = 300
    rows = np.round(rng.standard_normal((6, V)) * 2).astype(np.float32)   # few distinct values: ties everywhere
    rows[1, :] = 1.5                                                        # all equal
    rows[2, [7, 100, 299]] = 50.0                                           # a tie at the top
    targets = np.array([int(np.argmax(rows[0])), 150, 100, 3, 299, 0])
    rows[3, 3] = rows[3, 4] = rows[3, 5]                                    # target tied with neighbours on both sides
    for top_n in (0, 3, 20):
        _check_rows(rows, targets, top_n)
    g = SR.logprob_rows(rows[1:3], [150, 100], 20)
    assert g["rank"][0] == 151 and list(g["top_token"][0][:3]) == [0, 1, 2]   # ties rank by index
    assert g["rank"][1] == 2 and list(g["top_token"][1][:3]) == [7, 100, 299]


def test_statement_targets_below_the_cut():
    V = 1000
    row = np.zeros(V, np.float32)
    row[10] = 40.0
    row[20] = -200.0
    row[30] = np.float32(40.0 - 28.5)
    g = SR.logprob_rows(np.stack([row] * 3), [20, 30, 10], 5)
    _check_rows(np.stack([row] * 3), [20, 30, 10], 5)
    # a target far below the cut still gets its logit's value, not -inf
    assert math.isfinite(g["logprob"][0]) and abs(g["logprob"][0] - (-240.0)) < 1e-6
    assert abs(g["logprob"][1] - (-28.5)) < 1e-6


def test_statement_on_inf_and_nan_rows():
    V = 100
    rows = np.zeros((5, V), np.float32)
    rows[0, 7] = np.inf                     # +inf rank 0: NaN logprobs, rank 1 for it
    rows[1, 9] = np.nan                     # NaN ranks above +inf (the sampler's order)
    rows[2, :] = -np.inf                    # every logit -inf
    rows[3, 4] = -np.inf                    # a -inf target in a finite row
    rows[4, 2] = np.inf
    rows[4, 3] = np.nan
    targets = [7, 9, 0, 4, 5]
    _check_rows(rows, targets, 4)
    g = SR.logprob_rows(rows, targets, 4)
    assert g["rank"][0] == 1 and math.isnan(g["logprob"][0]) and all(math.isnan(x) for x in g["top_logprob"][0][:4])
    assert g["rank"][1] == 1 and math.isnan(g["logprob"][1])
    assert math.isnan(g["logprob"][2])
    assert g["logprob"][3] == -math.inf and g["rank"][3] == V
    assert g["rank"][4] == 6 and list(g["top_token"][4][:3]) == [3, 2, 0] and math.isnan(g["logprob"][4])   # NaN, +inf, then 0, 1, 4


def _bound(V: int) -> float:
    """the contract's distance from the exact log-softmax: f32 rounding of l - m (|l - m| <= 28: 2^-20), the floor of each
    weight (V 2^-40 against a sum >= 1), the cut at -28 (V e^-28)"""
    return 2.0 ** -20 + V * 2.0 ** -40 + V * math.exp(-28.0)


def _exact(row, t) -> float:
    r = [float(x) for x in row]
    m = max(r)
    return (r[t] - m) - math.log(math.fsum(math.exp(x - m) for x in r))


def _stress_rows():
    V = 128256
    rng = np.random.default_rng(9)
    out = []
    # f32 rounding of l - m: a top logit that makes every difference inexact, the mass spread near -1 .. -27
    row = (-rng.uniform(1.0, 27.0, V)).astype(np.float32)
    row[0] = np.float32(0.1)
    out.append(row)
    # the floor: most of the vocabulary just above the cut, where a weight is ~8
    row = np.full(V, np.float32(-27.9), np.float32)
    row[5] = 0.0
    out.append(row)
    # the cut: most of the vocabulary just below -28, where the contract drops e^-28 per token
    row = np.full(V, np.float32(-28.0001), np.float32)
    row[11] = 0.0
    out.append(row)
    return out


def test_contract_within_its_bound_of_the_exact_log_softmax():
    rows = _stress_rows()
    targets = [0, 5, 11]
    got = SR.logprob_rows(np.stack(rows), targets, 20)
    B = _bound(rows[0].shape[0])
    assert B < 1.3e-6
    worst = 0.0
    for r, (row, t) in enumerate(zip(rows, targets)):
        for j in range(20):
            tok = int(got["top_token"][r][j])
            err = abs(got["top_logprob"][r][j] - _exact(row, tok))
            worst = max(worst, err)
            assert err <= B, (r, j, err, B)
        assert abs(got["logprob"][r] - _exact(row, t)) <= B
    assert worst > 0.0


def test_a_broken_finish_fails_the_bound():
    """the bound check has teeth: dropping the 2^-40 scale of the sum (the ldexp) is caught"""
    row = _stress_rows()[0]
    t = 0
    m = float(row.max())
    keep = (row - np.float32(m)) >= np.float32(-28.0)
    e = SR.exp_det(np.where(keep, row - np.float32(m), 0).astype(np.float64))
    S = int(np.where(keep, np.floor(e * 2.0 ** 40), 0).astype(np.uint64).sum())
    broken = (float(row[t]) - m) - math.log(float(S))
    good = _finish(row[t], m, S)
    assert abs(good - _exact(row, t)) <= _bound(row.shape[0])
    assert abs(broken - _exact(row, t)) > _bound(row.shape[0])


# ---- the host loops' bookkeeping, against fake contexts that record what the library would -----------------------------

@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _engine(L, stop_id=999):
    class M:
        Vocabulary = L.model.Vocabulary(StopTokenIds=(stop_id,))
    return L.inference.InferenceEngine(M, L.model.InferenceArgs(0))


class _Records:
    """the library's record store: every emitted token of sequence k writes record (k, p_next); read_logprobs returns
    TokenLogprob(token, -p_next, ...) so a test can see which position it read"""

    def __init__(self):
        self.rec, self.top = {}, {}

    def set_logprobs(self, seq, top_n):
        self.top[seq] = top_n

    def write(self, k, p, tok):
        if self.top.get(k) is not None:
            self.rec[(k, p)] = tok

    def read_logprobs(self, seq, pos0, n):
        import lnb_b200
        return [lnb_b200.model.TokenLogprob(self.rec.get((seq, p), -1), -float(p), 1, []) for p in range(pos0, pos0 + n)]


class FakeSpecContext(_Records):
    def __init__(self, seq_len, tok):
        super().__init__()
        self.SequenceLength, self.max_rows, self.tok = seq_len, 8, tok

    def forward_speculative(self, segs):
        out, acc = [], []
        for s, p, t in segs:
            nxt = [self.tok(s, p + 1 + j) for j in range(len(t))]
            for j, x in enumerate(nxt):               # every row writes its record, accepted or not
                self.write(s, p + 1 + j, x)
            a = 0
            while a < len(t) - 1 and nxt[a] == t[a + 1]:
                a += 1
            out += nxt
            acc.append(a)
        return np.array(out, np.int32), np.array(acc, np.int32), None


def test_speculative_loop_collects_the_records_of_accepted_positions(L):
    seq_len = 40

    def tok(i, p):
        return 10 + p % 3 if i == 0 else 999 if p == 25 else 20 + p % 5

    prompts = [[10, 11, 12, 10, 11], [20, 21, 22, 23, 24, 20]]
    ctx = FakeSpecContext(seq_len, tok)
    for i in range(2):
        ctx.set_logprobs(i, 3)
    hists = [p + [tok(i, len(p))] for i, p in enumerate(prompts)]
    lp = [[], []]
    out = list(_engine(L)._generate_speculative(ctx, hists, [0, 1], L.inference.SpeculativeArgs(5), None, None, lp))
    for i, p in enumerate(prompts):
        emitted = [t for s, _, t in out if s == i]
        assert [r.Token for r in lp[i]] == emitted
        assert [-r.Logprob for r in lp[i]] == list(range(len(p) + 1, len(p) + 1 + len(emitted)))


class FakeContinuousContext(_Records):
    def __init__(self, seq_len, max_rows):
        super().__init__()
        self.SequenceLength, self.max_rows = seq_len, max_rows
        self.sampling = {}

    @staticmethod
    def tok(k, p):
        return 100 + (7 * k + 3 * p) % 50

    def forward_ragged(self, segs):
        out = []
        for k, start, toks in segs:
            p = start + len(toks)
            out.append(self.tok(k, p))
            self.write(k, p, out[-1])                 # also for a chunk that does not end its prompt
        return np.array(out, np.int32), None

    def forward_batch(self, toks, poss):
        out = [self.tok(k, p + 1) for k, p in enumerate(poss)]
        for k, p in enumerate(poss):
            self.write(k, p + 1, out[k])
        return np.array(out, np.int32), None


def test_continuous_loop_collects_one_record_per_emitted_token(L):
    prompts = [[1] * n for n in (3, 9, 1, 14, 5)]
    ctx = FakeContinuousContext(seq_len=24, max_rows=8)
    lp = []
    out = list(_engine(L)._generate_continuous(ctx, prompts, 2, 8, None, None, 4, lp))
    assert ctx.top == {0: 4, 1: 4}
    assert len(lp) == len(prompts)
    for i, p in enumerate(prompts):
        emitted = [t for s, _, t in out if s == i]
        assert len(emitted) == 24 - len(p)
        assert [r.Token for r in lp[i]] == emitted
        assert [-r.Logprob for r in lp[i]] == list(range(len(p), 24))


def test_continuous_loop_without_logprobs_reads_nothing(L):
    ctx = FakeContinuousContext(seq_len=12, max_rows=8)
    ctx.read_logprobs = None   # would fail if called
    lp = []
    out = list(_engine(L)._generate_continuous(ctx, [[1, 2], [3]], 2, 8, None, None, None, lp))
    assert out and lp == [] and ctx.top == {}
