"""Penalties and logit bias without a GPU (DESIGN.md §9e): the sequential C statement (orc_penalize_row in
oracle_sampling/lnb_sample_ref.c) against an independent numpy-float32 restatement, bit for bit, and the host loops'
first_pos and window bookkeeping against recording fake contexts."""
import numpy as np
import pytest

from oracle_sampling import sample_ref as SR

NAN = np.uint32(0x7FFFFFFF).view(np.float32)   # the NaN a step produces (penalty_det.h)


def _canon(x):
    x = np.asarray(x, np.float32)
    return np.where(np.isnan(x), NAN, x).astype(np.float32)


def _restate(row, p: dict, hist, p_next: int, fused: bool = False):
    """l' of the contract in numpy float32: every step one rounded f32 operation.  fused=True is a deliberately broken
    statement (c * fp + pp in one f64 rounding) that the checks below must reject."""
    row = np.asarray(row, np.float32)
    if p.get("rp", 1.0) == 1.0 and p.get("fp", 0.0) == 0.0 and p.get("pp", 0.0) == 0.0 and not p.get("bias"):
        return row.copy()   # neutral parameters: penalties off
    V = row.shape[0]
    hist = np.asarray(hist, np.int64)
    lo = p.get("first_pos", 0)
    if p.get("window", 0) > 0:
        lo = max(lo, p_next - p["window"])
    lo = max(lo, 0)
    h = hist[lo:p_next]
    h = h[(h >= 0) & (h < V)]
    c = np.bincount(h, minlength=V)
    out = row.copy()
    idx = c > 0
    rp, fp, pp = np.float32(p.get("rp", 1.0)), np.float32(p.get("fp", 0.0)), np.float32(p.get("pp", 0.0))
    with np.errstate(all="ignore"):
        a = row[idx]
        if rp != np.float32(1.0):
            a = _canon(np.where(a > 0, a / rp, a * rp))
        cf = c[idx].astype(np.float32)
        if fused:
            d = (cf.astype(np.float64) * np.float64(fp) + np.float64(pp)).astype(np.float32)
        else:
            d = _canon(cf * fp + pp)
        assert d.dtype == np.float32
        out[idx] = _canon(a - d)
        for t, b in p.get("bias", {}).items():
            b = np.float32(b)
            out[t] = -np.inf if b == -np.inf else _canon(out[t] + b)
    return out


def _params(p: dict):
    return SR.penalties(p.get("rp", 1.0), p.get("fp", 0.0), p.get("pp", 0.0), p.get("window", 0), p.get("first_pos", 0),
                        p.get("bias"))


def _check(rows, ps, hists, p_next, fused=False):
    rows = np.asarray(rows, np.float32)
    got = SR.penalize_rows(rows, [_params(p) for p in ps], hists, p_next)
    for r in range(rows.shape[0]):
        exp = _restate(rows[r], ps[r], hists[r], int(p_next[r]), fused)
        bad = np.flatnonzero(got[r].view(np.uint32) != exp.view(np.uint32))
        assert bad.size == 0, (r, bad[:8], got[r][bad[:8]], exp[bad[:8]])


def _random_case(rng, V, T, n):
    rows = rng.standard_normal((n, V)).astype(np.float32) * 4
    hists = rng.integers(-1, V, size=(n, T)).astype(np.int32)
    ps, pn = [], []
    for _ in range(n):
        bias_t = rng.choice(V, size=int(rng.integers(0, min(9, V + 1))), replace=False)
        ps.append(dict(rp=float(rng.choice([0.5, 1.0, 1.1, 1.3, 2.0])), fp=float(rng.uniform(-1, 1)), pp=float(rng.uniform(-1, 1)),
                       window=int(rng.choice([0, 1, 7, T])), first_pos=int(rng.integers(0, T // 2)),
                       bias={int(t): float(rng.choice([rng.uniform(-5, 5), -np.inf])) for t in bias_t}))
        pn.append(int(rng.integers(0, T + 1)))
    return rows, ps, hists, pn


@pytest.mark.parametrize("V,T", [(7, 5), (1000, 300), (4099, 2000)])
def test_statement_equals_restatement_on_random_rows(V, T):
    rng = np.random.default_rng(V)
    _check(*_random_case(rng, V, T, 6))


def test_statement_on_ties_and_negative_logits_under_rp():
    V, T = 64, 40
    row = np.repeat(np.float32([-3.0, -0.0, 0.0, 1.5, -1e-40, 2.0]), 11)[:V].astype(np.float32)
    row = np.concatenate([row, np.zeros(V - row.size, np.float32)])
    hist = (np.arange(T) % V).astype(np.int32)
    ps = [dict(rp=1.3), dict(rp=0.7, fp=0.25), dict(rp=1.3, pp=-0.5), dict(rp=3.0, fp=0.1, pp=0.3, bias={0: 1.0, 5: -np.inf})]
    _check(np.stack([row] * 4), ps, np.stack([hist] * 4), [T] * 4)


def test_statement_on_inf_and_nan():
    V, T = 16, 16
    row = np.array([np.inf, -np.inf, np.nan, 1.0, -1.0, 0.0, 3e38, -3e38] * 2, np.float32)
    row[9] = np.uint32(0xFFC00000).view(np.float32)      # a negative NaN (the x86 default NaN)
    row[10] = np.uint32(0x7FC00001).view(np.float32)     # a payload
    hist = np.arange(T, dtype=np.int32)
    ps = [dict(rp=1.5), dict(fp=2.0, pp=1.0), dict(rp=1e-30), dict(fp=3e38, pp=3e38),       # overflow to +-inf, then inf - inf
          dict(bias={0: -np.inf, 1: 5.0, 2: -np.inf, 9: 1.0, 10: 0.0, 3: -np.inf}),
          dict(rp=2.0, fp=1.0, bias={0: 1.0, 2: 2.0})]
    rows = np.stack([row] * len(ps))
    _check(rows, ps, np.stack([hist] * len(ps)), [T] * len(ps))
    got = SR.penalize_rows(rows[4:5], [_params(ps[4])], hist[None], [T])
    assert got[0][0] == -np.inf and got[0][2] == -np.inf   # -inf bias bans +inf and NaN logits too


def test_statement_counts_up_to_131072():
    V, T = 256, 131072
    rng = np.random.default_rng(3)
    row = rng.standard_normal(V).astype(np.float32)
    hists = [np.full(T, 7, np.int32), rng.integers(0, 3, T).astype(np.int32), np.where(np.arange(T) % 2 == 0, 5, -1).astype(np.int32)]
    ps = [dict(fp=0.1, pp=0.3), dict(rp=1.2, fp=1e-5, pp=0.0), dict(fp=-3.7e-6, pp=0.5)]
    _check(np.stack([row] * 3), ps, np.stack(hists), [T] * 3)
    got = SR.penalize_rows(row[None], [_params(ps[0])], hists[0][None], [T])
    assert got[0][7] == np.float32(row[7] - np.float32(np.float32(np.float32(T) * np.float32(0.1)) + np.float32(0.3)))


def test_statement_window_and_first_pos_edges():
    V, T = 32, 20
    rng = np.random.default_rng(5)
    row = rng.standard_normal(V).astype(np.float32)
    hist = rng.integers(0, V, T).astype(np.int32)
    hist[[3, 11]] = -1
    cases = []
    for pn in (0, 1, 10, T):
        for w in (0, 1, pn, pn + 1, 3):
            for fpos in (0, 1, pn - 1, pn, pn + 2):
                if fpos >= 0:
                    cases.append((dict(rp=1.4, fp=0.5, pp=0.25, window=w, first_pos=fpos), pn))
    ps = [c[0] for c in cases]
    pn = [c[1] for c in cases]
    _check(np.stack([row] * len(ps)), ps, np.stack([hist] * len(ps)), pn)
    # nothing counted: first_pos at p_next, or an empty window
    out = SR.penalize_rows(row[None], [_params(dict(rp=2.0, fp=1.0, first_pos=10))], hist[None], [10])
    assert np.array_equal(out[0].view(np.uint32), row.view(np.uint32))


def test_neutral_parameters_leave_the_row_unchanged():
    rng = np.random.default_rng(9)
    row = rng.standard_normal(500).astype(np.float32)
    row[3] = np.uint32(0xFFC00000).view(np.float32)
    hist = rng.integers(0, 500, 400).astype(np.int32)
    out = SR.penalize_rows(row[None], [SR.penalties()], hist[None], [400])
    assert np.array_equal(out[0].view(np.uint32), row.view(np.uint32))


def test_a_broken_statement_fails_the_check():
    V, T = 256, 131072
    rng = np.random.default_rng(3)
    row = rng.standard_normal(V).astype(np.float32)
    hist = rng.integers(0, V, T).astype(np.int32)
    ps = [dict(fp=0.1, pp=0.3)]
    _check(row[None], ps, hist[None], [T])
    with pytest.raises(AssertionError):
        _check(row[None], ps, hist[None], [T], fused=True)


# ---- host loops: first_pos and window bookkeeping ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _engine(L, stop_id=999):
    M = type("M", (), {})()
    M.Vocabulary = type("V", (), {"StopTokenIds": [stop_id], "PadId": -1})()
    return L.inference.InferenceEngine(M, L.model.InferenceArgs(0))


def test_penalty_args_first_pos_and_window(L):
    P = L.inference.PenaltyArgs
    c = P(1.2, 0.5, -0.25, 64, LogitBias={5: -np.inf, 9: 1.5}).c(17)
    assert (c.first_pos, c.window, c.n_bias) == (17, 64, 2)
    assert (c.bias_token[0], c.bias[0], c.bias_token[1], c.bias[1]) == (5, -np.inf, 9, 1.5)
    assert np.float32(c.repetition_penalty) == np.float32(1.2) and c.presence_penalty == -0.25
    assert P(1.2, CountPrompt=True).c(17).first_pos == 0
    n = P().c(3)
    assert (n.repetition_penalty, n.frequency_penalty, n.presence_penalty, n.n_bias) == (1.0, 0.0, 0.0, 0)
    with pytest.raises(L.ml.MlError):
        P(LogitBias={i: 1.0 for i in range(65)}).c(0)


class FakeContinuousContext:
    """records every set_penalties call with the lnb_penalties it would pass"""

    def __init__(self, seq_len, max_rows):
        self.SequenceLength, self.max_rows = seq_len, max_rows
        self.calls = []

    def set_penalties(self, seq, args, prompt_len):
        c = args.c(prompt_len)
        self.calls.append((seq, c.first_pos, c.window))

    @staticmethod
    def tok(k, p):
        return 100 + 10 * k + p

    def forward_ragged(self, segs):
        return [self.tok(k, p + len(t)) for k, p, t in segs], None

    def forward_batch(self, toks, poss):
        return [self.tok(k, p + 1) for k, p in enumerate(poss)], None


def test_continuous_loop_sets_first_pos_per_admitted_prompt(L):
    ctx = FakeContinuousContext(seq_len=7, max_rows=8)
    prompts = [[1, 2, 3], [4], [5, 6], [7, 8, 9, 10]]
    pen = L.inference.PenaltyArgs(1.3, Window=4)
    out = list(_engine(L)._generate_continuous(ctx, prompts, 2, 8, penalties=pen))
    assert out and {i for i, _, _ in out} == set(range(4))
    # one call per admission, before the prompt's first segment, with first_pos = that prompt's length
    assert sorted(c[1:] for c in ctx.calls) == sorted((len(p), 4) for p in prompts)
    assert [c[0] for c in ctx.calls[:2]] == [0, 1]
    ctx = FakeContinuousContext(seq_len=7, max_rows=8)
    list(_engine(L)._generate_continuous(ctx, prompts, 2, 8, penalties=L.inference.PenaltyArgs(1.3, CountPrompt=True)))
    assert [c[1] for c in ctx.calls] == [0] * 4
    ctx = FakeContinuousContext(seq_len=7, max_rows=8)
    list(_engine(L)._generate_continuous(ctx, prompts, 2, 8))
    assert ctx.calls == []


def test_reference_api_refuses_penalties(L):
    with pytest.raises(L.ml.MlError):
        next(_engine(L).GenerateTokens([1, 2], use_reference_api=True, penalties=L.inference.PenaltyArgs(1.2)))
