"""Seeded sampling without a GPU (DESIGN.md §9b): the shared exp against libm, the sequential C statement of the sampler
(oracle_sampling/lnb_sample_ref.c) against an independent restatement in Python integers, its distribution, and the
continuous scheduler's per-prompt seeds against a fake context."""
import math

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR

ONE = 1 << 40


def _ord(x: np.float32) -> int:
    u = int(np.float32(x).view(np.uint32))
    return (~u & 0xFFFFFFFF) if u & 0x80000000 else (u | 0x80000000)


def _splitmix(seed: int, i: int) -> int:
    M = (1 << 64) - 1
    z = (seed + (i + 1) * 0x9E3779B97F4A7C15) & M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
    return z ^ (z >> 31)


def _weights(row, T):
    """W_i of every index (Python ints): z = f32(f32(l - m) / T), W = floor(2^40 exp_det(z)) for z >= -28"""
    row = np.asarray(row, np.float32)
    m = row[max(range(len(row)), key=lambda i: (_ord(row[i]), -i))]
    z = (row - m) / np.float32(T)
    assert z.dtype == np.float32
    return [int(math.floor(math.ldexp(SR.exp_det(float(zi)), 40))) if zi >= -28.0 else 0 for zi in z]


def _kept(row, T, K, P):
    """rank order, the candidate set and the kept set of the contract (lists of indices in rank order)"""
    V = len(row)
    rank = sorted(range(V), key=lambda i: (-_ord(row[i]), i))
    W = _weights(row, T)
    C = rank[: (V if K == 0 or K >= V else K)]
    WC = sum(W[i] for i in C)
    if np.float32(P) >= 1.0 or WC == 0:
        return rank, C, list(C), W
    Q = min(max(math.ceil(float(np.float32(P)) * float(WC)), 1), WC)
    acc, kept = 0, []
    for i in C:
        kept.append(i)
        acc += W[i]
        if acc >= Q:
            break
    return rank, C, kept, W


def restated(row, T, K, P, seed, p_next):
    row = np.asarray(row, np.float32)
    if T == 0:
        return max(range(len(row)), key=lambda i: (_ord(row[i]), -i))
    rank, C, kept, W = _kept(row, T, K, P)
    if sum(W[i] for i in C) == 0:      # every weight 0 (top logit +inf or NaN): the rank-0 token
        return rank[0]
    ks = set(kept)
    Wk = sum(W[i] for i in kept)
    R = (_splitmix(seed & ((1 << 64) - 1), p_next) * Wk) >> 64
    acc = 0
    for i in range(len(row)):
        if i in ks:
            acc += W[i]
            if acc > R:
                return i
    raise AssertionError("no token drawn")


def test_exp_det_is_within_2_ulp_of_libm_on_every_f32_in_range():
    assert SR.exp_det(0.0) == 1.0 and SR.exp_det(-0.0) == 1.0
    # every non-positive f32 down to -1 (bit patterns 0x80000000 .. 0xBF800000), then every f32 in [-28, -1]
    assert SR.exp_det_max_ulp_f32(0x80000000, 0xBF800000) <= 2
    assert SR.exp_det_max_ulp_f32(0xBF800000, 0xC1E00000) <= 2
    rng = np.random.default_rng(5)
    z = -rng.uniform(1.0, 28.0, 10**6).astype(np.float32).astype(np.float64)
    got = SR.exp_det(z)
    ref = np.array([math.exp(v) for v in z])
    ulps = np.abs(got.view(np.int64) - ref.view(np.int64))
    assert ulps.max() <= 2


def _rows(rng, V):
    base = rng.normal(0.0, 2.0, V).astype(np.float32)
    ties = base.copy()
    ties[rng.choice(V, V // 3, replace=False)] = np.float32(ties.max() - 0.5)   # ties straddling any top-k boundary
    quant = np.round(base).astype(np.float32)                                   # many exact ties everywhere
    flat = np.full(V, np.float32(1.25))
    dominant = (rng.normal(0.0, 0.1, V)).astype(np.float32)
    dominant[V // 2] = np.float32(40.0)
    wide = rng.uniform(-60.0, 5.0, V).astype(np.float32)                        # many weights truncated to 0
    inf = base.copy()
    inf[V // 3] = np.float32(np.inf)                                            # l - m is NaN at the top: no weight
    return dict(base=base, ties=ties, quant=quant, flat=flat, dominant=dominant, wide=wide, inf=inf)


@pytest.mark.parametrize("T", [1e-3, 0.7, 1.0, 5.0])
def test_sample_row_equals_independent_restatement(T):
    rng = np.random.default_rng(int(T * 1000))
    V = 67
    for name, row in _rows(rng, V).items():
        for K in (0, 1, 2, 40, V - 1, V):
            for P in (1e-6, 0.5, 0.9, 1.0):
                for seed, pn in ((0, 1), (12345, 77), (2**64 - 1, 4096)):
                    want = restated(row, np.float32(T), K, P, seed, pn)
                    got = SR.sample_row(row, T, K, P, seed, pn)
                    assert got == want, (name, T, K, P, seed, pn)


def test_greedy_special_cases():
    rng = np.random.default_rng(9)
    for name, row in _rows(rng, 130).items():
        greedy = int(np.argmax(row))     # numpy keeps the first maximum, like ml.Argmax
        for seed in range(5):
            assert SR.sample_row(row, 0.0, 0, 1.0, seed, 3) == greedy, name
            assert SR.sample_row(row, 0.8, 1, 0.9, seed, 3) == greedy, name
            assert SR.sample_row(row, 0.8, 0, 1e-9, seed, 3) == greedy, name      # Q <= 2^40: rank 0 alone


def test_draw_depends_only_on_row_params_and_position():
    rng = np.random.default_rng(3)
    row = rng.normal(0, 1, 500).astype(np.float32)
    a = [SR.sample_row(row, 1.0, 0, 1.0, 42, p) for p in range(50)]
    assert a == [SR.sample_row(row.copy(), 1.0, 0, 1.0, 42, p) for p in range(50)]
    assert len(set(a)) > 10                                  # the position moves the draw
    assert a != [SR.sample_row(row, 1.0, 0, 1.0, 43, p) for p in range(50)]


@pytest.mark.parametrize("T,K,P", [(1.0, 0, 1.0), (0.7, 6, 1.0), (1.3, 0, 0.8), (1.0, 10, 0.9)])
def test_distribution_matches_renormalised_softmax(T, K, P):
    from scipy.stats import chisquare
    V = 16
    row = np.linspace(-2.5, 1.0, V).astype(np.float32)[np.random.default_rng(1).permutation(V)]
    rank, C, kept, W = _kept(row, np.float32(T), K, P)
    # the same sets from float64 probabilities
    p = np.exp((row.astype(np.float64) - row.max()) / np.float32(T))
    order = sorted(range(V), key=lambda i: (-row[i], i))
    c64 = order[: (V if K == 0 else K)]
    if P < 1.0:
        cum, k64 = 0.0, []
        tot = sum(p[i] for i in c64)
        for i in c64:
            k64.append(i)
            cum += p[i]
            if cum >= P * tot:
                break
    else:
        k64 = c64
    assert sorted(k64) == sorted(kept)
    counts = np.zeros(V)
    n = 20000
    for j in range(n):
        counts[SR.sample_row(row, T, K, P, 1000 + j // 100, j % 100)] += 1
    assert counts[[i for i in range(V) if i not in kept]].sum() == 0
    q = np.array([p[i] for i in kept])
    res = chisquare(counts[kept], q / q.sum() * n)
    assert res.pvalue > 1e-4, (res, counts[kept])


def test_continuous_scheduler_sets_each_prompts_seed_before_its_first_segment():
    import lnb_b200 as L
    from tests.test_ragged_cpu import FakeContext

    class SamplingFake(FakeContext):
        def set_sampling(self, seq, args):
            self.calls.append(("sampling", seq, args.Seed, args.Temperature))

    prompts = [[5, 6, 7], [8, 9], [10, 11, 12, 13], [14], [15, 16]]

    class M:
        Vocabulary = L.model.Vocabulary(StopTokenIds=(999,))
    eng = L.inference.InferenceEngine(M, L.model.InferenceArgs(16))
    ctx = SamplingFake(16, 8, 2, prompts, {0: {5}, 1: {4}, 2: {7}, 3: {3}}, 999)
    ctx.owner, ctx.started = {}, set()
    args = L.model.SamplingArgs(0.7, 40, 0.9, 100)
    out = list(eng._generate_continuous(ctx, prompts, 2, 8, None, args))
    assert sorted({i for i, _, _ in out}) == list(range(len(prompts)))
    seeds = {}   # slot -> seed set last
    first_seen = set()
    for c in ctx.calls:
        if c[0] == "sampling":
            seeds[c[1]] = c[2]
            assert c[3] == np.float32(0.7) or c[3] == 0.7
        elif c[0] == "ragged":
            for slot, start, _ in c[1]:
                pi = c[2][slot]
                if start == 0:
                    assert pi not in first_seen
                    first_seen.add(pi)
                assert seeds[slot] == 100 + pi, (slot, pi, seeds)
    assert first_seen == set(range(len(prompts)))
    assert len([c for c in ctx.calls if c[0] == "sampling" and c[1] == 0]) >= 2   # a refilled slot switches seeds


def test_reference_api_cannot_sample():
    import lnb_b200 as L

    class M:
        Vocabulary = L.model.Vocabulary(StopTokenIds=(999,))
    eng = L.inference.InferenceEngine(M, L.model.InferenceArgs(16))
    with pytest.raises(L.ml.MlError, match="Argmax"):
        next(eng.GenerateTokens([1, 2], use_reference_api=True, sampling=L.model.SamplingArgs(0.7, 0, 1.0, 1)))


def test_sampling_entry_points_validate_without_gpu():
    import ctypes as C
    import lnb_b200 as L
    lib = L._capi.lib
    assert lib.lnb_session_set_sampling(None, 0, None) == -1
    row = np.zeros(4, np.float32)
    out = np.zeros(1, np.int32)
    pn = np.ones(1, np.int32)
    bad = L._capi.SamplingC(1.0, 0, 0.0, 1)   # top_p outside (0, 1]
    assert lib.lnb_op_sample_f32(L._capi.ptr(row, L._capi.f32p), 1, 4, C.byref(bad), L._capi.ptr(pn, L._capi.i32p),
                                 L._capi.ptr(out, L._capi.i32p)) == -1
