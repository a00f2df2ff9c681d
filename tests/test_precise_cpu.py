"""The order-free references of tests/precise.py are sound (the reference order, and other fp32 orders, land inside the
intervals) and sharp (the mistakes tiled kernels make land outside them).  CPU only."""
import math

import numpy as np
import pytest

from oracle import oracle as O
from tests import precise as P
from tests.helpers import emulate_fast_linear, rand_bf16


def _t(x64):
    """a broken result as a kernel would store it: fp32 accumulator, truncated to bf16"""
    return O.bf16_bits(np.asarray(x64, np.float64).astype(np.float32))


def test_trunc_bf16_matches_the_bf16_conversion():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(10000) * np.exp(rng.uniform(-30, 30, 10000))).astype(np.float32)
    assert np.array_equal(P.trunc_bf16(x.astype(np.float64)), O.bf16_to_f32(O.bf16_bits(x)).astype(np.float64))


@pytest.mark.parametrize("S,K,N", [(3, 64, 16), (17, 512, 40), (5, 4096, 24), (2, 14336, 8)])
def test_linear_bounds_contain_every_summation_order(S, K, N):
    rng = np.random.default_rng(S * 7 + K)
    x = rand_bf16(rng, (S, K))
    w = rand_bf16(rng, (N, K), 1.0 / math.sqrt(K))
    lo, hi = P.linear_bounds(x, w)
    for name, got in (("reference order", O.linear_bf16(x, w)),
                      ("FAST GEMV order", emulate_fast_linear(x, w)),
                      ("reversed order", O.linear_bf16(x[:, ::-1].copy(), w[:, ::-1].copy())),
                      ("BLAS fp32", _t(O.bf16_to_f32(x).reshape(S, K) @ O.bf16_to_f32(w).reshape(N, K).T))):
        assert P.within(got, lo, hi).all(), f"{name}: {P.outside_report(got, lo, hi)}"


@pytest.mark.parametrize("K", [256, 512, 4096])
def test_linear_bounds_reject_broken_results(K):
    rng = np.random.default_rng(K)
    S, N = 8, 256
    x = rand_bf16(rng, (S, K))
    w = rand_bf16(rng, (N, K), 1.0 / math.sqrt(K))
    lo, hi = P.linear_bounds(x, w)
    xf = O.bf16_to_f32(x).astype(np.float64).reshape(S, K)
    wf = O.bf16_to_f32(w).astype(np.float64).reshape(N, K)
    exact = xf @ wf.T
    swapped = exact.copy()
    swapped[:, [5, 130]] = swapped[:, [130, 5]]                       # a wrong column (panel) index in the epilogue
    assert not P.within(_t(swapped), lo, hi)[:, [5, 130]].any()
    for k0 in (0, K // 2 - 64, K - 128):                              # one 128-wide k-tile dropped (a stale / skipped stage)
        keep = np.ones(K, bool)
        keep[k0:k0 + 128] = False
        dropped = xf[:, keep] @ wf[:, keep].T
        assert (~P.within(_t(dropped), lo, hi)).mean() > 0.8, k0
    doubled = exact + xf[:, :128] @ wf[:, :128].T                     # one k-tile accumulated twice (ring phase error)
    assert (~P.within(_t(doubled), lo, hi)).mean() > 0.8


def _attention_inputs(seed, S, T, nh, nkv, hd=128):
    rng = np.random.default_rng(seed)
    q, k = P.exact_score_qk(rng, S, T, nh, nkv, hd)
    v = rand_bf16(rng, (T, nkv, hd))
    return q, k, v


CASES = [(40, 40, 8, 2), (33, 100, 4, 4), (70, 70, 8, 8), (65, 129, 8, 2)]      # (S, T, nh, nkv); T - S is the start


@pytest.mark.parametrize("S,T,nh,nkv", CASES)
def test_attention_bounds_contain_the_reference(S, T, nh, nkv):
    q, k, v = _attention_inputs(S + T, S, T, nh, nkv)
    assert P.exact_score_inputs(q, k)
    pos0 = T - S
    lo, hi = P.attention_bounds(q, k, v, T, pos0)
    exp = O.attention(q, k, v, T, 1, q_pos0=pos0)
    assert P.within(exp, lo, hi).all(), P.outside_report(exp, lo, hi)
    if pos0 == 0:                                                      # the pinned entry point agrees
        assert np.array_equal(exp, O.attention(q, k, v, T, 1))
    lo0, hi0 = P.attention_bounds(q, k, v, T, 0, causal=False)
    exp0 = O.attention(q, k, v, T, 0)
    assert P.within(exp0, lo0, hi0).all(), P.outside_report(exp0, lo0, hi0)


def _broken_attention(q, k, v, T, vis):
    S, nh, hd = q.shape
    nkv = v.shape[1]
    p = P.attention_probs(q, k, T, vis)
    vv = np.repeat(O.bf16_to_f32(v[:T]).astype(np.float64).reshape(T, nkv, hd), nh // nkv, axis=1)
    return _t(np.einsum("sht,thd->shd", p, vv).reshape(S, nh * hd))


@pytest.mark.parametrize("S,T,nh,nkv", CASES)
def test_attention_bounds_reject_mask_and_position_errors(S, T, nh, nkv):
    q, k, v = _attention_inputs(S * 3 + T, S, T, nh, nkv)
    pos0 = T - S
    lo, hi = P.attention_bounds(q, k, v, T, pos0)
    rows = np.arange(S)
    vis = P.visible_keys(S, T, pos0)

    def rejected_rows(vis_bad):
        with np.errstate(invalid="ignore"):                            # a row that sees no key at all: p = 0 / 0
            bad = ~P.within(_broken_attention(q, k, v, T, vis_bad), lo, hi)
        return bad.any(1)

    no_diag = vis.copy()
    no_diag[rows, pos0 + rows] = False                                 # the diagonal key masked
    r = rejected_rows(no_diag)
    assert r[1:].all(), np.nonzero(~r)                                 # row 0 at pos0 0 has no other key: p is 0/0 there
    leak = vis.copy()
    fut = rows[pos0 + rows + 1 < T]
    leak[fut, pos0 + fut + 1] = True                                   # the first future key leaked
    assert rejected_rows(leak)[fut].all()
    for d in (1, -1):                                                  # start position off by one
        shifted = P.visible_keys(S, T, pos0 + d)
        changed = (shifted != vis).any(1) & shifted.any(1)
        assert changed.sum() >= S - 2
        assert rejected_rows(shifted)[changed].all(), d


def test_exact_score_inputs_are_checked():
    rng = np.random.default_rng(3)
    q, k = rand_bf16(rng, (4, 2, 128)), rand_bf16(rng, (8, 2, 128))
    assert not P.exact_score_inputs(q, k)
    with pytest.raises(ValueError):
        P.attention_bounds(q, k, k, 8, 4)
    qi, ki = P.exact_score_qk(rng, 4, 8, 2, 2, 128)
    assert P.exact_score_inputs(qi, ki)
