"""The order-free references of tests/precise.py are sound (the reference order, and other fp32 orders, land inside the
intervals) and sharp (the mistakes tiled kernels make land outside them).  CPU only."""
import math

import numpy as np
import pytest

from oracle import oracle as O
from tests import precise as P
from tests.helpers import bf, emulate_fast_linear, f32, rand_bf16


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


# ---- the stage references: one transformer layer at TINY and TINY128 widths --------------------------------------------------

# (dim, n_heads, n_kv_heads, head_dim, ffn) of synth.TINY and synth.TINY128
STAGE_WIDTHS = {"tiny": (256, 8, 2, 32, 512), "tiny128": (1024, 8, 2, 128, 1024)}
_SILU = None


def _silu():
    global _SILU
    if _SILU is None:
        _SILU = O.silu_table_bf16()
    return _SILU


def _layer_weights(name, seed=5):
    dim, nh, nkv, hd, ffn = STAGE_WIDTHS[name]
    rng = np.random.default_rng(seed)
    w = {"wq": rand_bf16(rng, (nh * hd, dim), dim ** -0.5), "wk": rand_bf16(rng, (nkv * hd, dim), dim ** -0.5),
         "wv": rand_bf16(rng, (nkv * hd, dim), dim ** -0.5), "wo": rand_bf16(rng, (dim, nh * hd), (nh * hd) ** -0.5),
         "w1": rand_bf16(rng, (ffn, dim), dim ** -0.5), "w3": rand_bf16(rng, (ffn, dim), dim ** -0.5),
         "w2": rand_bf16(rng, (dim, ffn), ffn ** -0.5), "out": rand_bf16(rng, (384, dim), dim ** -0.5),
         "attn_norm": bf(1 + 0.1 * rng.standard_normal(dim)), "ffn_norm": bf(1 + 0.1 * rng.standard_normal(dim)),
         "norm": bf(1 + 0.1 * rng.standard_normal(dim))}
    return w, O.rope_table(hd, 512, 500000.0, True)[1]


def _norm(x, w, parts):
    r = O.rms_scale_order(x, 1e-5, parts)
    return bf(f32(bf(f32(x) * r[:, None])) * f32(w)[None, :]).reshape(x.shape)


def _stages(name, x, pos0, order):
    """every stage of one layer over the rows x [S, dim] at positions pos0.. (cache rows [0, pos0) random), computed by the
    oracle's ops in the reference's order (order "ref") or in LNB_ACC_FAST's (order "fast")"""
    dim, nh, nkv, hd, ffn = STAGE_WIDTHS[name]
    w, cis = _layer_weights(name)
    S = x.shape[0]
    fast = order == "fast"
    lin = (lambda a, b: O.linear_order_bf16(a, b, 8)) if fast else O.linear_bf16
    parts = 256 if fast else 1
    rng = np.random.default_rng(pos0 + S)
    T = pos0 + S
    ck, cv = np.zeros((T, nkv, hd), np.uint16), np.zeros((T, nkv, hd), np.uint16)
    ck[:pos0], cv[:pos0] = rand_bf16(rng, (pos0, nkv, hd)), rand_bf16(rng, (pos0, nkv, hd))
    st = {"x": x, "xn": _norm(x, w["attn_norm"], parts)}
    st["q"] = O.rope_apply(lin(st["xn"], w["wq"]).reshape(S, nh, hd), cis, pos0)
    ck[pos0:] = O.rope_apply(lin(st["xn"], w["wk"]).reshape(S, nkv, hd), cis, pos0)
    cv[pos0:] = lin(st["xn"], w["wv"]).reshape(S, nkv, hd)
    st["ck"], st["cv"] = ck, cv
    st["attn"] = O.attention_order(st["q"], ck, cv, T, 1, pos0, O.ATTN_TREE if fast else O.ATTN_REF)
    st["post"] = O.add_bf16(x, lin(st["attn"], w["wo"]))
    st["xn2"] = _norm(st["post"], w["ffn_norm"], parts)
    sg = _silu()[lin(st["xn2"], w["w1"])]
    st["ffn"] = O.mul_bf16(sg, lin(st["xn2"], w["w3"]))
    st["out"] = O.add_bf16(st["post"], lin(st["ffn"], w["w2"]))
    st["xo"] = _norm(st["out"], w["norm"], parts)
    st["logits"] = f32(lin(st["xo"], w["out"]))
    return st, w, cis


def _stage_bounds(name, st, w, cis, pos0):
    """the admissible output of every stage, from that stage's own input"""
    dim, nh, nkv, hd, ffn = STAGE_WIDTHS[name]
    S = st["x"].shape[0]
    pos = pos0 + np.arange(S)
    b = {"q": [a.reshape(S, -1) for a in P.rope_bounds(*[a.reshape(S, nh, hd) for a in P.linear_bounds(st["xn"], w["wq"])], cis, pos)],
         "k": [a.reshape(S, -1) for a in P.rope_bounds(*[a.reshape(S, nkv, hd) for a in P.linear_bounds(st["xn"], w["wk"])], cis, pos)],
         "v": P.linear_bounds(st["xn"], w["wv"]),
         "attn": P.attention_bounds_general(st["q"], st["ck"], st["cv"], pos),
         "post": P.resid_bounds(st["x"], *P.linear_bounds(st["attn"], w["wo"])),
         "ffn": P.swiglu_set(*P.linear_bounds(st["xn2"], w["w1"]), *P.linear_bounds(st["xn2"], w["w3"]), _silu()),
         "out": P.resid_bounds(st["post"], *P.linear_bounds(st["ffn"], w["w2"])),
         "logits": P.linear_bounds(st["xo"], w["out"])}
    return b


def _stage_inside(st, b, pos0):
    S = st["x"].shape[0]
    return {"q": P.within(st["q"].reshape(S, -1), *b["q"]),
            "k": P.within(st["ck"][pos0:].reshape(S, -1), *b["k"]),
            "v": P.within(st["cv"][pos0:].reshape(S, -1), *b["v"]),
            "attn": P.within(st["attn"], *b["attn"]), "post": P.within(st["post"], *b["post"]),
            "ffn": P.in_set(st["ffn"], *b["ffn"]), "out": P.within(st["out"], *b["out"]),
            "logits": P.within_values(st["logits"], *b["logits"])}


STAGE_CASES = [("tiny", 40, 0), ("tiny", 40, 37), ("tiny128", 33, 0), ("tiny128", 40, 37)]


@pytest.mark.parametrize("order", ["ref", "fast"])
@pytest.mark.parametrize("name,S,pos0", STAGE_CASES)
def test_stage_bounds_contain_the_oracle(name, S, pos0, order):
    x = rand_bf16(np.random.default_rng(S * 3 + pos0), (S, STAGE_WIDTHS[name][0]))
    st, w, cis = _stages(name, x, pos0, order)
    b = _stage_bounds(name, st, w, cis, pos0)
    for k, ok in _stage_inside(st, b, pos0).items():
        assert ok.all(), f"{k}: {(~ok).sum()} of {ok.size} outside"


@pytest.mark.parametrize("name,S,pos0", STAGE_CASES)
def test_stage_bounds_reject_broken_stages(name, S, pos0):
    """each stage computed with one deliberate mistake, from the same inputs, is rejected on at least one element"""
    dim, nh, nkv, hd, ffn = STAGE_WIDTHS[name]
    x = rand_bf16(np.random.default_rng(S * 3 + pos0), (S, dim))
    st, w, cis = _stages(name, x, pos0, "fast")
    b = _stage_bounds(name, st, w, cis, pos0)

    def exact(a, m):
        return f32(a).astype(np.float64).reshape(a.shape) @ f32(m).astype(np.float64).reshape(m.shape).T

    rejected = {}
    # the residual epilogue without the inner t(): t(f32(x + acc))
    acc = exact(st["attn"], w["wo"]).astype(np.float32).astype(np.float64)
    rejected["residual without t(acc)"] = ~P.within(_t(f32(st["x"]).astype(np.float64) + acc), *b["post"])
    # SwiGLU with an untruncated up value, and with gate and up swapped within a half-panel
    g = O.linear_bf16(st["xn2"], w["w1"])
    u = O.linear_bf16(st["xn2"], w["w3"])
    sg = f32(_silu()[g]).astype(np.float64)
    u_acc = exact(st["xn2"], w["w3"]).astype(np.float32).astype(np.float64)
    rejected["SwiGLU with untruncated up"] = ~P.in_set(_t(sg * u_acc), *b["ffn"])
    rejected["SwiGLU with gate and up swapped"] = ~P.in_set(O.mul_bf16(_silu()[u], g), *b["ffn"])
    # logits without t()
    rejected["logits without t()"] = ~P.within_values(exact(st["xo"], w["out"]).astype(np.float32), *b["logits"])
    # q rotated at the neighbouring position
    q_raw = O.linear_bf16(st["xn"], w["wq"]).reshape(S, nh, hd)
    rejected["q at position + 1"] = ~P.within(O.rope_apply(q_raw, cis, pos0 + 1).reshape(S, -1), *b["q"])
    # a GEMM missing its last 64-wide k block (w2, K = ffn)
    short = exact(st["ffn"][:, :-64].copy(), w["w2"][:, :-64].copy())
    rejected["w2 without its last k block"] = ~P.within(_t(f32(st["post"]).astype(np.float64) + f32(_t(short)).astype(np.float64)),
                                                         *b["out"])
    # attention with one key too many: row s sees key pos0 + s + 1 (the last row has none to add)
    T = pos0 + S
    rejected["attention with one key too many"] = ~P.within(
        O.attention_order(st["q"], st["ck"], st["cv"], T, 1, pos0 + 1, O.ATTN_TREE)[:-1], b["attn"][0][:-1], b["attn"][1][:-1])
    for what, bad in rejected.items():
        assert bad.any(), f"{what}: every element inside its admissible set"


def test_bf16_values_enumerates_and_refuses_wide_intervals():
    lo = np.array([1.0, -1.0, -0.0, 0.5])
    hi = np.array([1.0078125, -0.9921875, 2.0 ** -130 * 0, 0.5])
    v = P.bf16_values(lo, hi)
    assert v.shape == (4, 3)
    assert list(v[0]) == [1.0, 1.0078125, 1.0078125]
    assert list(v[1]) == [-1.0, -0.99609375, -0.9921875]
    assert (v[2] == 0).all() and (v[3] == 0.5).all()
    with pytest.raises(ValueError):
        P.bf16_values(np.array([1.0]), np.array([2.0]), cap=16)
