"""Order-free references for the tensor-core kernels (gemm_tc.cuh, sdpa_tc.cuh).

The wgmma accumulation order belongs to the hardware, so a FAST tensor-core result cannot be emulated bit for bit.
These helpers bound it instead: the exact value of each sum in f64, widened by the worst error any fp32 summation
order can add, then truncated to bf16 at both ends.  Truncation toward zero is monotone, so an fp32 accumulator
anywhere inside [v - e, v + e] truncates to a bf16 value inside [t(v - e), t(v + e)].

    e = n * 2^-23 * sum_k |x_k * w_k|      n = number of terms

2^-23 is one fp32 ulp relative, not half of one: it allows an adder that truncates as well as one that rounds to
nearest, so no rounding mode of the tensor core's internal accumulation is assumed.  The products of two bf16 values
are exact in fp32 and in f64.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

_F32_MIN_NORMAL = 2.0 ** -126


def trunc_bf16(x) -> np.ndarray:
    """f64 values -> the bf16 value truncation toward zero gives (kept as f64): the top 8 significant bits.  For a value
    below fp32's normal range the real truncation lands closer to zero than this, so callers bounding from that side
    must widen to 0 (linear_bounds / attention_bounds do)."""
    b = np.ascontiguousarray(x, np.float64).view(np.uint64) & np.uint64(~((1 << 45) - 1) & (2 ** 64 - 1))
    return b.view(np.float64)


def _interval(v, a, n):
    """[t(v - e), t(v + e)] with e = n * 2^-23 * a; a little wider to cover the f64 rounding of v and a themselves"""
    e = np.asarray(n, np.float64) * 2.0 ** -23 * a * (1.0 + 2.0 ** -20)
    lo, hi = trunc_bf16(v - e), trunc_bf16(v + e)
    lo = np.where((lo > 0) & (lo < _F32_MIN_NORMAL), 0.0, lo)
    hi = np.where((hi < 0) & (hi > -_F32_MIN_NORMAL), 0.0, hi)
    return lo, hi


def linear_bounds(x_bits, w_bits):
    """x[S, K], w[N, K] bf16 bits -> (lo, hi) [S, N] f64: every fp32 accumulation order of sum_k x[s, k] * w[n, k],
    truncated to bf16, lies in [lo, hi] (n = K)"""
    x = O.bf16_to_f32(x_bits).astype(np.float64).reshape(np.shape(x_bits))
    w = O.bf16_to_f32(w_bits).astype(np.float64).reshape(np.shape(w_bits))
    return _interval(x @ w.T, np.abs(x) @ np.abs(w).T, x.shape[1])


def within(got_bits, lo, hi):
    """bool mask: the bf16 outputs that lie inside their intervals"""
    g = O.bf16_to_f32(got_bits).astype(np.float64).reshape(np.shape(lo))
    return (g >= lo) & (g <= hi)


def outside_report(got_bits, lo, hi) -> str:
    ok = within(got_bits, lo, hi)
    bad = np.argwhere(~ok)
    if not len(bad):
        return "all inside"
    g = O.bf16_to_f32(got_bits).astype(np.float64).reshape(np.shape(lo))
    i = tuple(bad[0])
    return f"{len(bad)} of {ok.size} outside; first at {i}: {g[i]!r} not in [{lo[i]!r}, {hi[i]!r}]"


# ---- attention --------------------------------------------------------------------------------------------------

def exact_score_inputs(q_bits, k_bits) -> bool:
    """True when every partial sum of every q.k dot product is exactly representable in fp32, whatever the order: all
    q values are integers times one power of two, all k values integers times another, and hd * max|q| * max|k|, in
    those units, stays below 2^24"""
    q = O.bf16_to_f32(q_bits).astype(np.float64)
    k = O.bf16_to_f32(k_bits).astype(np.float64)

    def unit(a):
        nz = np.abs(a[a != 0])
        if not len(nz):
            return 1.0, 0.0
        u = 2.0 ** np.floor(np.log2(nz.min()))
        while not np.all(np.mod(a / u, 1.0) == 0):
            u /= 2
        return u, np.abs(a).max() / u

    (uq, mq), (uk, mk) = unit(q), unit(k)
    return q_bits.shape[-1] * mq * mk < 2.0 ** 24


def attention_scale(hd: int) -> np.float32:
    """t(f32(sqrt(hd))) as the reference divides by it (llamatransformer.go:464)"""
    return O.bf16_to_f32(O.bf16_bits(np.float32(np.sqrt(np.float64(hd)))))[()]


def visible_keys(S: int, T: int, pos0: int, causal: bool = True) -> np.ndarray:
    """[S, T] bool: query row s (position pos0 + s) sees key t"""
    t = np.arange(T)[None, :]
    s = np.arange(S)[:, None]
    return (t <= pos0 + s) if causal else np.ones((S, T), bool)


def attention_probs(q_bits, k_bits, T: int, visible) -> np.ndarray:
    """p[S, nh, T] = t(f32(e / Z)) of the reference (llamatransformer.go:459-495) for exact-score inputs; `visible` is
    the [S, T] mask.  The scores are the reference's bits: each q.k sum is exact, then truncated to bf16, divided by
    t(sqrt(hd)) in fp32 and truncated again.  e = exp in f64 and Z is summed in f64, so only Z's order can differ from
    the kernel's; it moves Z by a few f64 ulps, and a p that flips across a bf16 boundary because of that has a
    probability of about 2^-45 per element."""
    S, nh, hd = q_bits.shape
    nkv = k_bits.shape[1]
    rep = nh // nkv
    q = O.bf16_to_f32(q_bits).astype(np.float64).reshape(S, nh, hd)
    k = O.bf16_to_f32(k_bits[:T]).astype(np.float64).reshape(T, nkv, hd)
    kk = np.repeat(k, rep, axis=1)                                       # expanded head H <- kv head H / n_rep
    raw = np.einsum("shd,thd->sht", q, kk)                               # exact (exact_score_inputs)
    sc = O.bf16_to_f32(O.bf16_bits(raw.astype(np.float32)))
    sc = O.bf16_to_f32(O.bf16_bits(sc / attention_scale(hd)))           # fp32 division, then t(.)
    e = np.where(visible[:, None, :], np.exp(sc.astype(np.float64)), 0.0)
    z = e.sum(-1, keepdims=True)
    return O.bf16_to_f32(O.bf16_bits((e / z).astype(np.float32))).astype(np.float64)


def attention_bounds(q_bits, k_bits, v_bits, T: int, pos0: int, causal: bool = True):
    """(lo, hi) [S, nh * hd] f64 for the attention output of q[S, nh, hd] over cache rows [0, T) of k, v [>= T, nkv, hd],
    query row s at position pos0 + s.  Only O = P . V is reordered by a tiled kernel; it is bounded with n = the
    number of keys row s sees.  Requires exact-score inputs (exact_score_inputs)."""
    if not exact_score_inputs(q_bits, k_bits):
        raise ValueError("q.k sums are not exact in fp32 for these inputs")
    S, nh, hd = q_bits.shape
    vis = visible_keys(S, T, pos0, causal)
    p = attention_probs(q_bits, k_bits, T, vis)
    nkv = v_bits.shape[1]
    v = np.repeat(O.bf16_to_f32(v_bits[:T]).astype(np.float64).reshape(T, nkv, hd), nh // nkv, axis=1)
    o = np.einsum("sht,thd->shd", p, v)
    a = np.einsum("sht,thd->shd", p, np.abs(v))
    n = vis.sum(1).astype(np.float64)[:, None, None]
    lo, hi = _interval(o, a, n)
    return lo.reshape(S, nh * hd), hi.reshape(S, nh * hd)


def attention_bounds_general(q_bits, k_bits, v_bits, positions):
    """(lo, hi) [S, nh * hd] f64 for the attention output of q[S, nh, hd] over the cache rows k, v [T, nkv, hd], query row s
    at position positions[s] (it sees the keys t <= positions[s]), for any data.  Every step is monotone, so interval ends
    carry through: the score t(q.k) in linear_bounds' interval, divided by t(sqrt(hd)) in fp32 and truncated; e = exp at
    both ends (widened by a few f64 ulps for the device's exp); Z in [sum e_lo, sum e_hi] widened by the f64 rounding of
    any order; p = t(f32(e / Z)) in [t(f32(e_lo / Z_hi)), t(f32(e_hi / Z_lo))]; O = sum p v over an interval of p, widened
    by n * 2^-23 * sum p_hi |v| for the fp32 accumulation (n = the keys the row sees).  Sound but looser than
    attention_bounds: it catches layout, head-mapping and position errors, not the last bit of the exact-score kernels."""
    S, nh, hd = q_bits.shape
    T, nkv = k_bits.shape[:2]
    rep = nh // nkv
    pos = np.asarray(positions, np.int64).reshape(S)
    if pos.max() >= T:
        raise ValueError(f"a row at position {pos.max()} needs more than the {T} cache rows given")
    q = O.bf16_to_f32(q_bits).astype(np.float64).reshape(S, nh, hd)
    k = np.repeat(O.bf16_to_f32(k_bits).astype(np.float64).reshape(T, nkv, hd), rep, axis=1)
    v = np.repeat(O.bf16_to_f32(v_bits).astype(np.float64).reshape(T, nkv, hd), rep, axis=1)
    vis = (np.arange(T)[None, :] <= pos[:, None])[:, None, :]                            # [S, 1, T]
    s_lo, s_hi = _interval(np.einsum("shd,thd->sht", q, k), np.einsum("shd,thd->sht", np.abs(q), np.abs(k)), hd)
    scale = attention_scale(hd)

    def scaled(sc):
        return trunc_bf16((sc.astype(np.float32) / scale).astype(np.float64))          # fp32 division (exact: sc is bf16)

    e_lo = np.where(vis, np.exp(scaled(s_lo)) * (1 - 2.0 ** -48), 0.0)
    e_hi = np.where(vis, np.exp(scaled(s_hi)) * (1 + 2.0 ** -48), 0.0)
    n = vis.sum(-1, keepdims=True).astype(np.float64)                                    # [S, 1, 1]
    z_lo = e_lo.sum(-1, keepdims=True) * (1 - (n + 2) * 2.0 ** -52)
    z_hi = e_hi.sum(-1, keepdims=True) * (1 + (n + 2) * 2.0 ** -52)
    p_lo = trunc_bf16((e_lo / z_hi * (1 - 2.0 ** -50)).astype(np.float32).astype(np.float64))
    p_hi = trunc_bf16((e_hi / z_lo * (1 + 2.0 ** -50)).astype(np.float32).astype(np.float64))
    o_lo = np.einsum("sht,thd->shd", p_lo, np.maximum(v, 0)) + np.einsum("sht,thd->shd", p_hi, np.minimum(v, 0))
    o_hi = np.einsum("sht,thd->shd", p_hi, np.maximum(v, 0)) + np.einsum("sht,thd->shd", p_lo, np.minimum(v, 0))
    e = n * 2.0 ** -23 * np.einsum("sht,thd->shd", p_hi, np.abs(v)) * (1.0 + 2.0 ** -20)
    lo, hi = trunc_bf16(o_lo - e), trunc_bf16(o_hi + e)
    lo = np.where((lo > 0) & (lo < _F32_MIN_NORMAL), 0.0, lo)
    hi = np.where((hi < 0) & (hi > -_F32_MIN_NORMAL), 0.0, hi)
    return lo.reshape(S, nh * hd), hi.reshape(S, nh * hd)


# ---- the epilogues and elementwise stages after a GEMM ---------------------------------------------------------------------
# Each takes the stage's input bits and the (lo, hi) intervals of the GEMM outputs it reads, and returns an interval or an
# admissible set of the stage's output.  Truncation toward zero and fp32 rounding are monotone, so an epilogue monotone in
# t(acc) maps the interval ends exactly; the others are evaluated on every bf16 value their inputs may take.

def resid_bounds(res_bits, lo, hi):
    """(lo, hi) of t(f32(res + t(acc))) for t(acc) in [lo, hi]: the residual epilogue (ml.Add(x, t(linear)))"""
    res = O.bf16_to_f32(res_bits).astype(np.float64).reshape(np.shape(lo))
    return (trunc_bf16((res + lo).astype(np.float32).astype(np.float64)),
            trunc_bf16((res + hi).astype(np.float32).astype(np.float64)))


def _key(bits):
    """the monotone integer key of bf16 bits (tests.helpers.bf16_ulp_diff's): -0 and +0 share key 0"""
    u = np.asarray(bits).astype(np.int32)
    return np.where(u & 0x8000, 0x8000 - u, u)


def bf16_values(lo, hi, cap: int = 16):
    """every bf16 value in [lo, hi] (bf16 values as f64), padded with hi to the widest interval: [..., n]; refuses (rather
    than silently widening) an interval of more than `cap` values"""
    k_lo = _key(O.bf16_bits(np.asarray(lo, np.float32)))
    k_hi = _key(O.bf16_bits(np.asarray(hi, np.float32)))
    cnt = k_hi - k_lo + 1
    if cnt.min() < 1:
        raise ValueError("an interval with lo > hi")
    n = int(cnt.max())
    if n > cap:
        raise ValueError(f"an interval holds {n} bf16 values, more than the cap of {cap}")
    k = k_lo[..., None] + np.minimum(np.arange(n), cnt[..., None] - 1)
    bits = np.where(k >= 0, k, 0x8000 - k).astype(np.uint16)
    return O.bf16_to_f32(bits).astype(np.float64).reshape(k.shape)


def _box(a_lo, a_hi, b_lo, b_hi):
    """[min, max] of a * b over a box: the product is linear in each factor, so its extremes are at the corners"""
    c = np.stack([a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi])
    return c.min(0), c.max(0)


_SILU_MONO = {}


def silu_monotone_from(silu_tab) -> float:
    """the least bf16 value g0 such that the table is non-decreasing over every bf16 value >= g0 (SiLU falls below its
    minimum near -1.28, rises above it)"""
    key = id(silu_tab)
    if key not in _SILU_MONO:
        k = np.arange(-0x7f80, 0x7f81)                                   # every finite bf16 value, in increasing order
        bits = np.where(k >= 0, k, 0x8000 - k).astype(np.uint16)
        v = O.bf16_to_f32(silu_tab[bits]).astype(np.float64)
        bad = np.nonzero(np.diff(v) < 0)[0]
        g0 = bits[bad[-1] + 1] if len(bad) else bits[0]
        _SILU_MONO[key] = float(O.bf16_to_f32(np.array([g0], np.uint16))[0])
    return _SILU_MONO[key]


def swiglu_set(glo, ghi, ulo, uhi, silu_tab, cap: int = 16):
    """(lo, hi) [..., n]: the SwiGLU stage t(f32(TABLE_SILU[t(g)] * t(u))) (llamatransformer.go:601-614) for t(g) in
    [glo, ghi] and t(u) in [ulo, uhi] lies in one of n intervals.  Each bf16 gate value g gives the interval
    [t(min), t(max)] of TABLE[g] * u over u's ends (the product of two bf16 values is exact in fp32, and t(s * u) is
    monotone in u).  A gate interval of more than `cap` values (one that crosses zero spans many binades) is taken whole
    where the table is non-decreasing, TABLE[glo] .. TABLE[ghi] then bounding TABLE[g]; anywhere else it is refused rather
    than widened."""
    glo, ghi = np.asarray(glo, np.float64), np.asarray(ghi, np.float64)
    wide = _key(O.bf16_bits(ghi.astype(np.float32))) - _key(O.bf16_bits(glo.astype(np.float32))) + 1 > cap
    if (wide & (glo < silu_monotone_from(silu_tab))).any():
        raise ValueError(f"a gate interval of more than {cap} values where the SiLU table is not monotone")
    g = bf16_values(glo, np.where(wide, glo, ghi), cap)                                 # wide intervals: below
    s = O.bf16_to_f32(silu_tab[O.bf16_bits(g.astype(np.float32))]).astype(np.float64)
    ul, uh = np.asarray(ulo, np.float64)[..., None], np.asarray(uhi, np.float64)[..., None]
    lo, hi = _box(s, s, ul, uh)
    s_lo = O.bf16_to_f32(silu_tab[O.bf16_bits(glo.astype(np.float32))]).astype(np.float64)[..., None]
    s_hi = O.bf16_to_f32(silu_tab[O.bf16_bits(ghi.astype(np.float32))]).astype(np.float64)[..., None]
    wlo, whi = _box(s_lo, s_hi, ul, uh)
    lo = np.where(wide[..., None], wlo, lo)
    hi = np.where(wide[..., None], whi, hi)
    return trunc_bf16(lo), trunc_bf16(hi)


def in_set(got_bits, lo, hi):
    """bool mask: the outputs inside one of their admissible intervals ((lo, hi) [..., n] as from swiglu_set)"""
    g = O.bf16_to_f32(got_bits).astype(np.float64).reshape(np.shape(lo)[:-1])[..., None]
    return ((g >= lo) & (g <= hi)).any(-1)


def set_single_fraction(lo, hi) -> float:
    """the fraction of admissible sets (swiglu_set) that hold one value only"""
    lo, hi = np.asarray(lo), np.asarray(hi)
    return float(np.mean(((lo == hi) & (lo == lo[..., :1])).all(-1)))


def rope_bounds(lo, hi, cis, positions):
    """(lo, hi) [S, H, hd] of RoPE's output (llamatransformer.go:374-403, O.rope_apply) for the pre-rotation values
    x[S, H, hd] in [lo, hi], row s at positions[s].  Each output of a pair, f2bf(f32(a c -+ b d)) in f64, is monotone in a
    and in b separately, so its extremes over the pair's box are among the four corners: the corners rotated by
    O.rope_apply bound every pair of bf16 values the intervals hold.  Covers q and the K cache."""
    S, H, hd = np.shape(lo)
    pos = np.asarray(positions, np.int64).reshape(S)
    outs = []
    for ea in (lo, hi):
        for eb in (lo, hi):
            x = np.empty((S, H, hd), np.float64)
            x[..., 0::2], x[..., 1::2] = ea[..., 0::2], eb[..., 1::2]
            xb = O.bf16_bits(x.astype(np.float32))
            if np.array_equal(pos, pos[0] + np.arange(S)):
                r = O.rope_apply(xb, cis, int(pos[0]))
            else:
                r = np.concatenate([O.rope_apply(np.ascontiguousarray(xb[s:s + 1]), cis, int(pos[s])) for s in range(S)])
            outs.append(O.bf16_to_f32(r).astype(np.float64))
    c = np.stack(outs)
    return c.min(0), c.max(0)


def within_values(got, lo, hi):
    """bool mask: f32 outputs (logits) inside their intervals"""
    g = np.asarray(got, np.float64).reshape(np.shape(lo))
    return (g >= lo) & (g <= hi)


def single_fraction(lo, hi) -> float:
    """the fraction of intervals that admit one bf16 value only"""
    return float(np.mean(np.asarray(lo) == np.asarray(hi)))


def exact_score_qk(rng, S, T, nh, nkv, hd, q_unit=0.5, k_unit=0.5, r=4):
    """random q[S, nh, hd], k[T, nkv, hd] bf16 bits: integers in [-r, r] times a power of two (exact q.k sums; scores
    of a few units, so the softmax is neither flat nor one-hot)"""
    q = O.bf16_bits((rng.integers(-r, r + 1, (S, nh, hd)) * q_unit).astype(np.float32))
    k = O.bf16_bits((rng.integers(-r, r + 1, (T, nkv, hd)) * k_unit).astype(np.float32))
    return q, k
