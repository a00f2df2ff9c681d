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


def exact_score_qk(rng, S, T, nh, nkv, hd, q_unit=0.5, k_unit=0.5, r=4):
    """random q[S, nh, hd], k[T, nkv, hd] bf16 bits: integers in [-r, r] times a power of two (exact q.k sums; scores
    of a few units, so the softmax is neither flat nor one-hot)"""
    q = O.bf16_bits((rng.integers(-r, r + 1, (S, nh, hd)) * q_unit).astype(np.float32))
    k = O.bf16_bits((rng.integers(-r, r + 1, (T, nkv, hd)) * k_unit).astype(np.float32))
    return q, k
