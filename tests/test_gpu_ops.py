"""GPU parity tests of the op-level C-ABI (what the src/ml shims bind) against the CPU oracle.
STRICT accumulation must be bit-identical to the oracle; FAST must be bit-identical to the NumPy
emulation of its documented order and within 1 bf16 ulp of the oracle."""
import math

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import bf, bf16_ulp_diff, emulate_fast_linear, emulate_fast_rms_scale, f32, rand_bf16, reference_vectors

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def test_device_present(L):
    assert L._capi.lib.lnb_device_count() >= 1


# ---- the reference's own golden cases, through the C-ABI (src/ml/operations_test.go:831-946) ----

def test_linear_bf16_reference_golden(L):
    ml = L.ml
    g = reference_vectors()["linear_bf16"]          # tests/golden: TestLinearTransformationBF16's literals
    w, x, exp = ml.Tensor.from_f32(g["weightVals"]), ml.Tensor.from_f32(g["inputVals"]), np.array(g["expected"], np.float32)
    got = ml.LinearTransformation(x, w)
    assert got.Size == [2, 4]
    assert np.abs(got.to_f32_array() - exp).max() <= 1e-3      # common.THRESHOLD_F32
    assert np.array_equal(got.RawData, O.linear_bf16(x.RawData, w.RawData))


def test_matmul_bf16_reference_golden(L):
    ml = L.ml
    g = reference_vectors()["matmul_bf16"]          # tests/golden: TestMatMulBF16's literals
    a, b, exp = ml.Tensor.from_f32(g["inputVals"]), ml.Tensor.from_f32(g["otherVals"]), np.array(g["expected"], np.float32)
    got = ml.MatMul(a, b)
    assert got.Size == [2, 2, 4]
    assert np.abs(got.to_f32_array() - exp).max() <= 1e-3
    assert np.array_equal(got.RawData, O.matmul_bf16(a.RawData, b.RawData))


def test_linear_shape_errors_like_reference(L):
    ml = L.ml
    with pytest.raises(ml.MlError, match="columns size"):
        ml.LinearTransformation(ml.Tensor.from_f32(np.zeros((2, 3))), ml.Tensor.from_f32(np.zeros((4, 5))))
    with pytest.raises(ml.MlError, match="same data type"):
        ml.LinearTransformation(ml.Tensor.from_f32(np.zeros((2, 3))), ml.Tensor.from_f32(np.zeros((4, 3)), ml.DT_F32))


# ---- panel GEMV vs oracle -------------------------------------------------------------------

@pytest.mark.parametrize("S,K,N", [(1, 64, 16), (1, 256, 48), (1, 4096, 4096), (2, 512, 32), (5, 1024, 96),
                                   (8, 4096, 1024), (11, 256, 64), (1, 14336, 512), (3, 14336, 64), (1, 264, 32),
                                   (1, 8, 16), (1, 1000, 20)])
def test_linear_strict_bit_exact(L, S, K, N):
    rng = np.random.default_rng(S * 1000003 + K * 101 + N)
    x = rand_bf16(rng, (S, K))
    w = rand_bf16(rng, (N, K), 1.0 / math.sqrt(K))
    ml = L.ml
    ml.ACC_MODE = L._capi.LNB_ACC_STRICT
    got = ml.LinearTransformation(ml.Tensor(x, ml.DT_BF16), ml.Tensor(w, ml.DT_BF16)).RawData
    exp = O.linear_bf16(x, w)
    assert np.array_equal(got, exp), f"{(got != exp).sum()} of {got.size} outputs differ"


@pytest.mark.parametrize("S,K,N", [(1, 64, 16), (1, 4096, 4096), (2, 512, 32), (8, 4096, 256), (1, 14336, 512),
                                   (1, 264, 32), (3, 72, 48)])
def test_linear_fast_matches_documented_order(L, S, K, N):
    rng = np.random.default_rng(S * 7 + K * 13 + N)
    x = rand_bf16(rng, (S, K))
    w = rand_bf16(rng, (N, K), 1.0 / math.sqrt(K))
    ml = L.ml
    ml.ACC_MODE = L._capi.LNB_ACC_FAST
    try:
        got = ml.LinearTransformation(ml.Tensor(x, ml.DT_BF16), ml.Tensor(w, ml.DT_BF16)).RawData
    finally:
        ml.ACC_MODE = L._capi.LNB_ACC_STRICT
    emu = emulate_fast_linear(x, w)
    assert np.array_equal(got, emu), f"{(got != emu).sum()} of {got.size} differ from the emulated FAST order"
    exp = O.linear_bf16(x, w)
    d = bf16_ulp_diff(got, exp)
    # reorder noise only: never more than 1 bf16 ulp unless the result is a cancellation near zero
    big = np.abs(f32(exp)) > 1e-2
    assert d[big].max(initial=0) <= 1
    assert (d > 0).mean() < 0.02


# ---- RMSNorm / RoPE / attention / elementwise ----------------------------------------------

@pytest.mark.parametrize("S,D", [(1, 4096), (3, 4096), (2, 256), (1, 1000)])
def test_rmsnorm_strict_bit_exact(L, S, D):
    rng = np.random.default_rng(D + S)
    x, w = rand_bf16(rng, (S, D), 2.0), bf(1 + 0.1 * rng.standard_normal(D))
    out = np.empty((S, D), np.uint16)
    c = L._capi
    c.check(c.lib.lnb_op_rmsnorm_bf16(c.ptr(x, c.u16p), c.ptr(w, c.u16p), c.ptr(out, c.u16p), S, D, 1e-5, c.LNB_ACC_STRICT))
    assert np.array_equal(out, O.rmsnorm(x, w, 1e-5))


def _adversarial_rows(rng, S, D):
    rows = []
    for s in range(S):
        k = s % 7
        if k == 0: v = rng.standard_normal(D) * 2.0
        elif k == 1: v = rng.standard_normal(D) * np.exp(rng.uniform(-20, 20, D))
        elif k == 2: v = np.where(rng.random(D) < 0.9, 0.0, rng.standard_normal(D))
        elif k == 3: v = rng.integers(1, 256, D).astype(np.float32) * 2.0 ** rng.integers(-8, 8)   # exact rounding ties
        elif k == 4: v = np.full(D, rng.uniform(0.1, 3.0))
        elif k == 5: v = rng.standard_normal(D) * np.linspace(1e-6, 1e3, D)
        else: v = rng.standard_normal(D) * np.linspace(1e3, 1e-6, D)
        rows.append(bf(np.asarray(v, np.float32)))
    return np.stack(rows)


@pytest.mark.parametrize("D", [4096, 8192, 256, 128, 64])
def test_rms_scale_scan_and_chain_bit_exact(L, D):
    """the two binade-scan kernels (csrc/seqsum.cuh) and the one-thread FADD chain all reproduce the reference's
    sequential fp32 mean of squares bit for bit, on rows built to hit rounding ties / binade jumps / zeros"""
    rng = np.random.default_rng(D)
    S = 28
    x = _adversarial_rows(rng, S, D)
    x[-1] = 0                                   # all-zero row: 1/sqrt(eps)
    exp = O.rms_scale(x, 1e-5)
    c = L._capi
    for algo in (4, 3, 2, 1, 0):                # 4 = the decode engine's in-CTA variant (warp-local runs, csrc/engine.cuh)
        if algo == 4 and D > 4096:
            continue                            # 256 threads x 16 squares
        r = np.empty(S, np.float32)
        c.check(c.lib.lnb_op_rms_scale_f32(c.ptr(x, c.u16p), c.ptr(r, c.f32p), S, D, 1e-5, algo))
        assert np.array_equal(r.view(np.uint32), exp.view(np.uint32)), (algo, np.nonzero(r != exp))


def test_rms_scale_scan_rejects_unfit_rows(L):
    c = L._capi
    x = np.zeros((1, 1000), np.uint16)
    r = np.empty(1, np.float32)
    with pytest.raises(c.LnbError):
        c.check(c.lib.lnb_op_rms_scale_f32(c.ptr(x, c.u16p), c.ptr(r, c.f32p), 1, 1000, 1e-5, 2))
    with pytest.raises(c.LnbError):
        c.check(c.lib.lnb_op_rms_scale_f32(c.ptr(x, c.u16p), c.ptr(r, c.f32p), 1, 1000, 1e-5, 3))
    c.check(c.lib.lnb_op_rms_scale_f32(c.ptr(x, c.u16p), c.ptr(r, c.f32p), 1, 1000, 1e-5, 0))   # falls back to the chain
    assert r[0] == O.rms_scale(x, 1e-5)[0]


def test_rmsnorm_fast_matches_documented_order(L):
    rng = np.random.default_rng(5)
    S, D = 2, 4096
    x, w = rand_bf16(rng, (S, D), 2.0), bf(1 + 0.1 * rng.standard_normal(D))
    out = np.empty((S, D), np.uint16)
    c = L._capi
    c.check(c.lib.lnb_op_rmsnorm_bf16(c.ptr(x, c.u16p), c.ptr(w, c.u16p), c.ptr(out, c.u16p), S, D, 1e-5, c.LNB_ACC_FAST))
    for s in range(S):
        r = emulate_fast_rms_scale(x[s], 1e-5)
        n1 = bf(f32(x[s]) * r)
        assert np.array_equal(out[s], bf(f32(n1) * f32(w)))
    assert bf16_ulp_diff(out, O.rmsnorm(x, w, 1e-5)).max() <= 1


def test_rope_bit_exact(L):
    rng = np.random.default_rng(6)
    _, cis = O.rope_table(128, 300, 500000.0, True)
    for S, H, pos in [(1, 32, 0), (1, 8, 137), (5, 32, 0), (3, 8, 255)]:
        x = rand_bf16(rng, (S, H, 128))
        out = np.empty_like(x)
        c = L._capi
        c.check(c.lib.lnb_op_rope_bf16(c.ptr(x, c.u16p), c.ptr(cis, c.f32p), c.ptr(out, c.u16p), S, H, 128, pos))
        assert np.array_equal(out, O.rope_apply(x, cis, pos))


@pytest.mark.parametrize("S,T,causal", [(1, 1, 0), (1, 37, 0), (1, 135, 0), (5, 5, 1), (8, 8, 1), (1, 300, 0), (70, 70, 1),
                                        (200, 200, 1)])
def test_attention_strict_bit_exact(L, S, T, causal):
    rng = np.random.default_rng(S * 31 + T)
    nh, nkv, hd = 32, 8, 128
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (T, nkv, hd)), rand_bf16(rng, (T, nkv, hd))
    out = np.empty((S, nh * hd), np.uint16)
    c = L._capi
    c.check(c.lib.lnb_op_attention_bf16(c.ptr(q, c.u16p), c.ptr(ck, c.u16p), c.ptr(cv, c.u16p), c.ptr(out, c.u16p),
                                        S, T, nh, nkv, hd, causal, c.LNB_ACC_STRICT))
    exp = O.attention(q, ck, cv, T, causal)
    assert np.array_equal(out, exp), f"{(out != exp).sum()} of {out.size} differ"
    c.check(c.lib.lnb_op_attention_bf16(c.ptr(q, c.u16p), c.ptr(ck, c.u16p), c.ptr(cv, c.u16p), c.ptr(out, c.u16p),
                                        S, T, nh, nkv, hd, causal, c.LNB_ACC_FAST))
    if S >= 32 and causal:
        # prompt-sized FAST attention runs sdpa_tc_kernel: q.k and p.v accumulate in the tensor core's order, so a score or an
        # output can land on the other side of a bf16 truncation boundary (a small fraction of the outputs, by at most one
        # bf16 ulp).  The order-free checks of both FAST prompt kernels are test_attention_fast_prompt_within_order_free_bounds
        # and test_attention_mask_probes below
        d = np.abs(O.bf16_to_f32(out).astype(np.float64) - O.bf16_to_f32(exp).astype(np.float64))
        assert d.max() <= 2.0 ** -7 and (out != exp).mean() < 5e-3
    else:
        # FAST only reorders the f64 softmax denominator
        assert bf16_ulp_diff(out, exp).max() <= 1 and (out != exp).mean() < 1e-3


def test_attention_mask_shape_error(L):
    c = L._capi
    z = np.zeros((2, 8, 32), np.uint16)
    k = np.zeros((5, 2, 32), np.uint16)
    out = np.zeros((2, 256), np.uint16)
    rc = c.lib.lnb_op_attention_bf16(c.ptr(z, c.u16p), c.ptr(k, c.u16p), c.ptr(k, c.u16p), c.ptr(out, c.u16p), 2, 5, 8, 2, 32, 1, 0)
    assert rc == -1 and b"T == S" in c.lib.lnb_last_error()


def test_elementwise_ops_bit_exact(L):
    ml = L.ml
    rng = np.random.default_rng(7)
    a, b = rand_bf16(rng, (3, 1000), 3.0), rand_bf16(rng, (3, 1000), 3.0)
    ta, tb = ml.Tensor(a, ml.DT_BF16), ml.Tensor(b, ml.DT_BF16)
    assert np.array_equal(ml.Add(ta, tb).RawData, O.add_bf16(a, b))
    assert np.array_equal(ml.MultiplyElementwise(ta, tb).RawData, O.mul_bf16(a, b))
    allbits = np.arange(65536, dtype=np.uint16)
    got, exp = ml.Silu(ml.Tensor(allbits, ml.DT_BF16)).RawData, O.silu_bf16(allbits)
    assert np.array_equal(got, exp)                       # every entry of TABLE_SILU


def test_softmax_argmax_getrows(L):
    ml = L.ml
    rng = np.random.default_rng(8)
    x = (rng.standard_normal((4, 135)) * 2).astype(np.float32)
    assert np.array_equal(ml.Softmax(ml.Tensor(x, ml.DT_F32), 1).RawData, O.softmax_f32(x))
    lg = f32(rand_bf16(rng, (3, 128256), 0.25)).reshape(3, 128256)
    lg[1, 500] = lg[1].max(); lg[1, 90000] = lg[1].max()              # tie -> lowest index
    lg[2, :] = np.nan
    got = ml.Argmax(ml.Tensor(lg, ml.DT_F32), 1).RawData
    assert list(got) == [O.argmax_f32(lg[0]), 500, -1]
    emb = rand_bf16(rng, (64, 256))
    tok = np.array([5, 0, 63, 5], np.int32)
    got = ml.Fwd_Get_Rows(ml.Tensor(emb, ml.DT_BF16), ml.Tensor(tok, ml.DT_INT32)).RawData
    assert np.array_equal(got, emb[tok])
    with pytest.raises(L._capi.LnbError):
        ml.Fwd_Get_Rows(ml.Tensor(emb, ml.DT_BF16), ml.Tensor(np.array([64], np.int32), ml.DT_INT32))


# ---- tensor-core prefill GEMM (wgmma) behind ml.LinearTransformation -------------------------

@pytest.mark.parametrize("S,K,N", [(32, 64, 128), (128, 128, 128), (200, 4096, 256), (256, 1024, 1024), (130, 14336, 128)])
def test_linear_tensor_core_prefill(L, S, K, N):
    """LNB_ACC_FAST with a prompt-sized S runs gemm_tc_kernel: same products, fp32 accumulation in the
    tensor core's own order -> at most 1 bf16 ulp away from the reference order (reorder noise only)."""
    rng = np.random.default_rng(S + K + N)
    x = rand_bf16(rng, (S, K))
    w = rand_bf16(rng, (N, K), 1.0 / math.sqrt(K))
    ml = L.ml
    ml.ACC_MODE = L._capi.LNB_ACC_FAST
    try:
        got = ml.LinearTransformation(ml.Tensor(x, ml.DT_BF16), ml.Tensor(w, ml.DT_BF16)).RawData
    finally:
        ml.ACC_MODE = L._capi.LNB_ACC_STRICT
    exp = O.linear_bf16(x, w)
    d = bf16_ulp_diff(got, exp)
    big = np.abs(f32(exp)).reshape(exp.shape) > 1e-2
    assert d[big].max(initial=0) <= 1, f"max ulp diff {d[big].max()}"
    assert (d > 0).mean() < 0.03, f"{(d > 0).mean():.4f} of outputs differ"
    # exactly representable case: small integers -> every accumulation order gives the same bits
    xi = bf(rng.integers(-3, 4, size=(S, K)).astype(np.float32)).reshape(S, K)
    wi = bf(rng.integers(-2, 3, size=(N, K)).astype(np.float32)).reshape(N, K)
    ml.ACC_MODE = L._capi.LNB_ACC_FAST
    try:
        got = ml.LinearTransformation(ml.Tensor(xi, ml.DT_BF16), ml.Tensor(wi, ml.DT_BF16)).RawData
    finally:
        ml.ACC_MODE = L._capi.LNB_ACC_STRICT
    assert np.array_equal(got, O.linear_bf16(xi, wi))


# ---- gemm_tc_kernel at its tile edges: exact data, order-free bounds, row independence --------------------------------

def _linear(L, x, w, acc):
    ml = L.ml
    ml.ACC_MODE = acc
    try:
        return ml.LinearTransformation(ml.Tensor(x, ml.DT_BF16), ml.Tensor(w, ml.DT_BF16)).RawData
    finally:
        ml.ACC_MODE = L._capi.LNB_ACC_STRICT


# M: one partial M tile, one row short of / exactly / one row past a 128-row tile, 16 tiles.  K in 128-wide k-tiles: 1, 2,
# 3 (= TC_NS, the ring fills exactly), 4 (first reuse of stage 0), 32 and 112 (the mbarrier phase flips many times).
# N: one, two and twelve 128-column tiles, and the stacked w1|w3 width.
TC_EDGES = [(32, 128, 128), (127, 256, 256), (128, 384, 128), (129, 512, 1536), (255, 4096, 256), (2048, 512, 256),
            (129, 14336, 128), (32, 4096, 28672), (128, 128, 1536), (255, 256, 128)]


@pytest.mark.parametrize("M,K,N", TC_EDGES)
def test_gemm_tc_edges_exact_bounded_and_row_independent(L, M, K, N):
    """lnb_op_linear_bf16 in FAST mode at M >= 32 runs gemm_tc_kernel (tc_eligible: N % 128 == 0, K % 128 == 0).
    (1) exact data: integers |x|, |w| <= 15, every row of X and every row of W scaled by its own power of two, so each
    output's partial sums are integers of one common unit below 2^22 -- exact in fp32 in any order: the result must be
    bit-identical to the oracle and to the f64 value truncated to bf16.  (2) random data: every output inside
    tests.precise.linear_bounds.  (3) a row's result does not depend on the other rows: a prefix of X gives the prefix of
    the output, and permuting X's rows permutes the output rows, bit for bit."""
    from tests import precise as P
    assert M >= 32 and N % 128 == 0 and K % 128 == 0
    fast = L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(M * 31 + K * 7 + N)
    rs = rng.integers(-6, 7, M).astype(np.float64)
    cs = rng.integers(-6, 7, N).astype(np.float64)
    xv = rng.integers(-15, 16, (M, K)) * 2.0 ** rs[:, None]
    wv = rng.integers(-15, 16, (N, K)) * 2.0 ** cs[:, None]
    xi, wi = bf(xv).reshape(M, K), bf(wv).reshape(N, K)
    assert np.array_equal(f32(xi).reshape(M, K), xv) and np.array_equal(f32(wi).reshape(N, K), wv)
    got = _linear(L, xi, wi, fast)
    exact = xv @ wv.T
    assert np.abs(exact / (2.0 ** (rs[:, None] + cs[None, :]))).max() < 2 ** 22
    assert np.array_equal(got, bf(exact).reshape(M, N)), f"{(got != bf(exact).reshape(M, N)).sum()} of {got.size} differ"
    assert np.array_equal(got, O.linear_bf16(xi, wi))

    x = rand_bf16(rng, (M, K))
    w = rand_bf16(rng, (N, K), 1.0 / math.sqrt(K))
    got = _linear(L, x, w, fast)
    lo, hi = P.linear_bounds(x, w)
    assert P.within(got, lo, hi).all(), P.outside_report(got, lo, hi)
    if M > 32:
        m1 = max(32, M // 2 + 1)
        assert np.array_equal(_linear(L, np.ascontiguousarray(x[:m1]), w, fast), got[:m1]), f"prefix of {m1} rows"
    perm = rng.permutation(M)
    assert np.array_equal(_linear(L, np.ascontiguousarray(x[perm]), w, fast), got[perm]), "permuted rows"


# ---- prompt attention: STRICT sdpa_kernel, FAST sdpa_tc_kernel and sdpa_prefill_kernel, with a start position ---------

def _attention(L, q, ck, cv, S, T, causal, acc):
    nh, hd = q.shape[1], q.shape[2]
    nkv = ck.shape[1]
    out = np.empty((S, nh * hd), np.uint16)
    c = L._capi
    c.check(c.lib.lnb_op_attention_bf16(c.ptr(q, c.u16p), c.ptr(ck, c.u16p), c.ptr(cv, c.u16p), c.ptr(out, c.u16p),
                                        S, T, nh, nkv, hd, causal, acc))
    return out


# (S, T - S, n_heads, n_kv): S on both sides of the 64-key tile, the 128-row query tile and the 32-row FMA tile; starts that
# are 0, 1, and multiples and non-multiples of 64; n_rep 1, 4 and 8
ATTN_CASES = [(32, 0, 8, 8), (63, 1, 32, 8), (64, 40, 32, 4), (65, 64, 8, 8), (127, 100, 32, 8), (128, 1, 8, 8),
              (129, 0, 32, 4), (200, 64, 8, 8), (513, 100, 32, 8), (129, 40, 8, 8), (64, 0, 32, 8), (200, 1, 32, 4)]
FAST_KERNELS = ["sdpa_tc", "sdpa_prefill"]


@pytest.mark.parametrize("S,dpos,nh,nkv", ATTN_CASES)
def test_attention_chunk_mask_strict_bit_exact(L, S, dpos, nh, nkv):
    """causal_mask = 2 (query row s at position T - S + s) in STRICT runs sdpa_kernel: the oracle's bits"""
    T, hd = S + dpos, 128
    rng = np.random.default_rng(S * 131 + dpos)
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (T, nkv, hd)), rand_bf16(rng, (T, nkv, hd))
    exp = O.attention(q, ck, cv, T, 1, q_pos0=dpos)
    got = _attention(L, q, ck, cv, S, T, 2, L._capi.LNB_ACC_STRICT)
    assert np.array_equal(got, exp), f"{(got != exp).sum()} of {got.size} differ"
    if dpos == 0:
        assert np.array_equal(_attention(L, q, ck, cv, S, T, 1, L._capi.LNB_ACC_STRICT), exp)


@pytest.mark.parametrize("kernel", FAST_KERNELS)
@pytest.mark.parametrize("S,dpos,nh,nkv", ATTN_CASES)
def test_attention_fast_prompt_within_order_free_bounds(L, S, dpos, nh, nkv, kernel, monkeypatch):
    """FAST prompt attention (S >= 32, causal_mask = 2) on sdpa_tc_kernel, and on sdpa_prefill_kernel with LNB_SDPA_TC=0.
    Exact-score inputs: every output inside tests.precise.attention_bounds (a statement about the exact softmax weights,
    not about the STRICT summation order).  Random inputs: the reorder statistics against the STRICT oracle."""
    from tests import precise as P
    if kernel == "sdpa_prefill":
        monkeypatch.setenv("LNB_SDPA_TC", "0")
    T, hd = S + dpos, 128
    fast = L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(S * 17 + dpos + nh)
    q, ck = P.exact_score_qk(rng, S, T, nh, nkv, hd)
    cv = rand_bf16(rng, (T, nkv, hd))
    got = _attention(L, q, ck, cv, S, T, 2, fast)
    lo, hi = P.attention_bounds(q, ck, cv, T, dpos)
    assert P.within(got, lo, hi).all(), P.outside_report(got, lo, hi)
    if dpos == 0:
        assert np.array_equal(_attention(L, q, ck, cv, S, T, 1, fast), got)
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (T, nkv, hd)), rand_bf16(rng, (T, nkv, hd))
    got = _attention(L, q, ck, cv, S, T, 2, fast)
    exp = O.attention(q, ck, cv, T, 1, q_pos0=dpos)
    d = np.abs(f32(got).astype(np.float64) - f32(exp).astype(np.float64))
    assert d.max() <= 2.0 ** -7 and (got != exp).mean() < 5e-3, (d.max(), (got != exp).mean())


def _mask_probe(T, nh, nkv, S, pos0, hd=128):
    """q, k, v for which the diagonal key (t = qpos) and the first masked key (t = qpos + 1) of every row score 512 / t(sqrt(128))
    and every other key at most half of that: key t is 16 at dimension t % 64 and 16 at 64 + t // 64; row qpos asks for
    both coordinates of qpos and of qpos + 1.  (Across a 64-key block boundary key qpos - 63 scores high too.)  v row t
    carries the bits of t as +-2 in dimensions 0..9, so the output names the keys a row attends to."""
    def onehot(t):
        e = np.zeros(hd, np.float32)
        e[t % 64] = 16
        e[64 + t // 64] = 16
        return e
    k1 = np.stack([onehot(t) for t in range(T)])
    q1 = np.stack([np.maximum(onehot(p), onehot(p + 1)) for p in range(pos0, pos0 + S)])
    v1 = np.zeros((T, hd), np.float32)
    for j in range(10):
        v1[:, j] = 4 * ((np.arange(T) >> j) & 1) - 2
    q = bf(np.repeat(q1[:, None, :], nh, 1)).reshape(S, nh, hd)
    k = bf(np.repeat(k1[:, None, :], nkv, 1)).reshape(T, nkv, hd)
    v = bf(np.repeat(v1[:, None, :], nkv, 1)).reshape(T, nkv, hd)
    return q, k, v


@pytest.mark.parametrize("kernel", FAST_KERNELS + ["strict"])
@pytest.mark.parametrize("S,pos0", [(200, 0), (129, 64), (129, 128), (150, 40), (96, 100), (64, 1), (40, 191)])
def test_attention_mask_probes(L, S, pos0, kernel, monkeypatch):
    """the causal boundary itself: with these inputs a leaked first future key, or a lost diagonal key, moves each row's
    output by at least 0.25 (shown on the exact softmax below), so any such row fails; starts on and off multiples of 64
    and 128"""
    from tests import precise as P
    if kernel == "sdpa_prefill":
        monkeypatch.setenv("LNB_SDPA_TC", "0")
    nh, nkv, T = 8, 2, S + pos0
    q, k, v = _mask_probe(T, nh, nkv, S, pos0)
    assert P.exact_score_inputs(q, k)
    acc = L._capi.LNB_ACC_STRICT if kernel == "strict" else L._capi.LNB_ACC_FAST
    got = f32(_attention(L, q, k, v, S, T, 2, acc)).reshape(S, nh, 128)[:, :, :10].astype(np.float64)
    vis = P.visible_keys(S, T, pos0)
    rows = np.arange(S)
    vf = f32(v).reshape(T, nkv, 128)[:, :1, :10].astype(np.float64)

    def out(visible):
        p = P.attention_probs(q[:, :1], k[:, :1], T, visible)
        return np.einsum("sht,thd->shd", p, vf)[:, 0]

    ok = out(vis)
    leak = vis.copy()
    fut = rows[pos0 + rows + 1 < T]
    leak[fut, pos0 + fut + 1] = True
    assert (np.abs(out(leak) - ok).max(1)[fut] >= 0.25).all()
    nodiag = vis.copy()
    nodiag[rows, pos0 + rows] = False
    probed = rows[pos0 + rows > 0]                                  # row at position 0 sees only its diagonal
    with np.errstate(invalid="ignore"):
        assert (np.abs(out(nodiag) - ok).max(1)[probed] >= 0.25).all()
    err = np.abs(got - ok[:, None, :]).max((1, 2))
    assert (err < 0.125).all(), f"rows {np.nonzero(err >= 0.125)[0][:10]} attend to the wrong keys (max err {err.max()})"
