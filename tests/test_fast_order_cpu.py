"""The oracle's statement of LNB_ACC_FAST's summation order (oracle/lnb_oracle.h, orc_order), without a GPU: each piece equals
an independent NumPy restatement of the kernel's order bit for bit, the reference order is untouched, and the FAST order
is far enough from the reference order that the GPU comparisons of tests/test_gpu_fast_order.py can fail."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import emulate_fast_linear, emulate_fast_rms_scale, emulate_z_stream, emulate_z_tree, host_tensors, \
    oracle_model, rand_bf16
from tests.test_gpu_ops import _adversarial_rows

# K: one chunk; 9 chunks (one round of 8 streams plus one); 33 chunks; 125 (not a multiple of 8 chunks); the TINY / 8B widths;
# 514 chunks (two past a multiple of 8); the 8B FFN width
KS = [8, 72, 264, 1000, 4096, 4112, 14336]


@pytest.mark.parametrize("K", KS)
def test_linear_ks8_equals_the_gemv_emulation(K):
    rng = np.random.default_rng(K)
    x = _adversarial_rows(rng, 7, K)
    w = rand_bf16(rng, (24, K), 1.0 / np.sqrt(K))
    got = O.linear_order_bf16(x, w, 8)
    assert np.array_equal(got, emulate_fast_linear(x, w)), f"{(got != emulate_fast_linear(x, w)).sum()} differ"
    assert np.array_equal(O.linear_order_bf16(x, w, 1), O.linear_bf16(x, w))    # ks = 1 is the reference's order
    assert np.array_equal(O.linear_order_bf16(x, w, 4), emulate_fast_linear(x, w, ks=4))


@pytest.mark.parametrize("K", KS)
def test_rms_scale_256_parts_equals_the_prologue_emulation(K):
    rng = np.random.default_rng(K + 1)
    x = _adversarial_rows(rng, 14, K)
    x[-1] = 0                                                   # all-zero row: 1/sqrt(eps)
    got = O.rms_scale_order(x, 1e-5, 256)
    exp = np.array([emulate_fast_rms_scale(r, 1e-5) for r in x], np.float32)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)), np.nonzero(got != exp)
    assert np.array_equal(O.rms_scale_order(x, 1e-5, 1).view(np.uint32), O.rms_scale(x, 1e-5).view(np.uint32))


def test_order_arguments_outside_the_statement_are_refused():
    x = np.zeros((1, 12), np.uint16)
    with pytest.raises(ValueError):
        O.linear_order_bf16(x, np.zeros((8, 12), np.uint16), 8)      # K % 8 != 0
    with pytest.raises(ValueError):
        O.rms_scale_order(x, 1e-5, 48)                               # not whole groups of 32


# T: one key; one short of, exactly and one past the 128 partials; the same around one 1024-key chunk; 3 chunks plus 1
ZT = [1, 127, 128, 129, 1023, 1024, 1025, 3 * 1024 + 1]


@pytest.mark.parametrize("T", ZT)
def test_z_orders_equal_their_numpy_restatement(T):
    rng = np.random.default_rng(T)
    sc = O.bf16_to_f32(rand_bf16(rng, (T,), 3.0))
    e = np.exp(sc.astype(np.float64))
    tree, stream = O.attention_z(e, O.ATTN_TREE), O.attention_z(e, O.ATTN_STREAM)
    assert tree == emulate_z_tree(e)
    assert stream == emulate_z_stream(e)
    ref = 0.0
    for v in e:
        ref += v
    assert O.attention_z(e, O.ATTN_REF) == ref
    if T <= 1024:
        assert stream == tree                                   # one chunk: the chunk sum is added to 0.0
    if T >= 1023:                                               # long sums: the orders give different f64 values
        assert tree != ref


@pytest.mark.parametrize("S,T,causal,q_pos0", [(1, 1, 0, 0), (1, 300, 0, 0), (5, 5, 1, 0), (3, 40, 1, 37), (2, 2100, 1, 2098),
                                               (4, 1030, 0, 0)])
def test_attention_orders_agree_with_the_reference_outside_z_and_chunks(S, T, causal, q_pos0):
    """TREE changes only Z, so it matches the reference wherever Z's last f64 bits do not reach a bf16 output; REF through the
    order entry point is attention's bits; STREAM over one chunk is TREE"""
    rng = np.random.default_rng(S * 7 + T)
    nh, nkv, hd = 8, 2, 32
    q = rand_bf16(rng, (S, nh, hd))
    ck, cv = rand_bf16(rng, (T, nkv, hd)), rand_bf16(rng, (T, nkv, hd))
    ref = O.attention(q, ck, cv, T, causal, q_pos0=q_pos0)
    assert np.array_equal(O.attention_order(q, ck, cv, T, causal, q_pos0, O.ATTN_REF), ref)
    tree = O.attention_order(q, ck, cv, T, causal, q_pos0, O.ATTN_TREE)
    stream = O.attention_order(q, ck, cv, T, causal, q_pos0, O.ATTN_STREAM)
    assert (tree != ref).mean() < 1e-3
    if T <= 1024 or (causal and q_pos0 + S <= 1024):
        assert np.array_equal(stream, tree)


# ---- whole model ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tiny():
    import lnb_b200
    args = dict(lnb_b200.synth.TINY)
    om = oracle_model(args, host_tensors(args, 1234))
    yield args, om
    om.close()


def _run(om, args, toks, order, seq=24):
    s = om.new_session(seq)
    try:
        lg, tr = s.forward(toks[:8], 0, all_rows=True, trace=True, order=order)
        out = [lg]
        for pos in range(8, 12):
            out.append(s.forward(toks[pos:pos + 1], pos, order=order))
        caches = [tuple(c.copy() for c in s.cache(l)) for l in range(args["n_layers"])]
        return np.concatenate(out), tr, caches
    finally:
        s.close()


def test_reference_order_through_the_order_entry_is_orc_forward(tiny):
    args, om = tiny
    toks = np.random.default_rng(3).integers(0, args["vocab_size"], size=24).astype(np.int32)
    a = _run(om, args, toks, None)
    b = _run(om, args, toks, O.ORDER_REF)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    for (ka, va), (kb, vb) in zip(a[2], b[2]):
        assert np.array_equal(ka, kb) and np.array_equal(va, vb)
    s1, s2 = om.new_session(24), om.new_session(24)
    try:
        s1.forward(toks[:8], 0, order=O.ORDER_REF); s2.forward(toks[:8], 0)
        assert np.array_equal(s1.forward_chunk(toks[8:13], 8, order=O.ORDER_REF), s2.forward_chunk(toks[8:13], 8))
    finally:
        s1.close(); s2.close()


def test_fast_statement_is_distinguishable_from_its_neighbours(tiny):
    """the FAST statement differs from the reference order and from 4 k-streams in a nonzero number of TINY logits, so a
    GPU route that sums its projections in either order fails the bit-for-bit comparisons.  The RMS and softmax orders are
    weaker levers: the scale r and Z enter the outputs only through t(x * r) and p = t(f32(e / Z)), so a change in their
    last bits reaches a bf16 value rarely (Z: about 2^-29 per element).  Those orders are pinned value for value by the
    tests above, and at model level only as far as they can be seen."""
    args, om = tiny
    toks = np.random.default_rng(4).integers(0, args["vocab_size"], size=24).astype(np.int32)
    fast = _run(om, args, toks, O.ORDER_FAST)[0]
    for other in (O.ORDER_REF, (4, 256, O.ATTN_TREE), (8, 1, O.ATTN_TREE), (8, 256, O.ATTN_REF)):
        n = int((_run(om, args, toks, other)[0] != fast).sum())
        print(f"{other}: {n} of {fast.size} logits differ from the FAST statement")
        if other[0] != 8:
            assert n > 0, other
