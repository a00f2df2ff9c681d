"""The MXFP8 KV cache's edge models without a GPU (tests/kv_cases.py): each builder reaches the blocks it claims, the
reference forward stays finite on them, and each of four decodes that are wrong only at the range's ends changes its
logits -- so the GPU tests that compare against that reference would see such a decode."""
import numpy as np
import pytest

import lnb_b200 as L
from oracle import oracle as O
from oracle_sampling import sample_ref as SR
from tests import kv_cases as K
from tests.model_shapes import CATALOGUE, create_error, ss_shape_ok
from tests.test_kvcache_cpu import RefSession

EXTREME = {"tiny": dict(L.synth.TINY), "tiny128": dict(L.synth.TINY128), "hd96": dict(CATALOGUE["hd96"])}
SEED = 23


@pytest.fixture(scope="module")
def extreme():
    made = {}

    def get(name):
        if name not in made:
            args = EXTREME[name]
            t, hot = K.extreme_kv_tensors(args, SEED)
            ref = RefSession(args, t, 48, True)
            p = K.extreme_prompt(args, hot, 40, 3)
            lg = ref.forward(p, 0)
            made[name] = (args, t, hot, p, ref, lg)
        return made[name]
    return get


def _blocks(pre, hd):
    c, s, _ = SR.kv_mxfp8_quantize(pre, hd)
    return c, s.astype(int) - 127


@pytest.mark.parametrize("name", list(EXTREME))
def test_extreme_models_reach_the_range_ends(extreme, name):
    args, _, hot, p, ref, _ = extreme(name)
    hd, n = args["head_dim"], len(p)
    assert hot and all(0 <= t < args["vocab_size"] for t in hot)
    # layer 0, head 0: K blocks at X >= 100, V blocks at X = 119 (elements >= 2^127), saturated codes among them
    ck, Xk = _blocks(ref.pre_k[0][:n], hd)
    cv, Xv = _blocks(ref.pre_v[0][:n], hd)
    assert Xk[:, 0].min() >= 100 and Xk[:, 0].max() <= 119
    assert 119 in set(Xv[:, 0].reshape(-1).tolist())
    assert (O.bf16_to_f32(ref.pre_v[0][:n, :hd]) >= 2.0 ** 127).any() or (O.bf16_to_f32(ref.pre_v[0][:n, :hd]) <= -2.0 ** 127).any()
    assert ((cv[:, :hd] & 0x7F) == 0x7E).any() and ((ck[:, :hd] & 0x7F) == 0x7E).any()
    # the last layer, head 0: every block clamped to X = -117, with subnormal codes and flushed (nonzero -> code 0) ones
    last = args["n_layers"] - 1
    for pre in (ref.pre_k[last][:n], ref.pre_v[last][:n]):
        c, X = _blocks(pre, hd)
        assert (X[:, 0] == -117).all()
        h0, raw = c[:, :hd] & 0x7F, pre[:, :hd] & 0x7FFF
        assert ((h0 > 0) & (h0 < 8)).any(), "no subnormal codes"
        assert ((h0 == 0) & (raw != 0)).any(), "no flushed codes"
        assert np.isfinite(O.bf16_to_f32(pre)).all()
    # ordinary heads beside them in the same rows
    for l in range(args["n_layers"]):
        for pre in (ref.pre_k[l][:n], ref.pre_v[l][:n]):
            X = _blocks(pre, hd)[1]
            assert (X[:, 1:] > -40).all() and (X[:, 1:] < 20).all()


@pytest.mark.parametrize("name", list(EXTREME))
def test_extreme_models_have_ordinary_logits(extreme, name):
    args, t, hot, p, ref, lg = extreme(name)
    assert np.isfinite(lg).all() and float(np.abs(lg).max()) < 100
    fast = RefSession(args, t, 48, True, order=O.ORDER_FAST_STREAM)
    lf = fast.forward(p, 0)
    assert np.isfinite(lf).all() and float(np.abs(lf - lg).max()) < 0.5
    for l in range(args["n_layers"]):            # both orders store finite rows
        assert np.isfinite(O.bf16_to_f32(fast.pre_v[l][:len(p)])).all()


def test_restated_decode_is_the_c_statement(extreme):
    args, _, _, p, ref, _ = extreme("tiny128")
    for l in range(args["n_layers"]):
        for pre in (ref.pre_k[l][:len(p)], ref.pre_v[l][:len(p)]):
            c, s, d = SR.kv_mxfp8_quantize(pre, args["head_dim"])
            assert np.array_equal(K.decode(c, s, args["head_dim"]), d)


BROKEN = {"subnormals flushed": dict(flush_subnormal=True), "X >= 100 one binade high": dict(high_from=100),
          "X = -117 one binade high": dict(high_at=-117), "0x7e read as 0x7d": dict(sat_as_7d=True)}


@pytest.mark.parametrize("broken", list(BROKEN))
@pytest.mark.parametrize("name", list(EXTREME))
def test_broken_decodes_change_the_logits(extreme, name, broken):
    args, t, _, p, _, lg = extreme(name)

    def dec(rows, hd):
        c, s, _ = SR.kv_mxfp8_quantize(rows, hd)
        return K.decode(c, s, hd, **BROKEN[broken])
    bad = RefSession(args, t, 48, True, decode=dec).forward(p, 0)
    assert not np.array_equal(bad.view(np.uint32), lg.view(np.uint32))


def test_nonfinite_model_stores_inf_at_the_token():
    args = dict(L.synth.TINY)
    tok = 77
    t, (jp, jn) = K.nonfinite_kv_tensors(args, SEED, tok)
    p = np.array([5, 9, 300, tok, 12, 40, tok, 3], np.int32)
    for order in (O.ORDER_REF, O.ORDER_FAST_STREAM):
        ref = RefSession(args, t, 16, True, order=order)
        with np.errstate(all="ignore"):
            ref.forward(p, 0)
        v = O.bf16_to_f32(ref.pre_v[0][:len(p)])
        at = np.flatnonzero(p == tok)
        assert (v[at, jp] == np.inf).all() and (v[at, jn] == -np.inf).all()
        others = np.flatnonzero(p != tok)
        assert np.isfinite(v[others]).all() and np.isfinite(O.bf16_to_f32(ref.pre_k[0][:len(p)])).all()
        c, s, _ = SR.kv_mxfp8_quantize(ref.pre_v[0][:len(p)], args["head_dim"])
        assert (c[at, jp] == 0x7E).all() and (c[at, jn] == 0xFE).all()
        assert (s[at, 0, 0] < 127 + 119).all()       # the block's scale comes from its finite elements


@pytest.mark.parametrize("name", list(K.SHAPES))
def test_extra_shapes_are_accepted_and_streamed(name):
    a = K.SHAPES[name]
    assert create_error(a) is None and ss_shape_ok(a)
    assert name not in CATALOGUE
    hd, rep = a["head_dim"], a["n_heads"] // a["n_kv_heads"]
    if name in ("hd40", "hd56"):
        assert hd % 32 in (8, 24)
    if name in ("hd80", "hd112"):
        assert hd % 32 == 16 and (hd // 2) % 32 not in (0,)         # STRICT d-range of hd / 2: a block spans two CTAs
    if name.startswith("rep"):
        assert rep == int(name[3:]) and hd == 32
    if name == "hd128_rep8":
        assert hd == 128 and rep == 8
