"""The persistent decode engine (csrc/engine.cuh: one kernel launch = n complete S=1 forwards, phases separated by grid
barriers) against the kernel chain it replaces (LNB_ENGINE=0: one launch per projection / attention / norm-scale) and
against the oracle.  Both paths evaluate the same expressions in the same order, so their logits, KV caches and greedy
tokens must be IDENTICAL in both accumulation modes; STRICT must in addition equal the oracle bit for bit."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module")
def tiny(L):
    args = dict(L.synth.TINY)
    tensors = host_tensors(args, 4321)
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    yield args, om, gm
    gm.Free()
    om.close()


def _context(L, gm, seq, acc, engine: bool, max_rows=8, **kw):
    old = os.environ.get("LNB_ENGINE")
    os.environ["LNB_ENGINE"] = "1" if engine else "0"      # read when the session first decodes
    try:
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=max_rows, acc_mode=acc, **kw)
        # force the probe now, while the variable is set
        gm.Transformer.forward_argmax(ctx, np.array([1], np.int32), 0)
    finally:
        if old is None:
            os.environ.pop("LNB_ENGINE", None)
        else:
            os.environ["LNB_ENGINE"] = old
    return ctx


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_engine_equals_kernel_chain_and_oracle(L, tiny, mode):
    args, om, gm = tiny
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    seq = 40
    prompt = np.array([1, 50, 999, 7, 300, 12, 64, 2], np.int32)
    ce, cc = _context(L, gm, seq, acc, True), _context(L, gm, seq, acc, False)
    osess = om.new_session(seq)
    try:
        l0 = ce.launch_count()
        fe, le = gm.Transformer.forward_argmax(ce, prompt, 0, want_logits="last")
        fc, lc = gm.Transformer.forward_argmax(cc, prompt, 0, want_logits="last")
        assert fe == fc and np.array_equal(le, lc)
        exp = osess.forward(prompt, 0, all_rows=False)
        nxt = O.argmax_f32(exp[0])
        for pos in range(8, 8 + 12):                         # host-driven S=1 steps, teacher-forced with the oracle's token
            te, le = gm.Transformer.forward_argmax(ce, np.array([nxt], np.int32), pos, want_logits="last")
            tc, lc = gm.Transformer.forward_argmax(cc, np.array([nxt], np.int32), pos, want_logits="last")
            assert np.array_equal(le, lc), f"engine and chain logits differ at position {pos}"
            assert te == tc
            exp = osess.forward(np.array([nxt], np.int32), pos, all_rows=False)
            if mode == "strict":
                assert np.array_equal(le, exp), f"position {pos}"
            else:
                assert float(np.abs(le - exp).max()) <= 1e-2
            nxt = O.argmax_f32(exp[0])
        for layer in range(args["n_layers"]):
            assert np.array_equal(ce.CacheK(layer).RawData[:20], cc.CacheK(layer).RawData[:20])
            assert np.array_equal(ce.CacheV(layer).RawData[:20], cc.CacheV(layer).RawData[:20])
        # 13 engine steps = 13 engine launches (+ state kernels); the chain needs an order of magnitude more
        assert ce.launch_count() - l0 < cc.launch_count() - l0
        # device-resident loop: ONE launch for all steps
        first = fe
        l1 = ce.launch_count()
        a, ms, _ = ce.decode_run(first, 8, seq - 9, use_graph=True)
        assert ce.launch_count() - l1 <= 3
        b, _, _ = cc.decode_run(first, 8, seq - 9, use_graph=True)
        assert list(a) == list(b) and ms > 0
        if mode == "strict":
            assert [first] + list(a) == list(om.generate(prompt, seq, stop_ids=(10**9,)))
    finally:
        ce.close(); cc.close(); osess.close()


def test_tensor_core_prompt_after_an_engine_step_reads_back_its_own_residual(L, tiny):
    """The engine keeps its residual row as tagged words; a FAST prompt of >= 32 rows on the tensor cores that follows an
    engine step must leave LNB_BUF_RESIDUAL holding the prompt's [S, dim] rows, equal to those of a session without the
    engine."""
    args, om, gm = tiny
    acc, seq, S = L._capi.LNB_ACC_FAST, 48, 40
    prompt = np.random.default_rng(11).integers(0, args["vocab_size"], size=S).astype(np.int32)
    ce = _context(L, gm, seq, acc, True, max_rows=S)     # _context runs one S=1 step: on the engine here
    cc = _context(L, gm, seq, acc, False, max_rows=S)
    try:
        assert ce.uses_engine() and not cc.uses_engine()
        n0 = ce.launch_count()
        te, le = gm.Transformer.forward_argmax(ce, prompt, 0, want_logits="last")
        # the tensor-core path: set_state, gather_rows, 8 kernels per layer (sdpa_kernel at head_dim 32), the last row's GEMV
        assert ce.launch_count() - n0 == 1 + 1 + 8 * args["n_layers"] + 1
        tc, lc = gm.Transformer.forward_argmax(cc, prompt, 0, want_logits="last")
        assert te == tc and np.array_equal(le, lc)
        assert np.array_equal(ce.residual(S), cc.residual(S))
    finally:
        ce.close(); cc.close()


def test_engine_follows_active_sequence_layer_limit_and_kept_logits(L, tiny):
    args, om, gm = tiny
    seq = 32
    ce = _context(L, gm, seq, L._capi.LNB_ACC_STRICT, True, n_seq=2)
    try:
        prompts = [[1, 50, 999, 7], [3, 4, 5, 6, 7, 8]]
        for i, p in enumerate(prompts):
            ce.set_active_sequence(i)
            first, _ = gm.Transformer.forward_argmax(ce, np.array(p, np.int32), 0)
            toks, _, _ = ce.decode_run(first, len(p), 8)
            assert [first] + list(toks) == list(om.generate(p, len(p) + 9, stop_ids=(10**9,))), i
        ce.set_active_sequence(0)
        ce.set_layer_limit(1)
        osess = om.new_session(seq)
        _, tr = osess.forward(np.array(prompts[0], np.int32), 0, all_rows=True, trace=True)
        gm.Transformer.forward_argmax(ce, np.array(prompts[0], np.int32), 0)
        _, tr1 = osess.forward(np.array([9], np.int32), 4, all_rows=True, trace=True)
        gm.Transformer.forward_argmax(ce, np.array([9], np.int32), 4)       # engine step with one layer only
        assert np.array_equal(ce.residual(1), tr1[1])
        ce.set_layer_limit(0)
        lg = gm.Transformer.Forward(ce, L.ml.Tensor(np.array([11], np.int32), L.ml.DT_INT32), 5)   # engine + kept logits
        exp = osess.forward(np.array([11], np.int32), 5, all_rows=True)
        # (layer-limited step above wrote layer-0 cache only: compare through a fresh pair instead)
        osess.close()
        o2 = om.new_session(seq)
        c2 = _context(L, gm, seq, L._capi.LNB_ACC_STRICT, True)
        e = o2.forward(np.array(prompts[1], np.int32), 0, all_rows=False)
        gm.Transformer.forward_argmax(c2, np.array(prompts[1], np.int32), 0)
        lg = gm.Transformer.Forward(c2, L.ml.Tensor(np.array([11], np.int32), L.ml.DT_INT32), 6)
        e = o2.forward(np.array([11], np.int32), 6, all_rows=True)
        assert int(L.ml.Argmax(lg.Slice([0], [1]), 1).Item()) == O.argmax_f32(e[0])
        assert np.array_equal(lg.RawData, e)
        c2.close(); o2.close()
    finally:
        ce.close()
