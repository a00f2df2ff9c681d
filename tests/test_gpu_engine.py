"""The persistent decode engine (csrc/engine.cuh: one kernel launch = n complete S=1 forwards, phases separated by grid
barriers) and the batch engine (csrc/engine_batch.cuh: one launch = one S=1 step of up to 8 sequences) against the kernel
chain they replace (LNB_ENGINE=0 / a session without the engines: one launch per projection / attention / norm-scale)
and against the oracle.  Both paths evaluate the same expressions in the same order, so their logits, KV caches and greedy
tokens must be IDENTICAL in both accumulation modes; STRICT must in addition equal the oracle bit for bit.

Which shapes reach which engine path (tests/engine_shapes.py restates the split; test_engine_shapes_cpu.py pins it at 132
SMs, and the `wide` fixture re-checks it at the device's SM count G):
- `tiny` (TINY): one panel per CTA and one k-tile per projection -- the engines' simplest schedule.
- `wide` (dim 1536, 32 x 64 heads over 8, ffn_dim 4 * (8G - 28) = 4112 at G = 132, vocab 32768): the LM head gives each
  CTA 31-32 panels, so STRICT row tiles of 16 + 15/16 panels and FAST tiles of 7-8 (the batch engine's activation re-fetch
  at rt > p0), with 12 / 6 k-tiles; w1|w3 gives 7-8 panels, so FAST's second chain runs full and partial; w2 has K = 4112,
  9 k-tiles of 512 with a 16-element tail (the STRICT generic chunk loop, the batch engine's short ktt); wq|wk|wv runs
  eng_chain_tile<16> over 3 k-tiles.  Batch attention of 8 sequences is 256 (head, sequence) items, so CTAs serve two.
  The engines accept SequenceLength <= 264 for this model.
- `tiny128` (TINY128): the 8B attention layout (head_dim 128, n_rep 4), engine limit 145 positions.
- `deep` (TINY with 32 layers): 161 phases per step, so one launch runs at most 403 steps and long runs split and wrap
  the 16-bit activation tags.  Engine limit 444 positions.
- `ties` (`wide` whose LM-head row i copies row (i // 2) % 64): every logit is tied with a row of its own panel, of another
  row tile of the same CTA and of other CTAs; every greedy path must return the lowest index."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import engine_shapes as ES
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


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _load(L, args, tensors):
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    return args, om, gm


@pytest.fixture(scope="module")
def wide_tensors(L, sms):
    ES.check_coverage(sms)                    # the widths below reach every engine path on this device's SM count
    args = ES.wide_args(sms)
    return args, host_tensors(args, 4321)


@pytest.fixture(scope="module")
def wide(L, wide_tensors):
    args, om, gm = _load(L, *wide_tensors)
    yield args, om, gm
    gm.Free()
    om.close()


@pytest.fixture(scope="module")
def ties(L, wide_tensors):
    args, tensors = wide_tensors
    t = dict(tensors)
    base = tensors["output.weight"]
    t["output.weight"] = np.ascontiguousarray(base[[ES.tie_base_row(i) for i in range(args["vocab_size"])]])
    args, om, gm = _load(L, args, t)
    yield args, om, gm
    gm.Free()
    om.close()


@pytest.fixture(scope="module")
def tiny128(L):
    args = dict(L.synth.TINY128)
    args, om, gm = _load(L, args, host_tensors(args, 4321))
    yield args, om, gm
    gm.Free()
    om.close()


@pytest.fixture(scope="module")
def deep(L):
    args = ES.deep_args()
    args, om, gm = _load(L, args, host_tensors(args, 4321))
    yield args, om, gm
    gm.Free()
    om.close()


def _acc(L, mode):
    return L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST


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
    check_engine_equals_kernel_chain_and_oracle(L, tiny, mode, fast_oracle_bound=1e-2)


@pytest.mark.parametrize("model", ["wide", "tiny128"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_engine_equals_kernel_chain_and_oracle_at_wide_shapes(L, request, model, mode):
    """the same at the shapes where a CTA owns several row tiles and k-tiles (`wide`) and at the 8B attention layout
    (`tiny128`): FAST is held to identity with the chain, which is pinned to the documented order elsewhere"""
    check_engine_equals_kernel_chain_and_oracle(L, request.getfixturevalue(model), mode)


def check_engine_equals_kernel_chain_and_oracle(L, model, mode, fast_oracle_bound=None):
    args, om, gm = model
    acc = _acc(L, mode)
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
            elif fast_oracle_bound is not None:
                assert float(np.abs(le - exp).max()) <= fast_oracle_bound
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


# ---- the batch engine ------------------------------------------------------------------------------------------------
BATCH_ENGINE_LAUNCHES = 1      # a greedy batched step on the batch engine: its one cooperative launch and nothing else
PROMPT = np.array([1, 50, 999, 7, 300, 12, 64, 2], np.int32)


def _greedy_row(lg):
    return O.argmax_f32(np.ascontiguousarray(lg, np.float32))


@pytest.mark.parametrize("model", ["wide", "tiny128"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_batch_engine_equals_chain_and_per_sequence_forwards(L, request, model, mode, monkeypatch):
    """steps of n = 8, 1, 2, 3, 8 sequences of an 8-sequence session, at different positions (one sequence starts at 0, one
    ends at the last position): the batch engine's logits, tokens and caches equal a session without the engines (batched
    kernel chain), each sequence's own S=1 chain forward, and in STRICT independent oracle sessions"""
    monkeypatch.delenv("LNB_BATCH_TC", raising=False)
    monkeypatch.delenv("LNB_BATCH_ENGINE", raising=False)
    args, om, gm = request.getfixturevalue(model)
    acc, strict = _acc(L, mode), mode == "strict"
    seq, steps = 32, (8, 1, 2, 3, 8)
    lens = (27, 5, 9, 1, 17, 2, 30, 0)          # sequence 0 ends at position 31, sequence 7 starts at 0; S < 32 (GEMV path)
    rng = np.random.default_rng(7)
    prompts = [rng.integers(0, args["vocab_size"], size=k).astype(np.int32) for k in lens]
    ce = _context(L, gm, seq, acc, True, max_rows=32, n_seq=8)      # batch engine
    cc = _context(L, gm, seq, acc, False, max_rows=32, n_seq=8)     # batched kernel chain
    cs = _context(L, gm, seq, acc, False, max_rows=32, n_seq=8)     # S=1 chain forwards, one sequence at a time
    osess = [om.new_session(seq) for _ in range(8)] if strict else []
    try:
        cur, pos = [], []
        for i, p in enumerate(prompts):
            if len(p) == 0:
                cur.append(int(rng.integers(0, args["vocab_size"]))); pos.append(0)
                continue
            got = []
            for ctx in (ce, cc, cs):
                ctx.set_active_sequence(i)
                got.append(gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last"))
            assert all(t == got[0][0] and np.array_equal(lg, got[0][1]) for t, lg in got), i
            if strict:
                assert np.array_equal(got[0][1], osess[i].forward(p, 0, all_rows=False))
            cur.append(got[0][0]); pos.append(len(p))
        for k, n in enumerate(steps):
            l0 = ce.launch_count()
            te, le = ce.forward_batch(cur[:n], pos[:n], want_logits=True)
            assert ce.launch_count() - l0 == BATCH_ENGINE_LAUNCHES, "the batch engine did not run"
            l0 = cc.launch_count()
            tc, lc = cc.forward_batch(cur[:n], pos[:n], want_logits=True)
            assert cc.launch_count() - l0 > BATCH_ENGINE_LAUNCHES
            assert np.array_equal(le, lc), f"step {k}: batch engine and batched chain logits differ"
            assert list(te) == list(tc)
            for i in range(n):
                cs.set_active_sequence(i)
                ts, ls = gm.Transformer.forward_argmax(cs, np.array([cur[i]], np.int32), pos[i], want_logits="last")
                assert np.array_equal(le[i], ls[0]), f"step {k}, sequence {i} at position {pos[i]}"
                assert te[i] == ts == _greedy_row(le[i])
                if strict:
                    exp = osess[i].forward(np.array([cur[i]], np.int32), pos[i], all_rows=False)
                    assert np.array_equal(le[i], exp[0]), f"step {k}, sequence {i}: oracle"
                cur[i] = int(te[i]); pos[i] += 1
        assert pos[0] == seq and pos[7] == 2
        for i in range(8):
            for ctx in (ce, cc, cs):
                ctx.set_active_sequence(i)
            for layer in range(args["n_layers"]):
                for rd in ("CacheK", "CacheV"):
                    e = getattr(ce, rd)(layer).RawData[:pos[i]]
                    assert np.array_equal(e, getattr(cc, rd)(layer).RawData[:pos[i]]), (i, layer, rd)
                    assert np.array_equal(e, getattr(cs, rd)(layer).RawData[:pos[i]]), (i, layer, rd)
                if strict:
                    ok, ov = osess[i].cache(layer)
                    assert np.array_equal(ce.CacheK(layer).RawData[:pos[i]], ok[:pos[i]])
                    assert np.array_equal(ce.CacheV(layer).RawData[:pos[i]], ov[:pos[i]])
    finally:
        ce.close(); cc.close(); cs.close()
        for o in osess:
            o.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_batch_engine_runs_the_predicted_k_tiles(L, wide, sms, mode, monkeypatch):
    """ties tests/engine_shapes.py to the kernel: the batch engine's per-CTA count of consumed k-tiles (LNB_ENGINE_PROF) is
    the count the restatement of eng_split / eng_kt predicts, mean and max over the CTAs"""
    monkeypatch.delenv("LNB_BATCH_TC", raising=False)
    monkeypatch.setenv("LNB_ENGINE_PROF", "1")
    args, om, gm = wide
    ctx = _context(L, gm, 16, _acc(L, mode), True, n_seq=8)
    try:
        ctx.engine_profile()                  # drop the counters of the decode-engine probe step
        ctx.forward_batch([1, 2, 3, 4, 5, 6, 7, 8], [0] * 8)
        mean, mx = ctx.engine_profile(batch=True)["tiles"]
        assert (mean, mx) == ES.k_tiles_per_step(args, sms, mode == "strict")
    finally:
        ctx.close()


# ---- position limit, tag wrap -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny128", "wide"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_engines_at_their_position_limit_and_one_past_it(L, request, model, mode):
    """SequenceLength = the engines' limit (eng_sdpa_smem): both engines run, to position limit - 1, and equal the chain (and
    the oracle in STRICT); one position more: the session falls back to the chain with the same bits"""
    args, om, gm = request.getfixturevalue(model)
    acc, strict = _acc(L, mode), mode == "strict"
    lim = ES.max_seq_len(args)
    assert lim == {"tiny128": 145, "wide": 264}[model]
    ref = None
    for seq in (lim, lim + 1):
        ce = _context(L, gm, seq, acc, True, n_seq=2)
        cc = _context(L, gm, seq, acc, False, n_seq=2)
        try:
            assert ce.uses_engine() == (seq == lim) and not cc.uses_engine()
            out = []
            for ctx in (ce, cc):
                first, _ = gm.Transformer.forward_argmax(ctx, PROMPT, 0)
                toks, _, _ = ctx.decode_run(first, 8, lim - 9, use_graph=False)        # positions 8 .. lim - 2
                toks = [first] + [int(t) for t in toks]
                t1, l1 = gm.Transformer.forward_argmax(ctx, np.array([toks[-1]], np.int32), lim - 1, want_logits="last")
                l0 = ctx.launch_count()
                tb, lb = ctx.forward_batch([toks[-1], 5], [lim - 1, 0], want_logits=True)
                launches = ctx.launch_count() - l0
                caches = [getattr(ctx, rd)(layer).RawData[:lim].copy() for layer in (0, args["n_layers"] - 1) for rd in ("CacheK", "CacheV")]
                out.append((toks + [t1], l1, list(tb), lb, caches, launches))
            (te, le, tbe, lbe, ke, ne), (tc, lc, tbc, lbc, kc, nc) = out
            assert te == tc and np.array_equal(le, lc), seq
            assert tbe == tbc and np.array_equal(lbe, lbc), seq
            assert np.array_equal(lbe[0], le[0]) and tbe[0] == te[-1]   # the batched row = the S=1 step at lim - 1
            assert all(np.array_equal(a, b) for a, b in zip(ke, kc)), seq
            assert (ne == BATCH_ENGINE_LAUNCHES) == (seq == lim) and nc > BATCH_ENGINE_LAUNCHES
            if ref is None:
                ref = (te, le, lbe, ke)
                if strict:
                    assert te == list(om.generate(PROMPT, lim + 1, stop_ids=(10**9,)))
            else:
                assert te == ref[0] and np.array_equal(le, ref[1]) and np.array_equal(lbe, ref[2])
                assert all(np.array_equal(a, b) for a, b in zip(ke, ref[3]))
        finally:
            ce.close(); cc.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_engine_splits_long_runs_and_wraps_its_tags(L, deep, mode):
    """`deep` has 161 phases per step: a 435-step decode_run is two engine launches (403 + 32) and the second zero-fills and
    restarts the 16-bit tags; a host-driven loop of 420 S=1 steps after it wraps them again.  Tokens and logits equal the
    chain's (and the oracle's in STRICT)."""
    args, om, gm = deep
    acc, seq = _acc(L, mode), ES.max_seq_len(args)
    assert seq == 444
    phases = ES.n_phases(args)
    ce = _context(L, gm, seq, acc, True)       # its probe step used tags [1, 1 + phases)
    cc = _context(L, gm, seq, acc, False)
    try:
        assert ce.uses_engine()
        plan, tag = ES.engine_launches(435, phases, 1 + phases)
        assert plan == [(403, False), (32, True)]
        first, _ = gm.Transformer.forward_argmax(ce, PROMPT, 0)
        fc, _ = gm.Transformer.forward_argmax(cc, PROMPT, 0)
        assert first == fc
        l0 = ce.launch_count()
        a, _, _ = ce.decode_run(first, 8, 435, use_graph=False)
        assert ce.launch_count() - l0 == 1 + len(plan)             # set_state + one launch per part
        b, _, _ = cc.decode_run(first, 8, 435, use_graph=True)
        toks = [first] + [int(t) for t in a]
        assert toks[1:] == [int(t) for t in b]
        if mode == "strict":
            assert toks == list(om.generate(PROMPT, 444, stop_ids=(10**9,)))
        wraps = 0
        for i in range(420):                                        # teacher-forced with the run's own tokens
            step, tag = ES.engine_launches(1, phases, tag)
            wraps += step[0][1]
            x = np.array([toks[i]], np.int32)
            t1, l1 = gm.Transformer.forward_argmax(ce, x, 8 + i, want_logits="last")
            t2, l2 = gm.Transformer.forward_argmax(cc, x, 8 + i, want_logits="last")
            assert np.array_equal(l1, l2), f"host step {i}"
            assert t1 == t2 == toks[i + 1]
        assert wraps == 1
    finally:
        ce.close(); cc.close()


# ---- greedy ties -----------------------------------------------------------------------------------------------------
class _Ties:
    def __init__(self, args, sms, strict):
        self.V, self.G, self.strict, self.kinds, self.n = args["vocab_size"], sms, strict, set(), 0

    def check(self, tok, lg, exp=None):
        """tok must be the lowest index of a real tie in lg (an even row below 128), argmax_f32(lg), and in STRICT the
        oracle's pick of logits equal to lg"""
        lg = np.ascontiguousarray(lg, np.float32).reshape(-1)
        group = np.flatnonzero(lg == lg.max())
        assert len(group) >= 3, "no tie"
        kinds = ES.tie_partner_kinds(int(group[0]), [int(g) for g in group], self.V, self.G, self.strict)
        assert {"panel", "cta"} <= kinds, kinds
        self.kinds |= kinds
        assert tok == group[0] == _greedy_row(lg) and tok % 2 == 0 and tok < 128, (tok, group[:4])
        if exp is not None:
            assert np.array_equal(lg, exp.reshape(-1)) and tok == _greedy_row(exp)
        self.n += 1


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_greedy_ties_pick_the_lowest_index_on_every_path(L, ties, sms, mode, monkeypatch):
    monkeypatch.delenv("LNB_BATCH_TC", raising=False)
    args, om, gm = ties
    acc, strict, seq = _acc(L, mode), mode == "strict", 32
    T = _Ties(args, sms, strict)
    ce, cc = _context(L, gm, seq, acc, True), _context(L, gm, seq, acc, False)
    be = _context(L, gm, seq, acc, True, n_seq=8)
    bc = _context(L, gm, seq, acc, False, n_seq=8)
    oss = [om.new_session(seq) for _ in range(9)] if strict else []     # 0..7: the batched sequences, 8: the single one
    try:
        # chain S=1 and decode engine, host-driven
        exp = oss[8].forward(PROMPT, 0, all_rows=False) if strict else None
        t, lg = gm.Transformer.forward_argmax(cc, PROMPT, 0, want_logits="last")
        T.check(t, lg, exp)
        t1, l1 = gm.Transformer.forward_argmax(ce, PROMPT, 0, want_logits="last")
        assert t1 == t and np.array_equal(l1, lg)
        host = [t]
        for pos in range(8, 14):
            x = np.array([host[-1]], np.int32)
            t1, l1 = gm.Transformer.forward_argmax(ce, x, pos, want_logits="last")
            t2, l2 = gm.Transformer.forward_argmax(cc, x, pos, want_logits="last")
            exp = oss[8].forward(x, pos, all_rows=False) if strict else None
            T.check(t1, l1, exp); T.check(t2, l2, exp)
            assert np.array_equal(l1, l2)
            host.append(t1)
        # decode_run: the engine's device loop, and the chain's captured graph
        a, _, _ = ce.decode_run(host[0], 8, 6, use_graph=True)
        b, _, g = cc.decode_run(host[0], 8, 6, use_graph=True)
        assert g and [int(v) for v in a] == [int(v) for v in b] == host[1:]
        # ml.Argmax of a kept Forward handle, engine and chain
        for ctx in (ce, cc):
            lgh = gm.Transformer.Forward(ctx, L.ml.Tensor(np.array([host[6]], np.int32), L.ml.DT_INT32), 14)
            am = int(L.ml.Argmax(lgh.Slice([0], [1]), 1).Item())
            T.check(am, lgh.RawData[0])
        # forward_batch on the batch engine and on the chain: 8 sequences, 3 steps
        rng = np.random.default_rng(9)
        prompts = [rng.integers(0, args["vocab_size"], size=k).astype(np.int32) for k in (8, 3, 5, 1, 2, 7, 4, 6)]
        cur, pos = [], []
        for i, p in enumerate(prompts):
            got = []
            for ctx in (be, bc):
                ctx.set_active_sequence(i)
                got.append(gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last"))
            (t, lg), (t2, l2) = got
            assert t == t2 and np.array_equal(lg, l2)
            exp = oss[i].forward(p, 0, all_rows=False) if strict else None
            T.check(t, lg, exp)
            cur.append(t); pos.append(len(p))
        for _ in range(3):
            l0 = be.launch_count()
            te, le = be.forward_batch(cur, pos, want_logits=True)
            assert be.launch_count() - l0 == BATCH_ENGINE_LAUNCHES
            tc, lc = bc.forward_batch(cur, pos, want_logits=True)
            assert np.array_equal(le, lc) and list(te) == list(tc)
            for i in range(8):
                exp = oss[i].forward(np.array([cur[i]], np.int32), pos[i], all_rows=False) if strict else None
                T.check(int(te[i]), le[i], exp)
                cur[i] = int(te[i]); pos[i] += 1
        # forward_ragged: decode rows of four sequences and a 3-token chunk of a fifth, in one forward
        segs = [(i, pos[i], [cur[i]]) for i in range(4)] + [(4, pos[4], [cur[4], 17, 23])]
        tr, lr = bc.forward_ragged(segs, want_logits=True)
        for k, (i, p0, tk) in enumerate(segs):
            exp = None
            if strict:
                exp = oss[i].forward_chunk(np.array(tk, np.int32), p0, all_rows=False) if len(tk) > 1 else \
                    oss[i].forward(np.array(tk, np.int32), p0, all_rows=False)
            T.check(int(tr[k]), lr[k], exp)
        assert "tile" in T.kinds, "no tie between two row tiles of one CTA was exercised"
    finally:
        for c in (ce, cc, be, bc):
            c.close()
        for o in oss:
            o.close()
