"""Speculative verification (lnb_forward_speculative): a sequence's last token plus k drafts as k + 1 rows of one forward.
Every row must carry the bits of its sequence's own S = 1 step at its position -- on the batch engine, on the kernel chain and
in the one-row path -- so that acceptance is exact and a speculative stream IS the plain stream, greedy or sampled, STRICT
(= the oracle) or FAST (= the plain FAST chain)."""
import os

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import engine_shapes as ES
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

PROMPT = [1, 50, 999, 7, 300, 12, 64, 2]
SAMPLING = (0.8, 40, 0.95, 77)         # Temperature, TopK, TopP, Seed
NO_STOP = (10**9,)


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _load(L, args):
    tensors = host_tensors(args, 4321)
    return args, oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)


@pytest.fixture(scope="module")
def tiny(L):
    m = _load(L, dict(L.synth.TINY))
    yield m
    m[2].Free(); m[1].close()


@pytest.fixture(scope="module")
def tiny128(L):
    m = _load(L, dict(L.synth.TINY128))
    yield m
    m[2].Free(); m[1].close()


@pytest.fixture(scope="module")
def wide(L):
    import torch
    m = _load(L, ES.wide_args(torch.cuda.get_device_properties(0).multi_processor_count))
    yield m
    m[2].Free(); m[1].close()


def _acc(L, mode):
    return L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST


def _ctx(L, gm, seq, acc, engine=None, n_seq=1, max_rows=8):
    """a session; engine True / False sets LNB_ENGINE while the engines are probed (None: the default)"""
    old = os.environ.get("LNB_ENGINE")
    if engine is not None:
        os.environ["LNB_ENGINE"] = "1" if engine else "0"
    try:
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)
        gm.Transformer.forward_argmax(ctx, np.array([1], np.int32), 0)     # probe now
    finally:
        if old is None:
            os.environ.pop("LNB_ENGINE", None)
        else:
            os.environ["LNB_ENGINE"] = old
    return ctx


def _plain_steps(L, gm, ctx, prompt, n_steps, seq=0):
    """greedy S = 1 steps of sequence `seq` after its prompt: tokens t[0..n] (t[0] from the prompt) and logits of every step"""
    if ctx.n_seq > 1:
        ctx.set_active_sequence(seq)
    t, _ = gm.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0)
    toks, logits = [t], []
    for j in range(n_steps):
        t, lg = gm.Transformer.forward_argmax(ctx, np.array([toks[-1]], np.int32), len(prompt) + j, want_logits="last")
        toks.append(t)
        logits.append(lg[0])
    return toks, logits


# ---- 1. every acceptance count ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny", "tiny128", "wide"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_every_acceptance_count(L, request, model, mode):
    """calls of 8 rows whose drafts are c correct tokens (0..7) and then wrong ones: n_accepted == c, rows 0..c give the plain
    steps' tokens and logits, one batch-engine launch per call"""
    args, om, gm = request.getfixturevalue(model)
    acc, V, k = _acc(L, mode), args["vocab_size"], 7
    seq = 64
    plain = _ctx(L, gm, seq, acc)
    spec = _ctx(L, gm, seq, acc)
    try:
        toks, logits = _plain_steps(L, gm, plain, PROMPT, 52)
        if mode == "strict":
            assert toks == list(om.generate(PROMPT, len(PROMPT) + len(toks), stop_ids=NO_STOP))
        first, _ = gm.Transformer.forward_argmax(spec, np.array(PROMPT, np.int32), 0)
        assert first == toks[0]
        p = len(PROMPT)                                   # position of the token fed next; toks[p - 8] is that token
        for c in range(k + 1):
            i0 = p - len(PROMPT)
            drafts = [toks[i0 + 1 + j] if j < c else (toks[i0 + 1 + j] + 1) % V for j in range(k)]
            l0 = spec.launch_count()
            nxt, na, lg = spec.forward_speculative([(0, p, [toks[i0]] + drafts)], want_logits=True)
            assert spec.launch_count() - l0 == 1, "one batch-engine launch per verify call"
            assert list(na) == [c]
            for j in range(c + 1):
                assert nxt[j] == toks[i0 + 1 + j], (c, j)
                assert np.array_equal(lg[j], logits[i0 + j]), (c, j)
            p += c + 1
    finally:
        plain.close(); spec.close()


# ---- 2. streams ---------------------------------------------------------------------------------------------------------
def _set_stop(gm, saved, stop):
    class V:
        StopTokenIds = (stop,)
        PadId = saved.PadId
    gm.Vocabulary = V


@pytest.mark.parametrize("model", ["tiny", "tiny128"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("sampled", [False, True])
def test_generate_streams_equal_plain_and_oracle(L, request, model, mode, sampled):
    """a prompt built to repeat (the drafter fires), the same prompt stopping on a stop id inside an accepted run, and
    prompts running to SequenceLength: speculative GenerateTokens == plain GenerateTokens (== orc_generate /
    orc_generate_sampled in STRICT)"""
    args, om, gm = request.getfixturevalue(model)
    seq = 48
    # max_rows 24: the repeating prompt prefills in one call; speculative calls still carry at most 8 rows
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=_acc(L, mode), max_rows=24)
    sp = L.model.SamplingArgs(*SAMPLING) if sampled else None
    spec = L.inference.SpeculativeArgs(7)
    rep = [3, 14, 15, 92, 65] * 4
    saved = gm.Vocabulary
    try:
        for prompt in (rep, PROMPT):
            _set_stop(gm, saved, NO_STOP[0])
            plain = [t for _, t in eng.GenerateTokens(prompt, sampling=sp)]
            stats = []
            got = list(eng.GenerateTokens(prompt, sampling=sp, speculative=spec, spec_stats=stats))
            assert [t for _, t in got] == plain and len(plain) == seq - len(prompt)
            assert got[-1][0] == L.inference.GSFinishedByReachingSeqLen
            if mode == "strict":
                exp = SR.generate_sampled(om, prompt, seq, *SAMPLING, stop_ids=NO_STOP) if sampled else \
                    om.generate(prompt, seq, stop_ids=NO_STOP)
                assert plain == list(exp)
            if prompt is not rep:
                continue
            assert sum(r for r, _ in stats) > len(stats), "no call carried a draft"
            # stop on a token emitted from an accepted draft row, before the call's last emitted token when it can
            idx, best = 1, (len(plain) // 2, 0)          # plain[0] came from the prompt; (stream index, accepted) of a call
            for _, a in stats:
                if a > best[1]:
                    best = (idx, a)
                idx += a + 1
            stop = plain[best[0] + best[1] // 2]
            _set_stop(gm, saved, stop)
            want = [t for _, t in eng.GenerateTokens(prompt, sampling=sp)]
            got = list(eng.GenerateTokens(prompt, sampling=sp, speculative=spec))
            assert [t for _, t in got] == want and want[-1] == stop
            assert got[-1][0] == L.inference.GSFinishedByReachingEOS
    finally:
        gm.Vocabulary = saved


# ---- 3. caches ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_caches_equal_the_plain_run(L, tiny128, mode):
    """after a speculative run, K/V of the first and last layer at every fed position equal the plain run's"""
    args, om, gm = tiny128
    acc, seq = _acc(L, mode), 40
    a, b = _ctx(L, gm, seq, acc), _ctx(L, gm, seq, acc)
    try:
        toks, _ = _plain_steps(L, gm, a, PROMPT, seq - len(PROMPT) - 1)
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=acc)
        hist = [PROMPT + [gm.Transformer.forward_argmax(b, np.array(PROMPT, np.int32), 0)[0]]]
        out = [t for _, _, t in eng._generate_speculative(b, hist, [0], L.inference.SpeculativeArgs(7))]
        assert [toks[0]] + out == toks
        last_fed = seq - 1
        for layer in (0, args["n_layers"] - 1):
            for rd in ("CacheK", "CacheV"):
                assert np.array_equal(getattr(a, rd)(layer).RawData[:last_fed], getattr(b, rd)(layer).RawData[:last_fed]), (layer, rd)
    finally:
        a.close(); b.close()


# ---- 4. routing ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_routing_at_the_engine_limit_and_beyond(L, tiny128, mode, monkeypatch):
    """n_seq == 1 at the engines' limit: one batch-engine launch per call.  At limit + 1 and with LNB_BATCH_ENGINE=0: the
    kernel chain, same bits.  A one-row call: the plain S = 1 path (its launch count and bits)."""
    args, om, gm = tiny128
    acc = _acc(L, mode)
    lim = ES.max_seq_len(args)
    ref = None
    for seq, env in ((lim, None), (lim + 1, None), (lim, "0")):
        if env is None:
            monkeypatch.delenv("LNB_BATCH_ENGINE", raising=False)
        else:
            monkeypatch.setenv("LNB_BATCH_ENGINE", env)
        plain, spec = _ctx(L, gm, seq, acc), _ctx(L, gm, seq, acc)
        try:
            n = lim - len(PROMPT) - 1                     # the last plain step feeds position lim - 2
            toks, logits = _plain_steps(L, gm, plain, PROMPT, n)
            gm.Transformer.forward_argmax(spec, np.array(PROMPT, np.int32), 0)
            p, rows = len(PROMPT), 8
            while p + rows - 1 <= lim - 2:
                i0 = p - len(PROMPT)
                l0 = spec.launch_count()
                nxt, na, lg = spec.forward_speculative([(0, p, toks[i0:i0 + rows])], want_logits=True)
                launches = spec.launch_count() - l0
                assert (launches == 1) == (seq == lim and env is None), (seq, env, launches)
                assert list(na) == [rows - 1] and list(nxt) == toks[i0 + 1:i0 + rows + 1]
                assert all(np.array_equal(lg[j], logits[i0 + j]) for j in range(rows))
                p += rows
            # one-row calls up to the end: the ordinary S = 1 step
            while p <= lim - 2:
                i0 = p - len(PROMPT)
                l0 = spec.launch_count()
                nxt, na, lg = spec.forward_speculative([(0, p, [toks[i0]])], want_logits=True)
                one = spec.launch_count() - l0
                l0 = plain.launch_count()
                gm.Transformer.forward_argmax(plain, np.array([toks[i0]], np.int32), p, want_logits="last")
                assert one == plain.launch_count() - l0
                assert list(nxt) == [toks[i0 + 1]] and list(na) == [0] and np.array_equal(lg[0], logits[i0])
                p += 1
            if ref is None:
                ref = (toks, logits)
            else:                                         # within sdpa_decode_kernel's fit FAST keeps its bits too
                assert toks == ref[0] and all(np.array_equal(x, y) for x, y in zip(logits, ref[1]))
        finally:
            plain.close(); spec.close()


# ---- 5. batch sessions --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny", "wide"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_batch_session_segments_and_generate_batch(L, request, model, mode):
    """segments of 3 sequences with different start positions and draft lengths in one call equal each sequence's plain steps;
    GenerateTokensBatch(speculative) equals the plain batch streams"""
    args, om, gm = request.getfixturevalue(model)
    acc, seq = _acc(L, mode), 40
    prompts = [PROMPT, [5, 6, 7], [9] * 6]
    ctx = _ctx(L, gm, seq, acc, n_seq=3)
    ref = _ctx(L, gm, seq, acc, n_seq=3)
    try:
        plain = [_plain_steps(L, gm, ref, p, 20, seq=i) for i, p in enumerate(prompts)]
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            gm.Transformer.forward_argmax(ctx, np.array(p, np.int32), 0)
        ctx.set_active_sequence(0)
        # sequence 2 first, then 0; sequence 1 sits this call out.  Drafts: 3 correct for seq 2, 1 correct + 1 wrong for seq 0
        t0, t2 = plain[0][0], plain[2][0]
        segs = [(2, len(prompts[2]), t2[0:4]), (0, len(prompts[0]), [t0[0], t0[1], (t0[2] + 1) % args["vocab_size"]])]
        nxt, na, lg = ctx.forward_speculative(segs, want_logits=True)
        assert list(na) == [3, 1]
        assert list(nxt[:4]) == t2[1:5] and list(nxt[4:6]) == t0[1:3]
        assert all(np.array_equal(lg[j], plain[2][1][j]) for j in range(4))
        assert all(np.array_equal(lg[4 + j], plain[0][1][j]) for j in range(2))
        # the next call continues where each stopped (sequence 0 overwrites its stale row)
        nxt, na, _ = ctx.forward_speculative([(0, len(prompts[0]) + 2, t0[2:5]), (1, len(prompts[1]), [plain[1][0][0]])])
        assert list(na) == [2, 0] and list(nxt[:3]) == t0[3:6] and nxt[3] == plain[1][0][1]
    finally:
        ctx.close(); ref.close()
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=acc)
    bprompts = [[3, 14, 15, 92] * 2, PROMPT, [5, 6], [7, 7, 7, 7]]
    want, got = {}, {}
    for i, _, t in eng.GenerateTokensBatch(bprompts):
        want.setdefault(i, []).append(t)
    stats = []
    for i, _, t in eng.GenerateTokensBatch(bprompts, speculative=L.inference.SpeculativeArgs(6), spec_stats=stats):
        got.setdefault(i, []).append(t)
    assert got == want
    assert all(r <= 8 for r, _ in stats)
    if mode == "strict":
        for i, p in enumerate(bprompts):
            assert want[i] == list(om.generate(p, seq, stop_ids=NO_STOP)), i


# ---- 6. validation ------------------------------------------------------------------------------------------------------
def test_invalid_calls_are_einval_and_the_session_stays_usable(L, tiny):
    args, om, gm = tiny
    c = L._capi
    seq = 24
    prompt = PROMPT[:5]
    ctx = _ctx(L, gm, seq, c.LNB_ACC_STRICT, n_seq=2, max_rows=6)
    try:
        gm.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0)
        base = ctx.launch_count()

        def call(n_segs, sq, st, nd, toks):
            a = [np.ascontiguousarray(x, np.int32) for x in (sq, st, nd, toks)]
            out = np.zeros(16, np.int32)
            na = np.zeros(8, np.int32)
            return c.lib.lnb_forward_speculative(ctx.h, n_segs, *[c.ptr(x, c.i32p) for x in a], None, c.ptr(out, c.i32p),
                                                 c.ptr(na, c.i32p))
        bad = [
            (0, [0], [8], [0], [1]),                          # n_segs < 1
            (3, [0, 1, 0], [8, 0, 9], [0, 0, 0], [1, 1, 1]),  # n_segs > n_seq
            (2, [0, 0], [8, 9], [0, 0], [1, 1]),              # repeated sequence
            (1, [2], [8], [0], [1]),                          # sequence out of range
            (1, [-1], [8], [0], [1]),
            (1, [0], [8], [-1], [1]),                         # n_draft < 0
            (1, [0], [-1], [0], [1]),                         # start_pos < 0
            (1, [0], [20], [4], [1] * 5),                     # start_pos + n_draft == seq_len
            (1, [0], [8], [6], [1] * 7),                      # 7 rows > max_rows 6
            (2, [0, 1], [8, 0], [3, 2], [1] * 7),             # 7 rows over two segments
            (1, [0], [8], [1], [1, args["vocab_size"]]),      # token id out of range
            (1, [0], [8], [1], [-1, 1]),
        ]
        for b in bad:
            assert call(*b) == -1, b                      # LNB_EINVAL
        assert ctx.launch_count() == base, "an invalid call enqueued work"
        ref = _ctx(L, gm, seq, c.LNB_ACC_STRICT)
        try:
            toks, _ = _plain_steps(L, gm, ref, prompt, 4)
        finally:
            ref.close()
        nxt, na, _ = ctx.forward_speculative([(0, len(prompt), toks[0:4])])
        assert list(na) == [3] and list(nxt) == toks[1:5]
    finally:
        ctx.close()


# ---- 7. the 8B model ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def m8b(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
    yield gm
    gm.Free()


def test_8b_strict_verify_call_and_fast_stream(L, m8b):
    """one STRICT call of 8 rows equals 8 plain S = 1 steps (logits, tokens); FAST GenerateTokens(speculative) of 32
    tokens equals the plain FAST stream"""
    gm = m8b
    prompt = list(L.synth.PROMPT_8)
    seq = len(prompt) + 33
    plain, spec = _ctx(L, gm, seq, L._capi.LNB_ACC_STRICT), _ctx(L, gm, seq, L._capi.LNB_ACC_STRICT)
    try:
        toks, logits = _plain_steps(L, gm, plain, prompt, 8)
        gm.Transformer.forward_argmax(spec, np.array(prompt, np.int32), 0)
        l0 = spec.launch_count()
        nxt, na, lg = spec.forward_speculative([(0, len(prompt), toks[:8])], want_logits=True)
        assert spec.launch_count() - l0 == 1
        assert list(na) == [7] and list(nxt) == toks[1:9]
        assert all(np.array_equal(lg[j], logits[j]) for j in range(8))
    finally:
        plain.close(); spec.close()
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=L._capi.LNB_ACC_FAST)
    want = [t for _, t in eng.GenerateTokens(prompt)]
    got = [t for _, t in eng.GenerateTokens(prompt, speculative=L.inference.SpeculativeArgs(7))]
    assert len(want) == 33 and got == want
