"""Token log-probabilities on the device (csrc/logprob.cuh, DESIGN.md §9d) against their sequential C statement
(orc_logprob_row, oracle_sampling/lnb_sample_ref.c): the op bit-exact on adversarial rows, STRICT scoring equal to the
statement on the oracle's logits (one shot and chunked), every emitting path writing the record of the token it emits
(equal to the statement on the logits the same call returned), the generate loops' records, sessions without logprobs
unchanged, validation, and the 8B vocabulary."""
import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 4321


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module", params=["TINY", "TINY128"])
def model(L, request):
    args = dict(getattr(L.synth, request.param))
    tensors = host_tensors(args, SEED)
    om, gm = oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)
    yield args, om, gm
    gm.Free()
    om.close()


def _op(L, rows, targets, top_n):
    rows = np.ascontiguousarray(rows, np.float32)
    t = np.ascontiguousarray(targets, np.int32)
    out = np.zeros(rows.shape[0], SR.LOGPROB_DTYPE)
    L._capi.check(L._capi.lib.lnb_op_logprobs_f32(L._capi.ptr(rows, L._capi.f32p), rows.shape[0], rows.shape[1],
                                                  L._capi.ptr(t, L._capi.i32p), top_n, out.ctypes.data))
    return out


def _same(a, b, what=""):
    """two LOGPROB_DTYPE arrays field for field, the doubles bit for bit"""
    for f in ("token", "rank", "n_top", "top_token"):
        assert np.array_equal(a[f], b[f]), (what, f, a[f], b[f])
    for f in ("logprob", "top_logprob"):
        assert np.array_equal(a[f].view(np.uint64), b[f].view(np.uint64)), (what, f, a[f], b[f])


def _adversarial(rng, V, n):
    rows = (rng.standard_normal((n, V)) * 3).astype(np.float32)
    k = 0
    for r in range(n):
        kind = r % 6
        if kind == 1:                                          # ties straddling every slice edge, at the top
            for e in range(4096, V, 4096):
                rows[r, e - 2:e + 2] = 30.0
        elif kind == 2:                                        # the top 20 spread over the slices
            idx = rng.choice(V, size=min(20, V), replace=False)
            rows[r, idx] = 20.0 + rng.integers(0, 4, size=idx.size)
        elif kind == 3:                                        # all equal
            rows[r, :] = -1.25
        elif kind == 4:                                        # few distinct values
            rows[r] = np.round(rows[r])
        elif kind == 5 and V > 40:                             # a long tail below the cut
            rows[r, :V // 2] = -100.0
        k += 1
    t = rng.integers(0, V, size=n)
    for r in range(n):
        if r % 3 == 0:
            t[r] = int(np.argmax(rows[r]))
        if r % 6 == 1 and V > 4096:
            t[r] = 4096                                        # a target tied with the slice edge
    return rows, t


@pytest.mark.parametrize("V,n", [(64, 8), (4097, 8), (12289, 8), (128256, 8), (4096, 1), (5000, 2048)])
@pytest.mark.parametrize("top_n", [0, 20])
def test_op_bit_exact(L, V, n, top_n):
    rng = np.random.default_rng(V + n + top_n)
    rows, t = _adversarial(rng, V, n)
    _same(_op(L, rows, t, top_n), SR.logprob_rows(rows, t, top_n), (V, n, top_n))


def test_op_inf_nan_rows(L):
    V = 5000
    rows = np.zeros((4, V), np.float32)
    rows[0, 4500] = np.inf
    rows[1, 9] = np.nan
    rows[2, :] = -np.inf
    rows[3, 4097] = -np.inf
    t = [4500, 9, 0, 4097]
    _same(_op(L, rows, t, 5), SR.logprob_rows(rows, t, 5))


@pytest.mark.parametrize("V", [64, 5000])
def test_op_device_nan_at_index_0(L, V):
    """logit bits 0x7FFFFFFF (the NaN the device's arithmetic makes) at index 0 have the largest key, ~0: rank 0, NaN logprobs"""
    nan = np.array([0x7FFFFFFF], np.uint32).view(np.float32)[0]
    rng = np.random.default_rng(V)
    rows = rng.standard_normal((3, V)).astype(np.float32)
    rows[0, 0] = nan                                           # alone in a finite row
    rows[1, :] = nan                                           # the whole row
    rows[2, 0] = nan
    rows[2, V - 1] = np.inf
    t = [0, V - 1, V - 1]
    for top_n in (0, 1, 20):
        got = _op(L, rows, t, top_n)
        _same(got, SR.logprob_rows(rows, t, top_n), (V, top_n))
        assert got["rank"][0] == 1 and np.isnan(got["logprob"]).all()
        if top_n:
            assert got["top_token"][0][0] == 0 and got["top_token"][1][0] == 0


def _ctx(L, gm, mode, seq_len=40, max_rows=8, n_seq=1):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq_len), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)


def _read(L, ctx, seq, pos0, n):
    out = np.zeros(n, SR.LOGPROB_DTYPE)
    L._capi.check(L._capi.lib.lnb_session_logprobs_read(ctx.h, seq, pos0, n, out.ctypes.data))
    return out


PROMPT = [1, 50, 999, 7, 300, 12, 64, 2, 5, 77, 31, 400, 8, 9, 1000, 3]


def test_strict_scoring_equals_the_statement_on_oracle_logits(L, model):
    args, om, gm = model
    toks = np.array(PROMPT, np.int32)
    sess = om.new_session(40)
    ref = sess.forward(toks[:-1], 0, all_rows=True)
    sess.close()
    want = SR.logprob_rows(ref, toks[1:], 7)
    ctx = _ctx(L, gm, "strict", max_rows=16)
    ctx.set_logprobs(0, 7)
    recs = gm.Transformer.score(ctx, toks, 0)
    assert [r.Token for r in recs] == list(toks[1:])
    _same(_read(L, ctx, 0, 1, len(toks) - 1), want, "one shot")
    # chunked: three calls of up to 6 rows, overlapping by one token
    ctx2 = _ctx(L, gm, "strict", max_rows=6)
    ctx2.allow_chunked_prefill(True)
    ctx2.set_logprobs(0, 7)
    for a, b in ((0, 7), (6, 13), (12, 16)):
        gm.Transformer.score(ctx2, toks[a:b], a)
    _same(_read(L, ctx2, 0, 1, len(toks) - 1), want, "chunked")
    ctx.close(); ctx2.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_fast_and_strict_scoring_equal_the_statement_on_their_logits(L, model, mode):
    _, _, gm = model
    toks = np.array(PROMPT * 3, np.int32)[:40]
    ctx = _ctx(L, gm, mode, seq_len=64, max_rows=48)
    ctx.set_logprobs(0, 20)
    gm.Transformer.score(ctx, toks, 0)
    got = _read(L, ctx, 0, 1, 39)
    _, lg = gm.Transformer.forward_argmax(ctx, toks[:-1], 0, want_logits="all")
    _same(got, SR.logprob_rows(lg, toks[1:], 20), mode)
    ctx.close()


def _oracle_records(om, prompt, stream, top_n):
    """the C statement on the oracle's logits, teacher-forced along `stream` (the tokens at positions len(prompt) ..)"""
    sess = om.new_session(40)
    rows = [sess.forward(np.asarray(prompt, np.int32), 0, all_rows=False)[0]]
    for i, t in enumerate(stream[:-1]):
        rows.append(sess.forward(np.array([t], np.int32), len(prompt) + i, all_rows=False)[0])
    sess.close()
    return SR.logprob_rows(np.stack(rows), stream, top_n)


def _check(L, ctx, seq, pos, logits_row, token, top_n, greedy):
    got = _read(L, ctx, seq, pos, 1)
    assert got["token"][0] == token, (got["token"][0], token)
    if greedy:
        assert got["rank"][0] == 1
    _same(got, SR.logprob_rows(np.asarray(logits_row, np.float32)[None], [token], top_n), (seq, pos))
    return got


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("sampled", [False, True])
def test_every_emitting_path_writes_the_emitted_tokens_record(L, model, mode, sampled):
    _, om, gm = model
    samp = L.model.SamplingArgs(0.9, 0, 1.0, 5) if sampled else None
    greedy = not sampled
    # lnb_forward (host logits), then the S = 1 step
    ctx = _ctx(L, gm, mode)
    ctx.set_sampling(0, samp)
    ctx.set_logprobs(0, 5)
    p = np.array(PROMPT[:8], np.int32)
    nxt, lg = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
    _check(L, ctx, 0, 8, lg[0], nxt, 5, greedy)
    nxt2, lg2 = gm.Transformer.forward_argmax(ctx, np.array([nxt], np.int32), 8, want_logits="last")
    _check(L, ctx, 0, 9, lg2[0], nxt2, 5, greedy)
    # lnb_forward_device (the reference-shaped Forward), then the logits through its handle
    lgd = gm.Transformer.Forward(ctx, L.ml.Tensor(np.array([nxt2], np.int32), L.ml.DT_INT32), 9).RawData
    rec = _read(L, ctx, 0, 10, 1)
    assert (rec["rank"][0] == 1) or sampled
    _same(rec, SR.logprob_rows(lgd[-1:], rec["token"], 5))
    # lnb_decode_run, without and with a graph: the same tokens and records as the host steps
    for use_graph in (False, True):
        c2 = _ctx(L, gm, mode)
        c2.set_sampling(0, samp)
        c2.set_logprobs(0, 5)
        n0, _ = gm.Transformer.forward_argmax(c2, p, 0)
        toks, _, _ = c2.decode_run(n0, 8, 6, use_graph=use_graph)
        c3 = _ctx(L, gm, mode)
        c3.set_sampling(0, samp)
        c3.set_logprobs(0, 5)
        gm.Transformer.forward_argmax(c3, p, 0)
        cur = n0
        for i in range(6):
            cur, lgi = gm.Transformer.forward_argmax(c3, np.array([cur], np.int32), 8 + i, want_logits="last")
            assert cur == toks[i]
            _check(L, c3, 0, 9 + i, lgi[0], cur, 5, greedy)
        _same(_read(L, c2, 0, 8, 7), _read(L, c3, 0, 8, 7), ("decode_run", use_graph))
        if mode == "strict":   # the C statement on the oracle's logits of the same stream (orc_generate / orc_generate_sampled)
            if sampled:
                stream = list(SR.generate_sampled(om, p, 15, 0.9, 0, 1.0, 5, stop_ids=(10**9,)))
            else:
                stream = list(om.generate(p, 15, stop_ids=(10**9,)))
            assert stream == [n0] + list(toks)
            _same(_read(L, c2, 0, 8, 7), _oracle_records(om, p, stream, 5), ("oracle", use_graph))
        c2.close(); c3.close()
    ctx.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("n", [1, 3, 8])
def test_batch_ragged_and_speculative_calls_write_their_records(L, model, mode, n):
    _, _, gm = model
    ctx = _ctx(L, gm, mode, n_seq=max(n, 2), max_rows=16)
    for i in range(ctx.n_seq):
        ctx.set_logprobs(i, 3)
        if i % 2:
            ctx.set_sampling(i, L.model.SamplingArgs(0.8, 0, 1.0, 11 + i))
    prompts = [PROMPT[i:i + 1 + i % 2] for i in range(ctx.n_seq)]
    segs = [(i, 0, p) for i, p in enumerate(prompts)]
    nxt, lg = ctx.forward_ragged(segs, want_logits=True)
    for i, p in enumerate(prompts):
        _check(L, ctx, i, len(p), lg[i], int(nxt[i]), 3, i % 2 == 0)
    toks, pos = [int(nxt[i]) for i in range(n)], [len(prompts[i]) for i in range(n)]
    nb, lb = ctx.forward_batch(toks, pos, want_logits=True)
    for i in range(n):
        _check(L, ctx, i, pos[i] + 1, lb[i], int(nb[i]), 3, i % 2 == 0)
    # speculative: sequence 0 with drafts, every acceptance count writes every row's record
    for a in range(0, 8):
        c = _ctx(L, gm, mode, max_rows=8)
        c.set_logprobs(0, 3)
        n0, _ = gm.Transformer.forward_argmax(c, np.array(prompts[0], np.int32), 0)
        plain, cur = [], n0
        for i in range(8):
            plain.append(cur)
            cur, _ = gm.Transformer.forward_argmax(c, np.array([cur], np.int32), len(prompts[0]) + i)
        plain.append(cur)
        want = _read(L, c, 0, len(prompts[0]) + 1, 8)
        c.close()
        c = _ctx(L, gm, mode, max_rows=8)
        c.set_logprobs(0, 3)
        gm.Transformer.forward_argmax(c, np.array(prompts[0], np.int32), 0)
        drafts = plain[1:1 + a] + ([(plain[1 + a] + 1) % 100] if a < 7 else [])   # a right drafts, then a wrong one
        nx, acc, lgs = c.forward_speculative([(0, len(prompts[0]), [plain[0]] + drafts)], want_logits=True)
        assert int(acc[0]) == a
        got = _read(L, c, 0, len(prompts[0]) + 1, a + 1)
        _same(got, want[:a + 1], ("speculative", a))
        for j in range(len(drafts) + 1):
            _check(L, c, 0, len(prompts[0]) + 1 + j, lgs[j], int(nx[j]), 3, True)
        c.close()
    ctx.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_generate_loops_collect_the_plain_records(L, model, mode):
    _, _, gm = model
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(32), acc_mode=acc, max_rows=16)
    prompts = [PROMPT[:8], PROMPT[3:5], PROMPT[5:10]]
    plain_tok, plain_lp = [], []
    for p in prompts:
        lp = []
        plain_tok.append([t for _, t in eng.GenerateTokens(p, logprobs=5, logprobs_out=lp)])
        assert plain_tok[-1] == [t for _, t in eng.GenerateTokens(p)]
        assert len(lp) == len(plain_tok[-1]) and [r.Token for r in lp] == plain_tok[-1]
        assert all(r.Rank == 1 and len(r.Top) == 5 and r.Top[0][0] == r.Token for r in lp)
        plain_lp.append(lp)
    lp = []
    spec = [t for _, t in eng.GenerateTokens(prompts[0], speculative=L.inference.SpeculativeArgs(4), logprobs=5, logprobs_out=lp)]
    assert spec == plain_tok[0] and lp == plain_lp[0]
    lp = []
    out = list(eng.GenerateTokensBatch(prompts, logprobs=5, logprobs_out=lp))
    for i in range(3):
        assert [t for s, _, t in out if s == i] == plain_tok[i] and lp[i] == plain_lp[i], i
    lp = []
    out = list(eng.GenerateTokensContinuous(prompts, slots=2, logprobs=5, logprobs_out=lp))
    for i in range(3):
        assert [t for s, _, t in out if s == i] == plain_tok[i] and lp[i] == plain_lp[i], i


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_nothing_changes_for_sequences_without_logprobs(L, model, mode):
    _, _, gm = model
    p = np.array(PROMPT[:8], np.int32)

    def run(ctx):
        l0 = ctx.launch_count()
        n0, lg0 = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
        nb, lb = ctx.forward_batch([n0], [8], want_logits=True)   # sequence 0 only
        ctx.set_active_sequence(0)
        toks, _, _ = ctx.decode_run(int(nb[0]), 9, 5, use_graph=True)
        toks2, _, _ = ctx.decode_run(int(toks[-1]), 14, 5, use_graph=True)
        return ctx.launch_count() - l0, n0, lg0, nb, lb, list(toks) + list(toks2)

    base = _ctx(L, gm, mode, n_seq=2)
    want = run(base)
    other = _ctx(L, gm, mode, n_seq=2)
    other.set_logprobs(1, 4)                     # another sequence has them on
    off = _ctx(L, gm, mode, n_seq=2)
    off.set_logprobs(0, 20)
    off.set_logprobs(0, None)                    # turned on, then off again
    for ctx in (other, off):
        got = run(ctx)
        assert got[0] == want[0] and got[1] == want[1] and got[5] == want[5]
        assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3]) and np.array_equal(got[4], want[4])
    # toggling re-captures the decode graph (the logprob job is part of the step); changing top_n does not
    on = _ctx(L, gm, mode, n_seq=2)
    gm.Transformer.forward_argmax(on, p, 0)
    on.decode_run(int(want[1]), 8, 3, use_graph=True)
    l0 = on.launch_count()
    on.decode_run(int(want[1]), 8, 3, use_graph=True)
    per_plain = on.launch_count() - l0
    on.set_logprobs(0, 2)
    l0 = on.launch_count()
    toks, _, graphed = on.decode_run(int(want[1]), 8, 3, use_graph=True)
    assert graphed and on.launch_count() - l0 > per_plain
    assert [r.Token for r in on.read_logprobs(0, 9, 3)] == list(toks)
    on.set_logprobs(0, 20)
    toks2, _, _ = on.decode_run(int(want[1]), 8, 3, use_graph=True)
    assert list(toks2) == list(toks) and all(len(r.Top) == 20 for r in on.read_logprobs(0, 9, 3))
    for c in (base, other, off, on):
        c.close()


def test_validation_leaves_the_session_usable(L, model):
    _, _, gm = model
    lib, E = L._capi.lib, L._capi.LnbError
    ctx = _ctx(L, gm, "strict", n_seq=2)
    for seq, n in ((-1, 0), (2, 0), (0, 21), (0, -2)):
        with pytest.raises(E) as e:
            ctx.set_logprobs(seq, n)
        assert e.value.code == -1
    t = np.array(PROMPT[:5], np.int32)
    with pytest.raises(E) as e:                   # logprobs off
        gm.Transformer.score(ctx, t, 0)
    assert e.value.code == -4
    ctx.set_logprobs(0, 2)
    for bad in (t[:1], np.array(PROMPT[:5] + [10**7], np.int32)):
        with pytest.raises(E):
            gm.Transformer.score(ctx, bad, 0)
    with pytest.raises(E):                        # start_pos > 0 without chunked prefill
        gm.Transformer.score(ctx, t, 3)
    with pytest.raises(E):                        # more than max_rows + 1 tokens
        gm.Transformer.score(ctx, np.array(PROMPT[:10], np.int32), 0)
    out = np.zeros(2, SR.LOGPROB_DTYPE)
    for seq, p0, n in ((0, 0, 1), (0, 40, 2), (0, 1, 0), (2, 1, 1)):
        assert lib.lnb_session_logprobs_read(ctx.h, seq, p0, n, out.ctypes.data) == -1
    recs = gm.Transformer.score(ctx, t, 0)
    assert [r.Token for r in recs] == list(t[1:])
    assert [r.Token for r in ctx.read_logprobs(1, 1, 3)] == [-1, -1, -1]
    assert [r.Token for r in ctx.read_logprobs(0, 6, 2)] == [-1, -1]
    ctx.close()


def test_8b_fast_scoring_of_2048_tokens(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    args = dict(L.synth.LLAMA31_8B)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    try:
        rng = np.random.default_rng(3)
        toks = rng.integers(0, args["vocab_size"], size=2049).astype(np.int32)
        ctx = _ctx(L, gm, "fast", seq_len=2064, max_rows=2048)
        ctx.set_logprobs(0, 20)
        t0 = gm.Transformer.score(ctx, toks, 0)
        assert len(t0) == 2048 and [r.Token for r in t0] == list(toks[1:])
        got = _read(L, ctx, 0, 1, 2048)
        # the same forward again, its logits kept on the device; 64 rows checked against the statement
        lg = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[:-1].copy(), L.ml.DT_INT32), 0)
        rows = sorted(set(rng.integers(0, 2048, size=62).tolist()) | {0, 2047})
        for r in rows:
            row = np.empty((1, args["vocab_size"]), np.float32)
            L._capi.check(L._capi.lib.lnb_session_logits_read(ctx.h, lg.generation, r, 1, L._capi.ptr(row, L._capi.f32p)))
            _same(got[r:r + 1], SR.logprob_rows(row, toks[r + 1:r + 2], 20), r)
        ctx.close()
    finally:
        gm.Free()


def test_enomem_leaves_the_session_usable(L):
    """records for 8 sequences of 131 073 positions (201 MB) with less device memory free: LNB_ENOMEM, nothing changed"""
    import torch
    args = dict(L.synth.TINY, max_seq_len=131072)
    gm = L.model.LoadModelFromTensors(args, host_tensors(args, SEED))
    ctx = _ctx(L, gm, "strict", seq_len=131072, n_seq=8)
    hog = None
    try:
        p = np.array(PROMPT[:8], np.int32)
        want, _ = gm.Transformer.forward_argmax(ctx, p, 0)
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        hog = torch.empty(max(0, free - (96 << 20)), dtype=torch.uint8, device="cuda")
        with pytest.raises(L._capi.LnbError) as e:
            ctx.set_logprobs(0, 5)
        assert e.value.code == -5 and "bytes" in str(e.value)
        del hog
        hog = None
        torch.cuda.empty_cache()
        assert [r.Token for r in ctx.read_logprobs(0, 1, 2)] == [-1, -1]   # nothing was allocated or switched on
        assert gm.Transformer.forward_argmax(ctx, p, 0)[0] == want
        ctx.set_logprobs(0, 5)
        assert gm.Transformer.forward_argmax(ctx, p, 0)[0] == want
        assert ctx.read_logprobs(0, 8, 1)[0].Token == want
    finally:
        del hog
        torch.cuda.empty_cache()
        ctx.close()
        gm.Free()


def test_8b_strict_sampled_decode_with_logprobs_equals_oracle(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    args = dict(L.synth.LLAMA31_8B)
    tensors = host_tensors(args, L.synth.SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    try:
        prompt = np.array(L.synth.PROMPT_8, np.int32)
        exp = list(SR.generate_sampled(om, prompt, 8 + 8, 0.8, 40, 0.95, 2024, stop_ids=(10**9,)))
        ctx = _ctx(L, gm, "strict", seq_len=136)
        ctx.set_sampling(0, L.model.SamplingArgs(0.8, 40, 0.95, 2024))
        ctx.set_logprobs(0, 20)
        first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
        toks, _, _ = ctx.decode_run(first, 8, 7, use_graph=True)
        assert [first] + list(toks) == exp
        sess = om.new_session(136)
        rows = [sess.forward(prompt, 0, all_rows=False)[0]]
        for i, t in enumerate(exp[:-1]):
            rows.append(sess.forward(np.array([t], np.int32), 8 + i, all_rows=False)[0])
        sess.close()
        _same(_read(L, ctx, 0, 8, 8), SR.logprob_rows(np.stack(rows), exp, 20), "8b")
        ctx.close()
    finally:
        gm.Free()
        om.close()


def _parse_lp(line):
    """'<tag> token rank logprob | t:lp ...' -> (token, rank, logprob, [(t, lp)])"""
    head, _, tail = line.partition("|")
    _, tok, rank, lp = head.split()
    return int(tok), int(rank), float(lp), [(int(a), float(b)) for a, b in (x.split(":") for x in tail.split())]


def _as_tuple(r):
    return r.Token, r.Rank, r.Logprob, [tuple(x) for x in r.Top]


def test_cli_logprobs_and_score_print_what_the_python_mirror_computes(L, tmp_path):
    """host/lnb_generate logprobs=3 (single and batch=3) and score=TEXT, STRICT: the printed values (%.17g, so exact) equal
    GenerateTokens / GenerateTokensBatch / Transformer.score on the same model"""
    import math
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    args = dict(L.synth.TINY)
    gm = L.model.LoadModelFromTensors(args, host_tensors(args, 7))     # lnb_generate's tiny model (seed 7)
    base = [1, 50, 999, 7, 300, 12, 64, 2]
    try:
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(24), acc_mode=L._capi.LNB_ACC_STRICT)
        out = subprocess.run([exe, "24", "strict", "tiny", "logprobs=3"], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        toks = [int(t) for t in [ln for ln in out.stdout.splitlines() if ln.startswith("tokens:")][0].split()[1:]]
        lines = [_parse_lp(ln) for ln in out.stdout.splitlines() if ln.startswith("logprob:")]
        lp = []
        assert [t for _, t in eng.GenerateTokens(base, logprobs=3, logprobs_out=lp)] == toks
        assert lines == [_as_tuple(r) for r in lp] and len(lines) == len(toks)
        out = subprocess.run([exe, "24", "strict", "tiny", "batch=3", "logprobs=3"], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        prompts = [[base[0]] + [(t + 977 * b) % 1000 for t in base[1:]] for b in range(3)]
        lpb = []
        list(eng.GenerateTokensBatch(prompts, logprobs=3, logprobs_out=lpb))
        for b in range(3):
            lines = [_parse_lp(ln) for ln in out.stdout.splitlines() if ln.startswith(f"logprob[{b}]:")]
            assert lines == [_as_tuple(r) for r in lpb[b]], b
    finally:
        gm.Free()
    # score=TEXT on a checkpoint directory with a tokenizer: chunks of 64 scored rows
    d = str(tmp_path)
    subprocess.check_call([exe, "--write-synthetic", d, "tiny"], stdout=subprocess.DEVNULL)
    text = "the quick brown fox jumps over the lazy dog; " * 4
    out = subprocess.run([exe, "200", "strict", d, "score=" + text], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    got = [ln.split() for ln in out.stdout.splitlines() if ln.startswith("score ")]
    m = L.model.LoadModel(d)
    try:
        ids = m.Vocabulary.TokenizeString(text)
        assert 66 < len(ids) <= 201, len(ids)          # more than one chunk
        ctx = _ctx(L, m, "strict", seq_len=200, max_rows=64)
        ctx.allow_chunked_prefill(True)
        ctx.set_logprobs(0, 0)
        recs = []
        for start in range(0, len(ids) - 1, 64):
            recs += m.Transformer.score(ctx, ids[start:start + 65], start)
        ctx.close()
        assert [(int(p), int(t), float(v)) for _, p, t, v in got] == [(i + 1, r.Token, r.Logprob) for i, r in enumerate(recs)]
        s = 0.0
        for r in recs:
            s += r.Logprob
        tail = {ln.split()[0]: float(ln.split()[1]) for ln in out.stdout.splitlines() if ln.startswith(("sum ", "perplexity "))}
        assert tail == {"sum": s, "perplexity": math.exp(-s / len(recs))}
    finally:
        m.Free()
