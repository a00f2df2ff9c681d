"""Penalties and logit bias on the device (csrc/penalty.cuh, DESIGN.md §9e) against their sequential C statement
(orc_penalize_row and orc_generate_processed, oracle_sampling/lnb_sample_ref.c): the op bit-exact on adversarial rows and
long histories, STRICT penalized streams equal to the statement on every path (greedy and sampled), chunking, batching
with other neighbours, banned tokens, neutral parameters and sessions without penalties unchanged, decode-graph
re-capture, validation, and the 8B model."""
import ctypes as C

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 4321
PROMPT = [1, 50, 999, 7, 300, 12, 64, 2]
PROMPTS = [PROMPT, [5, 6, 5, 6, 5], [900, 3, 4, 17, 22, 3, 4], [8]]
SEQ_LEN = 24
SAMP = (0.9, 0, 1.0, 5)   # temperature, top_k, top_p, seed


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


def _pens(L):
    P = L.model.PenaltyArgs
    return [P(1.3, 0.4, 0.2), P(0.8, -0.3, 0.5, Window=4, CountPrompt=True, LogitBias={3: 2.5, 7: -np.inf, 64: -1.0})]


def _oracle_pen(L, pen, prompt_len):
    return SR.Penalties.from_buffer_copy(bytes(pen.c(prompt_len)))


def _oracle(L, om, prompt, pen, sampled, seq_len=SEQ_LEN, seed_off=0):
    T, K, P, seed = SAMP if sampled else (0.0, 0, 1.0, 0)
    return list(SR.generate_processed(om, prompt, seq_len, T, K, P, seed + seed_off,
                                      None if pen is None else _oracle_pen(L, pen, len(prompt)), stop_ids=L.synth.STOP_IDS))


def _samp(L, sampled):
    return L.model.SamplingArgs(*SAMP) if sampled else None


def _ctx(L, gm, mode="strict", seq_len=SEQ_LEN, max_rows=8, n_seq=1):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq_len), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)


def _engine(L, gm, mode="strict", seq_len=SEQ_LEN, max_rows=8):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq_len), acc_mode=acc, max_rows=max_rows)


# ---- the op ---------------------------------------------------------------------------------------------------------
def _op(L, rows, params, hist, pos_next):
    rows = np.ascontiguousarray(rows, np.float32)
    n, V = rows.shape
    h = np.ascontiguousarray(hist, np.int32)
    pn = np.ascontiguousarray(pos_next, np.int32)
    par = (L._capi.PenaltiesC * n)(*[L._capi.PenaltiesC.from_buffer_copy(bytes(p)) for p in params])
    out = np.empty_like(rows)
    L._capi.check(L._capi.lib.lnb_op_penalize_f32(L._capi.ptr(rows, L._capi.f32p), n, V, par, L._capi.ptr(h, L._capi.i32p), h.shape[1],
                                                  L._capi.ptr(pn, L._capi.i32p), L._capi.ptr(out, L._capi.f32p)))
    return out


def _adversarial(rng, V, n, T):
    rows = (rng.standard_normal((n, V)) * 3).astype(np.float32)
    hist = rng.integers(-1, V, size=(n, T)).astype(np.int32)
    params, pn = [], []
    for r in range(n):
        kind = r % 8
        if kind == 1:
            hist[r] = 7 % V                                    # one token fills the whole history
        elif kind == 2:
            hist[r] = rng.integers(0, min(V, 5), T)            # a few tokens, long runs
            rows[r, : min(V, 5)] = [np.inf, -np.inf, np.nan, -0.0, 1e-42][: min(V, 5)]
        elif kind == 3:
            rows[r] = np.round(rows[r])                        # ties
        elif kind == 4:
            rows[r, ::3] = np.uint32(0xFFC00000).view(np.float32)   # negative NaNs (the x86 default NaN)
        nb = int(rng.integers(0, 65)) if r % 2 else 0
        bias = {int(t): float(rng.choice([rng.uniform(-8, 8), -np.inf])) for t in rng.choice(V, size=min(nb, V), replace=False)}
        rp = float(rng.choice([0.6, 1.0, 1.25, 2.0]))
        window = int(rng.choice([0, 1, 64, 4096, T]))
        params.append(SR.penalties(rp, float(rng.uniform(-1, 1)), float(rng.uniform(-1, 1)), window, int(rng.integers(0, 8)), bias))
        pn.append(T if r % 3 else int(rng.integers(0, T + 1)))
    params[0] = SR.penalties() if n > 1 else params[0]         # a neutral row beside the others: copied
    return rows, params, hist, pn


@pytest.mark.parametrize("V,n,T", [(64, 8, 50), (4097, 8, 4096), (128256, 1, 131072), (128256, 8, 131072), (32768, 8, 32768)])
def test_op_bit_exact(L, V, n, T):
    rng = np.random.default_rng(V + n + T)
    rows, params, hist, pn = _adversarial(rng, V, n, T)
    got = _op(L, rows, params, hist, pn)
    exp = SR.penalize_rows(rows, params, hist, pn)
    for r in range(n):
        bad = np.flatnonzero(got[r].view(np.uint32) != exp[r].view(np.uint32))
        assert bad.size == 0, (V, n, T, r, bad[:8], got[r][bad[:8]], exp[r][bad[:8]])


def test_op_counts_a_full_history_of_one_token(L):
    V, T = 128256, 131072
    row = np.zeros((1, V), np.float32)
    hist = np.full((1, T), 12345, np.int32)
    got = _op(L, row, [SR.penalties(1.0, 1.0, 0.5)], hist, [T])
    assert got[0, 12345] == np.float32(-(T + 0.5)) and np.count_nonzero(got) == 1


# ---- streams on every path ------------------------------------------------------------------------------------------
def _forward_device(L, ctx, toks, pos):
    t = np.ascontiguousarray(toks, np.int32)
    nxt, gen = C.c_int32(-1), C.c_int64(0)
    L._capi.check(L._capi.lib.lnb_forward_device(ctx.h, L._capi.ptr(t, L._capi.i32p), t.shape[0], pos, 1, C.byref(nxt), C.byref(gen)))
    return nxt.value


def _host_loop(L, gm, ctx, prompt, steps, device=False):
    """prefill, then one S = 1 forward per token through lnb_forward or lnb_forward_device"""
    fwd = (lambda t, p: _forward_device(L, ctx, t, p)) if device else (lambda t, p: gm.Transformer.forward_argmax(ctx, t, p)[0])
    out = [fwd(np.array(prompt, np.int32), 0)]
    for i in range(steps - 1):
        out.append(fwd(np.array([out[-1]], np.int32), len(prompt) + i))
    return out


@pytest.mark.parametrize("sampled", [False, True])
@pytest.mark.parametrize("which", [0, 1])
def test_strict_streams_equal_the_statement_on_every_path(L, model, sampled, which):
    _, om, gm = model
    pen = _pens(L)[which]
    want = _oracle(L, om, PROMPT, pen, sampled)
    n = len(want)
    eng = _engine(L, gm)
    # lnb_forward through the generate loop, one-shot and chunked prefill
    assert [t for _, t in eng.GenerateTokens(PROMPT, sampling=_samp(L, sampled), penalties=pen)] == want
    assert [t for _, t in eng.GenerateTokens(PROMPT, sampling=_samp(L, sampled), penalties=pen, prefill_chunk=3)] == want
    # lnb_forward and lnb_forward_device host loops
    for device in (False, True):
        ctx = _ctx(L, gm)
        ctx.set_sampling(0, _samp(L, sampled))
        ctx.set_penalties(0, pen, len(PROMPT))
        assert _host_loop(L, gm, ctx, PROMPT, n, device) == want, device
        ctx.close()
    # lnb_decode_run on an engine session, with and without a graph
    for use_graph in (False, True):
        ctx = _ctx(L, gm)
        ctx.set_sampling(0, _samp(L, sampled))
        ctx.set_penalties(0, pen, len(PROMPT))
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        toks, _, graphed = ctx.decode_run(first, len(PROMPT), n - 1, use_graph=use_graph)
        assert [first] + list(toks) == want and graphed == use_graph
        assert "penalized" in L._capi.lib.lnb_last_error().decode() or sampled
        ctx.close()
    # speculative generation (prompt lookup) and the batch / continuous loops
    spec = [t for _, t in eng.GenerateTokens(PROMPT, sampling=_samp(L, sampled), penalties=pen, speculative=L.inference.SpeculativeArgs(4))]
    assert spec == want
    wants = [want] + [_oracle(L, om, p, pen, sampled, seed_off=i + 1) for i, p in enumerate(PROMPTS[1:])]
    out = list(eng.GenerateTokensBatch(PROMPTS, sampling=_samp(L, sampled), penalties=pen))
    for i in range(len(PROMPTS)):
        assert [t for s, _, t in out if s == i] == wants[i], ("batch", i)
    out = list(eng.GenerateTokensBatch(PROMPTS, sampling=_samp(L, sampled), penalties=pen, speculative=L.inference.SpeculativeArgs(3)))
    for i in range(len(PROMPTS)):
        assert [t for s, _, t in out if s == i] == wants[i], ("batch speculative", i)
    out = list(eng.GenerateTokensContinuous(PROMPTS, slots=2, step_tokens=4, sampling=_samp(L, sampled), penalties=pen))
    for i in range(len(PROMPTS)):
        assert [t for s, _, t in out if s == i] == wants[i], ("continuous", i)


@pytest.mark.parametrize("sampled", [False, True])
def test_speculative_calls_with_perfect_and_wrong_drafts(L, model, sampled):
    _, om, gm = model
    pen = _pens(L)[1]
    want = _oracle(L, om, PROMPT, pen, sampled)
    p0 = len(PROMPT)
    for wrong in (False, True):
        ctx = _ctx(L, gm)
        ctx.set_sampling(0, _samp(L, sampled))
        ctx.set_penalties(0, pen, p0)
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
        assert first == want[0]
        got, pos = [first], p0
        while len(got) < len(want):
            k = min(7, len(want) - len(got), SEQ_LEN - 2 - pos)
            drafts = list(want[len(got):len(got) + k])
            if wrong and drafts:
                drafts[len(drafts) // 2] = (drafts[len(drafts) // 2] + 1) % 1024   # rejected from there on
            nxt, acc, _ = ctx.forward_speculative([(0, pos, [got[-1]] + drafts)])
            a = int(acc[0])
            assert a == (len(drafts) if not wrong else len(drafts) // 2)
            got += [int(t) for t in nxt[:a + 1]]
            pos += a + 1
        assert got[:len(want)] == want, wrong
        ctx.close()


def test_batched_with_neighbours_equals_alone(L, model):
    """sequence 0 with penalties A, greedy; sequence 1 with penalties B, sampled; sequence 2 plain: forward_batch steps"""
    _, om, gm = model
    pa, pb = _pens(L)
    prompts = [PROMPT, PROMPTS[2], PROMPTS[1]]
    wants = [_oracle(L, om, prompts[0], pa, False), _oracle(L, om, prompts[1], pb, True), _oracle(L, om, prompts[2], None, False)]
    ctx = _ctx(L, gm, n_seq=3)
    ctx.set_penalties(0, pa, len(prompts[0]))
    ctx.set_penalties(1, pb, len(prompts[1]))
    ctx.set_sampling(1, _samp(L, True))
    cur, pos, got = [], [], [[], [], []]
    for i, p in enumerate(prompts):
        ctx.set_active_sequence(i)
        t, _ = gm.Transformer.forward_argmax(ctx, np.array(p, np.int32), 0)
        cur.append(t)
        pos.append(len(p))
        got[i].append(t)
    while min(pos) < SEQ_LEN - 1:
        nxt, _ = ctx.forward_batch(cur, pos)
        for i in range(3):
            if pos[i] < SEQ_LEN - 1:
                got[i].append(int(nxt[i]))
                cur[i], pos[i] = int(nxt[i]), pos[i] + 1
    for i in range(3):
        assert got[i] == wants[i][:len(got[i])], i
    ctx.close()


def test_banned_tokens_are_never_emitted(L, model):
    _, om, gm = model
    eng = _engine(L, gm)
    for sampled in (False, True):
        plain = [t for _, t in eng.GenerateTokens(PROMPT, sampling=_samp(L, sampled))]
        ban = sorted(set(plain))[:64]
        pen = L.model.PenaltyArgs(LogitBias={t: -np.inf for t in ban})
        got = [t for _, t in eng.GenerateTokens(PROMPT, sampling=_samp(L, sampled), penalties=pen)]
        assert not set(got) & set(ban) and got == _oracle(L, om, PROMPT, pen, sampled)


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_neutral_and_unused_penalties_change_nothing(L, model, mode):
    _, _, gm = model
    p = np.array(PROMPT, np.int32)

    def run(ctx):
        l0 = ctx.launch_count()
        n0, lg0 = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
        nb, lb = ctx.forward_batch([n0], [8], want_logits=True)   # sequence 0 only
        ctx.set_active_sequence(0)
        toks, _, _ = ctx.decode_run(int(nb[0]), 9, 5, use_graph=True)
        toks2, _, _ = ctx.decode_run(int(toks[-1]), 14, 5, use_graph=False)
        nr, _ = ctx.forward_ragged([(0, 19, [int(toks2[-1])])])
        return ctx.launch_count() - l0, n0, lg0, nb, lb, list(toks) + list(toks2) + [int(nr[0])]

    base = _ctx(L, gm, mode, n_seq=2)
    want = run(base)
    neutral = _ctx(L, gm, mode, n_seq=2)
    neutral.set_penalties(0, L.model.PenaltyArgs(1.0, 0.0, 0.0, Window=5, CountPrompt=True), 8)
    other = _ctx(L, gm, mode, n_seq=2)
    other.set_penalties(1, _pens(L)[0], 3)          # another sequence is penalized
    off = _ctx(L, gm, mode, n_seq=2)
    off.set_penalties(0, _pens(L)[1], 8)
    off.set_penalties(0, None)                       # turned on, then off again
    for ctx in (neutral, other, off):
        got = run(ctx)
        assert got[0] == want[0] and got[1] == want[1] and got[5] == want[5]
        assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3]) and np.array_equal(got[4], want[4])
    eng = _engine(L, gm, mode)
    assert [t for _, t in eng.GenerateTokens(PROMPT, penalties=L.model.PenaltyArgs())] == [t for _, t in eng.GenerateTokens(PROMPT)]
    for c in (base, neutral, other, off):
        c.close()


def test_graph_recaptures_on_a_toggle_not_on_a_value_change(L, model):
    _, om, gm = model
    pa, pb = _pens(L)
    p = np.array(PROMPT, np.int32)
    ctx = _ctx(L, gm)
    first, _ = gm.Transformer.forward_argmax(ctx, p, 0)
    ctx.decode_run(first, 8, 3, use_graph=True)
    l0 = ctx.launch_count()
    plain, _, _ = ctx.decode_run(first, 8, 3, use_graph=True)
    per_plain = ctx.launch_count() - l0

    def penalized_run(pen):
        ctx.set_penalties(0, pen, 8)
        f, _ = gm.Transformer.forward_argmax(ctx, p, 0)   # records the prompt (the enable cleared the history)
        l1 = ctx.launch_count()
        toks, _, graphed = ctx.decode_run(f, 8, 6, use_graph=True)
        assert graphed
        assert [f] + list(toks) == _oracle(L, om, PROMPT, pen, False)[:7]
        return ctx.launch_count() - l1

    per_a = penalized_run(pa)
    assert per_a > 2 * per_plain   # toggled on: the step records, penalizes and samples
    ctx.set_sampling(0, None)
    assert penalized_run(pb) == per_a   # a value change replays the same graph, which reads the new slot
    ctx.set_penalties(0, None)
    l0 = ctx.launch_count()
    toks, _, _ = ctx.decode_run(first, 8, 3, use_graph=True)
    assert ctx.launch_count() - l0 == per_plain and list(toks) == list(plain)
    ctx.close()


def test_validation(L, model):
    args, _, gm = model
    V = args["vocab_size"]
    ctx = _ctx(L, gm, n_seq=2)
    P = L.model.PenaltyArgs
    bad = [P(0.0), P(-1.0), P(float("inf")), P(float("nan")), P(1.0, float("inf")), P(1.0, float("nan")), P(1.0, 0.0, float("-inf")),
           P(1.2, Window=-1), P(1.2, LogitBias={V: 1.0}), P(1.2, LogitBias={-1: 1.0}), P(LogitBias={3: float("inf")}),
           P(LogitBias={3: float("nan")})]
    for b in bad:
        with pytest.raises(L._capi.LnbError) as e:
            ctx.set_penalties(0, b, 0)
        assert e.value.code == -1, b
    with pytest.raises(L._capi.LnbError):
        ctx.set_penalties(0, P(1.2), -1)                    # first_pos < 0
    with pytest.raises(L._capi.LnbError):
        ctx.set_penalties(2, P(1.2), 0)                     # sequence out of range
    c = L._capi.PenaltiesC.from_buffer_copy(bytes(P(1.0, LogitBias={3: 1.0, 4: 2.0}).c(0)))
    c.bias_token[1] = 3                                      # a repeated bias token
    with pytest.raises(L._capi.LnbError):
        L._capi.check(L._capi.lib.lnb_session_set_penalties(ctx.h, 0, C.byref(c)))
    c.bias_token[1] = 4
    c.n_bias = 65
    with pytest.raises(L._capi.LnbError):
        L._capi.check(L._capi.lib.lnb_session_set_penalties(ctx.h, 0, C.byref(c)))
    # nothing was switched on: the session launches what a fresh one does
    fresh = _ctx(L, gm, n_seq=2)
    counts = []
    for x in (ctx, fresh):
        l0 = x.launch_count()
        n0, _ = gm.Transformer.forward_argmax(x, np.array(PROMPT, np.int32), 0)
        x.decode_run(n0, 8, 4, use_graph=False)
        counts.append((x.launch_count() - l0, n0))
    assert counts[0] == counts[1]
    # the op's own checks
    row = np.zeros((1, 16), np.float32)
    with pytest.raises(L._capi.LnbError):
        _op(L, row, [SR.penalties(1.2)], np.zeros((1, 4), np.int32), [5])   # pos_next beyond the history
    with pytest.raises(L._capi.LnbError):
        _op(L, np.zeros((9, 16), np.float32), [SR.penalties(1.2)] * 9, np.zeros((9, 4), np.int32), [4] * 9)
    ctx.close(); fresh.close()


# ---- 8B --------------------------------------------------------------------------------------------------------------
def test_8b_strict_batch_and_fast_decode_with_penalties(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    args = dict(L.synth.LLAMA31_8B)
    tensors = host_tensors(args, L.synth.SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    try:
        prompts = [list(L.synth.PROMPT_8), [int(t) for t in L.synth.PROMPT_8[:5]]]
        plain = [t for _, t in _engine(L, gm, "strict", seq_len=16).GenerateTokens(prompts[0])]
        pen = L.model.PenaltyArgs(1.3, 0.5, 0.25, Window=64, LogitBias={plain[0]: -np.inf, 128000: -np.inf})
        want0 = _oracle(L, om, prompts[0], pen, False, seq_len=16)
        assert want0[0] != plain[0]
        out = list(_engine(L, gm, "strict", seq_len=16).GenerateTokensBatch(prompts, penalties=pen))
        assert [t for s, _, t in out if s == 0] == want0
        alone = [t for _, t in _engine(L, gm, "strict", seq_len=16).GenerateTokens(prompts[1], penalties=pen)]
        assert [t for s, _, t in out if s == 1] == alone
        # FAST: the device-resident decode equals the host loop, both penalized and sampled
        for sampled in (False, True):
            c1 = _ctx(L, gm, "fast", seq_len=32)
            c1.set_sampling(0, _samp(L, sampled))
            c1.set_penalties(0, pen, 8)
            host = _host_loop(L, gm, c1, prompts[0], 16)
            c2 = _ctx(L, gm, "fast", seq_len=32)
            c2.set_sampling(0, _samp(L, sampled))
            c2.set_penalties(0, pen, 8)
            f, _ = gm.Transformer.forward_argmax(c2, np.array(prompts[0], np.int32), 0)
            toks, _, graphed = c2.decode_run(f, 8, 15, use_graph=True)
            assert graphed and [f] + list(toks) == host and plain[0] not in host
            c1.close(); c2.close()
    finally:
        gm.Free()
        om.close()


def test_cli_penalties_print_what_the_python_mirror_generates(L):
    """host/lnb_generate rep= freq= pres= last_n= (single, batch=3 and slots=2), STRICT: the ids GenerateTokens /
    GenerateTokensBatch / GenerateTokensContinuous generate with the same penalties on the same model"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    args = dict(L.synth.TINY)
    gm = L.model.LoadModelFromTensors(args, host_tensors(args, 7))     # lnb_generate's tiny model (seed 7)
    base = [1, 50, 999, 7, 300, 12, 64, 2]
    pen = L.model.PenaltyArgs(1.5, 0.5, 0.25, Window=6)
    flags = ["rep=1.5", "freq=0.5", "pres=0.25", "last_n=6"]
    try:
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(24), acc_mode=L._capi.LNB_ACC_STRICT)
        out = subprocess.run([exe, "24", "strict", "tiny"] + flags, capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        toks = [int(t) for t in [ln for ln in out.stdout.splitlines() if ln.startswith("tokens:")][0].split()[1:]]
        assert [t for _, t in eng.GenerateTokens(base, penalties=pen)] == toks
        prompts = [[base[0]] + [(t + 977 * b) % 1000 for t in base[1:]] for b in range(3)]
        for extra, run in ((["batch=3"], lambda: eng.GenerateTokensBatch(prompts, penalties=pen)),
                           (["batch=3", "slots=2"], lambda: eng.GenerateTokensContinuous(prompts, slots=2, step_tokens=64, penalties=pen))):
            out = subprocess.run([exe, "24", "strict", "tiny"] + extra + flags, capture_output=True, text=True, timeout=120)
            assert out.returncode == 0, out.stderr
            got = list(run())
            for b in range(3):
                line = [ln for ln in out.stdout.splitlines() if ln.startswith(f"tokens[{b}]:")][0]
                assert [int(t) for t in line.split()[1:]] == [t for s, _, t in got if s == b], (extra, b)
    finally:
        gm.Free()
