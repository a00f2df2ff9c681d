"""Ragged forwards (lnb_forward_ragged): one forward whose rows belong to several sequences at their own positions --
prompts, prompt chunks and decode rows side by side -- and continuous batching on top of it
(InferenceEngine.GenerateTokensContinuous).  STRICT: every segment is bit-identical to an independent oracle
InferenceContext fed the same calls.  FAST: a segment's bits do not depend on its neighbours, and it stays within pinned
ulps of the oracle."""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import f32, host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 1234


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _load(L, args):
    tensors = host_tensors(args, SEED)
    return args, tensors, oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors)


@pytest.fixture(scope="module", params=["TINY", "TINY128"])
def model(L, request):
    m = _load(L, dict(getattr(L.synth, request.param)))
    yield m
    m[3].Free()
    m[2].close()


@pytest.fixture(scope="module")
def tiny(L):
    m = _load(L, dict(L.synth.TINY))
    yield m
    m[3].Free()
    m[2].close()


@pytest.fixture(scope="module")
def tiny128(L):
    m = _load(L, dict(L.synth.TINY128))
    yield m
    m[3].Free()
    m[2].close()


def _ctx(L, gm, seq_len, n_seq, max_rows, mode):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq_len), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)


def _oracle_segment(osess, start, toks):
    """the oracle's Forward for one segment: last-row logits [V]"""
    toks = np.asarray(toks, np.int32)
    if start == 0 or len(toks) == 1:
        return osess.forward(toks, start, all_rows=False)[0]
    return osess.forward_chunk(toks, start, all_rows=False)[0]


def _ulps(got, exp):
    """distance in bf16 ulps of the element (of 2^-6 of the largest magnitude for smaller elements), as in test_gpu_model"""
    g, e = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    floor = 2.0 ** -6 * max(np.abs(e).max(), 2.0 ** -100)
    return np.abs(g - e) / 2.0 ** (np.floor(np.log2(np.maximum(np.abs(e), floor))) - 7)


# (seq, start_pos, len) of each segment, in the order the call lists them.  Prompts at 0 of lengths 1, 7 and 33 (and 20, 12),
# continuation chunks at start_pos > 0, single decode rows, sequences idle in some calls, segments out of sequence order.
SCRIPT = [
    [(1, 0, 7), (0, 0, 33)],
    [(2, 0, 1), (3, 0, 20), (1, 7, 1)],
    [(4, 0, 12), (3, 20, 13), (0, 33, 1), (2, 1, 1)],
    [(3, 33, 1), (1, 8, 1), (4, 12, 1)],
    [(3, 34, 1), (0, 34, 1), (4, 13, 1), (1, 9, 1), (2, 2, 1)],
    [(2, 3, 5), (0, 35, 1)],
]


def _run_script(L, gm, ctx, osess, args, rng, mode, ulps=None):
    """feeds SCRIPT to ctx and (when given) to one oracle session per sequence; returns the final positions"""
    pos = [0] * 5
    for call in SCRIPT:
        segs = []
        for sq, start, n in call:
            assert start == pos[sq]
            segs.append((sq, start, rng.integers(0, args["vocab_size"], size=n).astype(np.int32)))
            pos[sq] += n
        nxt, lg = ctx.forward_ragged(segs, want_logits=True)
        assert lg.shape == (len(segs), args["vocab_size"])
        for i, (sq, start, toks) in enumerate(segs):
            if osess is None:
                continue
            exp = _oracle_segment(osess[sq], start, toks)
            if mode == "strict":
                assert np.array_equal(lg[i], exp), (call, i)
                assert nxt[i] == O.argmax_f32(exp), (call, i)
            else:
                ulps["logits"] = max(ulps["logits"], _ulps(lg[i], exp).max())
                assert nxt[i] == int(np.argmax(lg[i]))
    return pos


def _check_caches(ctx, osess, pos, args, exact=True, ulps=None):
    for sq in range(len(pos)):
        ctx.set_active_sequence(sq)
        for layer in range(args["n_layers"]):
            ok, ov = osess[sq].cache(layer)
            gk, gv = ctx.CacheK(layer).RawData[:pos[sq]], ctx.CacheV(layer).RawData[:pos[sq]]
            if exact:
                assert np.array_equal(gk, ok[:pos[sq]]), (sq, layer)
                assert np.array_equal(gv, ov[:pos[sq]]), (sq, layer)
            else:
                ulps["cache"] = max(ulps["cache"], _ulps(f32(gk), f32(ok[:pos[sq]])).max(), _ulps(f32(gv), f32(ov[:pos[sq]])).max())


def test_strict_ragged_calls_equal_independent_oracle_contexts(L, model):
    """six ragged calls over five sequences (prompts, continuation chunks, decode rows, idle sequences, segments out of
    sequence order): every segment's last-row logits and greedy token are bit-identical to an independent oracle session
    fed the same calls, and so is every layer's K/V cache of every sequence up to its position"""
    args, _, om, gm = model
    seq = 48
    ctx = _ctx(L, gm, seq, 5, 64, "strict")
    osess = [om.new_session(seq) for _ in range(5)]
    try:
        ctx.set_active_sequence(3)
        pos = _run_script(L, gm, ctx, osess, args, np.random.default_rng(11), "strict")
        # the ragged calls left the active sequence alone
        assert np.array_equal(ctx.CacheK(0).RawData[:pos[3]], osess[3].cache(0)[0][:pos[3]])
        _check_caches(ctx, osess, pos, args)
        assert ctx.residual(6).shape == (6, args["dim"])   # the last call's rows: [sum(len), dim]
    finally:
        ctx.close()
        for o in osess:
            o.close()


def test_strict_ragged_call_on_a_single_sequence_session(L, tiny):
    """any session takes ragged calls: a single-sequence one without lnb_session_set_chunked_prefill, prompt then chunk"""
    args, _, om, gm = tiny
    ctx = _ctx(L, gm, 32, 1, 16, "strict")
    osess = om.new_session(32)
    try:
        rng = np.random.default_rng(5)
        for start, n in ((0, 9), (9, 6), (15, 1)):
            toks = rng.integers(0, args["vocab_size"], size=n).astype(np.int32)
            nxt, lg = ctx.forward_ragged([(0, start, toks)], want_logits=True)
            exp = _oracle_segment(osess, start, toks)
            assert np.array_equal(lg[0], exp) and nxt[0] == O.argmax_f32(exp)
        _check_caches(ctx, [osess], [16], args)
        assert ctx.residual(1).shape == (1, args["dim"])
    finally:
        ctx.close()
        osess.close()


# Neighbour independence: segment X is run alone (sequence 0), with other segments (sequence 2) and with them in another
# order (sequence 4).  Its last-row logits and cache rows must be bit-identical in all three.  FAST compares calls on the
# same side of the 32-row threshold: (first call) X of 40 rows, all calls >= 32 rows (the tensor-core path);
# (second call) a decode row plus a 3-row chunk of X's sequence next, all calls < 32 rows (GEMV chain).
def _independence(L, model, mode, x_len, others):
    args, _, _, gm = model
    rng = np.random.default_rng(x_len)
    x1 = rng.integers(0, args["vocab_size"], size=x_len).astype(np.int32)
    x2 = rng.integers(0, args["vocab_size"], size=1).astype(np.int32)
    o = [rng.integers(0, args["vocab_size"], size=n).astype(np.int32) for n in others]
    runs = []
    for place, layout in ((0, "alone"), (2, "with"), (4, "permuted")):
        ctx = _ctx(L, gm, 64, 5, 64, mode)
        try:
            oth = [s for s in range(5) if s != place][:len(o)]
            segs1 = [(place, 0, x1)] + [(s, 0, t) for s, t in zip(oth, o)] if layout != "alone" else [(place, 0, x1)]
            segs2 = [(place, x_len, x2)] + [(s, len(t), t[:3]) for s, t in zip(oth, o)] if layout != "alone" else [(place, x_len, x2)]
            if layout == "permuted":
                segs1, segs2 = segs1[::-1], segs2[1:] + segs2[:1]
            out = []
            for segs in (segs1, segs2):
                _, lg = ctx.forward_ragged(segs, want_logits=True)
                out.append(lg[[i for i, s in enumerate(segs) if s[0] == place][0]])
            ctx.set_active_sequence(place)
            out.append([(ctx.CacheK(l).RawData[:x_len + 1].copy(), ctx.CacheV(l).RawData[:x_len + 1].copy())
                        for l in range(args["n_layers"])])
            runs.append((layout, sum(len(s[2]) for s in segs1), sum(len(s[2]) for s in segs2), out))
        finally:
            ctx.close()
    return runs


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_segment_bits_do_not_depend_on_neighbours(L, model, mode):
    runs = _independence(L, model, mode, 40, (10, 5, 8))
    ref = runs[0][3]
    for layout, rows1, rows2, out in runs:
        assert rows1 >= 32 and rows2 < 32   # each call pair stays on one side of the tensor-core threshold
        assert np.array_equal(out[0], ref[0]), (layout, "first call logits")
        assert np.array_equal(out[1], ref[1]), (layout, "second call logits")
        for l, ((k, v), (rk, rv)) in enumerate(zip(out[2], ref[2])):
            assert np.array_equal(k, rk) and np.array_equal(v, rv), (layout, l)


# FAST against the oracle, per element in ulps (_ulps), pinned at about 1.5x the largest value measured on an H100 80GB HBM3
# (700 W power limit): TINY logits 50, caches 24; TINY128 logits 83, caches 59.5.
FAST_ULPS = {"TINY": dict(logits=75, cache=36), "TINY128": dict(logits=128, cache=90)}


def test_fast_ragged_calls_within_pinned_ulps_of_the_oracle(L, model):
    """SCRIPT in FAST (first call: 40 rows on the tensor cores on TINY128; the other calls on the GEMV chain): every
    segment's last-row logits and every cache row within FAST_ULPS of the oracle fed the same calls"""
    args, _, om, gm = model
    name = "TINY128" if args["head_dim"] == 128 else "TINY"
    ctx = _ctx(L, gm, 48, 5, 64, "fast")
    osess = [om.new_session(48) for _ in range(5)]
    try:
        m = dict(logits=0.0, cache=0.0)
        pos = _run_script(L, gm, ctx, osess, args, np.random.default_rng(11), "fast", ulps=m)
        _check_caches(ctx, osess, pos, args, exact=False, ulps=m)
        print(f"ragged FAST {name}: " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(m.items())))
        for k, v in m.items():
            assert v <= FAST_ULPS[name][k], (k, v)
    finally:
        ctx.close()
        for o in osess:
            o.close()


def test_strict_segment_whose_keys_cross_a_chunk_edge(L, tiny128):
    """TINY128 with a 2048-position RoPE table: sequence 0 reaches 1043 positions in three ragged calls beside another
    sequence, so its last rows' keys cross the streamed kernels' 1024-key chunk edge; STRICT stays bit-exact"""
    args = dict(L.synth.TINY128, max_seq_len=2048)
    tensors = tiny128[1]
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    seq = 1100
    ctx = _ctx(L, gm, seq, 2, 528, "strict")
    osess = [om.new_session(seq) for _ in range(2)]
    try:
        rng = np.random.default_rng(1043)
        pos = [0, 0]
        for call in ([(0, 0, 520)], [(1, 0, 8), (0, 520, 520)], [(0, 1040, 3), (1, 8, 1)]):
            segs = [(sq, st, rng.integers(0, args["vocab_size"], size=n).astype(np.int32)) for sq, st, n in call]
            nxt, lg = ctx.forward_ragged(segs, want_logits=True)
            for i, (sq, st, toks) in enumerate(segs):
                exp = _oracle_segment(osess[sq], st, toks)
                assert np.array_equal(lg[i], exp) and nxt[i] == O.argmax_f32(exp), (sq, st)
                pos[sq] = st + len(toks)
        _check_caches(ctx, osess, pos, args)
    finally:
        ctx.close()
        for o in osess:
            o.close()
        gm.Free()
        om.close()


def test_invalid_ragged_calls_are_refused_and_leave_the_session_usable(L, tiny):
    args, _, om, gm = tiny
    ctx = _ctx(L, gm, 32, 3, 16, "strict")
    osess = om.new_session(32)
    try:
        t = lambda n: np.arange(1, n + 1, dtype=np.int32)
        bad = [
            [],                                           # n_segs < 1
            [(0, 0, t(1)), (1, 0, t(1)), (2, 0, t(1)), (0, 1, t(1))],   # n_segs > n_seq
            [(3, 0, t(2))], [(-1, 0, t(2))],              # sequence out of range
            [(0, 0, t(2)), (0, 2, t(1))],                 # one segment per sequence
            [(0, 0, t(0))],                               # empty segment
            [(0, 0, t(10)), (1, 0, t(7))],                # more than max_rows rows
            [(0, -1, t(2))], [(1, 31, t(2))],             # positions outside [0, seq_len)
            [(0, 0, np.array([1, args["vocab_size"]], np.int32))], [(0, 0, np.array([-1], np.int32))],   # token ids
        ]
        for segs in bad:
            with pytest.raises(L._capi.LnbError):
                ctx.forward_ragged(segs)
        # after every refusal a valid call is still bit-exact
        toks = t(5) * 7
        nxt, lg = ctx.forward_ragged([(1, 0, toks)], want_logits=True)
        exp = _oracle_segment(osess, 0, toks)
        assert np.array_equal(lg[0], exp) and nxt[0] == O.argmax_f32(exp)
        # a forward_device handle is stale after a ragged call
        h = gm.Transformer.Forward(ctx, L.ml.Tensor(t(3), L.ml.DT_INT32), 0)
        ctx.forward_ragged([(2, 0, t(2))])
        with pytest.raises(L._capi.LnbError) as e:
            h.RawData
        assert e.value.code == -4                                                                  # LNB_ESTATE
        c, out = L._capi, np.empty((1, args["vocab_size"]), np.float32)
        assert c.lib.lnb_session_logits_read(ctx.h, h.generation, 0, 1, c.ptr(out, c.f32p)) == -4    # LNB_ESTATE
    finally:
        ctx.close()
        osess.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_generate_tokens_continuous_equals_per_prompt_generation(L, tiny, mode):
    """11 prompts of 1..70 tokens through 4 slots with 48-row steps: long prompts are chunked beside decode rows, finished
    slots are refilled, one prompt stops early on an EOS id.  STRICT: every prompt's stream is the single-prompt loop's
    (oracle: orc_generate); FAST: every stream is complete and well formed"""
    args, _, om, gm = tiny
    lens = [1, 70, 7, 33, 2, 48, 15, 64, 5, 29, 11]
    rng = np.random.default_rng(70)
    prompts = [rng.integers(0, args["vocab_size"], size=n).astype(np.int32).tolist() for n in lens]
    seq = 96
    free = [list(om.generate(p, seq, stop_ids=(10**9,))) for p in prompts]
    stop = int(free[2][4])
    exp = [list(om.generate(p, seq, stop_ids=(stop,))) for p in prompts]
    assert len(exp[2]) <= 5 and any(len(e) == seq - len(p) for e, p in zip(exp, prompts))
    saved = gm.Vocabulary.StopTokenIds
    gm.Vocabulary.StopTokenIds = (stop,)
    try:
        acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=acc)
        got, last_state = [[] for _ in prompts], {}
        for i, state, tok in eng.GenerateTokensContinuous(prompts, slots=4, step_tokens=48):
            assert last_state.get(i, L.inference.GSInProgress) == L.inference.GSInProgress      # nothing after the end
            got[i].append(tok)
            last_state[i] = state
        assert sorted(last_state) == list(range(len(prompts)))
        assert all(s != L.inference.GSInProgress for s in last_state.values())
        if mode == "strict":
            assert got == exp
            for i, e in enumerate(exp):
                assert last_state[i] == (L.inference.GSFinishedByReachingEOS if e[-1] == stop else L.inference.GSFinishedByReachingSeqLen)
        else:
            for g, p, s in zip(got, prompts, (last_state[i] for i in range(len(prompts)))):
                assert 1 <= len(g) <= seq - len(p)
                assert (g[-1] == stop) == (s == L.inference.GSFinishedByReachingEOS)
                assert s == L.inference.GSFinishedByReachingEOS or len(g) == seq - len(p)
        with pytest.raises(L.ml.MlError):
            list(eng.GenerateTokensContinuous([list(range(seq))], slots=2, step_tokens=8))
    finally:
        gm.Vocabulary.StopTokenIds = saved


def test_cpp_continuous_generation_matches_the_oracle(L):
    """host/lnb_generate batch=5 slots=2: inference::GenerateTokensContinuous, every prompt's stream = the oracle's"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    out = subprocess.run([exe, "24", "strict", "tiny", "batch=5", "slots=2"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    args = dict(L.synth.TINY)
    om = oracle_model(args, host_tensors(args, 7))
    base = [1, 50, 999, 7, 300, 12, 64, 2]
    try:
        for b in range(5):
            prompt = [base[0]] + [(t + 977 * b) % 1000 for t in base[1:]]
            line = [l for l in out.stdout.splitlines() if l.startswith(f"tokens[{b}]:")][0]
            assert [int(t) for t in line.split()[1:]] == list(om.generate(prompt, 24, stop_ids=(10**9,))), b
    finally:
        om.close()


# ---- the 8B model (synthetic checkpoint): once ---------------------------------------------------------------------

def test_8b_ragged_admission(L):
    """the 8 synth.batch_prompt prompts admitted in ONE ragged call: STRICT logits bit-identical to 8 serial lnb_forward
    prefills; FAST (64 rows: the tensor-core path) within 0.05 of the oracle's last-row logits, the bound of the 8B
    prefill test"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    args = dict(L.synth.LLAMA31_8B)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    prompts = [np.array(L.synth.batch_prompt(b), np.int32) for b in range(8)]
    segs = [(b, 0, p) for b, p in enumerate(prompts)]
    try:
        ctx = _ctx(L, gm, 64, 8, 64, "strict")
        try:
            nxt, lg = ctx.forward_ragged(segs, want_logits=True)
            for b, p in enumerate(prompts):
                ctx.set_active_sequence(b)
                n1, l1 = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
                assert np.array_equal(lg[b], l1[0]) and nxt[b] == n1, b
        finally:
            ctx.close()
        ctx = _ctx(L, gm, 64, 8, 64, "fast")
        try:
            _, lf = ctx.forward_ragged(segs, want_logits=True)
        finally:
            ctx.close()
    finally:
        gm.Free()
    tensors = host_tensors(args, L.synth.SEED)
    om = oracle_model(args, tensors)
    try:
        worst = 0.0
        for b, p in enumerate(prompts):
            s = om.new_session(16)
            exp = s.forward(p, 0, all_rows=False)[0]
            s.close()
            worst = max(worst, float(np.abs(lf[b] - exp).max()))
        print(f"8B ragged FAST admission: max |logit - oracle| {worst:.4f}")
        assert worst <= 0.05, worst
    finally:
        om.close()
        del tensors
