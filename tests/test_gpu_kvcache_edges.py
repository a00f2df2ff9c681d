"""The MXFP8 KV cache at its edges (DESIGN.md §9j), bit for bit against the reference forward with decoded cache rows
(RefSession of tests/test_kvcache_cpu.py): blocks at the ends of the E8M0 range and non-finite values written by the
forward's own writer and read by the attention's decode (tests/kv_cases.py), head shapes beyond the main suite's, the
last positions of a 131 072-position session and the reads of its cache, the calls that rewrite or reorder cache rows,
and the FAST tensor-core prompt stage by stage."""
import ctypes as C

import numpy as np
import pytest

import lnb_b200 as L
from lnb_b200._capi import LNB_ACC_FAST, LNB_ACC_STRICT, lib
from oracle import oracle as O
from oracle_sampling import sample_ref as SR
from tests import kv_cases as K
from tests import precise as P
from tests.helpers import host_tensors
from tests.model_shapes import CATALOGUE
from tests.test_gpu_kvcache import _bits, _ctx, _forward, _own_caches, _prompt
from tests.test_gpu_logprobs import _read, _same
from tests.test_gpu_tc_stages import _inside, _norm, _probes
from tests.test_kvcache_cpu import RefSession

pytestmark = pytest.mark.gpu

SEED = 23
SHAPES = {"tiny": dict(L.synth.TINY), "tiny128": dict(L.synth.TINY128), "hd96": dict(CATALOGUE["hd96"]),
          "tiny_long": dict(L.synth.TINY, max_seq_len=4096), "tiny128_long": dict(L.synth.TINY128, max_seq_len=4096),
          "tiny_far": dict(L.synth.TINY, max_seq_len=131072), "gqa8_far": dict(CATALOGUE["gqa8"], max_seq_len=131072),
          **{k: dict(v) for k, v in K.SHAPES.items()}}
EXTREME = ["tiny", "tiny128", "hd96"]
NONFINITE_TOKEN = 77


@pytest.fixture(scope="module")
def models():
    made = {}

    def get(name, kind="plain"):
        """(args, tensors, hot tokens or the non-finite elements, model)"""
        key = (name, kind)
        if key not in made:
            args = dict(SHAPES[name])
            extra = None
            if kind == "extreme":
                tensors, extra = K.extreme_kv_tensors(args, SEED)
            elif kind == "nonfinite":
                tensors, extra = K.nonfinite_kv_tensors(args, SEED, NONFINITE_TOKEN)
            else:
                tensors = host_tensors(args, SEED)
            made[key] = (args, tensors, extra, L.model.LoadModelFromTensors(args, tensors))
        return made[key]

    yield get
    for *_, gm in made.values():
        gm.Free()


def _order(mode):
    return O.ORDER_REF if mode == LNB_ACC_STRICT else O.ORDER_FAST_STREAM


def _clone(ref: RefSession) -> RefSession:
    c = RefSession(ref.a, ref.t, ref.seq_len, ref.kv_mx, order=(ref.ks, ref.parts, ref.attn), decode=ref.decode)
    for n in ("ck", "cv", "pre_k", "pre_v"):
        setattr(c, n, [a.copy() for a in getattr(ref, n)])
    return c


def _check_caches(ctx, refs, args, seq, n, layers=None):
    """every listed sequence's decoded caches equal its reference's, and its raw blocks of positions [0, n) are the C
    statement's blocks of the reference's rows before quantization (and decode to the session's rows)"""
    kvd, hd = args["n_kv_heads"] * args["head_dim"], args["head_dim"]
    for q, ref in refs.items():
        ctx.set_active_sequence(q)
        for layer in (range(args["n_layers"]) if layers is None else layers):
            for w, cache, pre, dec in (("k", ctx.CacheK, ref.pre_k, ref.ck), ("v", ctx.CacheV, ref.pre_v, ref.cv)):
                got = cache(layer).RawData.reshape(seq, kvd)
                assert np.array_equal(got, dec[layer]), (q, layer, w)
                codes, scales = ctx.kv_read(q, layer, w, 0, n)
                c, s, _ = SR.kv_mxfp8_quantize(pre[layer][:n], hd)
                assert np.array_equal(scales, s), (q, layer, w, np.argwhere(scales != s)[:4])
                assert np.array_equal(codes, c), (q, layer, w, np.argwhere(codes != c)[:4])
                assert np.array_equal(K.decode(codes, scales, hd), got[:n])
    ctx.set_active_sequence(0)


# ---- blocks at the ends of the range, written and read inside forwards ---------------------------------------------------
@pytest.mark.parametrize("name", EXTREME)
@pytest.mark.parametrize("plen", [1, 40])
def test_extreme_blocks_strict_prompt_and_steps(models, name, plen):
    args, t, hot, gm = models(name, "extreme")
    seq = 48
    ref = RefSession(args, t, seq, True)
    ctx = _ctx(gm, seq)
    try:
        p = K.extreme_prompt(args, hot, plen, 3)
        assert np.array_equal(_bits(_forward(ctx, p, 0)), _bits(ref.forward(p, 0)))
        tok, pos = int(hot[-1]), plen
        for _ in range(3):
            lg = ref.forward([tok], pos)
            assert np.array_equal(_bits(_forward(ctx, [tok], pos)), _bits(lg)), pos
            tok, pos = int(np.argmax(lg[0])), pos + 1
        _check_caches(ctx, {0: ref}, args, seq, pos)
    finally:
        ctx.close()


@pytest.mark.parametrize("name", EXTREME)
def test_extreme_blocks_batched_steps(models, name):
    args, t, hot, gm = models(name, "extreme")
    seq, n = 32, 3
    refs = {i: RefSession(args, t, seq, True) for i in range(n)}
    ctx = _ctx(gm, seq, n_seq=n)
    try:
        lens = [5, 9, 13]
        toks = []
        for i in range(n):
            ctx.set_active_sequence(i)
            p = K.extreme_prompt(args, hot, lens[i], 10 + i)
            lg = _forward(ctx, p, 0)
            assert np.array_equal(_bits(lg), _bits(refs[i].forward(p, 0)))
            toks.append(int(hot[i % len(hot)]))
        pos = list(lens)
        for _ in range(2):
            nxt, lg = ctx.forward_batch(toks, pos, want_logits=True)
            for i in range(n):
                assert np.array_equal(_bits(lg[i]), _bits(refs[i].forward([toks[i]], pos[i])[0])), i
            toks, pos = [int(x) for x in nxt], [q + 1 for q in pos]
        _check_caches(ctx, refs, args, seq, min(pos))
    finally:
        ctx.close()


@pytest.mark.parametrize("name", EXTREME)
def test_extreme_blocks_fast_chain(models, name):
    args, t, hot, gm = models(name, "extreme")
    seq = 48
    ref = RefSession(args, t, seq, True, order=O.ORDER_FAST_STREAM)
    ctx = _ctx(gm, seq, mode=LNB_ACC_FAST, max_rows=31)
    try:
        p = K.extreme_prompt(args, hot, 12, 6)
        assert np.array_equal(_bits(_forward(ctx, p, 0)), _bits(ref.forward(p, 0)))
        tok = int(hot[0])
        for i in range(3):
            e = ref.forward([tok], 12 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], 12 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
        _check_caches(ctx, {0: ref}, args, seq, 15)
    finally:
        ctx.close()


@pytest.mark.parametrize("mode", [LNB_ACC_STRICT, LNB_ACC_FAST])
def test_nonfinite_values_keep_their_blocks(models, mode):
    """+inf and -inf in one V head of layer 0 at two positions: that layer's raw blocks are the C statement's (saturated
    codes, the scale of the finite elements); the logits after it are not compared"""
    args, t, (jp, jn), gm = models("tiny", "nonfinite")
    seq = 16
    ref = RefSession(args, t, seq, True, order=_order(mode))
    ctx = _ctx(gm, seq, mode=mode, max_rows=31)
    try:
        p = np.array([5, 9, 300, NONFINITE_TOKEN, 12, 40, NONFINITE_TOKEN, 3], np.int32)
        with np.errstate(all="ignore"):
            ref.forward(p, 0)
            ref.forward([8], len(p))
        _forward(ctx, p, 0)
        _forward(ctx, [8], len(p))
        n = len(p) + 1
        c, s, _ = SR.kv_mxfp8_quantize(ref.pre_v[0][:n], args["head_dim"])
        assert c[3, jp] == 0x7E and c[3, jn] == 0xFE and c[6, jp] == 0x7E and s[3, 0, 0] < 127 + 119
        for w, pre in (("k", ref.pre_k[0]), ("v", ref.pre_v[0])):
            codes, scales = ctx.kv_read(0, 0, w, 0, n)
            c, s, _ = SR.kv_mxfp8_quantize(pre[:n], args["head_dim"])
            assert np.array_equal(scales, s), (w, np.argwhere(scales != s)[:4])
            bad = np.argwhere(codes != c)
            assert not bad.size, (w, bad[:4], codes[codes != c], c[codes != c], pre[:n][codes != c])
    finally:
        ctx.close()


# ---- head shapes beyond the main suite's -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(K.SHAPES))
def test_shape_strict_batched_and_fast(models, name):
    args, t, _, gm = models(name)
    seq = 48
    ref = RefSession(args, t, seq, True)
    ctx = _ctx(gm, seq)
    try:                                                   # STRICT prompt and steps
        p = _prompt(args, 40)
        lg = _forward(ctx, p, 0)
        assert np.array_equal(_bits(lg), _bits(ref.forward(p, 0)))
        tok = int(np.argmax(lg[-1]))
        for i in range(2):
            e = ref.forward([tok], 40 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], 40 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
        _check_caches(ctx, {0: ref}, args, seq, 42, layers=[0, args["n_layers"] - 1])
    finally:
        ctx.close()
    refs = {i: RefSession(args, t, seq, True) for i in range(3)}
    ctx = _ctx(gm, seq, n_seq=3)
    try:                                                   # three sequences, batched steps
        toks, pos = [], [3, 6, 9]
        for i in range(3):
            ctx.set_active_sequence(i)
            p = _prompt(args, pos[i], seed=20 + i)
            lg = _forward(ctx, p, 0)
            assert np.array_equal(_bits(lg), _bits(refs[i].forward(p, 0)))
            toks.append(int(np.argmax(lg[-1])))
        for _ in range(2):
            nxt, lg = ctx.forward_batch(toks, pos, want_logits=True)
            for i in range(3):
                assert np.array_equal(_bits(lg[i]), _bits(refs[i].forward([toks[i]], pos[i])[0])), i
            toks, pos = [int(x) for x in nxt], [q + 1 for q in pos]
    finally:
        ctx.close()
    ref = RefSession(args, t, seq, True, order=O.ORDER_FAST_STREAM)
    ctx = _ctx(gm, seq, mode=LNB_ACC_FAST, max_rows=31)
    try:                                                   # FAST chain
        p = _prompt(args, 9, seed=6)
        lg = _forward(ctx, p, 0)
        assert np.array_equal(_bits(lg), _bits(ref.forward(p, 0)))
        tok = int(np.argmax(lg[-1]))
        for i in range(2):
            e = ref.forward([tok], 9 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], 9 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
    finally:
        ctx.close()


@pytest.mark.parametrize("name", list(K.LONG_SHAPES))
def test_shape_long_cache(models, name):
    """a cache of 1 100 positions: two FAST chunks (1 024 keys) and several V stages"""
    args, t, _, gm = models(name)
    T0 = 1100
    seq = T0 + 4
    p = _prompt(args, T0, seed=8)
    ref = RefSession(args, t, seq, True)
    ctx = _ctx(gm, seq, max_rows=T0)
    try:
        e = ref.forward(p, 0)
        assert np.array_equal(_bits(_forward(ctx, p, 0)), _bits(e))
        tok = int(np.argmax(e[-1]))
        for i in range(2):
            e = ref.forward([tok], T0 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], T0 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
    finally:
        ctx.close()
    ref = RefSession(args, t, seq, True, order=O.ORDER_FAST_STREAM)
    ctx = _ctx(gm, seq, mode=LNB_ACC_FAST, max_rows=T0)
    try:          # the prompt (tensor cores where the shape allows), then steps over the session's own caches
        lg = _forward(ctx, p, 0)
        ref.load_caches(*_own_caches(ctx, args, seq), T0)
        tok = int(np.argmax(lg[-1]))
        for i in range(2):
            e = ref.forward([tok], T0 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], T0 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
    finally:
        ctx.close()


# ---- the last positions of a 131 072-position session -------------------------------------------------------------------
FAR = 131072


def _read_bytes(ctx, which, layer, nbytes, total):
    out = np.full(total, 0xA5, np.uint8)
    L._capi.check(lib.lnb_session_read(ctx.h, which, layer, out.ctypes.data_as(C.c_void_p), nbytes))
    return out


@pytest.mark.parametrize("mode", [LNB_ACC_STRICT, LNB_ACC_FAST])
@pytest.mark.parametrize("name", ["tiny_far", "gqa8_far"])
def test_far_positions(models, name, mode):
    args, t, _, gm = models(name)
    order, hd = _order(mode), args["head_dim"]
    kvd = args["n_kv_heads"] * hd
    refs = {i: RefSession(args, t, FAR, True, order=order) for i in range(4)}
    ctx = _ctx(gm, FAR, mode=mode, n_seq=4, max_rows=31 if mode == LNB_ACC_FAST else 40)
    ctx.allow_chunked_prefill(True)
    rng = np.random.default_rng(31)
    tk = lambda k: rng.integers(0, args["vocab_size"], k).astype(np.int32)   # noqa: E731
    try:
        # sequence 0: a 40-row prompt at 131 000 (FAST: two chunks, below the tensor-core cut), then steps up to the end
        p = tk(40)
        for a, b in (((0, 40),) if mode == LNB_ACC_STRICT else ((0, 20), (20, 40))):
            assert np.array_equal(_bits(_forward(ctx, p[a:b], 131000 + a)), _bits(refs[0].forward(p[a:b], 131000 + a)))
        for pos in (131040, 131041, 131071):
            tok = int(tk(1)[0])
            assert np.array_equal(_bits(_forward(ctx, [tok], pos)), _bits(refs[0].forward([tok], pos))), pos
        # batched rows of four sequences, then a ragged call of prompt chunks and a decode row
        toks, pos = tk(4), [131042, 131000, 131035, 131070]
        _, lg = ctx.forward_batch(toks, pos, want_logits=True)
        for i in range(4):
            assert np.array_equal(_bits(lg[i]), _bits(refs[i].forward([toks[i]], pos[i])[0])), i
        segs = [(1, 131001, tk(3)), (2, 131036, tk(1)), (3, 131064, tk(5)), (0, 131043, tk(2))]
        _, lg = ctx.forward_ragged(segs, want_logits=True)
        for i, (q, p0, tt) in enumerate(segs):
            assert np.array_equal(_bits(lg[i]), _bits(refs[q].forward(tt, p0)[-1])), (q, p0)
        # lnb_session_read of whole caches (32 chunks of 4 096 rows), of a non-active sequence, and of a byte count
        # that ends inside a row; unwritten records decode to 0
        last = args["n_layers"] - 1
        for q in (0, 2):
            ctx.set_active_sequence(q)
            for layer in (0, last):
                for w, which, dec in (("k", L._capi.LNB_BUF_CACHE_K, refs[q].ck), ("v", L._capi.LNB_BUF_CACHE_V, refs[q].cv)):
                    got = (ctx.CacheK if w == "k" else ctx.CacheV)(layer).RawData.reshape(FAR, kvd)
                    assert np.array_equal(got, dec[layer]), (q, layer, w)
                    codes, scales = ctx.kv_read(q, layer, w, 0, FAR)
                    assert np.array_equal(K.decode(codes, scales, hd), got)
                    nb = (131001 * kvd + 3) * 2
                    part = _read_bytes(ctx, which, layer, nb, FAR * kvd * 2)
                    assert np.array_equal(part[:nb], dec[layer].view(np.uint8).reshape(-1)[:nb]) and (part[nb:] == 0xA5).all()
        ctx.set_active_sequence(0)
        c, s, _ = SR.kv_mxfp8_quantize(refs[3].pre_v[last][131064:131069], hd)
        codes, scales = ctx.kv_read(3, last, "v", 131064, 6)
        assert np.array_equal(codes[:5], c) and np.array_equal(scales[:5], s)
        assert not codes[5].any() and not scales[5].any()          # an unwritten record is zero
    finally:
        ctx.close()


# ---- calls that write or move rows --------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [LNB_ACC_STRICT, LNB_ACC_FAST])
def test_speculative_rows_and_the_calls_that_overwrite_them(models, mode):
    args, t, _, gm = models("tiny")
    seq = 32
    refs = {i: RefSession(args, t, seq, True, order=_order(mode)) for i in range(2)}
    ctx = _ctx(gm, seq, mode=mode, n_seq=2, max_rows=31)
    try:
        last = []
        for i, n in enumerate((7, 5)):
            ctx.set_active_sequence(i)
            p = _prompt(args, n, seed=40 + i)
            lg = _forward(ctx, p, 0)
            assert np.array_equal(_bits(lg), _bits(refs[i].forward(p, 0)))
            last.append(int(np.argmax(lg[-1])))
        peek = _clone(refs[0]).forward([last[0]], 7)
        g1 = int(np.argmax(peek[0]))
        peek = _clone(refs[0]).forward([last[0], g1], 7)
        bad0 = (int(np.argmax(peek[1])) + 1) % args["vocab_size"]
        peek = _clone(refs[1]).forward([last[1]], 5)
        bad1 = (int(np.argmax(peek[0])) + 1) % args["vocab_size"]
        d0, d1 = [last[0], g1, bad0, 17], [last[1], bad1, 23]
        nxt, acc, lg = ctx.forward_speculative([(0, 7, d0), (1, 5, d1)], want_logits=True)
        e0, e1 = refs[0].forward(d0, 7), refs[1].forward(d1, 5)    # the rejected rows stay in both caches
        assert np.array_equal(_bits(lg), _bits(np.vstack([e0, e1])))
        assert acc.tolist() == [1, 0]
        # the next calls overwrite the rejected rows from the first position after the accepted ones
        toks, pos = [int(nxt[1]), int(nxt[len(d0)])], [9, 6]
        for _ in range(2):
            nx, lg = ctx.forward_batch(toks, pos, want_logits=True)
            for i in range(2):
                assert np.array_equal(_bits(lg[i]), _bits(refs[i].forward([toks[i]], pos[i])[0])), i
            toks, pos = [int(x) for x in nx], [q + 1 for q in pos]
        _check_caches(ctx, {0: refs[0]}, args, seq, 11)           # the positions each sequence has written
        _check_caches(ctx, {1: refs[1]}, args, seq, 8)
    finally:
        ctx.close()


def test_copy_sequences_cycles_fanout_and_offsets(models):
    args, t, _, gm = models("tiny")
    seq, n = 32, 4
    refs = {i: RefSession(args, t, seq, True) for i in range(n)}
    ctx = _ctx(gm, seq, n_seq=n)
    layers = range(args["n_layers"])

    def blocks():
        return {(q, l, w): ctx.kv_read(q, l, w, 0, seq) for q in range(n) for l in layers for w in "kv"}

    def step(lens, seed):
        toks = np.random.default_rng(seed).integers(0, args["vocab_size"], n).astype(np.int32)
        _, lg = ctx.forward_batch(toks, lens, want_logits=True)
        for i in range(n):
            assert np.array_equal(_bits(lg[i]), _bits(refs[i].forward([toks[i]], lens[i])[0])), i
        return [q + 1 for q in lens]
    try:
        lens = [6, 8, 10, 12]
        for i in range(n):
            ctx.set_active_sequence(i)
            p = _prompt(args, lens[i], seed=50 + i)
            assert np.array_equal(_bits(_forward(ctx, p, 0)), _bits(refs[i].forward(p, 0)))
        ctx.set_active_sequence(0)
        # a 3-cycle of positions [5, seq): each destination keeps [0, 5) and takes its source's rows from 5 on
        src, dst, p0 = [0, 1, 2], [1, 2, 0], 5
        before = blocks()
        ctx.copy_sequences(src, dst, p0, seq)
        after = blocks()
        moved = dict(zip(dst, src))
        for (q, l, w), (c, s) in after.items():
            o = moved.get(q, q)
            bc, bs = before[(q, l, w)]
            sc, ss = before[(o, l, w)]
            assert np.array_equal(c[:p0], bc[:p0]) and np.array_equal(s[:p0], bs[:p0]), (q, l, w)
            assert np.array_equal(c[p0:], sc[p0:]) and np.array_equal(s[p0:], ss[p0:]), (q, l, w)
        new = {}
        for q in range(n):
            o = moved.get(q, q)
            r = _clone(refs[q])
            for name in ("ck", "cv", "pre_k", "pre_v"):
                for l in layers:
                    getattr(r, name)[l][p0:] = getattr(refs[o], name)[l][p0:]
            new[q] = r
        refs = new
        lens = step([lens[moved.get(q, q)] for q in range(n)], 60)
        # a fan-out of the whole window: every sequence becomes sequence 0
        ctx.copy_sequences([0, 0, 0], [1, 2, 3], 0, seq)
        after = blocks()
        for (q, l, w), (c, s) in after.items():
            c0, s0 = after[(0, l, w)]
            assert np.array_equal(c, c0) and np.array_equal(s, s0), (q, l, w)
        refs = {q: _clone(refs[0]) for q in range(n)}
        lens = step([lens[0]] * n, 61)
        _check_caches(ctx, refs, args, seq, lens[0])
    finally:
        ctx.close()


@pytest.mark.parametrize("off", [37, 129])
def test_chunked_prefill(models, off):
    args, t, _, gm = models("tiny_long")
    seq = 192
    ref = RefSession(args, t, seq, True)
    ctx = _ctx(gm, seq, max_rows=off)
    ctx.allow_chunked_prefill(True)
    try:
        p = _prompt(args, off + 24, seed=off)
        assert np.array_equal(_bits(_forward(ctx, p[:off], 0)), _bits(ref.forward(p[:off], 0)))
        assert np.array_equal(_bits(_forward(ctx, p[off:], off)), _bits(ref.forward(p[off:], off)))
        _check_caches(ctx, {0: ref}, args, seq, off + 24)
    finally:
        ctx.close()


@pytest.mark.parametrize("mode", [LNB_ACC_STRICT, LNB_ACC_FAST])
def test_score_and_logprobs(models, mode):
    args, t, _, gm = models("tiny")
    ref = RefSession(args, t, 40, True, order=_order(mode))
    ctx = _ctx(gm, 40, mode=mode, max_rows=31)
    try:
        toks = _prompt(args, 24, seed=70)
        ctx.set_logprobs(0, 7)
        recs = gm.Transformer.score(ctx, toks, 0)
        assert [r.Token for r in recs] == toks[1:].tolist()
        _same(_read(L, ctx, 0, 1, len(toks) - 1), SR.logprob_rows(ref.forward(toks[:-1], 0), toks[1:], 7), "score")
    finally:
        ctx.close()


def _greedy(args, t, prompt, seq):
    ref = RefSession(args, t, seq, True)
    tok = int(np.argmax(ref.forward(prompt, 0)[-1]))
    out = [tok]
    for pos in range(len(prompt), seq - 1):
        tok = int(np.argmax(ref.forward([tok], pos)[0]))
        out.append(tok)
    return out


def test_engine_generation(models):
    """continuous batching, speculative generation and beam search with kv_format="mxfp8" (STRICT): the greedy streams of
    the reference, and every beam's logprobs those of the reference's logits along its tokens"""
    args, t, _, gm = models("tiny")
    seq = 24
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=LNB_ACC_STRICT, max_rows=24, kv_format="mxfp8")
    prompts = [_prompt(args, n, seed=80 + n).tolist() for n in (3, 9, 5)]
    got = [[] for _ in prompts]
    for i, _, tok in eng.GenerateTokensContinuous(prompts, slots=2, step_tokens=8):
        got[i].append(tok)
    assert got == [_greedy(args, t, p, seq) for p in prompts]
    rep = [3, 14, 15, 92, 65] * 3
    spec = [tk for _, tk in eng.GenerateTokens(rep, speculative=L.inference.SpeculativeArgs(4))]
    assert spec == _greedy(args, t, rep, seq)
    hyps = eng.GenerateBeams(prompts[1], L.inference.BeamSearchArgs(2, NumReturn=2))
    assert len(hyps) == 2
    for h in hyps:
        ref = RefSession(args, t, seq, True)
        rows = [ref.forward(prompts[1], 0)[-1]]
        for i, tok in enumerate(h.Tokens[:-1]):
            rows.append(ref.forward([tok], len(prompts[1]) + i)[0])
        want = SR.logprob_rows(np.stack(rows), h.Tokens, 0)["logprob"]
        assert list(h.Logprobs) == want.tolist()


# ---- the FAST tensor-core prompt, stage by stage -------------------------------------------------------------------------
class _Stages:
    def __init__(self, args, tensors):
        self.args, self.w = args, tensors
        self.cis = O.rope_table(args["head_dim"], args["max_seq_len"], args["rope_theta"], bool(args["use_scaled_rope"]))[1]
        self.silu = O.silu_table_bf16()

    def lw(self, l, name):
        return self.w[f"layers.{l}.{name}"]


def _check_mx_layer(m, l, x_in, pr, ck, cv, start):
    """layer l of a FAST tensor-core prompt over a quantized cache: the attention probe bit for bit the stream order's
    attention over the probed q and the session's decoded caches; the other stages inside their order-free bounds"""
    a = m.args
    S, nh, hd = x_in.shape[0], a["n_heads"], a["head_dim"]
    pos = start + np.arange(S)
    xn = _norm(x_in, m.lw(l, "attention_norm.weight"))
    lo, hi = P.rope_bounds(*[v.reshape(S, nh, hd) for v in P.linear_bounds(xn, m.lw(l, "attention.wq.weight"))], m.cis, pos)
    _inside("mx q", P.within(pr["q"], lo.reshape(S, -1), hi.reshape(S, -1)), lo, hi)
    att = O.attention_order(np.ascontiguousarray(pr["q"].reshape(S, nh, hd)), ck, cv, start + S, S > 1, start, O.ORDER_FAST_STREAM[2])
    att = att.reshape(S, -1)
    assert np.array_equal(pr["attn"], att), f"attention: {(pr['attn'] != att).sum()} of {att.size} differ, first at {np.argwhere(pr['attn'] != att)[0]}"
    lo, hi = P.resid_bounds(x_in, *P.linear_bounds(pr["attn"], m.lw(l, "attention.wo.weight")))
    _inside("mx post-attention", P.within(pr["post"], lo, hi), lo, hi)
    xn2 = _norm(pr["post"], m.lw(l, "ffn_norm.weight"))
    assert np.array_equal(pr["normed"], xn2)
    slo, shi = P.swiglu_set(*P.linear_bounds(xn2, m.lw(l, "feed_forward.w1.weight")),
                            *P.linear_bounds(xn2, m.lw(l, "feed_forward.w3.weight")), m.silu)
    _inside("mx SwiGLU", P.in_set(pr["ffn"], slo, shi))
    lo, hi = P.resid_bounds(pr["post"], *P.linear_bounds(pr["ffn"], m.lw(l, "feed_forward.w2.weight")))
    _inside("mx output residual", P.within(pr["out"], lo, hi), lo, hi)


@pytest.mark.parametrize("name,S,start", [("tiny128_long", 40, 0), ("tiny128_long", 300, 0), ("tiny128_long", 2048, 0),
                                          ("tiny128_long", 40, 37), ("hd128_rep8", 40, 0), ("hd128_rep8", 300, 0),
                                          ("hd128_rep8", 40, 37)])
def test_fast_tensor_core_prompt_stage_by_stage(models, name, S, start):
    args, t, _, gm = models(name)
    m = _Stages(args, t)
    seq = max(48, start + S)
    nl, kvs = args["n_layers"], (args["n_kv_heads"], args["head_dim"])
    toks = np.random.default_rng(S * 7 + start).integers(0, args["vocab_size"], size=start + S).astype(np.int32)
    ctx = _ctx(gm, seq, mode=LNB_ACC_FAST, max_rows=max(S, start, 32))
    ctx.allow_chunked_prefill(True)
    try:
        if start:
            gm.Transformer.forward_argmax(ctx, toks[:start], 0)
        chunk = toks[start:]
        x_in = t["tok_embeddings.weight"][chunk]
        for l in range(nl):
            ctx.set_layer_limit(l + 1)
            gm.Transformer.forward_argmax(ctx, chunk, start, want_logits="last")
            pr = _probes(ctx, S)
            ck = ctx.CacheK(l).RawData.reshape(seq, *kvs)
            cv = ctx.CacheV(l).RawData.reshape(seq, *kvs)
            _check_mx_layer(m, l, x_in, pr, ck, cv, start)
            x_in = pr["out"]
        ctx.set_layer_limit(0)
        _, lg = gm.Transformer.forward_argmax(ctx, chunk, start, want_logits="all")
        xo = _norm(ctx.residual(S), t["norm.weight"])
        rows = sorted({0, 1, min(127, S - 2), min(128, S - 2), S - 2, S - 1})
        lo, hi = P.linear_bounds(xo[rows], t["output.weight"])
        _inside("mx logits", P.within_values(lg[rows], lo, hi), lo, hi)
    finally:
        ctx.close()


# ---- 8B: the attention at position 131 000 ---------------------------------------------------------------------------------
def test_8b_attention_at_the_end_of_the_window():
    """four sequences of an 8B session of 131 072 positions step at 131 000 with layer limit 1: each row's attention probe
    is the stream order's attention over its probed q and its sequence's decoded layer-0 caches"""
    import torch
    if torch.cuda.mem_get_info()[1] < (79 << 30):
        pytest.skip("sized for an 80 GB card")
    args = dict(L.synth.LLAMA31_8B, max_seq_len=FAR)
    gm = L.model.LoadSyntheticModel(args)
    try:
        ctx = _ctx(gm, FAR, mode=LNB_ACC_FAST, n_seq=4, max_rows=4)
        try:
            ctx.set_layer_limit(1)
            ctx.forward_batch([1, 2, 3, 4], [131000] * 4)
            q, att = ctx.stage("q", 4), ctx.stage("attn", 4)
            nh, hd = args["n_heads"], args["head_dim"]
            for i in (0, 3):
                ctx.set_active_sequence(i)
                ck, cv = ctx.CacheK(0).RawData, ctx.CacheV(0).RawData
                assert ck[131000].any() and not ck[131001:].any()
                e = O.attention_order(np.ascontiguousarray(q[i].reshape(1, nh, hd)), ck, cv, 131001, False, 131000,
                                      O.ORDER_FAST_STREAM[2])
                assert np.array_equal(att[i], e.reshape(-1)), i
        finally:
            ctx.close()
    finally:
        gm.Free()
