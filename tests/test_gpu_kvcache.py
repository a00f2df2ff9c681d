"""The MXFP8 KV cache on the GPU (DESIGN.md §9j): the cache writer's block rule against the C statement, STRICT calls bit
for bit against the reference forward whose stored K and V rows are replaced by their decoded blocks (RefSession of
tests/test_kvcache_cpu.py), the raw blocks, forks, routing, refusals and launch counts."""
import ctypes as C

import numpy as np
import pytest

import lnb_b200 as L
from lnb_b200._capi import LNB_ACC_FAST, LNB_ACC_STRICT, LnbError, lib, ptr
from oracle import oracle as O
from oracle_sampling import sample_ref as SR
from tests.helpers import host_tensors
from tests.model_shapes import CATALOGUE
from tests.test_kvcache_cpu import HEAD_DIMS, RefSession, case_rows, non_finite_rows

pytestmark = pytest.mark.gpu

SHAPES = {"tiny": dict(L.synth.TINY), "tiny128": dict(L.synth.TINY128),
          **{k: CATALOGUE[k] for k in ("mha", "gqa3", "gqa8", "hd96", "stories")}}


@pytest.fixture(scope="module")
def models():
    made = {}

    def get(name, weight_format="bf16"):
        key = (name, weight_format)
        if key not in made:
            args = dict(SHAPES[name])
            tensors = host_tensors(args, 23)
            gm = L.model.LoadModelFromTensors(args, tensors, weight_format=weight_format)
            if weight_format != "bf16":   # the reference runs on the dequantized weights D(W)
                tensors = dict(tensors)
                for n in tensors:
                    if n.startswith("layers.") and n.endswith(".weight") and "norm" not in n or n == "output.weight":
                        rd = gm.Transformer.mxfp8_read if weight_format == "mxfp8" else gm.Transformer.mxfp4_read
                        c, s = rd(n)
                        tensors[n] = (SR.mxfp8_dequantize(c, s) if weight_format == "mxfp8" else SR.mxfp4_dequantize(c, s))
            made[key] = (args, tensors, gm)
        return made[key]

    yield get
    for _, _, gm in made.values():
        gm.Free()


def _ctx(gm, seq_len, mode=LNB_ACC_STRICT, n_seq=1, max_rows=64, kv="mxfp8"):
    return L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq_len), acc_mode=mode, n_seq=n_seq,
                                    max_rows=max_rows, kv_format=kv)


def _forward(ctx, toks, pos):
    toks = np.ascontiguousarray(toks, np.int32)
    lg = np.empty((len(toks), ctx.transformer.args.VocabSize), np.float32)
    nxt = np.zeros(1, np.int32)
    L._capi.check(lib.lnb_forward(ctx.h, ptr(toks, L._capi.i32p), len(toks), pos, ptr(lg, L._capi.f32p), 1, ptr(nxt, L._capi.i32p)))
    return lg


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _prompt(args, n, seed=3):
    return np.random.default_rng(seed).integers(0, args["vocab_size"], n).astype(np.int32)


# ---- op level --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_device_quantizer_equals_statement(hd):
    for rows in (case_rows(hd), non_finite_rows(hd)):
        n, kv = rows.shape
        nb = (hd + 31) // 32
        codes = np.empty((n, kv), np.uint8)
        scales = np.empty((n, kv // hd, nb), np.uint8)
        deq = np.empty((n, kv), np.uint16)
        L._capi.check(lib.lnb_op_kv_quantize_bf16(ptr(rows, L._capi.u16p), n, hd, kv // hd, codes.ctypes.data_as(C.c_void_p),
                                                  scales.ctypes.data_as(C.c_void_p), ptr(deq, L._capi.u16p)))
        c, s, d = SR.kv_mxfp8_quantize(rows, hd)
        assert np.array_equal(scales, s)
        assert np.array_equal(codes, c), np.argwhere(codes != c)[:8]
        assert np.array_equal(deq, d)


# ---- STRICT, bit for bit ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("plen", [1, 7, 40])
def test_strict_prompt_steps_and_caches(models, name, plen):
    args, tensors, gm = models(name)
    seq = 48
    ref = RefSession(args, tensors, seq, True)
    ctx = _ctx(gm, seq)
    try:
        p = _prompt(args, plen)
        assert np.array_equal(_bits(_forward(ctx, p, 0)), _bits(ref.forward(p, 0)))
        tok, pos = int(p[-1]), plen
        for _ in range(3):                                  # host-driven steps: each row reads the row it just wrote
            lg = ref.forward([tok], pos)
            assert np.array_equal(_bits(_forward(ctx, [tok], pos)), _bits(lg))
            tok, pos = int(np.argmax(lg[0])), pos + 1
        kvd = args["n_kv_heads"] * args["head_dim"]
        for layer in (0, args["n_layers"] - 1):
            assert np.array_equal(ctx.CacheK(layer).RawData.reshape(seq, kvd), ref.ck[layer])
            assert np.array_equal(ctx.CacheV(layer).RawData.reshape(seq, kvd), ref.cv[layer])
            for w, pre in (("k", ref.pre_k[layer]), ("v", ref.pre_v[layer])):   # the raw blocks of the pre-quantization rows
                codes, scales = ctx.kv_read(0, layer, w, 0, pos)
                c, s, _ = SR.kv_mxfp8_quantize(pre[:pos], args["head_dim"])
                assert np.array_equal(codes, c) and np.array_equal(scales, s)
    finally:
        ctx.close()


@pytest.mark.parametrize("weights", ["bf16", "mxfp8", "mxfp4"])
@pytest.mark.parametrize("graph", [False, True])
def test_strict_decode_run(models, weights, graph):
    args, tensors, gm = models("tiny", weights)
    ref = RefSession(args, tensors, 40, True)
    ctx = _ctx(gm, 40)
    try:
        p = _prompt(args, 9, seed=4)
        lg = _forward(ctx, p, 0)
        assert np.array_equal(_bits(lg), _bits(ref.forward(p, 0)))
        first = int(np.argmax(lg[-1]))
        toks, _, _ = ctx.decode_run(first, 9, 12, use_graph=graph)
        exp, tok = [], first
        for i in range(12):
            tok = int(np.argmax(ref.forward([tok], 9 + i)[0]))
            exp.append(tok)
        assert toks.tolist() == exp
    finally:
        ctx.close()


@pytest.mark.parametrize("n_seq", [3, 8])
def test_strict_batched_steps_and_forks(models, n_seq):
    args, tensors, gm = models("tiny")
    seq = 32
    refs = [RefSession(args, tensors, seq, True) for _ in range(n_seq)]
    ctx = _ctx(gm, seq, n_seq=n_seq)
    try:
        lens = [3 + 2 * i for i in range(n_seq)]
        toks = []
        for i in range(n_seq):
            ctx.set_active_sequence(i)
            p = _prompt(args, lens[i], seed=10 + i)
            lg = _forward(ctx, p, 0)
            assert np.array_equal(_bits(lg), _bits(refs[i].forward(p, 0)))
            toks.append(int(np.argmax(lg[-1])))
        pos = list(lens)
        for _ in range(3):
            nxt, lg = ctx.forward_batch(toks, pos, want_logits=True)
            for i in range(n_seq):
                e = refs[i].forward([toks[i]], pos[i])
                assert np.array_equal(_bits(lg[i]), _bits(e[0])), i
            toks, pos = [int(t) for t in nxt], [q + 1 for q in pos]
        # a fork copies the blocks bit for bit; the forked sequence then steps exactly like its source's reference
        ctx.copy_sequences([0], [1], 0, pos[0])
        for layer in range(args["n_layers"]):
            for w in ("k", "v"):
                assert all(np.array_equal(a, b) for a, b in zip(ctx.kv_read(0, layer, w, 0, pos[0]), ctx.kv_read(1, layer, w, 0, pos[0])))
        ctx.set_active_sequence(1)
        assert np.array_equal(_bits(_forward(ctx, [toks[0]], pos[0])), _bits(refs[0].forward([toks[0]], pos[0])))
    finally:
        ctx.close()


# ---- FAST, bit for bit against the stream order ---------------------------------------------------------------------
def _own_caches(ctx, args, seq):
    kvd = args["n_kv_heads"] * args["head_dim"]
    ck = [ctx.CacheK(l).RawData.reshape(seq, kvd) for l in range(args["n_layers"])]
    cv = [ctx.CacheV(l).RawData.reshape(seq, kvd) for l in range(args["n_layers"])]
    return ck, cv


@pytest.mark.parametrize("name", ["tiny", "gqa8", "hd96"])
def test_fast_chain_equals_the_stream_order(models, name):
    """FAST prompts below the tensor-core cut (max_rows 31: the kernel chain) and steps, bit for bit against the oracle ops
    in ORDER_FAST_STREAM with every stored row replaced by its decoded blocks"""
    args, tensors, gm = models(name)
    ref = RefSession(args, tensors, 48, True, order=O.ORDER_FAST_STREAM)
    ctx = _ctx(gm, 48, mode=LNB_ACC_FAST, max_rows=31)
    try:
        p = _prompt(args, 7, seed=6)
        assert np.array_equal(_bits(_forward(ctx, p, 0)), _bits(ref.forward(p, 0)))
        tok = int(p[-1])
        for i in range(4):
            e = ref.forward([tok], 7 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], 7 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
        ck, cv = _own_caches(ctx, args, 48)
        assert np.array_equal(ck[0], ref.ck[0]) and np.array_equal(cv[-1], ref.cv[-1])
    finally:
        ctx.close()


@pytest.mark.parametrize("name", ["tiny", "tiny128"])
def test_fast_tensor_core_prompt_then_steps_bit_for_bit(models, name):
    """a 40-row FAST prompt (projections on the tensor cores, attention streamed); its logits near the stream-order
    reference; then, from the session's own decoded caches, steps bit for bit against the stream order"""
    args, tensors, gm = models(name)
    seq = 48
    ref = RefSession(args, tensors, seq, True, order=O.ORDER_FAST_STREAM)
    ctx = _ctx(gm, seq, mode=LNB_ACC_FAST)
    try:
        p = _prompt(args, 40, seed=6)
        lg, e = _forward(ctx, p, 0), ref.forward(p, 0)
        assert np.isfinite(lg).all() and float(np.abs(lg - e).max()) <= 5e-2
        ref.load_caches(*_own_caches(ctx, args, seq), 40)
        tok = int(np.argmax(lg[-1]))
        for i in range(4):
            e = ref.forward([tok], 40 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], 40 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
    finally:
        ctx.close()


# ---- long caches: many K tiles (128 keys), both V stages (256 keys), several FAST chunks (1024 keys) --------------------
LONG = {"tiny_long": dict(L.synth.TINY, max_seq_len=4096), "gqa8_long": dict(CATALOGUE["gqa8"], max_seq_len=4096)}
SHAPES.update(LONG)


@pytest.mark.parametrize("name", list(LONG))
@pytest.mark.parametrize("T0", [300, 2500])
def test_long_cache_strict_and_fast(models, name, T0):
    args, tensors, gm = models(name)
    seq = T0 + 8
    p = _prompt(args, T0, seed=8)
    # STRICT: the whole prompt and two steps, bit for bit
    ref = RefSession(args, tensors, seq, True)
    ctx = _ctx(gm, seq, max_rows=T0)
    try:
        lg, e = _forward(ctx, p, 0), ref.forward(p, 0)
        assert np.array_equal(_bits(lg), _bits(e))
        tok = int(np.argmax(e[-1]))
        for i in range(2):
            e = ref.forward([tok], T0 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], T0 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
    finally:
        ctx.close()
    # FAST: the prompt on the tensor cores, then three steps over every chunk of the session's own caches, bit for bit
    ref = RefSession(args, tensors, seq, True, order=O.ORDER_FAST_STREAM)
    ctx = _ctx(gm, seq, mode=LNB_ACC_FAST, max_rows=T0)
    try:
        lg = _forward(ctx, p, 0)
        ref.load_caches(*_own_caches(ctx, args, seq), T0)
        tok = int(np.argmax(lg[-1]))
        for i in range(3):
            e = ref.forward([tok], T0 + i)
            assert np.array_equal(_bits(_forward(ctx, [tok], T0 + i)), _bits(e)), i
            tok = int(np.argmax(e[0]))
    finally:
        ctx.close()


# ---- ragged calls -----------------------------------------------------------------------------------------------------
def test_strict_ragged_calls(models):
    """prompts, a prompt chunk and decode rows of three sequences in one forward: each segment's last-row logits"""
    args, tensors, gm = models("tiny")
    seq = 48
    rng = np.random.default_rng(24)
    t = lambda k: rng.integers(0, args["vocab_size"], size=k).astype(np.int32)   # noqa: E731
    refs = [RefSession(args, tensors, seq, True) for _ in range(3)]
    ctx = _ctx(gm, seq, n_seq=3)
    pos, last = [0, 0, 0], {}
    try:
        for call in [[(0, t(7)), (1, t(5))], [(0, None), (1, t(3)), (2, t(9))], [(0, None), (1, None), (2, t(2))]]:
            segs = [(q, pos[q], np.array([last[q]], np.int32) if tk is None else tk) for q, tk in call]
            nxt, lg = ctx.forward_ragged(segs, want_logits=True)
            for i, (q, p0, tk) in enumerate(segs):
                e = refs[q].forward(tk, p0)[-1]
                assert np.array_equal(_bits(lg[i]), _bits(e)), (q, p0)
                pos[q] += len(tk); last[q] = int(nxt[i])
        for q in range(3):
            ctx.set_active_sequence(q)
            assert np.array_equal(ctx.CacheK(1).RawData.reshape(seq, -1), refs[q].ck[1])
    finally:
        ctx.close()


# ---- routing and refusals ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine_env", [None, "1"])
def test_engines_refuse_and_session_stays_usable(models, monkeypatch, engine_env):
    if engine_env:
        monkeypatch.setenv("LNB_ENGINE", engine_env)
    args, tensors, gm = models("tiny")
    ctx = _ctx(gm, 32, n_seq=2)
    try:
        assert lib.lnb_session_decode_engine(ctx.h) == 0
        assert b"MXFP8 KV cache" in lib.lnb_last_error()
        ctx.set_active_sequence(0)
        ref = RefSession(args, tensors, 32, True)
        p = _prompt(args, 5)
        assert np.array_equal(_bits(_forward(ctx, p, 0)), _bits(ref.forward(p, 0)))
        fmt, nbytes = ctx.kv_info()
        rowb = args["n_kv_heads"] * args["head_dim"] + ((4 * args["n_kv_heads"] + 15) // 16) * 16
        assert fmt == "mxfp8" and nbytes == 2 * args["n_layers"] * 2 * 32 * rowb
    finally:
        ctx.close()


def test_refusals_allocate_nothing(models):
    import torch
    args, _, gm = models("tiny")
    h = C.c_void_p()
    shaped = {n: L.model.LoadModelFromTensors(dict(CATALOGUE[n]), host_tensors(dict(CATALOGUE[n]), 2)) for n in ("hd256", "rep16")}
    try:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        assert lib.lnb_session_create_kv(gm.Transformer.h, 32, 1, 8, LNB_ACC_STRICT, 7, C.byref(h)) == -1
        assert b"unknown KV cache format" in lib.lnb_last_error()
        for m in shaped.values():
            assert lib.lnb_session_create_kv(m.Transformer.h, 64, 1, 8, LNB_ACC_STRICT, 1, C.byref(h)) == -1
            assert b"streamed kernels" in lib.lnb_last_error()
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0 and not h.value
        for m in shaped.values():
            with pytest.raises(LnbError):
                L.model.InferenceContext(m.Transformer, L.model.InferenceArgs(64), kv_format="mxfp8")
    finally:
        for m in shaped.values():
            m.Free()
    with pytest.raises(ValueError):
        L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(32), kv_format="fp8")


def test_bf16_create_kv_is_the_plain_session(models):
    args, tensors, gm = models("tiny")
    a, b = _ctx(gm, 32, kv="bf16"), _ctx(gm, 32, kv="bf16", n_seq=3)
    c = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(32), acc_mode=LNB_ACC_STRICT, max_rows=64)
    try:
        p = _prompt(args, 6)
        assert np.array_equal(_bits(_forward(a, p, 0)), _bits(_forward(c, p, 0)))
        assert a.kv_info() == ("bf16", 2 * 2 * 32 * 64 * 2) and b.kv_info()[1] == 3 * a.kv_info()[1]
    finally:
        a.close(); b.close(); c.close()


def test_step_launches_one_writer_per_layer_more_than_the_streamed_route(models, monkeypatch):
    """a batched step of a session whose caches the shared-memory decode kernel cannot hold streams its attention in
    both formats: the MXFP8 step launches exactly one more kernel (the cache writer) per layer"""
    monkeypatch.setenv("LNB_ENGINE", "0")
    args, _, gm = models("tiny_long")
    counts = []
    for kv in ("bf16", "mxfp8"):
        ctx = _ctx(gm, 2048, kv=kv, n_seq=2)
        try:
            ctx.forward_batch([3, 4], [0, 0])
            n0 = ctx.launch_count()
            ctx.forward_batch([5, 6], [1, 1])
            counts.append(ctx.launch_count() - n0)
        finally:
            ctx.close()
    assert counts[1] - counts[0] == args["n_layers"], counts


# ---- 8B: capacity and long-context steps -------------------------------------------------------------------------------
def test_8b_mxfp8_cache_fits_sequences_bf16_refuses():
    """n_seq x 131 072 positions that a bf16 cache cannot hold next to the 8B weights (LNB_ENOMEM), created with the
    MXFP8 cache, run batched steps near the end of the window"""
    import torch
    if torch.cuda.mem_get_info()[1] < (79 << 30):
        pytest.skip("sized for an 80 GB card")
    args = dict(L.synth.LLAMA31_8B, max_seq_len=131072)
    gm = L.model.LoadSyntheticModel(args)
    try:
        h = C.c_void_p()
        assert lib.lnb_session_create_kv(gm.Transformer.h, 131072, 4, 4, LNB_ACC_FAST, 0, C.byref(h)) == -5   # LNB_ENOMEM
        ctx = _ctx(gm, 131072, mode=LNB_ACC_FAST, n_seq=4, max_rows=4)
        try:
            assert ctx.kv_info() == ("mxfp8", 2 * 32 * 4 * 131072 * 1056)
            for i in range(3):
                nxt, lg = ctx.forward_batch([1, 2, 3, 4], [131000 + i] * 4, want_logits=True)
                assert np.isfinite(lg).all() and ((0 <= nxt) & (nxt < args["vocab_size"])).all()
        finally:
            ctx.close()
    finally:
        gm.Free()
