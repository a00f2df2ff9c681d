"""MXFP8 linear weights on the GPU (DESIGN.md §9h).  The quantizer against the C statement (orc_mxfp8_quantize), bit for
bit; then the identity the format promises: an MXFP8 model returns the bits of the bf16 model D(W) whose linear weights
are the dequantized values (orc_mxfp8_dequantize) on every route -- prompts on the FMA pipes and on the tensor cores,
host-driven and device-resident decode, batched, ragged, speculative and chunked calls, streamed attention and the
generate loops -- in STRICT and FAST; STRICT against the CPU oracle of D(W); and the routing: the engines and the packed
stream refuse MXFP8 and say why."""
import ctypes
import os

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import engine_shapes as ES
from tests import model_shapes as MS
from tests import mx_cases as MC
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

PROMPT = [1, 50, 999, 7, 300, 12, 64, 2]
NO_STOP = (10**9,)
SEED = 2718
LAYER_LINEAR = ("attention.wq.weight", "attention.wk.weight", "attention.wv.weight", "attention.wo.weight",
                "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight")


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def linear_names(args):
    return [f"layers.{l}.{n}" for l in range(args["n_layers"]) for n in LAYER_LINEAR] + ["output.weight"]


def dequantized(args, tensors):
    """D(W): the checkpoint with every linear weight replaced by its dequantized MXFP8 value (the C statement)"""
    out = dict(tensors)
    for name in linear_names(args):
        codes, scales = SR.mxfp8_quantize(tensors[name])
        out[name] = SR.mxfp8_dequantize(codes, scales)
    return out


class Pair:
    """an MXFP8 model and the bf16 model of its D(W), from one synthetic checkpoint"""

    def __init__(self, L, args, tensors=None):
        self.args = args
        self.tensors = host_tensors(args, SEED) if tensors is None else tensors
        self.dw_tensors = dequantized(args, self.tensors)
        self.mx = L.model.LoadModelFromTensors(args, self.tensors, weight_format="mxfp8")
        self.dw = L.model.LoadModelFromTensors(args, self.dw_tensors)

    def close(self):
        self.mx.Free()
        self.dw.Free()


def _pair(L, args):
    p = Pair(L, args)
    yield p
    p.close()


@pytest.fixture(scope="module")
def tiny(L):
    yield from _pair(L, dict(L.synth.TINY))


@pytest.fixture(scope="module")
def tiny128(L):
    yield from _pair(L, dict(L.synth.TINY128))


@pytest.fixture(scope="module")
def wide(L):
    import torch
    yield from _pair(L, ES.wide_args(torch.cuda.get_device_properties(0).multi_processor_count))   # w2: K % 32 == 16


@pytest.fixture(scope="module")
def tail16(L):
    # ffn_dim % 32 == 16: w2's last block of every row is 16 wide; w1|w3 hold 33 blocks of 16 rows
    yield from _pair(L, dict(MS.CATALOGUE["one_layer"], ffn_dim=528))


@pytest.fixture(scope="module")
def tiny128_8k(L):
    # prompts past one 128-row tile: the layer GEMMs span several M tiles, and the LM head runs in 2048-row slices
    yield from _pair(L, dict(L.synth.TINY128, vocab_size=8192))


def case_args(L, model):
    """the shapes whose every linear matrix is built from tests/mx_cases.py"""
    import torch
    if model == "wide":
        return ES.wide_args(torch.cuda.get_device_properties(0).multi_processor_count)
    if model == "tail16":
        return dict(MS.CATALOGUE["one_layer"], ffn_dim=528)
    return dict(L.synth.TINY if model == "tiny" else L.synth.TINY128)


def check_case_matrices(L, fmt, args):
    """a model whose every linear matrix is built from the format's edge and tie blocks: the device quantizer's codes and
    scales against the C statement.  No forward runs: these weights make no meaningful activations."""
    tensors = host_tensors(args, SEED)
    names = linear_names(args)
    for i, name in enumerate(names):
        tensors[name] = MC.matrix(fmt, *tensors[name].shape, shift=7 * i)
    m = L.model.LoadModelFromTensors(args, tensors, weight_format=fmt)
    try:
        for name in names:
            codes, scales = getattr(m.Transformer, f"{fmt}_read")(name)
            want_c, want_s = (SR.mxfp8_quantize if fmt == "mxfp8" else SR.mxfp4_quantize)(tensors[name])
            assert np.array_equal(scales, want_s), (name, np.argwhere(scales != want_s)[:4])
            assert np.array_equal(codes, want_c), (name, np.argwhere(codes != want_c)[:4])
    finally:
        m.Free()


def check_extreme_head(L, p):
    """the MX and D(W) models of mx_cases.extreme_head, bit for bit: host-driven decode steps (the 1-row LM-head configs),
    a ragged call of 8 segments and batched steps of 2 and 8 rows, and a 40-row prompt whose FAST LM head runs as
    dequantized tensor-core slices; STRICT prompt logits also against the oracle of D(W)"""
    om = oracle_model(p.args, p.dw_tensors)
    try:
        toks = np.random.default_rng(5).integers(0, p.args["vocab_size"], 40).astype(np.int32)
        for mode in ("strict", "fast"):
            acc = _acc(L, mode)
            a, b = _ctx(L, p.mx, 64, acc), _ctx(L, p.dw, 64, acc, engine=False)
            try:
                ta, la = _steps(p.mx, a, 6)
                tb, lb = _steps(p.dw, b, 6)
                assert ta == tb and np.array_equal(la, lb), mode
                assert np.isfinite(la).all() and (np.abs(la[:, 0::MC.HEAD_CLASSES]) > 2.0 ** 90).mean() > 0.9, mode
            finally:
                a.close(); b.close()
            res = []
            for m in (p.mx, p.dw):
                ctx = _ctx(L, m, 64, acc, n_seq=8, max_rows=40, engine=False if m is p.dw else None)
                try:
                    n1, l1 = ctx.forward_ragged([(s, 0, PROMPT[:2 + s % 6]) for s in range(8)], want_logits=True)
                    n2, l2 = ctx.forward_batch([int(t) for t in n1[:2]], [2, 3], want_logits=True)
                    n3, l3 = ctx.forward_batch([int(t) for t in n1], [2 + s % 6 + (s < 2) for s in range(8)], want_logits=True)
                    res.append((n1, l1, n2, l2, n3, l3))
                finally:
                    ctx.close()
            for i, (x, y) in enumerate(zip(*res)):
                assert np.array_equal(np.asarray(x), np.asarray(y)), (mode, i)
            a, b = _ctx(L, p.mx, 64, acc, max_rows=40), _ctx(L, p.dw, 64, acc, max_rows=40, engine=False)
            try:
                la0, lb0 = a.launch_count(), b.launch_count()
                ga = p.mx.Transformer.forward_argmax(a, toks, 0, want_logits="all")
                gb = p.dw.Transformer.forward_argmax(b, toks, 0, want_logits="all")
                assert ga[0] == gb[0] and np.array_equal(ga[1], gb[1]), mode
                assert np.isfinite(ga[1]).all()
                extra = _tc_extra(p.args, 40, mode == "strict", 40)
                assert (a.launch_count() - la0) - (b.launch_count() - lb0) == extra, mode
                if mode == "fast":
                    assert extra - 4 * p.args["n_layers"] == 2 * (p.args["vocab_size"] // 2048) - 1, "the LM head did not run in slices"
                else:
                    os_ = om.new_session(64)
                    try:
                        assert np.array_equal(os_.forward(toks, 0), ga[1])
                    finally:
                        os_.close()
            finally:
                a.close(); b.close()
    finally:
        om.close()


def _acc(L, mode):
    return L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST


def _ctx(L, m, seq, acc, n_seq=1, max_rows=8, engine=None):
    old = os.environ.get("LNB_ENGINE")
    if engine is not None:
        os.environ["LNB_ENGINE"] = "1" if engine else "0"
    try:
        ctx = L.model.InferenceContext(m.Transformer, L.model.InferenceArgs(seq), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)
        ctx.uses_engine()   # probe while LNB_ENGINE is set
    finally:
        if old is None:
            os.environ.pop("LNB_ENGINE", None)
        else:
            os.environ["LNB_ENGINE"] = old
    return ctx


def _caches_equal(args, a, b, n, seqs=(0,)):
    for s in seqs:
        for ctx in (a, b):
            if ctx.n_seq > 1:
                ctx.set_active_sequence(s)
        for layer in range(args["n_layers"]):
            for rd in ("CacheK", "CacheV"):
                assert np.array_equal(getattr(a, rd)(layer).RawData[:n], getattr(b, rd)(layer).RawData[:n]), (s, layer, rd)


# ---- quantizer ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny", "tiny128", "wide", "tail16"])
def test_quantizer_equals_the_c_statement(L, request, model):
    p = request.getfixturevalue(model)
    for name in linear_names(p.args):
        codes, scales = p.mx.Transformer.mxfp8_read(name)
        want_c, want_s = SR.mxfp8_quantize(p.tensors[name])
        assert np.array_equal(scales, want_s), name
        assert np.array_equal(codes, want_c), name


@pytest.mark.parametrize("model", ["tiny", "tiny128", "wide", "tail16"])
def test_quantizer_on_edge_and_tie_matrices(L, model):
    check_case_matrices(L, "mxfp8", case_args(L, model))


@pytest.mark.parametrize("vocab", [4096, 8192, 16384])
def test_decoders_at_extreme_scales_through_the_lm_head(L, vocab):
    args = dict(L.synth.TINY128, vocab_size=vocab)
    p = Pair(L, args, MC.extreme_head("mxfp8", host_tensors(args, SEED)))
    try:
        check_extreme_head(L, p)
    finally:
        p.close()


@pytest.mark.parametrize("name,row,col,bits", [("layers.1.feed_forward.w3.weight", 5, 17, 0x7F80),
                                               ("layers.0.attention.wk.weight", 40, 3, 0xFFC0),
                                               ("output.weight", 1000, 255, 0xFF80)])
def test_non_finite_weight_fails_finalize_with_its_index(L, name, row, col, bits):
    args = dict(L.synth.TINY)
    tensors = host_tensors(args, SEED)
    tensors[name] = tensors[name].copy()
    tensors[name][row, col] = bits
    m = L.model.Model(L.model.ModelArgs.from_c_dict(args), weight_format="mxfp8")
    try:
        for k, v in tensors.items():
            m.Transformer.upload_tensor(k, v)
        with pytest.raises(L._capi.LnbError, match=f'"{name}" has a non-finite weight at row {row}, column {col}') as e:
            m.Transformer.finalize()
        assert e.value.code == -1
    finally:
        m.Free()


# ---- identity: prompts ----------------------------------------------------------------------------------------------------
def _tc_extra(args, S, strict, max_rows):
    """the launches an MX prompt adds on the tensor-core route: one dequantization per GEMM, and an LM head in n row slices
    runs n dequantizations and n GEMMs where the bf16 model runs one GEMM"""
    if not MS.forward_tc(args, S, strict, max_rows):
        return 0
    w = MS.widths(args)
    d, q, kv, f, v = args["dim"], w["q_l"], w["kv_l"], w["ffn_l"], w["vocab_l"]
    elems = max((q + 2 * kv) * d, d * q, 2 * f * d, d * f, 128 * d)
    slice_rows = min(v, elems // d // 128 * 128)
    slices = -(-v // slice_rows) if v % 128 == 0 and S > 1 else 0
    return 4 * args["n_layers"] + max(2 * slices - 1, 0)


@pytest.mark.parametrize("model", ["tiny", "tiny128", "wide", "tail16", "tiny128_8k"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_prompt_logits_and_caches(L, request, model, mode):
    p = request.getfixturevalue(model)
    # tiny128_8k: prompts past one 128-row tile (S = 129: two M tiles in the layer GEMMs, one full tile in the LM head;
    # 130 and 300: an LM head of 129 and 299 rows, two and three tiles, in 2048-row slices), each followed by decode steps
    sizes, rows = ((129, 130, 300), 300) if model == "tiny128_8k" else ((1, 7, 40), 40)
    acc, seq = _acc(L, mode), max(64, rows + 8)
    rng = np.random.default_rng(3)
    for S in sizes:
        toks = rng.integers(0, p.args["vocab_size"], S).astype(np.int32)
        # the bf16 session on the kernel chain too, so that launch counts compare (the engine's bits are the chain's)
        a, b = _ctx(L, p.mx, seq, acc, max_rows=rows), _ctx(L, p.dw, seq, acc, max_rows=rows, engine=False)
        try:
            la, lb = a.launch_count(), b.launch_count()
            ga = p.mx.Transformer.Forward(a, L.ml.Tensor(toks, L.ml.DT_INT32), 0).RawData
            gb = p.dw.Transformer.Forward(b, L.ml.Tensor(toks, L.ml.DT_INT32), 0).RawData
            assert np.array_equal(ga, gb), (S, np.abs(ga - gb).max())
            _caches_equal(p.args, a, b, S)
            extra = _tc_extra(p.args, S, mode == "strict", rows)
            assert (a.launch_count() - la) - (b.launch_count() - lb) == extra, S
            if model.startswith("tiny128") and mode == "fast" and S >= 40:
                assert extra > 0, "the tensor-core route was not taken"
            if model == "tiny128_8k":
                t = int(np.argmax(ga[-1]))
                for j in range(3):
                    ta, da = p.mx.Transformer.forward_argmax(a, np.array([t], np.int32), S + j, want_logits="last")
                    tb, db = p.dw.Transformer.forward_argmax(b, np.array([t], np.int32), S + j, want_logits="last")
                    assert ta == tb and np.array_equal(da, db), (S, j)
                    t = ta
                _caches_equal(p.args, a, b, S + 3)
        finally:
            a.close(); b.close()


def test_chunked_prefill(L, tiny128):
    """the second plan's last chunk runs 263 rows from position 37: its GEMMs and its sliced LM head cross the 128-row tile
    edges at an offset.  Each plan ends with a decode step."""
    p = tiny128
    for chunks in (((0, 5), (5, 38), (38, 45)), ((0, 5), (5, 37), (37, 300))):
        end, rows = chunks[-1][1], max(s1 - s0 for s0, s1 in chunks)
        for mode in ("strict", "fast"):
            a, b = _ctx(L, p.mx, end + 8, _acc(L, mode), max_rows=rows), _ctx(L, p.dw, end + 8, _acc(L, mode), max_rows=rows)
            try:
                out = []
                for ctx, m in ((a, p.mx), (b, p.dw)):
                    ctx.allow_chunked_prefill()
                    toks = np.arange(3, 3 + end, dtype=np.int32)
                    lg = []
                    for s0, s1 in chunks:
                        lg.append(m.Transformer.Forward(ctx, L.ml.Tensor(toks[s0:s1], L.ml.DT_INT32), s0).RawData)
                    nxt = np.array([int(np.argmax(lg[-1][-1]))], np.int32)
                    t, d = m.Transformer.forward_argmax(ctx, nxt, end, want_logits="last")
                    out.append((np.concatenate(lg), t, d))
                assert np.array_equal(out[0][0], out[1][0]), (chunks, mode)
                assert out[0][1] == out[1][1] and np.array_equal(out[0][2], out[1][2]), (chunks, mode)
                _caches_equal(p.args, a, b, end + 1)
            finally:
                a.close(); b.close()


# ---- identity: decode ---------------------------------------------------------------------------------------------------
def _steps(m, ctx, n):
    t, _ = m.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
    toks, logits = [t], []
    for j in range(n):
        t, lg = m.Transformer.forward_argmax(ctx, np.array([toks[-1]], np.int32), len(PROMPT) + j, want_logits="last")
        toks.append(t)
        logits.append(lg[0])
    return toks, np.array(logits)


@pytest.mark.parametrize("model", ["tiny", "tiny128", "wide"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_decode_host_driven_and_device_resident(L, request, model, mode):
    p = request.getfixturevalue(model)
    acc, seq, n = _acc(L, mode), 48, 24
    a, b = _ctx(L, p.mx, seq, acc), _ctx(L, p.dw, seq, acc)
    try:
        ta, la = _steps(p.mx, a, n)
        tb, lb = _steps(p.dw, b, n)
        assert ta == tb
        assert np.array_equal(la, lb)
        _caches_equal(p.args, a, b, len(PROMPT) + n)
    finally:
        a.close(); b.close()
    for use_graph in (False, True):
        got = []
        for m in (p.mx, p.dw):
            ctx = _ctx(L, m, seq, acc, engine=False if m is p.dw else None)
            first, _ = m.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
            toks, _, _ = ctx.decode_run(first, len(PROMPT), n, use_graph=use_graph)
            got.append([first] + list(toks))
            ctx.close()
        assert got[0] == got[1], use_graph


@pytest.mark.parametrize("n_seq", [3, 8])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_batched_steps(L, tiny128, n_seq, mode):
    p = tiny128
    acc, seq = _acc(L, mode), 40
    prompts = [[1 + i, 50 + 3 * i, 999 - i, 7, 300 + i] for i in range(n_seq)]
    res = []
    ctxs = [_ctx(L, p.mx, seq, acc, n_seq=n_seq), _ctx(L, p.dw, seq, acc, n_seq=n_seq)]
    try:
        for ctx, m in zip(ctxs, (p.mx, p.dw)):
            last = []
            for s, pr in enumerate(prompts):
                ctx.set_active_sequence(s)
                last.append(m.Transformer.forward_argmax(ctx, np.array(pr, np.int32), 0)[0])
            lg = []
            for j in range(6):
                nxt, l = ctx.forward_batch(last, [len(prompts[0]) + j] * n_seq, want_logits=True)
                last = list(nxt)
                lg.append(l)
            res.append(np.array(lg))
        assert np.array_equal(res[0], res[1])
        _caches_equal(p.args, ctxs[0], ctxs[1], len(prompts[0]) + 6, seqs=range(n_seq))
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_ragged_and_speculative_calls(L, tiny128, mode):
    p = tiny128
    acc, seq = _acc(L, mode), 64
    res = []
    for m in (p.mx, p.dw):
        ctx = _ctx(L, m, seq, acc, n_seq=3, max_rows=40)
        try:
            n1, l1 = ctx.forward_ragged([(0, 0, PROMPT), (1, 0, PROMPT[:3]), (2, 0, list(range(5, 30)))], want_logits=True)
            n2, l2 = ctx.forward_ragged([(0, 8, [int(n1[0])]), (1, 3, PROMPT[3:]), (2, 25, [int(n1[2])])], want_logits=True)
            nx, na, l3 = ctx.forward_speculative([(0, 9, [int(n2[0]), 5, 6, 7]), (2, 26, [int(n2[2]), 11, 12])], want_logits=True)
            res.append((n1, l1, n2, l2, nx, na, l3))
        finally:
            ctx.close()
    for x, y in zip(*res):
        assert np.array_equal(np.asarray(x), np.asarray(y))


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_streamed_attention_past_the_decode_kernel(L, mode):
    """batched steps of a session one key past sdpa_decode_kernel's fit run the streamed kernels"""
    args = dict(L.synth.TINY, max_seq_len=4096)
    seq = MS.sdpa_decode_fit(args) + 1
    assert not MS.sdpa_smem_decode(args, seq)
    p = Pair(L, args)
    try:
        res = []
        for m in (p.mx, p.dw):
            ctx = _ctx(L, m, seq, _acc(L, mode), n_seq=2)
            last = []
            for s in range(2):
                ctx.set_active_sequence(s)
                last.append(m.Transformer.forward_argmax(ctx, np.array(PROMPT[s:], np.int32), 0)[0])
            lg = []
            for j in range(4):
                nxt, l = ctx.forward_batch(last, [len(PROMPT) - s + j for s in range(2)], want_logits=True)
                last = list(nxt)
                lg.append(l)
            res.append(np.array(lg))
            ctx.close()
        assert np.array_equal(res[0], res[1])
    finally:
        p.close()


# ---- identity: generate loops -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_generate_loops(L, tiny, mode, tmp_path):
    p = tiny
    acc, seq = _acc(L, mode), 40
    path = str(tmp_path / "tokenizer.model")
    L._capi.check(L._capi.lib.lnb_vocab_write_synthetic(path.encode(), p.args["vocab_size"] - 256))
    vocab = L.vocabulary.Load(path)
    runs = []
    for m in (p.mx, p.dw):
        saved = m.Vocabulary
        m.Vocabulary = vocab
        try:
            eng = L.inference.InferenceEngine(m, L.model.InferenceArgs(seq), acc_mode=acc)
            out = {}
            out["sampled"] = [t for _, t in eng.GenerateTokens(PROMPT, sampling=L.model.SamplingArgs(0.8, 40, 0.95, 77))]
            out["penalized"] = [t for _, t in eng.GenerateTokens(PROMPT, penalties=L.model.PenaltyArgs(1.3, 0.4, 0.2))]
            lp = []
            out["logprobs"] = [t for _, t in eng.GenerateTokens(PROMPT, logprobs=5, logprobs_out=lp)]
            out["logprob_records"] = [repr(r) for r in lp]
            g = L.model.Grammar(m.Transformer, r"[a-z]+( [a-z]+)*\.", vocab)
            out["grammar"] = [t for _, t in eng.GenerateTokens(PROMPT, grammar=g)]
            g.close()
            out["beams"] = [repr(h) for h in eng.GenerateBeams(PROMPT, L.inference.BeamSearchArgs(3, NumReturn=3))]
            runs.append(out)
        finally:
            m.Vocabulary = saved
    for k in runs[0]:
        assert runs[0][k] == runs[1][k], k
        assert len(runs[0][k]) > 0, k


# ---- oracle ---------------------------------------------------------------------------------------------------------------
def test_strict_equals_the_oracle_of_dw(L, tiny):
    p = tiny
    om = oracle_model(p.args, p.dw_tensors)
    try:
        want = list(om.generate(PROMPT, 40, stop_ids=NO_STOP))
        eng = L.inference.InferenceEngine(p.mx, L.model.InferenceArgs(40), acc_mode=L._capi.LNB_ACC_STRICT)
        saved = p.mx.Vocabulary

        class V:
            StopTokenIds = NO_STOP
            PadId = saved.PadId
        p.mx.Vocabulary = V
        try:
            assert [t for _, t in eng.GenerateTokens(PROMPT)] == want
        finally:
            p.mx.Vocabulary = saved
        os_ = om.new_session(40)
        ctx = _ctx(L, p.mx, 40, L._capi.LNB_ACC_STRICT)
        try:
            lo = os_.forward(np.array(PROMPT, np.int32), 0)
            lg = p.mx.Transformer.Forward(ctx, L.ml.Tensor(np.array(PROMPT, np.int32), L.ml.DT_INT32), 0).RawData
            assert np.array_equal(lo, lg)
        finally:
            ctx.close(); os_.close()
    finally:
        om.close()


def test_cli_and_load_model_take_the_weight_format(L, tmp_path):
    """host/lnb_generate <seq_len> strict <dir> weights=mxfp8 (the C++ mirror's LoadModel) prints the tokens of the Python
    mirror's LoadModel(dir, weight_format="mxfp8"), which are those of the bf16 model of its D(W)"""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    d = str(tmp_path)
    subprocess.run([exe, "--write-synthetic", d, "tiny"], check=True, capture_output=True, timeout=120)
    mx = L.model.LoadModel(d, weight_format="mxfp8")
    dw = None
    try:
        args = mx.Transformer.args.to_c_dict()
        dw = L.model.Model(mx.Transformer.args)
        lin = set(linear_names(args))
        with L.torch_reader.TorchModelReader(os.path.join(d, "consolidated.00.pth")) as r:
            for name, t in r.Load().items():
                if name in L.synth.tensor_shapes(args):
                    dw.Transformer.upload_tensor(name, SR.mxfp8_dequantize(*mx.Transformer.mxfp8_read(name)) if name in lin
                                                 else np.asarray(t.RawData).view(np.uint16).reshape(t.Size))
        dw.Transformer.finalize()
        want = []
        for m in (mx, dw):
            m.Vocabulary = L.model.Vocabulary(StopTokenIds=NO_STOP)   # the CLI's stop set below the 8B vocabulary
            eng = L.inference.InferenceEngine(m, L.model.InferenceArgs(32), acc_mode=L._capi.LNB_ACC_STRICT)
            want.append([t for _, t in eng.GenerateTokens(PROMPT)])
        assert want[0] == want[1] and want[0]
        out = subprocess.run([exe, "32", "strict", d, "weights=mxfp8"], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        line = next(ln for ln in out.stdout.splitlines() if ln.startswith("tokens:"))
        assert [int(t) for t in line.split()[1:]] == want[0]
        bad = subprocess.run([exe, "32", "strict", d, "weights=fp4"], capture_output=True, text=True, timeout=120)
        assert bad.returncode != 0 and "weights=fp4" in bad.stderr
    finally:
        mx.Free()
        if dw is not None:
            dw.Free()


# ---- routing ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("env", [None, True])
def test_engines_refuse_and_the_session_stays_usable(L, tiny128, mode, env):
    p = tiny128
    acc = _acc(L, mode)
    a = _ctx(L, p.mx, 40, acc, engine=env)
    b = _ctx(L, p.dw, 40, acc, engine=False)
    try:
        assert not a.uses_engine()
        assert "MXFP8" in L._capi.lib.lnb_last_error().decode()
        ta, la = _steps(p.mx, a, 4)
        tb, lb = _steps(p.dw, b, 4)
        assert ta == tb and np.array_equal(la, lb)
    finally:
        a.close(); b.close()
    # batched and speculative calls take the kernel chain: one launch per call would be the batch engine
    c = _ctx(L, p.mx, 40, acc, n_seq=2, engine=env)
    try:
        for s in range(2):
            c.set_active_sequence(s)
            p.mx.Transformer.forward_argmax(c, np.array(PROMPT, np.int32), 0)
        l0 = c.launch_count()
        c.forward_batch([3, 4], [8, 8])
        assert c.launch_count() - l0 > 1
    finally:
        c.close()


def test_packed_stream_refuses(L, tiny128):
    info = (ctypes.c_int64 * 5)()
    assert L._capi.lib.lnb_model_wpack_read(tiny128.mx.Transformer.h, -1, None, None, None, info) == 0
    assert "MXFP8" in L._capi.lib.lnb_last_error().decode()


def test_weight_format_errors_and_weight_info(L, tiny128):
    p = tiny128
    lib = L._capi.lib
    assert lib.lnb_model_set_weight_format(p.mx.Transformer.h, L._capi.LNB_WEIGHTS_BF16) == -4      # LNB_ESTATE
    m = L.model.Model(L.model.ModelArgs.from_c_dict(p.args))
    try:
        assert lib.lnb_model_set_weight_format(m.Transformer.h, 7) == -1                             # LNB_EINVAL
        assert lib.lnb_model_set_weight_format(m.Transformer.h, L._capi.LNB_WEIGHTS_MXFP8) == 0
    finally:
        m.Free()
    with pytest.raises(ValueError):
        L.model.Model(L.model.ModelArgs.from_c_dict(p.args), weight_format="fp4")
    a, b = p.mx.Transformer.weight_info(), p.dw.Transformer.weight_info()
    assert a["format"] == "mxfp8" and b["format"] == "bf16"
    w = MS.widths(p.args)
    d, q, kv, f, v = p.args["dim"], w["q_l"], w["kv_l"], w["ffn_l"], w["vocab_l"]
    mats = [(q + 2 * kv, d), (d, q), (2 * f, d), (d, f)] * p.args["n_layers"] + [(v, d)]
    drop = sum(N * K * 2 - (N * K + N // 8 * ((-(-K // 32) + 1) & ~1) * 8) for N, K in mats)
    assert b["device_bytes"] - a["device_bytes"] == drop
    assert b["step_bytes"] - a["step_bytes"] == drop
    # the tensor-parallel refusal is in lnb_model_set_weight_format (this suite has one GPU): read it there
    src = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "llama-nuts-and-bolts_b200", "csrc", "api.cu")).read()
    body = src[src.index('extern "C" int lnb_model_set_weight_format'):]
    body = body[:body.index("\n}\n")]
    assert "m->tp_size > 1" in body and "LNB_EINVAL" in body


# ---- 8B ---------------------------------------------------------------------------------------------------------------------
def test_8b_mxfp8_equals_its_dequantized_model(L):
    """synthetic 8B: the LM head's and layer 0's codes against the C statement; then an MXFP8 model against the bf16 model of
    its D(W), built tensor by tensor from the library's own codes (both fit in 80 GB): FAST 8-token prompt and 32 decode
    steps, STRICT 8 + 10 with the first and last layer's caches, and a FAST 2048-token prompt"""
    args = dict(L.synth.LLAMA31_8B)
    mx = L.model.LoadSyntheticModel(args, weight_format="mxfp8")
    dw = None
    try:
        for name in ["output.weight"] + [f"layers.0.{n}" for n in LAYER_LINEAR]:
            w = L.synth.fill_host(args, name)
            codes, scales = mx.Transformer.mxfp8_read(name)
            wc, ws = SR.mxfp8_quantize(w)
            assert np.array_equal(scales, ws) and np.array_equal(codes, wc), name
            del w, wc, ws
        dw = L.model.Model(L.model.ModelArgs.from_c_dict(args))
        lin = set(linear_names(args))
        for name in L.synth.tensor_shapes(args):
            if name in lin:
                codes, scales = mx.Transformer.mxfp8_read(name)
                dw.Transformer.upload_tensor(name, SR.mxfp8_dequantize(codes, scales))
            else:
                dw.Transformer.upload_tensor(name, L.synth.fill_host(args, name))
        dw.Transformer.finalize()
        prompt = L.synth.PROMPT_8
        for mode, n in (("fast", 32), ("strict", 10)):
            a, b = _ctx(L, mx, 64, _acc(L, mode)), _ctx(L, dw, 64, _acc(L, mode), engine=False)
            try:
                ta, la = [], []
                for m, ctx in ((mx, a), (dw, b)):
                    t, lg0 = m.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0, want_logits="last")
                    toks, lgs = [t], [lg0[0]]
                    for j in range(n):
                        t, lg = m.Transformer.forward_argmax(ctx, np.array([toks[-1]], np.int32), len(prompt) + j, want_logits="last")
                        toks.append(t)
                        lgs.append(lg[0])
                    ta.append(toks)
                    la.append(np.array(lgs))
                assert ta[0] == ta[1], mode
                assert np.array_equal(la[0], la[1]), mode
                if mode == "strict":
                    for layer in (0, args["n_layers"] - 1):
                        for rd in ("CacheK", "CacheV"):
                            assert np.array_equal(getattr(a, rd)(layer).RawData[:len(prompt) + n],
                                                  getattr(b, rd)(layer).RawData[:len(prompt) + n]), (layer, rd)
            finally:
                a.close(); b.close()
        # the benchmark's prefill2048 workload: a FAST prompt of 2048 tokens on the tensor cores, every layer GEMM over 16 M
        # tiles of the dequantized scratch; its last row, and the first and last layer's caches at every position
        S = 2048
        toks = np.random.default_rng(0).integers(0, 128000, size=S).astype(np.int32)
        a, b = _ctx(L, mx, S, _acc(L, "fast"), max_rows=S), _ctx(L, dw, S, _acc(L, "fast"), max_rows=S, engine=False)
        try:
            ta, lga = mx.Transformer.forward_argmax(a, toks, 0, want_logits="last")
            tb, lgb = dw.Transformer.forward_argmax(b, toks, 0, want_logits="last")
            assert ta == tb and np.array_equal(lga, lgb), "prefill2048"
            for layer in (0, args["n_layers"] - 1):
                for rd in ("CacheK", "CacheV"):
                    assert np.array_equal(getattr(a, rd)(layer).RawData[:S], getattr(b, rd)(layer).RawData[:S]), (layer, rd)
        finally:
            a.close(); b.close()
    finally:
        mx.Free()
        if dw is not None:
            dw.Free()
