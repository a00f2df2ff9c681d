"""The tensor-core routes stage by stage: each stage's output, read through lnb_session_read's stage probes, against an
order-free reference of that stage computed from the GPU's own input to it (tests/precise.py).

The accumulation order of a tensor-core GEMM belongs to the hardware, so these routes cannot be restated bit for bit.  But
with the stage's input fixed, the exact f64 value of every sum, widened by the worst fp32 reordering error, brackets the
accumulator, and every epilogue after it is monotone in t(acc) or has few admissible inputs.  So a truncation point missing
from an epilogue (the residual without t(acc), SwiGLU on an untruncated up value, untruncated logits) or a position, layout
or head-mapping slip lands outside the admissible set on some elements, where the model-level tolerances cannot see it.
The intervals are single values on a large share of elements at these widths (the tests print the share per stage); at 8B
widths they are several ulps wide and the checks would say little, so they run on the small shapes.

Routes: the FAST tensor-core prompt path (enqueue_forward_tc) on TINY, TINY128 and every catalogue shape whose prompts
take it, MXFP8 and MXFP4 prompts whose LM head runs in row slices, and the batch engine's tensor-core form
(LNB_BATCH_TC=1).  The probes themselves are first checked bit for bit on the STRICT routes, where every stage can be
recomputed exactly."""
import time

import numpy as np
import pytest

from oracle import oracle as O
from tests import precise as P
from tests.engine_shapes import eng_split, wide_args
from tests.helpers import bf, f32, host_tensors, oracle_model
from tests.model_shapes import CATALOGUE, forward_tc

pytestmark = pytest.mark.gpu

SEED = 1234
STATS = {}      # stage -> [elements, single-value elements]
_WALL = {}


@pytest.fixture(autouse=True)
def _wall_time(request):
    t0 = time.perf_counter()
    yield
    _WALL[request.node.name] = time.perf_counter() - t0


def teardown_module(module):
    print("\nstage checks: elements checked, and the share whose admissible set is a single value")
    for k, (n, one) in sorted(STATS.items()):
        print(f"  {k:28s} {n:10d} elements, {one / max(n, 1):6.1%} single-valued")
    print(f"wall time, all tests: {sum(_WALL.values()):.1f} s")


def _stat(key, n, one):
    s = STATS.setdefault(key, [0, 0])
    s[0] += int(n)
    s[1] += int(one)


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# shapes: TINY, TINY128, `wide`, and the catalogue entries whose FAST prompts run on the tensor cores
TC_CATALOGUE = sorted(n for n, a in CATALOGUE.items() if forward_tc(a, 40, False, 40))


def _shape(name, sms):
    import lnb_b200
    if name == "wide":
        return wide_args(sms)
    a = dict(lnb_b200.synth.TINY) if name == "tiny" else dict(lnb_b200.synth.TINY128) if name == "tiny128" else dict(CATALOGUE[name])
    a["max_seq_len"] = max(a["max_seq_len"], 512)      # room for a 300-row prompt and a chunk at 37 (RoPE table only)
    return a


class Model:
    def __init__(self, L, args, weight_format="bf16"):
        self.args = args
        self.tensors = host_tensors(args, SEED)
        self.gm = L.model.LoadModelFromTensors(args, self.tensors, weight_format=weight_format)
        self.cis = O.rope_table(args["head_dim"], args["max_seq_len"], args["rope_theta"], bool(args["use_scaled_rope"]))[1]
        self.silu = O.silu_table_bf16()
        # the weights the stages read: D(W) for an MXFP8 or MXFP4 model (the bf16 model of its dequantized weights)
        self.w = self.tensors
        if weight_format == "mxfp8":
            from tests.test_gpu_mxfp8 import dequantized
            self.w = dequantized(args, self.tensors)
        elif weight_format == "mxfp4":
            from tests.test_gpu_mxfp4 import dequantized
            self.w = dequantized(args, self.tensors)

    def lw(self, l, name):
        return self.w[f"layers.{l}.{name}"]

    def close(self):
        self.gm.Free()


_MODELS = {}


def _model(L, name, sms):
    if name not in _MODELS:
        _MODELS[name] = Model(L, _shape(name, sms))
    return _MODELS[name]


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    for m in _MODELS.values():
        m.close()
    _MODELS.clear()


def _ctx(L, m, seq, max_rows, acc, n_seq=1):
    return L.model.InferenceContext(m.gm.Transformer, L.model.InferenceArgs(seq), max_rows=max_rows, acc_mode=acc, n_seq=n_seq)


def _norm(x, w, eps=1e-5):
    """RMSNorm with the scale summed in 256 interleaved parts (rmsnorm_x8_kernel, the batch engine's SCALE phase): exact"""
    r = O.rms_scale_order(np.ascontiguousarray(x), eps, 256)
    return bf(f32(bf(f32(x) * r[:, None])) * f32(w)[None, :]).reshape(x.shape)


def _inside(what, ok, lo=None, hi=None):
    if lo is not None:
        _stat(what, ok.size, np.sum(np.asarray(lo) == np.asarray(hi)))
    assert ok.all(), f"{what}: {(~ok).sum()} of {ok.size} outside their admissible sets; first at {np.argwhere(~ok)[0]}"


def _check_layer(m, l, x_in, pr, kv, seq, pos, route, normed="ffn"):
    """every stage of layer l for rows x_in [S, dim] (sequence seq[r] at position pos[r]) against its reference from its own
    probed input.  pr: the probes after the layer (q, attn, post, normed, ffn, out); kv: sequence -> (K, V) cache rows of
    layer l.  normed: "ffn" -- the probe holds the w1|w3 input; "output" -- the output norm of pr["out"] (the batch engine's
    last SCALE phase); None -- not readable."""
    a = m.args
    S, nh, nkv, hd = x_in.shape[0], a["n_heads"], a["n_kv_heads"], a["head_dim"]
    xn = _norm(x_in, m.lw(l, "attention_norm.weight"))
    lo, hi = P.rope_bounds(*[v.reshape(S, nh, hd) for v in P.linear_bounds(xn, m.lw(l, "attention.wq.weight"))], m.cis, pos)
    _inside(f"{route} q", P.within(pr["q"], lo.reshape(S, -1), hi.reshape(S, -1)), lo, hi)
    klo, khi = P.rope_bounds(*[v.reshape(S, nkv, hd) for v in P.linear_bounds(xn, m.lw(l, "attention.wk.weight"))], m.cis, pos)
    vlo, vhi = P.linear_bounds(xn, m.lw(l, "attention.wv.weight"))
    k_rows = np.stack([kv[q][0][p] for q, p in zip(seq, pos)]).reshape(S, -1)
    v_rows = np.stack([kv[q][1][p] for q, p in zip(seq, pos)]).reshape(S, -1)
    _inside(f"{route} K cache", P.within(k_rows, klo.reshape(S, -1), khi.reshape(S, -1)), klo, khi)
    _inside(f"{route} V cache", P.within(v_rows, vlo, vhi), vlo, vhi)
    alo, ahi = np.zeros((S, nh * hd)), np.zeros((S, nh * hd))
    for q in sorted(set(seq)):
        r = np.array([i for i in range(S) if seq[i] == q])
        T = int(max(pos[i] for i in r)) + 1
        lo_, hi_ = P.attention_bounds_general(pr["q"][r].reshape(len(r), nh, hd), kv[q][0][:T], kv[q][1][:T], np.asarray(pos)[r])
        alo[r], ahi[r] = lo_, hi_
    _inside(f"{route} attention", P.within(pr["attn"], alo, ahi), alo, ahi)
    lo, hi = P.resid_bounds(x_in, *P.linear_bounds(pr["attn"], m.lw(l, "attention.wo.weight")))
    _inside(f"{route} post-attention", P.within(pr["post"], lo, hi), lo, hi)
    xn2 = _norm(pr["post"], m.lw(l, "ffn_norm.weight"))
    if normed == "ffn":
        assert np.array_equal(pr["normed"], xn2), f"{route} ffn norm: {(pr['normed'] != xn2).sum()} of {xn2.size} differ"
    elif normed == "output":
        exp = _norm(pr["out"], m.w["norm.weight"])
        assert np.array_equal(pr["normed"], exp), f"{route} output norm: {(pr['normed'] != exp).sum()} of {exp.size} differ"
    slo, shi = P.swiglu_set(*P.linear_bounds(xn2, m.lw(l, "feed_forward.w1.weight")),
                            *P.linear_bounds(xn2, m.lw(l, "feed_forward.w3.weight")), m.silu)
    ok = P.in_set(pr["ffn"], slo, shi)
    _stat(f"{route} SwiGLU", ok.size, ok.size * P.set_single_fraction(slo, shi))
    _inside(f"{route} SwiGLU", ok)
    lo, hi = P.resid_bounds(pr["post"], *P.linear_bounds(pr["ffn"], m.lw(l, "feed_forward.w2.weight")))
    _inside(f"{route} output residual", P.within(pr["out"], lo, hi), lo, hi)


def _probes(ctx, S, normed=True):
    out = {k: ctx.stage(k, S) for k in ("q", "attn", "post_attn", "ffn")}
    out["post"] = out.pop("post_attn")
    out["normed"] = ctx.stage("normed", S) if normed else None
    out["out"] = ctx.residual(S)
    return out


def _caches(ctx, l, seqs):
    kv = {}
    for q in seqs:
        ctx.set_active_sequence(q)
        kv[q] = (ctx.CacheK(l).RawData.copy(), ctx.CacheV(l).RawData.copy())
    ctx.set_active_sequence(0)
    return kv


# ---- 1. the probes on the STRICT routes: every stage recomputed bit for bit from its probed input ---------------------------

def _strict_stages(m, l, x_in, pr, kv, seq, pos, fma_normed=True):
    a = m.args
    S, nh, nkv, hd = x_in.shape[0], a["n_heads"], a["n_kv_heads"], a["head_dim"]
    xn = O.rmsnorm(np.ascontiguousarray(x_in), m.lw(l, "attention_norm.weight"), a["norm_eps"])
    for i in range(S):
        q_exp = O.rope_apply(O.linear_bf16(xn[i:i + 1], m.lw(l, "attention.wq.weight")).reshape(1, nh, hd), m.cis, int(pos[i]))
        assert np.array_equal(pr["q"][i], q_exp.reshape(-1)), f"q, row {i}"
        k_exp = O.rope_apply(O.linear_bf16(xn[i:i + 1], m.lw(l, "attention.wk.weight")).reshape(1, nkv, hd), m.cis, int(pos[i]))
        assert np.array_equal(kv[seq[i]][0][pos[i]], k_exp[0]), f"K cache, row {i}"
        T = int(pos[i]) + 1
        att = O.attention(pr["q"][i].reshape(1, nh, hd), kv[seq[i]][0][:T], kv[seq[i]][1][:T], T, 1, q_pos0=int(pos[i]))
        assert np.array_equal(pr["attn"][i], att[0]), f"attention, row {i}"
    assert np.array_equal(pr["post"], O.add_bf16(x_in, O.linear_bf16(pr["attn"], m.lw(l, "attention.wo.weight"))))
    xn2 = O.rmsnorm(pr["post"], m.lw(l, "ffn_norm.weight"), a["norm_eps"])
    g = O.linear_bf16(xn2, m.lw(l, "feed_forward.w1.weight"))
    u = O.linear_bf16(xn2, m.lw(l, "feed_forward.w3.weight"))
    assert np.array_equal(pr["ffn"], O.mul_bf16(m.silu[g], u))
    assert np.array_equal(pr["out"], O.add_bf16(pr["post"], O.linear_bf16(pr["ffn"], m.lw(l, "feed_forward.w2.weight"))))


def test_strict_chain_probes_equal_the_stages_recomputed(L, sms):
    m = _model(L, "tiny", sms)
    nl, S = m.args["n_layers"], 6
    toks = np.random.default_rng(1).integers(0, m.args["vocab_size"], size=S).astype(np.int32)
    ctx = _ctx(L, m, 32, 8, L._capi.LNB_ACC_STRICT)
    try:
        x_in = m.tensors["tok_embeddings.weight"][toks]
        for l in range(nl):
            ctx.set_layer_limit(l + 1)
            m.gm.Transformer.forward_argmax(ctx, toks, 0)
            with pytest.raises(L._capi.LnbError, match="prologue"):
                ctx.stage("normed", S)
            pr = _probes(ctx, S, normed=False)
            _strict_stages(m, l, x_in, pr, _caches(ctx, l, [0]), [0] * S, np.arange(S))
            x_in = pr["out"]
    finally:
        ctx.close()


@pytest.mark.parametrize("n", [3, 8])
def test_strict_batch_engine_probes_and_residual(L, sms, n, monkeypatch):
    """after a STRICT batch-engine step LNB_BUF_RESIDUAL holds each sequence's row of the oracle's trace (it used to return
    the rows of the last kernel-chain forward), and every probe equals its stage recomputed bit for bit"""
    monkeypatch.delenv("LNB_BATCH_ENGINE", raising=False)
    m = _model(L, "tiny", sms)
    a = m.args
    nl, seq_len = a["n_layers"], 32
    om = oracle_model(a, m.tensors)
    ctx = _ctx(L, m, seq_len, 8, L._capi.LNB_ACC_STRICT, n_seq=8)
    rng = np.random.default_rng(n)
    prompts = [rng.integers(0, a["vocab_size"], size=2 + i % 7).astype(np.int32) for i in range(n)]
    osess = [om.new_session(seq_len) for _ in range(n)]
    try:
        assert ctx.uses_engine()
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            m.gm.Transformer.forward_argmax(ctx, p, 0)
            osess[i].forward(p, 0)
        ctx.set_active_sequence(0)
        toks = rng.integers(0, a["vocab_size"], size=n).astype(np.int32)
        pos = np.array([len(p) for p in prompts], np.int32)
        ctx.forward_batch(toks, pos)                                   # after kernel-chain forwards of more rows
        res = ctx.residual(n)
        for i in range(n):
            _, tr = osess[i].forward(toks[i:i + 1], int(pos[i]), trace=True)
            assert np.array_equal(res[i], tr[-1][0]), f"sequence {i}: the residual row is not the batch step's"
        with pytest.raises(L._capi.LnbError, match="rows"):
            ctx.residual(n + 1)
        x_in = m.tensors["tok_embeddings.weight"][toks]
        for l in range(nl):
            ctx.set_layer_limit(l + 1)
            ctx.forward_batch(toks, pos)
            with pytest.raises(L._capi.LnbError, match="prologue"):
                ctx.stage("normed", n)
            pr = _probes(ctx, n, normed=False)
            _strict_stages(m, l, x_in, pr, _caches(ctx, l, range(n)), list(range(n)), pos)
            x_in = pr["out"]
        ctx.set_layer_limit(0)
    finally:
        ctx.close()
        for o in osess:
            o.close()
        om.close()


def test_refused_reads_leave_the_session_usable(L, sms):
    m = _model(L, "tiny", sms)
    a = m.args
    toks = np.arange(1, 6, dtype=np.int32)
    ctx = _ctx(L, m, 32, 8, L._capi.LNB_ACC_STRICT)
    try:
        with pytest.raises(L._capi.LnbError, match="no forward"):
            ctx.stage("q", 1)
        t0, lg0 = m.gm.Transformer.forward_argmax(ctx, toks, 0, want_logits="last")
        with pytest.raises(L._capi.LnbError, match="rows"):
            ctx.stage("ffn", 6)
        with pytest.raises(L._capi.LnbError, match="rows"):
            ctx.residual(6)
        c = L._capi
        buf = np.zeros(16, np.uint16)
        with pytest.raises(c.LnbError, match="bad buffer"):
            c.check(c.lib.lnb_session_read(ctx.h, 99, 0, c.ptr(buf, c.u16p), buf.nbytes))
        if ctx.uses_engine():
            t1, _ = m.gm.Transformer.forward_argmax(ctx, np.array([t0], np.int32), 5)
            with pytest.raises(L._capi.LnbError, match="tagged words"):
                ctx.stage("q", 1)
            assert ctx.residual(1).shape == (1, a["dim"])
        t2, lg2 = m.gm.Transformer.forward_argmax(ctx, toks, 0, want_logits="last")
        assert t2 == t0 and np.array_equal(lg2, lg0)
        assert ctx.stage("q", 5).shape == (5, a["n_heads"] * a["head_dim"])
    finally:
        ctx.close()


# ---- 2. the tensor-core prompt path, stage by stage ---------------------------------------------------------------------------

PROMPTS = [(32, 0), (129, 0), (300, 0), (40, 37)]      # (rows, start): one row past a tile, several tiles, a chunk at 37


def _prefill_stages(L, m, S, start, route):
    a = m.args
    nl = a["n_layers"]
    seq_len = min(a["max_seq_len"], 512)
    if start + S > seq_len:
        pytest.skip(f"{start + S} positions exceed the shape's {seq_len}")
    toks = np.random.default_rng(S * 7 + start).integers(0, a["vocab_size"], size=start + S).astype(np.int32)
    ctx = _ctx(L, m, seq_len, max(S, start, 32), L._capi.LNB_ACC_FAST)
    try:
        ctx.allow_chunked_prefill(True)
        if start:
            m.gm.Transformer.forward_argmax(ctx, toks[:start], 0)
        chunk = toks[start:]
        pos = start + np.arange(S)
        x_in = m.tensors["tok_embeddings.weight"][chunk]
        for l in range(nl):
            ctx.set_layer_limit(l + 1)
            m.gm.Transformer.forward_argmax(ctx, chunk, start, want_logits="last")
            pr = _probes(ctx, S)
            _check_layer(m, l, x_in, pr, _caches(ctx, l, [0]), [0] * S, pos, route)
            x_in = pr["out"]
        ctx.set_layer_limit(0)
        _, lg = m.gm.Transformer.forward_argmax(ctx, chunk, start, want_logits="all")
        res = ctx.residual(S)
        xo = _norm(res, m.w["norm.weight"])
        rows = sorted({0, 1, min(127, S - 2), min(128, S - 2), S - 2})
        lo, hi = P.linear_bounds(xo[rows], m.w["output.weight"])
        _inside(f"{route} logits (f32 of t(acc))", P.within_values(lg[rows], lo, hi), lo, hi)
        last = f32(O.linear_order_bf16(xo[-1:], m.w["output.weight"], 8))
        assert np.array_equal(lg[-1:], last), "the last row's logits are not the GEMV's (ks = 8) bits"
    finally:
        ctx.close()


@pytest.mark.parametrize("S,start", PROMPTS)
@pytest.mark.parametrize("name", ["tiny", "tiny128"] + TC_CATALOGUE)
def test_tensor_core_prompt_stage_by_stage(L, sms, name, S, start):
    m = _model(L, name, sms)
    assert forward_tc(m.args, S, False, max(S, 32))
    _prefill_stages(L, m, S, start, "prefill")


def _sliced_head_prompt(L, sms, fmt, S):
    a = dict(_shape("tiny128", sms), vocab_size=8192)
    dim = a["dim"]
    assert forward_tc(a, S, False, S)
    w_elems = max([(a["n_heads"] + 2 * a["n_kv_heads"]) * a["head_dim"] * dim, dim * a["n_heads"] * a["head_dim"],
                   2 * a["ffn_dim"] * dim, dim * a["ffn_dim"], 128 * dim])
    assert a["vocab_size"] > w_elems // dim, "the LM head must run in row slices"
    m = Model(L, a, weight_format=fmt)
    try:
        _prefill_stages(L, m, S, 0, f"{fmt} prefill")
    finally:
        m.close()


def test_mxfp8_prompt_with_a_sliced_lm_head_stage_by_stage(L, sms):
    """an MXFP8 FAST prompt of 40 rows whose LM head is dequantized and run in row slices (TINY128 with a vocabulary of
    8192: the largest layer matrix, w1|w3, holds 2048 rows of dim; `wide` slices too, but its FFN is off the 128-wide tiles,
    so its prompts stay on the kernel chain): every stage against D(W), the bf16 values of the dequantized weights"""
    _sliced_head_prompt(L, sms, "mxfp8", 40)


@pytest.mark.parametrize("fmt,S", [("mxfp8", 300), ("mxfp4", 40), ("mxfp4", 300)])
def test_mx_prompt_with_a_sliced_lm_head_stage_by_stage(L, sms, fmt, S):
    """the test above for MXFP4, and for prompts of 300 rows: three M tiles in every GEMM over the dequantized scratch,
    and a sliced LM head of 299 rows"""
    _sliced_head_prompt(L, sms, fmt, S)


# ---- 3. the batch engine's tensor-core form ------------------------------------------------------------------------------------

def _tiles(N, G):
    """panel counts of the row tiles of every CTA for a projection of N rows (eng_split, 16-panel tiles)"""
    out = []
    for b in range(G):
        p0, p1 = eng_split(N // 8, b, G)
        out += [min(16, p1 - rt) for rt in range(p0, p1, 16)]
    return out


@pytest.mark.parametrize("name", ["tiny", "tiny128", "wide"])
def test_batch_engine_tensor_core_form_stage_by_stage(L, sms, name, monkeypatch):
    monkeypatch.setenv("LNB_BATCH_TC", "1")
    monkeypatch.delenv("LNB_BATCH_ENGINE", raising=False)
    m = _model(L, name, sms)
    a = m.args
    nl, seq_len = a["n_layers"], 64
    rng = np.random.default_rng(len(name))
    prompts = [rng.integers(0, a["vocab_size"], size=3 + i % 6).astype(np.int32) for i in range(8)]
    ctx = _ctx(L, m, seq_len, 8, L._capi.LNB_ACC_FAST, n_seq=8)
    try:
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            m.gm.Transformer.forward_argmax(ctx, p, 0)
        ctx.set_active_sequence(0)
        calls = []
        for n in (1, 3, 8):
            toks = rng.integers(0, a["vocab_size"], size=n).astype(np.int32)
            calls.append(("batch", list(range(n)), np.array([len(prompts[i]) for i in range(n)]), toks))
        # speculative rows: sequence 2 with two drafts after its prompt, sequence 5 with one
        spec = [(2, len(prompts[2]), rng.integers(0, a["vocab_size"], size=3).astype(np.int32)),
                (5, len(prompts[5]), rng.integers(0, a["vocab_size"], size=2).astype(np.int32))]
        calls.append(("speculative", [2, 2, 2, 5, 5], np.array([spec[0][1] + j for j in range(3)] + [spec[1][1] + j for j in range(2)]),
                      np.concatenate([spec[0][2], spec[1][2]])))
        for kind, seqs, pos, toks in calls:
            rows = len(toks)

            def run():
                if kind == "batch":
                    ctx.forward_batch(toks, pos)
                else:
                    ctx.forward_speculative(spec)

            x_in = m.tensors["tok_embeddings.weight"][toks]
            for l in range(nl):
                ctx.set_layer_limit(l + 1)
                run()
                pr = _probes(ctx, rows)            # NORMED reads: the tensor-core form ran (the FMA form refuses them)
                _check_layer(m, l, x_in, pr, _caches(ctx, l, sorted(set(seqs))), seqs, pos, f"batch TC {kind}", normed="output")
                x_in = pr["out"]
            ctx.set_layer_limit(0)
    finally:
        ctx.close()


def test_batch_engine_tiling_reaches_partial_and_multi_slice_tiles(L, sms):
    """the shapes above give some CTA a tile whose panel count is not a multiple of 4, and some a tile of several 32-row
    slices (ceil(np / 4) > 1)"""
    off4, multi = False, False
    for name in ("tiny", "tiny128", "wide"):
        a = _shape(name, sms)
        q_l, kv_l, f = a["n_heads"] * a["head_dim"], a["n_kv_heads"] * a["head_dim"], a["ffn_dim"]
        for N in (q_l + 2 * kv_l, a["dim"], 2 * f, a["vocab_size"]):
            t = _tiles(N, sms)
            off4 |= any(x % 4 for x in t)
            multi |= any(x > 4 for x in t)
    assert off4 and multi


def test_speculative_rows_have_the_bits_of_batched_steps(L, sms, monkeypatch):
    """under LNB_BATCH_TC=1 a speculative call's rows equal, bit for bit, the batched steps that feed the same tokens one
    position at a time (lnb.h)"""
    monkeypatch.setenv("LNB_BATCH_TC", "1")
    monkeypatch.delenv("LNB_BATCH_ENGINE", raising=False)
    m = _model(L, "tiny128", sms)
    a = m.args
    rng = np.random.default_rng(9)
    prompt = rng.integers(0, a["vocab_size"], size=7).astype(np.int32)
    draft = rng.integers(0, a["vocab_size"], size=4).astype(np.int32)
    got = []
    for mode in ("speculative", "batched"):
        ctx = _ctx(L, m, 64, 8, L._capi.LNB_ACC_FAST, n_seq=2)
        try:
            m.gm.Transformer.forward_argmax(ctx, prompt, 0)
            if mode == "speculative":
                _, _, lg = ctx.forward_speculative([(0, 7, draft)], want_logits=True)
            else:
                lg = np.stack([ctx.forward_batch(draft[j:j + 1], np.array([7 + j], np.int32), want_logits=True)[1][0]
                               for j in range(len(draft))])
            got.append((lg, ctx.CacheK(a["n_layers"] - 1).RawData[:11].copy()))
        finally:
            ctx.close()
    assert np.array_equal(got[0][0], got[1][0]), "logits"
    assert np.array_equal(got[0][1], got[1][1]), "K cache"
