"""GPU parity of the model-level C-ABI (LlamaTransformer.Forward / generate loop) against the CPU
oracle on a structurally identical miniature of Llama-3.1 (all fusion paths, GQA, RoPE, KV cache).
STRICT mode must reproduce the oracle bit for bit; FAST the oracle run in FAST's summation order (tests/test_gpu_fast_order.py),
and within north_star's tolerance of the reference order."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import bf16_ulp_diff, f32, host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 1234


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


@pytest.fixture(scope="module")
def tiny(L):
    args = dict(L.synth.TINY)
    tensors = host_tensors(args, SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)       # the reference's flow: host tensors -> upload
    yield args, tensors, om, gm
    gm.Free()
    om.close()


def test_tables_match_oracle(L, tiny):
    args, _, _, gm = tiny
    _, cis = O.rope_table(args["head_dim"], args["max_seq_len"] * 2, args["rope_theta"], bool(args["use_scaled_rope"]))
    assert np.array_equal(gm.Transformer.rope_table(), cis)
    assert np.array_equal(gm.Transformer.silu_table(), O.silu_table_bf16())


def test_device_generator_equals_host_generator(L, tiny):
    args, tensors, om, gm = tiny
    g2 = L.model.LoadSyntheticModel(args, seed=SEED)        # generated directly in HBM
    try:
        toks = np.array([3, 77, 1000, 5, 9], np.int32)
        c1 = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(16), acc_mode=L._capi.LNB_ACC_STRICT)
        c2 = L.model.InferenceContext(g2.Transformer, L.model.InferenceArgs(16), acc_mode=L._capi.LNB_ACC_STRICT)
        l1 = gm.Transformer.Forward(c1, L.ml.Tensor(toks, L.ml.DT_INT32), 0).RawData
        l2 = g2.Transformer.Forward(c2, L.ml.Tensor(toks, L.ml.DT_INT32), 0).RawData
        assert np.array_equal(l1, l2)
        c1.close(); c2.close()
    finally:
        g2.Free()
    # and the host twin inside the product library
    name = "layers.1.feed_forward.w2.weight"
    assert np.array_equal(L.synth.fill_host(args, name, SEED), tensors[name])


@pytest.mark.parametrize("prompt_len", [1, 5, 8])
def test_forward_strict_bit_exact(L, tiny, prompt_len):
    check_forward_strict(L, tiny, prompt_len)


def check_forward_strict(L, model, prompt_len):
    args, _, om, gm = model
    rng = np.random.default_rng(prompt_len)
    seq = 24
    toks = rng.integers(0, args["vocab_size"], size=seq).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), acc_mode=L._capi.LNB_ACC_STRICT)
    osess = om.new_session(seq)
    try:
        # prefill
        exp, tr = osess.forward(toks[:prompt_len], 0, all_rows=True, trace=True)
        got = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[:prompt_len], L.ml.DT_INT32), 0).RawData
        assert np.array_equal(ctx.residual(prompt_len), tr[-1]), "residual stream after the last layer differs"
        assert np.array_equal(got, exp)
        # decode steps
        for pos in range(prompt_len, prompt_len + 6):
            exp = osess.forward(toks[pos:pos + 1], pos)
            got = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[pos:pos + 1], L.ml.DT_INT32), pos).RawData
            assert np.array_equal(got, exp), f"logits differ at position {pos}"
        for layer in range(args["n_layers"]):
            ok, ov = osess.cache(layer)
            assert np.array_equal(ctx.CacheK(layer).RawData, ok)
            assert np.array_equal(ctx.CacheV(layer).RawData, ov)
    finally:
        ctx.close(); osess.close()


def test_forward_per_layer_trace_strict(L, tiny):
    args, _, om, gm = tiny
    toks = np.array([1, 2, 3], np.int32)
    osess = om.new_session(8)
    _, tr = osess.forward(toks, 0, trace=True)
    osess.close()
    for n in range(1, args["n_layers"] + 1):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(8), acc_mode=L._capi.LNB_ACC_STRICT)
        ctx.set_layer_limit(n)
        gm.Transformer.forward_argmax(ctx, toks, 0)
        assert np.array_equal(ctx.residual(3), tr[n]), f"layer {n}"
        ctx.close()


def test_forward_fast_equals_the_fast_order_statement(L, tiny):
    """FAST through the reference-shaped Forward: every prompt row and every decode step is the oracle run in FAST's
    summation order (O.ORDER_FAST) bit for bit -- and so within north_star's tolerance of the reference order"""
    args, _, om, gm = tiny
    rng = np.random.default_rng(11)
    seq = 24
    toks = rng.integers(0, args["vocab_size"], size=seq).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), acc_mode=L._capi.LNB_ACC_FAST)
    osess, oref = om.new_session(seq), om.new_session(seq)
    try:
        exp = osess.forward(toks[:8], 0, order=O.ORDER_FAST)
        got = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[:8], L.ml.DT_INT32), 0).RawData
        assert np.array_equal(got, exp)
        assert np.abs(got - oref.forward(toks[:8], 0)).max() <= 1e-2                      # north_star tolerance
        for pos in range(8, 16):
            exp = osess.forward(toks[pos:pos + 1], pos, order=O.ORDER_FAST)
            got = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[pos:pos + 1], L.ml.DT_INT32), pos).RawData
            assert np.array_equal(got, exp), f"position {pos}"
            assert np.abs(got - oref.forward(toks[pos:pos + 1], pos)).max() <= 1e-2
    finally:
        ctx.close(); osess.close(); oref.close()


def test_forward_errors_like_reference(L, tiny):
    args, _, _, gm = tiny
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(8))
    T = L.ml.Tensor
    with pytest.raises(L.ml.MlError, match="empty token array"):
        gm.Transformer.Forward(ctx, T(np.zeros(0, np.int32), L.ml.DT_INT32), 0)
    with pytest.raises(L._capi.LnbError, match="SequenceLength"):
        gm.Transformer.Forward(ctx, T(np.zeros(1, np.int32), L.ml.DT_INT32), 8)
    with pytest.raises(L._capi.LnbError, match="out of range"):
        gm.Transformer.Forward(ctx, T(np.array([args["vocab_size"]], np.int32), L.ml.DT_INT32), 0)
    with pytest.raises(L._capi.LnbError, match="startPos 0"):
        gm.Transformer.Forward(ctx, T(np.zeros(2, np.int32), L.ml.DT_INT32), 3)
    ctx.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_generate_loop_matches_oracle(L, tiny, mode):
    args, _, om, gm = tiny
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    prompt = [1, 50, 999, 7, 300, 12, 64, 2]
    seq = 40
    exp = om.generate(prompt, seq, stop_ids=(10**9,))
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=acc)
    got_ref_api = [t for _, t in eng.GenerateTokens(prompt, use_reference_api=True)]
    got_fused = [t for _, t in eng.GenerateTokens(prompt, use_reference_api=False)]
    assert got_ref_api == got_fused
    assert len(got_fused) == seq - len(prompt)
    if mode == "strict":
        assert got_fused == list(exp)
    else:
        n = next((i for i, (a, b) in enumerate(zip(got_fused, exp)) if a != b), len(exp))
        assert n >= 1  # first token must agree; the full-size statistics live in test_gpu_8b.py


def test_generate_stops_on_eos(L, tiny):
    args, _, om, gm = tiny
    prompt = [1, 50, 999]
    free = list(om.generate(prompt, 20, stop_ids=(10**9,)))
    stop = free[4]
    gm.Vocabulary.StopTokenIds = (stop,)
    try:
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(20), acc_mode=L._capi.LNB_ACC_STRICT)
        out = list(eng.GenerateTokens(prompt))
        k = free.index(stop)
        assert [t for _, t in out] == free[:k + 1]
        assert out[-1][0] == L.inference.GSFinishedByReachingEOS
        assert list(om.generate(prompt, 20, stop_ids=(stop,))) == free[:k + 1]
    finally:
        gm.Vocabulary.StopTokenIds = L.synth.STOP_IDS


@pytest.mark.parametrize("use_graph", [False, True])
def test_device_resident_decode_equals_host_loop(L, tiny, use_graph):
    args, _, om, gm = tiny
    prompt = [1, 50, 999, 7, 300, 12, 64, 2]
    seq = 40
    exp = list(om.generate(prompt, seq, stop_ids=(10**9,)))
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), acc_mode=L._capi.LNB_ACC_STRICT)
    try:
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0)
        assert first == exp[0]
        toks, ms, graphed = ctx.decode_run(first, len(prompt), seq - len(prompt) - 1, use_graph=use_graph)
        assert list(toks) == exp[1:]
        assert ms > 0
        assert graphed == use_graph
        assert ctx.launch_count() > 0
    finally:
        ctx.close()


def test_prefill_tensor_core_path(L, tiny):
    """LNB_ACC_FAST with a prompt of >= 32 tokens runs the tensor-core prefill path (gemm_tc.cuh + X8
    elementwise kernels); it must agree with the oracle up to fp32 summation order, and the KV cache it
    leaves must drive the ordinary decode path."""
    args, _, om, gm = tiny
    rng = np.random.default_rng(40)
    S, seq = 40, 48
    toks = rng.integers(0, args["vocab_size"], size=seq).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=S, acc_mode=L._capi.LNB_ACC_FAST)
    osess = om.new_session(seq)
    try:
        exp, tr = osess.forward(toks[:S], 0, all_rows=True, trace=True)
        nxt, got = gm.Transformer.forward_argmax(ctx, toks[:S], 0, want_logits="all")
        assert got.shape == exp.shape
        assert np.abs(got - exp).max() <= 1e-2
        assert (np.argmax(got, -1) == np.argmax(exp, -1)).mean() >= 0.95
        assert nxt == int(np.argmax(got[-1]))
        from tests.helpers import f32
        r_got, r_exp = f32(ctx.residual(S)).reshape(S, -1), f32(tr[-1]).reshape(S, -1)
        assert np.abs(r_got - r_exp).max() <= 2.0 ** -5 * max(1.0, np.abs(r_exp).max())   # a few bf16 ulps of the largest entry
        assert (r_got != r_exp).mean() < 0.3
        for layer in range(args["n_layers"]):
            ok, ov = osess.cache(layer)
            for got_c, exp_c in ((ctx.CacheK(layer).RawData[:S], ok[:S]), (ctx.CacheV(layer).RawData[:S], ov[:S])):
                g_, e_ = f32(got_c).reshape(-1), f32(exp_c).reshape(-1)
                assert np.abs(g_ - e_).max() <= 2.0 ** -6 * max(1.0, np.abs(e_).max())
        for pos in range(S, S + 4):     # decode continues on the cache written by the prefill kernels
            e = osess.forward(toks[pos:pos + 1], pos)
            g = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[pos:pos + 1], L.ml.DT_INT32), pos).RawData
            assert np.abs(g - e).max() <= 1e-2
    finally:
        ctx.close(); osess.close()


def test_prefill_strict_stays_bit_exact_for_long_prompts(L, tiny):
    args, _, om, gm = tiny
    rng = np.random.default_rng(41)
    S = 36
    toks = rng.integers(0, args["vocab_size"], size=S).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), max_rows=S, acc_mode=L._capi.LNB_ACC_STRICT)
    osess = om.new_session(40)
    try:
        exp = osess.forward(toks, 0, all_rows=True)
        got = gm.Transformer.Forward(ctx, L.ml.Tensor(toks, L.ml.DT_INT32), 0).RawData
        assert np.array_equal(got, exp)
    finally:
        ctx.close(); osess.close()


def test_cpp_host_mirror_generates_the_oracle_tokens(L):
    """host/lnb_generate: the C++ mirror of src/ml + src/model + src/inference (reference-shaped loop:
    Forward -> logits to host -> Slice -> ml.Argmax) over the C-ABI, on the device-generated tiny model."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    out = subprocess.run([exe, "24", "strict", "tiny"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    line = [l for l in out.stdout.splitlines() if l.startswith("tokens:")][0]
    got = [int(t) for t in line.split()[1:]]
    args = dict(L.synth.TINY)
    om = oracle_model(args, host_tensors(args, 7))
    exp = list(om.generate([1, 50, 999, 7, 300, 12, 64, 2], 24, stop_ids=(10**9,)))
    om.close()
    assert got == exp
    # the same through model.LoadModel: `--write-synthetic` writes params.json + consolidated.00.pth (host-only),
    # the second run maps that file and uploads it (SURVEY 8f-1)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        subprocess.check_call([exe, "--write-synthetic", d, "tiny"])
        out = subprocess.run([exe, "24", "strict", d], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        line = [l for l in out.stdout.splitlines() if l.startswith("tokens:")][0]
        assert [int(t) for t in line.split()[1:]] == exp
    # inference::GenerateTokensBatch: 3 prompts generated together, each gets its single-prompt stream
    out = subprocess.run([exe, "24", "strict", "tiny", "batch=3"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    base = [1, 50, 999, 7, 300, 12, 64, 2]
    om = oracle_model(args, host_tensors(args, 7))
    for b in range(3):
        prompt = [base[0]] + [(t + 977 * b) % 1000 for t in base[1:]]
        line = [l for l in out.stdout.splitlines() if l.startswith(f"tokens[{b}]:")][0]
        assert [int(t) for t in line.split()[1:]] == list(om.generate(prompt, 24, stop_ids=(10**9,))), b
    om.close()


@pytest.mark.parametrize("mode", ["strict", "fast", "fast_tc"])
def test_batched_decode_equals_independent_contexts(L, tiny, mode, monkeypatch):
    """config 5: n_seq sequences stepped together through one pass over the weights; STRICT: every sequence is
    bit-identical to its own oracle InferenceContext (different prompt lengths, different positions).  fast_tc: the
    batch engine's tensor-core form (LNB_BATCH_TC=1)."""
    if mode == "fast_tc":
        monkeypatch.setenv("LNB_BATCH_TC", "1")
    check_batched_decode(L, tiny, mode)


@pytest.fixture(scope="module")
def wide(L):
    """TINY with a 4096-wide FFN and a 16384-entry vocabulary: on any GPU with at most 256 SMs a CTA of the batch engine owns
    more than 4 panels (32 rows) of w1|w3 and of the LM head, so the tensor-core form issues several 32-row slices per tile"""
    args = dict(L.synth.TINY, ffn_dim=4096, vocab_size=16384)
    tensors = host_tensors(args, SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    yield args, tensors, om, gm
    gm.Free()
    om.close()


def test_batch_engine_tensor_core_form_on_wide_projections(L, wide, monkeypatch):
    """the tensor-core form of the batch engine (LNB_BATCH_TC=1) with several 32-row slices per row tile: every sequence's
    logits stay within FAST's tolerance of its own oracle context"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    args = wide[0]
    assert -(-(2 * args["ffn_dim"] // 8) // sms) > 4 and -(-(args["vocab_size"] // 8) // sms) > 4
    monkeypatch.setenv("LNB_BATCH_TC", "1")
    check_batched_decode(L, wide, "fast_tc")


def check_batched_decode(L, model, mode):
    args, _, om, gm = model
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(55)
    seq, nseq = 32, 5
    prompts = [rng.integers(0, args["vocab_size"], size=k).astype(np.int32) for k in (3, 8, 1, 6, 8)]
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=8, acc_mode=acc, n_seq=nseq)
    # FAST on the FMA pipe: every batched row must equal its sequence's own S=1 forward on the kernel chain (a single-GPU FAST
    # session's S=1 default); the tensor-core form's order is the hardware's and keeps the tolerance
    own = None
    if mode == "fast":
        own = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=8, acc_mode=acc, n_seq=nseq)
    osess = [om.new_session(seq) for _ in range(nseq)]
    try:
        cur, pos = [], []
        for i, p in enumerate(prompts):                      # prefill every sequence through the ordinary Forward
            ctx.set_active_sequence(i)
            nxt, lg = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
            if own is not None:
                own.set_active_sequence(i)
                assert not own.uses_engine()
                assert np.array_equal(gm.Transformer.forward_argmax(own, p, 0, want_logits="last")[1], lg)
            exp = osess[i].forward(p, 0, all_rows=False)
            if mode == "strict":
                assert np.array_equal(lg, exp)
            cur.append(int(np.argmax(exp[0]))); pos.append(len(p))
            assert mode != "strict" or nxt == cur[-1]
        for step in range(6):
            nxt, lg = ctx.forward_batch(cur, pos, want_logits=True)
            for i in range(nseq):
                exp = osess[i].forward(np.array([cur[i]], np.int32), pos[i])
                if mode == "strict":
                    assert np.array_equal(lg[i], exp[0]), f"sequence {i} step {step}"
                    assert nxt[i] == O.argmax_f32(exp[0])
                else:
                    assert np.abs(lg[i] - exp[0]).max() <= 1e-2
                if own is not None:
                    own.set_active_sequence(i)
                    t1, l1 = gm.Transformer.forward_argmax(own, np.array([cur[i]], np.int32), pos[i], want_logits="last")
                    assert np.array_equal(lg[i], l1[0]), f"sequence {i} step {step}: batched row != its own S=1 forward"
                    assert nxt[i] == t1
                cur[i] = int(np.argmax(exp[0])); pos[i] += 1   # teacher-forced with the oracle's token
        if mode == "strict":
            for i in range(nseq):                            # caches of every sequence, all layers
                ctx.set_active_sequence(i)
                for layer in range(args["n_layers"]):
                    ok, ov = osess[i].cache(layer)
                    assert np.array_equal(ctx.CacheK(layer).RawData[:pos[i]], ok[:pos[i]])
                    assert np.array_equal(ctx.CacheV(layer).RawData[:pos[i]], ov[:pos[i]])
        with pytest.raises(L._capi.LnbError):
            ctx.forward_batch([1] * (nseq + 1), [0] * (nseq + 1))
        with pytest.raises(L._capi.LnbError):
            ctx.set_active_sequence(nseq)
    finally:
        ctx.close()
        if own is not None:
            own.close()
        for o in osess:
            o.close()


def test_load_model_from_checkpoint_directory(L, tiny, tmp_path):
    """SURVEY 8f-1: model.LoadModel(modelDir) -- params.json + consolidated.00.pth go from the file mapping straight
    to HBM (lnb_model_load_pth) and the model is bit-identical to the one built from host tensors / the oracle"""
    import json
    from lnb_b200.torch_reader import TorchModelWriter, write_synthetic_checkpoint
    args, tensors, om, gm = tiny
    write_synthetic_checkpoint(str(tmp_path / "consolidated.00.pth"), L.synth.args_c(args), SEED)
    # a params.json that derives TINY's widths the reference's way: head_dim = dim / n_heads,
    # ffn = multiple_of * ceil(int(mult * int(2 * 4 dim / 3)) / multiple_of) = 256 * ceil(511 / 256) = 512
    (tmp_path / "params.json").write_text(json.dumps({
        "dim": args["dim"], "n_layers": args["n_layers"], "n_heads": args["n_heads"], "n_kv_heads": args["n_kv_heads"],
        "ffn_dim_multiplier": 0.75, "multiple_of": 256, "norm_eps": 1e-05, "rope_theta": 500000.0, "use_scaled_rope": True}))
    d = L.model.load_model_args(str(tmp_path), max_seq_len=args["max_seq_len"])
    assert d["ffn_dim"] == args["ffn_dim"] and d["head_dim"] == args["head_dim"] and d["vocab_size"] == -1
    m = L.model.LoadModel(str(tmp_path), max_seq_len=args["max_seq_len"])     # vocab from tok_embeddings rows
    try:
        assert m.ModelArgs.VocabSize == args["vocab_size"]
        toks = np.array([3, 77, 1000, 5, 9], np.int32)
        ctx = L.model.InferenceContext(m.Transformer, L.model.InferenceArgs(16), acc_mode=L._capi.LNB_ACC_STRICT)
        so = om.new_session(16)
        got = m.Transformer.Forward(ctx, L.ml.Tensor(toks, L.ml.DT_INT32), 0).RawData
        assert np.array_equal(got, so.forward(toks, 0))
        nxt, lg = m.Transformer.forward_argmax(ctx, np.array([int(np.argmax(got[-1]))], np.int32), 5, want_logits="last")
        assert np.array_equal(lg, so.forward(np.array([int(np.argmax(got[-1]))], np.int32), 5))
        ctx.close(); so.close()
    finally:
        m.Free()
    # a checkpoint with a missing tensor / a wrong shape / a non-bf16 tensor is refused the reference's way
    def variant(mutate):
        w = TorchModelWriter(str(tmp_path / "consolidated.00.pth"))
        for name, arr in tensors.items():
            r = mutate(name, arr)
            if r is not None:
                w.Add(name, *r)
        w.Finish()
    variant(lambda n, a: None if n == "layers.1.ffn_norm.weight" else (a,))
    with pytest.raises(L._capi.LnbError) as e:
        L.model.LoadModel(str(tmp_path), max_seq_len=args["max_seq_len"])
    assert "missing" in str(e.value)
    variant(lambda n, a: (a[:-1],) if n == "norm.weight" else (a,))
    with pytest.raises(L._capi.LnbError) as e:
        L.model.LoadModel(str(tmp_path), max_seq_len=args["max_seq_len"])
    assert "norm.weight" in str(e.value) and "shape" in str(e.value)
    variant(lambda n, a: (a.astype(np.float32),) if n == "norm.weight" else (a,))
    with pytest.raises(L._capi.LnbError) as e:
        L.model.LoadModel(str(tmp_path), max_seq_len=args["max_seq_len"])
    assert "float32" in str(e.value)


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_generate_tokens_batch_equals_per_prompt_generation(L, tiny, mode):
    """SURVEY 8f-4: the batched generate loop -- every prompt gets exactly the stream the single-prompt loop of
    generateTokensInternal gives it (oracle: orc_generate), with different prompt lengths and one sequence that
    stops early on an EOS id while the others run to SequenceLength"""
    args, _, om, gm = tiny
    prompts = [[1, 50, 999, 7, 300, 12, 64, 2], [5, 6, 7], [1000], [3, 3, 3, 3, 3]]
    seq = 24
    free = [list(om.generate(p, seq, stop_ids=(10**9,))) for p in prompts]
    stop = int(free[1][4])                                   # sequence 1 will hit it at its 5th token at the latest
    exp = [list(om.generate(p, seq, stop_ids=(stop,))) for p in prompts]
    assert len(exp[1]) <= 5 and any(len(e) == seq - len(p) for e, p in zip(exp, prompts))
    saved = gm.Vocabulary.StopTokenIds
    gm.Vocabulary.StopTokenIds = (stop,)
    try:
        acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=acc)
        got, last_state = [[] for _ in prompts], {}
        for i, state, tok in eng.GenerateTokensBatch(prompts):
            assert last_state.get(i, L.inference.GSInProgress) == L.inference.GSInProgress      # nothing after the end
            got[i].append(tok); last_state[i] = state
        if mode == "strict":
            assert got == exp
            for i, e in enumerate(exp):
                assert last_state[i] == (L.inference.GSFinishedByReachingEOS if e[-1] == stop else L.inference.GSFinishedByReachingSeqLen)
        else:   # FAST may flip a near-tie; the streams must at least be complete and well-formed
            assert all(len(g) >= 1 and s != L.inference.GSInProgress for g, s in zip(got, last_state.values()))
        one = [tok for _, _, tok in eng.GenerateTokensBatch([prompts[2]])]                       # n = 1 delegates
        assert mode != "strict" or one == exp[2]
        with pytest.raises(L.ml.MlError):
            list(eng.GenerateTokensBatch([list(range(seq))]))
    finally:
        gm.Vocabulary.StopTokenIds = saved


def test_captured_decode_graph_follows_active_sequence_and_layer_limit(L, tiny):
    """round-1 advisor finding: the decode graph bakes in the active sequence's cache pointers and the layer count;
    changing either must re-capture, not silently replay the first capture"""
    args, _, om, gm = tiny
    seq = 32
    prompts = [[1, 50, 999, 7], [3, 4, 5, 6, 7, 8]]
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=8, acc_mode=L._capi.LNB_ACC_STRICT, n_seq=2)
    try:
        firsts = []
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            first, _ = gm.Transformer.forward_argmax(ctx, np.array(p, np.int32), 0)
            firsts.append(first)
        for i, p in enumerate(prompts):                      # graph captured on sequence 0, then used on sequence 1
            ctx.set_active_sequence(i)
            toks, _, graphed = ctx.decode_run(firsts[i], len(p), 8, use_graph=True)
            assert graphed
            exp = list(om.generate(p, len(p) + 9, stop_ids=(10**9,)))
            assert [firsts[i]] + list(toks) == exp, f"sequence {i}"
        ctx.set_active_sequence(0)
        ctx.set_layer_limit(1)                               # one layer only: the graph path must agree with the eager path
        a, _, _ = ctx.decode_run(firsts[0], len(prompts[0]), 4, use_graph=True)
        b, _, _ = ctx.decode_run(firsts[0], len(prompts[0]), 4, use_graph=False)
        assert list(a) == list(b)
        ctx.set_layer_limit(0)
        c, _, _ = ctx.decode_run(firsts[0], len(prompts[0]), 8, use_graph=True)
        assert [firsts[0]] + list(c) == list(om.generate(prompts[0], len(prompts[0]) + 9, stop_ids=(10**9,)))
    finally:
        ctx.close()
    # single-GPU FAST sessions decode on the kernel chain, so decode_run replays the captured graph: under a layer limit
    # the replays must count the kernels the eager steps launch
    fast = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), acc_mode=L._capi.LNB_ACC_FAST)
    try:
        first, _ = gm.Transformer.forward_argmax(fast, np.array(prompts[0], np.int32), 0)
        assert not fast.uses_engine()
        fast.set_layer_limit(1)
        n0 = fast.launch_count()
        a, _, graphed = fast.decode_run(first, len(prompts[0]), 4, use_graph=True)
        n1 = fast.launch_count()
        b, _, _ = fast.decode_run(first, len(prompts[0]), 4, use_graph=False)
        assert graphed and list(a) == list(b)
        assert n1 - n0 == fast.launch_count() - n1
    finally:
        fast.close()


def test_forward_returns_a_device_handle_that_reads_like_the_host_tensor(L, tiny):
    """Transformer.Forward keeps the [S, vocab] logits in HBM (ml.DeviceLogits): Size / Slice / ml.Argmax work on the handle,
    RawData copies the rows out, and the handle dies with the context's next Forward (inference.go:202-216 never needs more)"""
    args, _, om, gm = tiny
    toks = np.array([1, 50, 999, 7, 300], np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(16), acc_mode=L._capi.LNB_ACC_STRICT)
    osess = om.new_session(16)
    try:
        exp = osess.forward(toks, 0, all_rows=True)
        lg = gm.Transformer.Forward(ctx, L.ml.Tensor(toks, L.ml.DT_INT32), 0)
        assert isinstance(lg, L.ml.DeviceLogits) and lg.Size == [5, args["vocab_size"]] and lg.on_device()
        last = lg.Slice([4], [5])
        assert last.Size == [1, args["vocab_size"]] and last.on_device()
        assert int(L.ml.Argmax(last, 1).Item()) == O.argmax_f32(exp[4])          # fused argmax of the kept last row
        mid = lg.Slice([1], [4])
        assert L.ml.Argmax(mid, 1).RawData.tolist() == [O.argmax_f32(exp[r]) for r in (1, 2, 3)]   # device argmax of kept rows
        assert np.array_equal(mid.RawData, exp[1:4]) and not mid.on_device()      # materialised on first touch
        assert np.array_equal(lg.RawData, exp)
        lg2 = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[:1] + 1, L.ml.DT_INT32), 5)
        stale = lg.Slice([0], [1])                                                # lg itself was read: still a host tensor
        assert np.array_equal(stale.RawData, exp[0:1])
        lg3 = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[:1] + 2, L.ml.DT_INT32), 6)
        with pytest.raises(L.ml.MlError):
            lg2.RawData                                                           # never read, and a newer Forward ran
        assert lg3.Size == [1, args["vocab_size"]]
        gm.Transformer.forward_argmax(ctx, toks[:1] + 3, 7, want_logits="last")  # any forward ends the handle
        c, out = L._capi, np.empty((1, args["vocab_size"]), np.float32)
        assert c.lib.lnb_session_logits_read(ctx.h, lg3.generation, 0, 1, c.ptr(out, c.f32p)) == -4    # LNB_ESTATE
    finally:
        ctx.close()
        osess.close()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_chunked_prefill_extension_equals_one_shot_prefill(L, tiny, mode):
    """SURVEY 8f-4 (beyond the reference): S > 1 at startPos > 0 with the [S,T] causal mask.  The library refuses it by
    default exactly like the reference's [S,S] mask would fail; with the switch on, a prompt fed in chunks leaves the caches
    and logits of the one-shot prefill (bit-identical in STRICT, and equal to the oracle's extension)."""
    check_chunked_prefill(L, tiny, mode)


def check_chunked_prefill(L, model, mode):
    args, _, om, gm = model
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    rng = np.random.default_rng(8)
    prompt = rng.integers(0, args["vocab_size"], size=19).astype(np.int32)
    seq = 40
    one = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=24, acc_mode=acc)
    chk = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=24, acc_mode=acc)
    o1, o2 = om.new_session(seq), om.new_session(seq)
    try:
        with pytest.raises(L._capi.LnbError, match="startPos 0"):
            gm.Transformer.forward_argmax(chk, prompt[8:12], 8)
        chk.allow_chunked_prefill(True)
        n1, l1 = gm.Transformer.forward_argmax(one, prompt, 0, want_logits="last")
        exp = o1.forward(prompt, 0, all_rows=False)
        pos = 0
        for size in (8, 5, 6):                                  # 8 + 5 + 6 = 19, unequal chunks
            n2, l2 = gm.Transformer.forward_argmax(chk, prompt[pos:pos + size], pos, want_logits="all")
            e2 = o2.forward(prompt[pos:pos + size], pos, all_rows=True) if pos == 0 else o2.forward_chunk(prompt[pos:pos + size], pos)
            if mode == "strict":
                assert np.array_equal(l2, e2), f"chunk at {pos}"
            else:
                assert float(np.abs(l2 - e2).max()) <= 1e-2
            pos += size
        if mode == "strict":
            assert np.array_equal(l2[-1:], l1) and np.array_equal(l1, exp) and n1 == n2      # chunked == one-shot == reference
            for layer in range(args["n_layers"]):
                assert np.array_equal(chk.CacheK(layer).RawData[:19], one.CacheK(layer).RawData[:19])
                assert np.array_equal(chk.CacheV(layer).RawData[:19], one.CacheV(layer).RawData[:19])
        # the generate loop with a chunked prompt emits the same stream (a prompt longer than max_rows becomes possible)
        eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=acc, max_rows=8)
        got = [t for _, t in eng.GenerateTokens(list(prompt), prefill_chunk=8)]
        if mode == "strict":
            assert got == list(om.generate(prompt, seq, stop_ids=gm.Vocabulary.StopTokenIds))
    finally:
        one.close(); chk.close(); o1.close(); o2.close()


# ---- the tensor-core prefill on a head_dim-128 miniature: gemm_tc_kernel + sdpa_tc_kernel inside a model forward --------

@pytest.fixture(scope="module")
def tiny128(L):
    """synth.TINY128: head_dim 128 and every tensor-core tiling condition of the prefill path (forward_tc_ok) hold, so a FAST
    prompt of >= 32 tokens runs gemm_tc_kernel for every projection and sdpa_tc_kernel for attention"""
    args = dict(L.synth.TINY128)
    tensors = host_tensors(args, SEED)
    om = oracle_model(args, tensors)
    gm = L.model.LoadModelFromTensors(args, tensors)
    yield args, tensors, om, gm
    gm.Free()
    om.close()


# Largest distance from the oracle of a FAST tensor-core prefill of tiny128, per element, in bf16 ulps of the element
# (of 2^-6 of the tensor's largest magnitude for smaller elements, where cancellation makes an ulp meaningless).
# The reorder noise is close to absolute (a few ulps of the tensor's large entries), so small elements show the most ulps.
# Pinned at about 1.5x the largest of S = 32, 129, 300 and both attention kernels, measured on an H100 SXM (80 GB):
# logits 105.5 (chunked prefill: 66), residual after layer 1 32, after the last layer 64, K/V caches 58, decode steps 86.25.
TC_ULPS = dict(logits=160, residual1=48, residual=96, cache=88, decode=128)


def _ulps(got, exp):
    g, e = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    floor = 2.0 ** -6 * max(np.abs(e).max(), 2.0 ** -100)
    return np.abs(g - e) / 2.0 ** (np.floor(np.log2(np.maximum(np.abs(e), floor))) - 7)


def _tc_launches(n_layers, S, all_rows):
    """kernels the tensor-core path (enqueue_forward_tc) launches for one forward on one GPU, plus the set_state_kernel of
    the call: gather_rows, then per layer rmsnorm_x8, gemm_tc (wq|wk|wv), rope_kv, the attention kernel of launch_attention,
    gemm_tc (wo + residual), rmsnorm_x8, gemm_tc (w1|w3 + SwiGLU), gemm_tc (w2 + residual); all-rows logits add
    rmsnorm_x8 + gemm_tc for rows < S - 1; the last row's LM head GEMV"""
    return 1 + 1 + 8 * n_layers + (2 if all_rows and S > 1 else 0) + 1


def _kernel_env(monkeypatch, kernel):
    if kernel == "sdpa_prefill":
        monkeypatch.setenv("LNB_SDPA_TC", "0")
    else:
        monkeypatch.delenv("LNB_SDPA_TC", raising=False)


def test_tiny128_prefill_runs_the_tensor_core_path(L, tiny128, monkeypatch):
    """the path the other tiny128 tests claim to cover is the one that runs: on the tensor-core path (enqueue_forward_tc),
    head_dim 128 selects the sdpa_tc_kernel branch of launch_attention, the launch count of one forward is that path's, and
    LNB_SDPA_TC=0 (sdpa_prefill_kernel) gives different bits"""
    args, _, _, gm = tiny128
    monkeypatch.delenv("LNB_SDPA_TC", raising=False)
    assert args["head_dim"] == 128
    q_l, kv_l = args["n_heads"] * 128, args["n_kv_heads"] * 128
    assert (q_l + 2 * kv_l) % 128 == 0 and args["dim"] % 128 == 0 and (2 * args["ffn_dim"]) % 128 == 0 and args["ffn_dim"] % 128 == 0
    toks = np.random.default_rng(3).integers(0, args["vocab_size"], size=300).astype(np.int32)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(320), max_rows=300, acc_mode=L._capi.LNB_ACC_FAST)
    try:
        for S, want in ((32, "all"), (129, "last"), (300, "all"), (200, "none")):
            n0 = ctx.launch_count()
            gm.Transformer.forward_argmax(ctx, toks[:S], 0, want_logits=want)
            assert ctx.launch_count() - n0 == _tc_launches(args["n_layers"], S, want == "all"), (S, want)
        ctx.set_layer_limit(1)
        n0 = ctx.launch_count()
        gm.Transformer.forward_argmax(ctx, toks[:64], 0, want_logits="all")
        assert ctx.launch_count() - n0 == _tc_launches(1, 64, True)
        ctx.set_layer_limit(0)
        _, a = gm.Transformer.forward_argmax(ctx, toks[:129], 0, want_logits="all")
        monkeypatch.setenv("LNB_SDPA_TC", "0")
        _, b = gm.Transformer.forward_argmax(ctx, toks[:129], 0, want_logits="all")
        assert not np.array_equal(a, b)
    finally:
        ctx.close()


@pytest.mark.parametrize("kernel", ["sdpa_tc", "sdpa_prefill"])
@pytest.mark.parametrize("S", [32, 129, 300])
def test_tiny128_fast_prefill_within_pinned_ulps_of_the_oracle(L, tiny128, S, kernel, monkeypatch):
    """one-shot FAST prefill at S = 32 (one tile of everything), 129 (one row past a 128-row tile) and 300 (three query
    tiles, five key tiles) against the oracle: logits of every row, the residual stream after layer 1 and after the last
    layer, both caches of every layer, and four decode steps on the caches the prefill wrote -- every element within
    TC_ULPS.  Measured on an H100 SXM, largest over both kernels (ulps): S = 32: logits 105.5, residual1 24, residual 50,
    cache 58, decode 86.25; S = 129: 52.5, 24, 64, 33, 64; S = 300: 70.1, 32, 64, 43, 79."""
    _kernel_env(monkeypatch, kernel)
    args, _, om, gm = tiny128
    rng = np.random.default_rng(S + 128)
    toks = rng.integers(0, args["vocab_size"], size=S + 4).astype(np.int32)
    osess = om.new_session(S + 4)
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(S + 4), max_rows=S, acc_mode=L._capi.LNB_ACC_FAST)
    one = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(S + 4), max_rows=S, acc_mode=L._capi.LNB_ACC_FAST)
    try:
        exp, tr = osess.forward(toks[:S], 0, all_rows=True, trace=True)
        nxt, got = gm.Transformer.forward_argmax(ctx, toks[:S], 0, want_logits="all")
        assert nxt == int(np.argmax(got[-1]))
        m = dict(logits=_ulps(got, exp).max(), residual=_ulps(f32(ctx.residual(S)), f32(tr[-1])).max(), cache=0.0, decode=0.0)
        for layer in range(args["n_layers"]):
            ok, ov = osess.cache(layer)
            m["cache"] = max(m["cache"], _ulps(f32(ctx.CacheK(layer).RawData[:S]), f32(ok[:S])).max(),
                             _ulps(f32(ctx.CacheV(layer).RawData[:S]), f32(ov[:S])).max())
        one.set_layer_limit(1)
        gm.Transformer.forward_argmax(one, toks[:S], 0)
        m["residual1"] = _ulps(f32(one.residual(S)), f32(tr[1])).max()
        for pos in range(S, S + 4):
            e = osess.forward(toks[pos:pos + 1], pos)
            g = gm.Transformer.Forward(ctx, L.ml.Tensor(toks[pos:pos + 1], L.ml.DT_INT32), pos).RawData
            m["decode"] = max(m["decode"], _ulps(g, e).max())
        print(f"tiny128 S={S} {kernel}: " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(m.items())))
        for k, v in m.items():
            assert v <= TC_ULPS[k], (k, v)
    finally:
        ctx.close(); one.close(); osess.close()


@pytest.mark.parametrize("kernel", ["sdpa_tc", "sdpa_prefill"])
@pytest.mark.parametrize("S1,S2", [(40, 300), (129, 200)])
def test_tiny128_prefill_rows_do_not_depend_on_later_rows(L, tiny128, S1, S2, kernel, monkeypatch):
    """prefill prompt[:S1] and prompt[:S2]: each row's GEMM and attention arithmetic is independent of the other rows (masked
    keys add exact zeros; Z is split over threads by absolute key index), so every layer's K/V rows < S1, the residual rows
    < S1 and the logits rows < S1 - 1 are bit-identical (row S1 - 1 of the shorter run comes from the LM-head GEMV)"""
    _kernel_env(monkeypatch, kernel)
    args, _, _, gm = tiny128
    toks = np.random.default_rng(S1 * S2).integers(0, args["vocab_size"], size=S2).astype(np.int32)
    a = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(S2), max_rows=S1, acc_mode=L._capi.LNB_ACC_FAST)
    b = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(S2), max_rows=S2, acc_mode=L._capi.LNB_ACC_FAST)
    try:
        _, la = gm.Transformer.forward_argmax(a, toks[:S1], 0, want_logits="all")
        _, lb = gm.Transformer.forward_argmax(b, toks, 0, want_logits="all")
        for layer in range(args["n_layers"]):
            assert np.array_equal(a.CacheK(layer).RawData[:S1], b.CacheK(layer).RawData[:S1]), f"K cache, layer {layer}"
            assert np.array_equal(a.CacheV(layer).RawData[:S1], b.CacheV(layer).RawData[:S1]), f"V cache, layer {layer}"
        assert np.array_equal(a.residual(S1), b.residual(S2)[:S1])
        assert np.array_equal(la[:S1 - 1], lb[:S1 - 1])
    finally:
        a.close(); b.close()


@pytest.mark.parametrize("kernel", ["sdpa_tc", "sdpa_prefill"])
def test_tiny128_chunked_fast_prefill_equals_one_shot(L, tiny128, kernel, monkeypatch):
    """a 300-token prompt in chunks of 40 + 100 + 33 + 127 (starts 0, 40, 140, 173: on and off multiples of 64 and 128, so
    the query tiles no longer line up with the key tiles) on the tensor-core path: caches and the residual are bit-identical
    to the one-shot prefill, and so are the logits except each earlier chunk's last row (GEMV there, GEMM in the one-shot
    run); every chunk is within TC_ULPS of the oracle's chunk extension"""
    _kernel_env(monkeypatch, kernel)
    args, _, om, gm = tiny128
    n = 300
    prompt = np.random.default_rng(77).integers(0, args["vocab_size"], size=n).astype(np.int32)
    one = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(n + 4), max_rows=n, acc_mode=L._capi.LNB_ACC_FAST)
    chk = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(n + 4), max_rows=127, acc_mode=L._capi.LNB_ACC_FAST)
    osess = om.new_session(n + 4)
    try:
        chk.allow_chunked_prefill(True)
        n1, l1 = gm.Transformer.forward_argmax(one, prompt, 0, want_logits="all")
        r1 = one.residual(n)
        pos, worst = 0, 0.0
        chunks = (40, 100, 33, 127)
        for i, size in enumerate(chunks):
            n2, l2 = gm.Transformer.forward_argmax(chk, prompt[pos:pos + size], pos, want_logits="all")
            last = i == len(chunks) - 1
            assert np.array_equal(l2 if last else l2[:-1], l1[pos:pos + size] if last else l1[pos:pos + size - 1]), f"chunk at {pos}"
            e2 = osess.forward(prompt[:size], 0, all_rows=True) if pos == 0 else osess.forward_chunk(prompt[pos:pos + size], pos)
            worst = max(worst, _ulps(l2, e2).max())
            pos += size
        assert n2 == n1
        assert np.array_equal(chk.residual(127), r1[n - 127:])
        for layer in range(args["n_layers"]):
            assert np.array_equal(chk.CacheK(layer).RawData[:n], one.CacheK(layer).RawData[:n]), f"K cache, layer {layer}"
            assert np.array_equal(chk.CacheV(layer).RawData[:n], one.CacheV(layer).RawData[:n]), f"V cache, layer {layer}"
        print(f"tiny128 chunked {kernel}: logits {worst:.2f} ulps from the oracle")
        assert worst <= TC_ULPS["logits"]
    finally:
        one.close(); chk.close(); osess.close()


@pytest.mark.parametrize("prompt_len", [1, 8])
def test_forward_strict_bit_exact_head_dim_128(L, tiny128, prompt_len):
    """test_forward_strict_bit_exact on tiny128: the persistent decode engine's head_dim-128 attention, bit for bit"""
    check_forward_strict(L, tiny128, prompt_len)


def test_chunked_prefill_strict_head_dim_128(L, tiny128):
    check_chunked_prefill(L, tiny128, "strict")
