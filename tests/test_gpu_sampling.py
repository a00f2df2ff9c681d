"""Seeded sampling on the device (csrc/sample.cuh, DESIGN.md §9b) against its sequential C statement
(oracle_sampling/lnb_sample_ref.c): the op bit-exact on any row, STRICT sampled streams token for token equal to the oracle's
generate loop on every path (host loop, decode run with and without graph, batch, continuous batching, engine session),
FAST sampled tokens equal to the statement applied to the logits the GPU returned, greedy sessions unchanged, validation."""
import ctypes as C

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

SEED = 1234
ARGS = (0.8, 40, 0.95, 77)       # Temperature, TopK, TopP, Seed


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


def _op(L, rows, params, pos):
    rows = np.ascontiguousarray(rows, np.float32)
    n, V = rows.shape
    p = (L._capi.SamplingC * n)(*[L._capi.SamplingC(float(t), int(k), float(q), int(s) & (2**64 - 1)) for t, k, q, s in params])
    pn = np.ascontiguousarray(pos, np.int32)
    out = np.empty(n, np.int32)
    L._capi.check(L._capi.lib.lnb_op_sample_f32(L._capi.ptr(rows, L._capi.f32p), n, V, p, L._capi.ptr(pn, L._capi.i32p),
                                                L._capi.ptr(out, L._capi.i32p)))
    return out


def _grid_rows(rng, V):
    from tests.test_sampling_cpu import _rows
    return list(_rows(rng, V).values())


@pytest.mark.parametrize("V", [67, 1000, 1025, 3001])
def test_op_bit_exact_on_the_cpu_grid(L, V):
    rng = np.random.default_rng(V)
    rows = _grid_rows(rng, V)
    todo = []
    for r in rows:
        for T in (1e-3, 0.7, 1.0, 5.0):
            for K in (0, 1, 2, 40, V - 1, V):
                for P in (1e-6, 0.5, 0.9, 1.0):
                    todo.append((r, (T, K, P, int(rng.integers(0, 2**63))), int(rng.integers(1, 10**6))))
    for j in range(0, len(todo), 8):
        chunk = todo[j:j + 8]
        got = _op(L, np.stack([c[0] for c in chunk]), [c[1] for c in chunk], [c[2] for c in chunk])
        for g, (r, (T, K, P, s), pn) in zip(got, chunk):
            assert g == SR.sample_row(r, T, K, P, s, pn), (V, T, K, P, s, pn)


def test_op_bit_exact_at_the_8b_vocabulary(L):
    V = 128256
    rng = np.random.default_rng(7)
    rows = rng.normal(0.0, 3.0, (8, V)).astype(np.float32)
    rows[3, ::7] = rows[3].max()                     # ties at the top
    params = [(0.8, 40, 0.95, 1), (1.0, 0, 1.0, 2), (0.7, 0, 0.9, 3), (1.5, 1000, 1.0, 4), (0.0, 0, 1.0, 5), (5.0, 0, 0.5, 6),
              (1e-3, 2, 1.0, 7), (1.0, V - 1, 0.99, 8)]
    pos = [9, 100, 4000, 77, 5, 131071, 1, 2]
    got = _op(L, rows, params, pos)
    for i in range(8):
        assert got[i] == SR.sample_row(rows[i], *params[i], pos[i]), i


def _sampling(L, a=ARGS, seed_off=0):
    return L.model.SamplingArgs(a[0], a[1], a[2], a[3] + seed_off)


def _eng(L, gm, seq_len, mode, max_rows=8):
    acc = L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST
    return L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq_len), acc_mode=acc, max_rows=max_rows)


PROMPTS = [[1, 50, 999, 7, 300, 12, 64, 2], [5, 6], [900, 3, 4, 17, 22], [8]]


def test_strict_generate_equals_oracle(L, model):
    args, _, om, gm = model
    eng = _eng(L, gm, 40, "strict")
    for i, p in enumerate(PROMPTS[:3]):
        exp = list(SR.generate_sampled(om, p, 40, *ARGS[:3], ARGS[3] + i, stop_ids=(10**9,)))
        got = [t for _, t in eng.GenerateTokens(p, sampling=_sampling(L, seed_off=i))]
        assert got == exp, i
    # a stream that stops on an EOS id: make the 5th sampled token a stop id
    exp = list(SR.generate_sampled(om, PROMPTS[0], 40, *ARGS, stop_ids=(10**9,)))
    stop = exp[4]

    saved = gm.Vocabulary

    class V:
        StopTokenIds = (stop,)
        PadId = saved.PadId
    gm.Vocabulary = V
    try:
        got = list(eng.GenerateTokens(PROMPTS[0], sampling=_sampling(L)))
    finally:
        gm.Vocabulary = saved
    want = list(SR.generate_sampled(om, PROMPTS[0], 40, *ARGS, stop_ids=(stop,)))
    assert [t for _, t in got] == want and got[-1][0] == L.inference.GSFinishedByReachingEOS


def test_strict_decode_run_equals_host_loop(L, model):
    args, _, om, gm = model
    exp = list(SR.generate_sampled(om, PROMPTS[0], 40, *ARGS, stop_ids=(10**9,)))
    for graph in (True, False):
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), acc_mode=L._capi.LNB_ACC_STRICT)
        try:
            ctx.set_sampling(0, _sampling(L))
            first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPTS[0], np.int32), 0)
            toks, _, used = ctx.decode_run(first, 8, 20, use_graph=graph)
            assert used == graph
            assert [first] + list(toks) == exp[:21]
            if ctx.uses_engine():
                assert b"kernel chain" in L._capi.lib.lnb_last_error()
            # again from the same state: the replayed graph reads the (unchanged) parameters from the device
            toks2, _, _ = ctx.decode_run(first, 8, 20, use_graph=graph)
            assert list(toks2) == list(toks)
        finally:
            ctx.close()


def test_strict_batch_and_continuous_equal_per_prompt_streams(L, model):
    args, _, om, gm = model
    prompts = [PROMPTS[i % 4] + [i + 1] * (i % 3) for i in range(11)]
    exp = {i: list(SR.generate_sampled(om, p, 24, *ARGS[:3], ARGS[3] + i, stop_ids=(10**9,))) for i, p in enumerate(prompts)}
    eng = _eng(L, gm, 24, "strict")
    got = {}
    for i, _, t in eng.GenerateTokensBatch(prompts[:4], sampling=_sampling(L)):
        got.setdefault(i, []).append(t)
    assert got == {i: exp[i] for i in range(4)}
    got = {}
    for i, _, t in eng.GenerateTokensContinuous(prompts, slots=4, step_tokens=12, sampling=_sampling(L)):
        got.setdefault(i, []).append(t)
    assert got == exp


def test_engine_session_s1_forward_samples(L, model):
    args, _, om, gm = model
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), acc_mode=L._capi.LNB_ACC_STRICT)
    try:
        if not ctx.uses_engine():
            pytest.skip("this session's S=1 steps use the kernel chain")
        osess = om.new_session(40)
        ctx.set_sampling(0, _sampling(L))
        lo = osess.forward(np.array(PROMPTS[0], np.int32), 0, all_rows=False)[0]
        tok, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPTS[0], np.int32), 0)
        assert tok == SR.sample_row(lo, *ARGS, 8)
        for pos in range(8, 14):
            lo = osess.forward(np.array([tok], np.int32), pos, all_rows=False)[0]
            nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), pos, want_logits="last")
            assert np.array_equal(lg[0], lo)
            assert nxt == SR.sample_row(lo, *ARGS, pos + 1)
            tok = nxt
        osess.close()
    finally:
        ctx.close()


def test_fast_every_path_samples_the_logits_it_returned(L, model):
    args, _, om, gm = model
    acc = L._capi.LNB_ACC_FAST
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), max_rows=16, acc_mode=acc, n_seq=3)
    try:
        for k in range(3):
            ctx.set_sampling(k, _sampling(L, seed_off=k))
        toks, pos = [], []
        for k in range(3):   # single-sequence forwards (prefill) on each sequence
            ctx.set_active_sequence(k)
            p = np.array(PROMPTS[k], np.int32)
            nxt, lg = gm.Transformer.forward_argmax(ctx, p, 0, want_logits="last")
            assert nxt == SR.sample_row(lg[0], *ARGS[:3], ARGS[3] + k, len(p))
            toks.append(nxt); pos.append(len(p))
        for _ in range(4):   # batched steps
            nxt, lg = ctx.forward_batch(toks, pos, want_logits=True)
            for k in range(3):
                assert nxt[k] == SR.sample_row(lg[k], *ARGS[:3], ARGS[3] + k, pos[k] + 1)
            toks = [int(t) for t in nxt]; pos = [p + 1 for p in pos]
        for _ in range(3):   # ragged steps: two decode rows and one two-token chunk
            segs = [(0, pos[0], [toks[0]]), (2, pos[2], [toks[2]]), (1, pos[1], [toks[1], 5])]
            nxt, lg = ctx.forward_ragged(segs, want_logits=True)
            for j, (k, s, t) in enumerate(segs):
                assert nxt[j] == SR.sample_row(lg[j], *ARGS[:3], ARGS[3] + k, s + len(t))
            toks = [int(nxt[0]), int(nxt[2]), int(nxt[1])]
            pos = [pos[0] + 1, pos[1] + 2, pos[2] + 1]
        ctx.set_active_sequence(0)   # single decode: sampled from the kept logits row
        nxt, lg = gm.Transformer.forward_argmax(ctx, np.array([toks[0]], np.int32), pos[0], want_logits="last")
        assert nxt == SR.sample_row(lg[0], *ARGS, pos[0] + 1)
    finally:
        ctx.close()


def test_greedy_unchanged_after_a_cleared_sampler(L, model):
    args, _, om, gm = model
    for mode in (L._capi.LNB_ACC_STRICT, L._capi.LNB_ACC_FAST):
        runs = []
        for sample_first in (False, True):
            ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), acc_mode=mode)
            try:
                if sample_first:
                    ctx.set_sampling(0, _sampling(L))
                    ctx.set_sampling(0, None)
                first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPTS[0], np.int32), 0)
                toks, _, _ = ctx.decode_run(first, 8, 12, use_graph=True)
                nxt, _ = gm.Transformer.forward_argmax(ctx, np.array([toks[-1]], np.int32), 20)
                runs.append(([first] + list(toks) + [nxt], ctx.launch_count()))
            finally:
                ctx.close()
        assert runs[0] == runs[1]
        if mode == L._capi.LNB_ACC_STRICT:
            assert runs[0][0][:13] == list(om.generate(PROMPTS[0], 40, stop_ids=(10**9,)))[:13]


def test_only_the_sampled_sequence_of_a_batch_changes(L, model):
    args, _, om, gm = model
    for mode in (L._capi.LNB_ACC_STRICT, L._capi.LNB_ACC_FAST):
        outs = []
        for samp in (False, True):
            ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), acc_mode=mode, n_seq=3)
            try:
                if samp:
                    ctx.set_sampling(1, L.model.SamplingArgs(5.0, 0, 1.0, 3))
                toks, pos = [], []
                for k in range(3):
                    ctx.set_active_sequence(k)
                    nxt, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPTS[k], np.int32), 0)
                    toks.append(nxt); pos.append(len(PROMPTS[k]))
                seqs = [[t] for t in toks]
                for _ in range(6):
                    nxt, _ = ctx.forward_batch(toks, pos)
                    for k in range(3):
                        seqs[k].append(int(nxt[k]))
                    toks = [int(t) for t in nxt]; pos = [p + 1 for p in pos]
                outs.append(seqs)
            finally:
                ctx.close()
        assert outs[0][0] == outs[1][0] and outs[0][2] == outs[1][2]
        assert outs[0][1] != outs[1][1]   # temperature 5 over the whole vocabulary leaves greedy at once


def test_logits_argmax_stays_greedy(L, model):
    args, _, om, gm = model
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), acc_mode=L._capi.LNB_ACC_STRICT)
    try:
        ctx.set_sampling(0, L.model.SamplingArgs(5.0, 0, 1.0, 11))
        p = np.array(PROMPTS[0], np.int32)
        tok, gen = C.c_int32(-1), C.c_int64(0)
        L._capi.check(L._capi.lib.lnb_forward_device(ctx.h, L._capi.ptr(p, L._capi.i32p), len(p), 0, 1, C.byref(tok), C.byref(gen)))
        lo = om.new_session(40)
        exp = lo.forward(p, 0, all_rows=False)[0]
        lo.close()
        greedy = np.empty(1, np.int32)
        L._capi.check(L._capi.lib.lnb_session_logits_argmax(ctx.h, gen.value, 0, 1, L._capi.ptr(greedy, L._capi.i32p)))
        assert greedy[0] == int(np.argmax(exp))
        assert tok.value == SR.sample_row(exp, 5.0, 0, 1.0, 11, 8)
    finally:
        ctx.close()


def test_validation_leaves_the_session_usable(L, model):
    args, _, om, gm = model
    lib = L._capi.lib
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(40), acc_mode=L._capi.LNB_ACC_STRICT, n_seq=2)
    try:
        S = L._capi.SamplingC
        bad = [(0, S(float("nan"), 0, 1.0, 1)), (0, S(float("inf"), 0, 1.0, 1)), (0, S(-0.5, 0, 1.0, 1)), (0, S(1.0, -1, 1.0, 1)),
               (0, S(1.0, 0, 0.0, 1)), (0, S(1.0, 0, 1.5, 1)), (0, S(1.0, 0, float("nan"), 1)), (2, S(1.0, 0, 1.0, 1)),
               (-1, S(1.0, 0, 1.0, 1))]
        for seq, p in bad:
            assert lib.lnb_session_set_sampling(ctx.h, seq, C.byref(p)) == -1, (seq, p.temperature, p.top_k, p.top_p)
        first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPTS[0], np.int32), 0)
        assert first == list(om.generate(PROMPTS[0], 40, stop_ids=(10**9,)))[0]   # still greedy
    finally:
        ctx.close()


def test_8b_strict_sampled_decode_equals_oracle(L):
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
        exp = list(SR.generate_sampled(om, prompt, 8 + 16, 0.8, 40, 0.95, 2024, stop_ids=(10**9,)))
        ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(136), max_rows=8, acc_mode=L._capi.LNB_ACC_STRICT)
        try:
            ctx.set_sampling(0, L.model.SamplingArgs(0.8, 40, 0.95, 2024))
            first, _ = gm.Transformer.forward_argmax(ctx, prompt, 0)
            toks, _, _ = ctx.decode_run(first, 8, 15, use_graph=True)
            assert [first] + list(toks) == exp
        finally:
            ctx.close()
    finally:
        gm.Free()
        om.close()


def test_cpp_cli_samples_like_the_python_stream(L):
    """host/lnb_generate temp= top_k= top_p= seed= (tiny, STRICT): single, batch and continuous streams = the oracle's"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])
    flags = ["temp=0.8", "top_k=40", "top_p=0.95", "seed=77"]
    args = dict(L.synth.TINY)
    om = oracle_model(args, host_tensors(args, 7))
    base = [1, 50, 999, 7, 300, 12, 64, 2]
    try:
        out = subprocess.run([exe, "24", "strict", "tiny"] + flags, capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        line = [ln for ln in out.stdout.splitlines() if ln.startswith("tokens:")][0]
        assert [int(t) for t in line.split()[1:]] == list(SR.generate_sampled(om, base, 24, 0.8, 40, 0.95, 77, stop_ids=(10**9,)))
        for extra in (["batch=3"], ["batch=5", "slots=2"]):
            out = subprocess.run([exe, "24", "strict", "tiny"] + extra + flags, capture_output=True, text=True, timeout=120)
            assert out.returncode == 0, out.stderr
            for b in range(int(extra[0][6:])):
                prompt = [base[0]] + [(t + 977 * b) % 1000 for t in base[1:]]
                line = [ln for ln in out.stdout.splitlines() if ln.startswith(f"tokens[{b}]:")][0]
                exp = list(SR.generate_sampled(om, prompt, 24, 0.8, 40, 0.95, 77 + b, stop_ids=(10**9,)))
                assert [int(t) for t in line.split()[1:]] == exp, (extra, b)
    finally:
        om.close()
