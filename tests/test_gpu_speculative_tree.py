"""Tree speculative verification (lnb_forward_speculative_tree).  Every row of a tree call must carry the bits of the last
row of lnb_forward_speculative over its path (root .. row as a chain) on the same session state, the walk must follow the
rows' next tokens, and after the call the cache rows start .. start + a must equal those the chain call over the accepted
path leaves -- on every route, in STRICT and FAST, on bf16 and MXFP8 caches and weights."""
import itertools
import os
import subprocess

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import engine_shapes as ES
from tests import model_shapes as MS
from tests.helpers import host_tensors, oracle_model

pytestmark = pytest.mark.gpu

PROMPT = [1, 50, 999, 7, 300, 12, 64, 2]
SAMPLING = (0.8, 40, 0.95, 77)
NO_STOP = (10**9,)


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _load(L, args, weight_format="bf16"):
    tensors = host_tensors(args, 4321)
    return args, oracle_model(args, tensors), L.model.LoadModelFromTensors(args, tensors, weight_format=weight_format)


_MODELS = {}


@pytest.fixture(scope="module")
def models(L):
    yield _MODELS
    for args, om, gm in _MODELS.values():
        gm.Free(); om.close()
    _MODELS.clear()


def _model(L, models, name):
    if name not in models:
        import torch
        if name == "wide":
            args = ES.wide_args(torch.cuda.get_device_properties(0).multi_processor_count)
        elif name in MS.CATALOGUE:
            args = dict(MS.CATALOGUE[name])
        else:
            args = dict(getattr(L.synth, name.upper().replace("_MX8", "")))
        models[name] = _load(L, args, "mxfp8" if name.endswith("_mx8") else "bf16")
    return models[name]


def _acc(L, mode):
    return L._capi.LNB_ACC_STRICT if mode == "strict" else L._capi.LNB_ACC_FAST


def _ctx(L, gm, seq, acc, n_seq=1, kv_format="bf16"):
    ctx = L.model.InferenceContext(gm.Transformer, L.model.InferenceArgs(seq), max_rows=8, acc_mode=acc, n_seq=n_seq,
                                   kv_format=kv_format)
    return ctx


def all_trees(max_rows):
    """every recursive tree of 1 .. max_rows rows: parent[j] in [0, j) (parent[0] = -1)"""
    for n in range(1, max_rows + 1):
        for par in itertools.product(*[range(j) for j in range(1, n)]):
            yield [-1] + list(par)


def random_trees(rng, n, count):
    return [[-1] + [int(rng.integers(0, j)) for j in range(1, n)] for _ in range(count)]


def _path(par, j):
    p = [j]
    while p[-1] > 0:
        p.append(par[p[-1]])
    return p[::-1]


def _cache_rows(ctx, layer, p, n, kv_format):
    if kv_format == "mxfp8":
        return [x for w in ("k", "v") for x in ctx.kv_read(0, layer, w, p, n)]
    return [ctx.CacheK(layer).RawData[p:p + n].copy(), ctx.CacheV(layer).RawData[p:p + n].copy()]


class TreeChecker:
    """checks tree calls on sequence 0 of ctx at position p (rows [0, p) hold the prompt): the chain calls run on the same
    sequence first (they only write rows >= p), then the tree call"""

    def __init__(self, L, args, ctx, p, root, kv_format="bf16", rng=None):
        self.L, self.args, self.ctx, self.p, self.root, self.kv = L, args, ctx, p, root, kv_format
        self.rng = rng or np.random.default_rng(0)
        self.chain = {}

    def chain_call(self, toks):
        key = tuple(toks)
        if key not in self.chain:
            nxt, na, lg = self.ctx.forward_speculative([(0, self.p, list(toks))], want_logits=True)
            self.chain[key] = (nxt.copy(), lg.copy())
        return self.chain[key]

    def tokens_for(self, par):
        """tokens of the tree: each node either carries its parent's predicted next token (an acceptable branch) or a
        random one, siblings distinct"""
        V = self.args["vocab_size"]
        toks = [self.root]
        for j in range(1, len(par)):
            pt = [toks[r] for r in _path(par, par[j])]
            want = int(self.chain_call(pt)[0][-1])
            sib = {toks[k] for k in range(1, j) if par[k] == par[j]}
            t = want if (want not in sib and self.rng.random() < 0.6) else int(self.rng.integers(0, V))
            while t in sib:
                t = (t + 1) % V
            toks.append(t)
        return toks

    def check(self, par, layers):
        n = len(par)
        toks = self.tokens_for(par)
        # expected rows: the chain over each row's path (the root: row 0 of a two-row chain when there is one, so every
        # expected row comes from the same route as the tree call)
        exp_next, exp_lg = [], []
        for j in range(n):
            path = _path(par, j) if (j > 0 or n == 1) else [0, 1]
            nxt, lg = self.chain_call([toks[r] for r in path])
            k = len(_path(par, j)) - 1
            exp_next.append(int(nxt[k])); exp_lg.append(lg[k])
        walk = [0]
        while True:
            c = [j for j in range(1, n) if par[j] == walk[-1] and toks[j] == exp_next[walk[-1]]]
            if not c:
                break
            walk.append(c[0])
        a = len(walk) - 1
        acc_path = walk if (a > 0 or n == 1) else [0, 1]
        l0 = self.ctx.launch_count()
        self.ctx.forward_speculative([(0, self.p, [toks[r] for r in acc_path])])
        chain_launches = self.ctx.launch_count() - l0
        want_cache = {l: _cache_rows(self.ctx, l, self.p, a + 1, self.kv) for l in layers}
        if len(acc_path) != n:      # the launches of a chain call of n rows (the tree call's row count)
            l0 = self.ctx.launch_count()
            self.ctx.forward_speculative([(0, self.p, toks)])
            chain_launches = self.ctx.launch_count() - l0
        l0 = self.ctx.launch_count()
        nxt, na, paths, lg = self.ctx.forward_speculative_tree([(0, self.p, toks, par)], want_logits=True)
        launches = self.ctx.launch_count() - l0
        branching = any(par[j] != j - 1 for j in range(1, n))
        assert launches == chain_launches + (1 if branching else 0), (par, launches, chain_launches)
        assert [int(x) for x in nxt] == exp_next, par
        for j in range(n):
            assert np.array_equal(lg[j], exp_lg[j]), (par, j)
        assert list(na) == [a] and paths == [walk], (par, list(na), paths, walk)
        for l in layers:
            got = _cache_rows(self.ctx, l, self.p, a + 1, self.kv)
            assert all(np.array_equal(x, y) for x, y in zip(got, want_cache[l])), (par, l)
        return a


def _prefilled(L, gm, seq, acc, kv_format="bf16"):
    ctx = _ctx(L, gm, seq, acc, kv_format=kv_format)
    first, _ = gm.Transformer.forward_argmax(ctx, np.array(PROMPT, np.int32), 0)
    return ctx, int(first)


# ---- 1. every tree shape up to 6 rows, random trees of 7 and 8 --------------------------------------------------------
@pytest.mark.parametrize("model", ["tiny", "tiny128", "wide"])
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_every_tree_shape(L, models, model, mode):
    args, om, gm = _model(L, models, model)
    ctx, first = _prefilled(L, gm, 64, _acc(L, mode))
    try:
        rng = np.random.default_rng(11)
        tc = TreeChecker(L, args, ctx, len(PROMPT), first, rng=rng)
        layers = (0, args["n_layers"] - 1)
        accepted = [tc.check(par, layers) for par in list(all_trees(6)) + random_trees(rng, 7, 6) + random_trees(rng, 8, 6)]
        assert max(accepted) >= 3
    finally:
        ctx.close()


# ---- 2. routes, shapes and formats ------------------------------------------------------------------------------------
ROUTES = ["engine_limit", "batch_engine_off", "past_engine_limit", "streamed", "batch_tc", "gqa8", "hd96", "kv_mxfp8",
          "weights_mxfp8"]


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_routes(L, models, monkeypatch, route, mode):
    monkeypatch.delenv("LNB_BATCH_ENGINE", raising=False)
    monkeypatch.delenv("LNB_BATCH_TC", raising=False)
    name = {"gqa8": "gqa8", "hd96": "hd96", "weights_mxfp8": "tiny_mx8"}.get(route, "tiny128")
    args, om, gm = _model(L, models, name)
    lim = ES.max_seq_len(args)
    seq, kv = 64, "bf16"
    if route == "engine_limit":
        seq = lim
    elif route == "batch_engine_off":
        monkeypatch.setenv("LNB_BATCH_ENGINE", "0")
    elif route == "past_engine_limit":
        seq = lim + 1
    elif route == "streamed":
        seq = MS.sdpa_decode_fit(args) + 1
    elif route == "batch_tc":
        if mode == "strict":
            pytest.skip("LNB_BATCH_TC selects the FAST batch engine's tensor-core form")
        monkeypatch.setenv("LNB_BATCH_TC", "1")
    elif route == "kv_mxfp8":
        kv = "mxfp8"
    ctx, first = _prefilled(L, gm, seq, _acc(L, mode), kv)
    try:
        rng = np.random.default_rng(5)
        p = seq - 10 if route in ("engine_limit", "past_engine_limit", "streamed") else len(PROMPT)
        tok = first
        if p > len(PROMPT):                  # walk the prompt's continuation up to p with plain steps
            for q in range(len(PROMPT), p):
                tok, _ = gm.Transformer.forward_argmax(ctx, np.array([tok], np.int32), q)
                tok = int(tok)
        tc = TreeChecker(L, args, ctx, p, tok, kv, rng)
        layers = (0, args["n_layers"] - 1)
        trees = list(all_trees(4)) + random_trees(rng, 6, 3) + random_trees(rng, 8, 4)
        assert max(tc.check(par, layers) for par in trees) >= 2
    finally:
        ctx.close()


# ---- 3. several segments ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_three_segments(L, models, mode):
    """three sequences with different trees (a chain, a branching tree, a lone root) in one call equal each segment alone"""
    args, om, gm = _model(L, models, "tiny")
    acc, seq = _acc(L, mode), 48
    prompts = [PROMPT, [5, 6, 7], [9] * 6]
    ctx = _ctx(L, gm, seq, acc, n_seq=3)
    try:
        firsts = []
        for i, p in enumerate(prompts):
            ctx.set_active_sequence(i)
            firsts.append(int(gm.Transformer.forward_argmax(ctx, np.array(p, np.int32), 0)[0]))
        ctx.set_active_sequence(0)
        V = args["vocab_size"]
        # each sequence's own single-segment tree calls first (at the same positions: the later call overwrites the rows)
        n2, _, _ = ctx.forward_speculative([(2, len(prompts[2]), [firsts[2]])])
        n0, _, _ = ctx.forward_speculative([(0, len(prompts[0]), [firsts[0]])])
        segs = [(2, len(prompts[2]), [firsts[2], int(n2[0]), 17 % V], [-1, 0, 1]),
                (0, len(prompts[0]), [firsts[0], (int(n0[0]) + 1) % V, int(n0[0]), 3 % V], [-1, 0, 0, 2]),
                (1, len(prompts[1]), [firsts[1]], [-1])]
        alone = [ctx.forward_speculative_tree([s], want_logits=True) for s in segs]
        nxt, na, paths, lg = ctx.forward_speculative_tree(segs, want_logits=True)
        r0 = 0
        for k, (nx, a, pa, lga) in enumerate(alone):
            n = len(segs[k][2])
            assert list(nxt[r0:r0 + n]) == list(nx) and na[k] == a[0] and paths[k] == pa[0], k
            assert all(np.array_equal(lg[r0 + j], lga[j]) for j in range(n)), k
            r0 += n
        assert na[1] >= 1 and paths[1][1] == 2          # sequence 0 accepted through its second branch
    finally:
        ctx.close()


# ---- 4. streams -------------------------------------------------------------------------------------------------------
def _set_stop(gm, saved, stop):
    class V:
        StopTokenIds = (stop,)
        PadId = saved.PadId
    gm.Vocabulary = V


@pytest.mark.parametrize("branches", [2, 4])
@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("sampled", [False, True])
def test_generate_streams(L, models, branches, mode, sampled):
    """GenerateTokens and GenerateTokensBatch with spec=7 and Branches: the plain streams (STRICT: the oracle's)"""
    args, om, gm = _model(L, models, "tiny128")
    seq = 56
    eng = L.inference.InferenceEngine(gm, L.model.InferenceArgs(seq), acc_mode=_acc(L, mode), max_rows=24)
    sp = L.model.SamplingArgs(*SAMPLING) if sampled else None
    spec = L.inference.SpeculativeArgs(7, Branches=branches)
    saved = gm.Vocabulary
    rep = [3, 14, 15, 92, 65, 3, 14, 15, 7, 8, 3, 14, 15, 92]
    try:
        _set_stop(gm, saved, NO_STOP[0])
        for prompt in (rep, PROMPT):
            plain = [t for _, t in eng.GenerateTokens(prompt, sampling=sp)]
            stats = []
            got = [t for _, t in eng.GenerateTokens(prompt, sampling=sp, speculative=spec, spec_stats=stats)]
            assert got == plain
            if mode == "strict":
                exp = SR.generate_sampled(om, prompt, seq, *SAMPLING, stop_ids=NO_STOP) if sampled else \
                    om.generate(prompt, seq, stop_ids=NO_STOP)
                assert plain == list(exp)
        bprompts = [rep, PROMPT, [5, 6]]
        want, got = {}, {}
        for i, _, t in eng.GenerateTokensBatch(bprompts, sampling=sp):
            want.setdefault(i, []).append(t)
        for i, _, t in eng.GenerateTokensBatch(bprompts, sampling=sp, speculative=spec):
            got.setdefault(i, []).append(t)
        assert got == want
    finally:
        gm.Vocabulary = saved


# ---- 5. refusals ------------------------------------------------------------------------------------------------------
def test_refusals_enqueue_nothing(L, models):
    args, om, gm = _model(L, models, "tiny")
    c = L._capi
    seq = 24
    ctx = _ctx(L, gm, seq, c.LNB_ACC_STRICT, n_seq=2)
    ref = _ctx(L, gm, seq, c.LNB_ACC_STRICT)
    try:
        prompt = PROMPT[:5]
        first = int(gm.Transformer.forward_argmax(ctx, np.array(prompt, np.int32), 0)[0])
        ctx.set_penalties(1, L.model.PenaltyArgs(RepetitionPenalty=1.3), 0)
        base = ctx.launch_count()
        V, p = args["vocab_size"], len(prompt)

        def call(segs):
            seq_ = np.array([s[0] for s in segs], np.int32)
            st = np.array([s[1] for s in segs], np.int32)
            nn = np.array([len(s[2]) - 1 for s in segs], np.int32)
            tk = np.array([t for s in segs for t in s[2]], np.int32)
            pa = np.array([q for s in segs for q in s[3]], np.int32)
            out = np.zeros(16, np.int32)
            return c.lib.lnb_forward_speculative_tree(ctx.h, len(segs), *[c.ptr(x, c.i32p) for x in (seq_, st, nn, pa, tk)], None,
                                                      c.ptr(out, c.i32p), c.ptr(out, c.i32p), c.ptr(out, c.i32p))
        bad = [
            [],                                                       # n_segs < 1
            [(0, p, [1, 2, 3], [-1, 0, 2])],                          # parent[j] == j
            [(0, p, [1, 2, 3], [-1, 0, 5])],                          # parent[j] > j
            [(0, p, [1, 2, 3], [-1, -1, 0])],                         # parent[j] < 0
            [(0, p, [1, 2, 2], [-1, 0, 0])],                          # siblings with one token
            [(0, seq - 2, [1, 2, 3], [-1, 0, 0])],                    # slot start + n_nodes == seq_len
            [(0, p, [1] + list(range(2, 10)), [-1] + [0] * 8)],       # 9 rows > 8
            [(0, p, [1, V], [-1, 0])],                                # token id out of range
            [(0, p, [1, 2], [-1, 0]), (0, p, [1], [-1])],             # repeated sequence
            [(1, p, [1, 2, 3], [-1, 0, 0])],                          # a branching tree on a penalized sequence
        ]
        for b in bad:
            assert call(b) == -1, b
        assert b"not built" in c.lib.lnb_last_error()
        assert ctx.launch_count() == base, "an invalid call enqueued work"
        want, lw = gm.Transformer.forward_argmax(ref, np.array(prompt, np.int32), 0)
        w2, lw2 = gm.Transformer.forward_argmax(ref, np.array([want], np.int32), p, want_logits="last")
        g2, lg2 = gm.Transformer.forward_argmax(ctx, np.array([first], np.int32), p, want_logits="last")
        assert first == want and g2 == w2 and np.array_equal(lg2, lw2)
    finally:
        ctx.close(); ref.close()


# ---- 6. the 8B model --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def m8b(L):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GB of free HBM")
    gm = L.model.LoadSyntheticModel(dict(L.synth.LLAMA31_8B), seed=L.synth.SEED)
    yield gm
    gm.Free()


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_8b_branching_call_near_position_1000(L, m8b, mode):
    gm = m8b
    args = dict(L.synth.LLAMA31_8B)
    seq = 1040
    ctx = _ctx(L, gm, seq, _acc(L, mode))
    try:
        rng = np.random.default_rng(3)
        prompt = [int(t) for t in rng.integers(0, args["vocab_size"], size=1000)]
        ctx.allow_chunked_prefill(True)
        for q in range(0, 1000, 8):
            tok, _ = gm.Transformer.forward_argmax(ctx, np.array(prompt[q:q + 8], np.int32), q)
        tc = TreeChecker(L, args, ctx, 1000, int(tok), rng=rng)
        tc.check([-1, 0, 0, 1, 1, 2, 3, 3], (0, args["n_layers"] - 1))
    finally:
        ctx.close()


# ---- 7. the CLI -------------------------------------------------------------------------------------------------------
def test_cli_tree_prints_the_plain_run(L):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "host", "lnb_generate")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(root, "host"), "-s"])

    def ids(flags):
        out = subprocess.run([exe, "40", "strict", "tiny"] + flags, capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        lines = [ln for ln in out.stdout.splitlines() if ln.startswith("tokens")]
        assert lines, out.stdout
        return lines
    plain = ids([])
    assert ids(["spec=7", "branches=4"]) == plain
    assert ids(["spec=7", "branches=2", "batch=3"]) == ids(["batch=3"])
