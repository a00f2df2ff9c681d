"""Tree speculative decoding without a GPU: the tree drafter against a brute-force restatement and against its C++ twin, the
host loop's tree calls, emitted paths and stops against a fake context that records its calls, and the C-ABI entry's
binding."""
import os
import re
import subprocess

import numpy as np
import pytest


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def _tree_brute(h, max_nodes, branches, nmax, nmin):
    """the definition, literally: the continuations in preference order, distinct, at most `branches`; every distinct
    prefix of them is a node; nodes ordered by (depth, rank of the first continuation having that prefix), cut to max_nodes;
    a node's parent is the node of its prefix one shorter (the root, row 0, for depth 1)"""
    L_ = len(h)
    if max_nodes <= 0 or branches <= 0:
        return [], []
    conts = []
    for n in range(nmax, nmin - 1, -1):
        for j in reversed(range(L_)):
            if j + n < L_ and list(h[j:j + n]) == list(h[L_ - n:]):
                c = [int(t) for t in h[j + n:min(j + n + max_nodes, L_)]]
                if c not in conts and len(conts) < branches:
                    conts.append(c)
    keys = []
    for c in conts:
        for d in range(1, len(c) + 1):
            if tuple(c[:d]) not in keys:
                keys.append(tuple(c[:d]))
    rank = {k: min(r for r, c in enumerate(conts) if tuple(c[:len(k)]) == k) for k in keys}
    keys = sorted(keys, key=lambda k: (len(k), rank[k]))[:max_nodes]
    toks = [k[-1] for k in keys]
    par = [0 if len(k) == 1 else 1 + keys.index(k[:-1]) for k in keys]
    return toks, par


def _random_history(rng, seed):
    n = int(rng.integers(0, 40))
    alphabet = int(rng.integers(1, 5)) if seed % 2 else int(rng.integers(2, 40))
    return [int(t) for t in rng.integers(0, alphabet, size=n)]


@pytest.mark.parametrize("seed", range(6))
def test_tree_drafter_equals_brute_force(L, seed):
    rng = np.random.default_rng(100 + seed)
    for _ in range(300):
        h = _random_history(rng, seed)
        mn, br, nmax = int(rng.integers(0, 9)), int(rng.integers(1, 6)), int(rng.integers(1, 5))
        nmin = int(rng.integers(1, nmax + 1))
        toks, par = L.inference.prompt_lookup_tree(h, mn, br, nmax, nmin)
        assert (toks, par) == _tree_brute(h, mn, br, nmax, nmin), (h, mn, br, nmax, nmin)
        assert len(toks) == len(par) <= max(mn, 0)                       # the budget
        for i, p in enumerate(par):
            assert 0 <= p <= i                                            # row i + 1's parent precedes it
        sib = [(p, t) for p, t in zip(par, toks)]
        assert len(set(sib)) == len(sib)                                  # siblings carry distinct tokens
        if br == 1:
            d = L.inference.prompt_lookup_drafts(h, mn, nmax, nmin)
            assert toks == d and par == list(range(len(d)))


def test_tree_drafter_examples(L):
    t = L.inference.prompt_lookup_tree
    # "1 2" is followed by 3 (j = 4, most recent) and by 9 (j = 0); the trigram never matches
    h = [1, 2, 9, 7, 1, 2, 3, 5, 1, 2]
    assert t(h, 8, 1) == ([3, 5, 1, 2], [0, 1, 2, 3])
    assert t(h, 8, 2) == ([3, 9, 5, 7, 1, 1, 2, 2], [0, 0, 1, 2, 3, 4, 5, 6])
    assert t(h, 3, 2) == ([3, 9, 5], [0, 0, 1])                         # breadth first: both branches survive the cut
    assert t(h, 0, 4) == ([], []) and t([4], 5, 3) == ([], [])
    # the bigram "6 1" matches at j = 4 and j = 1; the unigram's matches repeat those continuations (kept once)
    assert t([5, 6, 1, 8, 6, 1, 9, 6, 1], 4, 3, 2, 1) == ([9, 8, 6, 6], [0, 0, 1, 2])


def test_tree_drafter_cpp_twin(L, tmp_path):
    """model::PromptLookupTree (host/lnb_host.hpp) equals prompt_lookup_tree on random histories"""
    root = os.path.join(os.path.dirname(__file__), "..")
    src = tmp_path / "tree.cpp"
    src.write_text(r'''
#include "lnb_host.hpp"
#include <iostream>
int main() {
  int n;
  while (std::cin >> n) {
    std::vector<int32_t> h(n);
    for (auto& x : h) std::cin >> x;
    int mn, br, nmax, nmin;
    std::cin >> mn >> br >> nmax >> nmin;
    std::vector<int32_t> t, p;
    lnb_host::model::PromptLookupTree(h, mn, br, nmax, nmin, t, p);
    std::cout << t.size();
    for (size_t i = 0; i < t.size(); i++) std::cout << ' ' << t[i] << ' ' << p[i];
    std::cout << '\n';
  }
}
''')
    exe = tmp_path / "tree"
    subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-I", os.path.join(root, "host"), "-I", os.path.join(root, "include"),
                           str(src), "-o", str(exe), "-ldl"])
    rng = np.random.default_rng(7)
    cases, lines = [], []
    for k in range(2000):
        h = _random_history(rng, k)
        mn, br, nmax = int(rng.integers(0, 9)), int(rng.integers(1, 6)), int(rng.integers(1, 5))
        nmin = int(rng.integers(1, nmax + 1))
        cases.append((h, mn, br, nmax, nmin))
        lines.append(" ".join(map(str, [len(h)] + h + [mn, br, nmax, nmin])))
    out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.split("\n")
    for (h, mn, br, nmax, nmin), line in zip(cases, out):
        v = [int(x) for x in line.split()]
        toks, par = L.inference.prompt_lookup_tree(h, mn, br, nmax, nmin)
        assert v[0] == len(toks) and v[1::2] == toks and v[2::2] == par, (h, mn, br, nmax, nmin)


class FakeTreeContext:
    """'model': the token at position p of sequence i is tok(i, p).  forward_speculative_tree checks the call like the
    C-ABI (row budget, parents, distinct siblings, the slot bound) and returns every row's prediction (the token after its
    path), the accepted depths and paths."""

    def __init__(self, seq_len, max_rows, tok):
        self.SequenceLength, self.max_rows, self.tok = seq_len, max_rows, tok
        self.calls = []

    def forward_speculative(self, segs):
        raise AssertionError("Branches > 1 issues tree calls only")

    def forward_speculative_tree(self, segs):
        rows = sum(len(t) for _, _, t, _ in segs)
        assert rows <= min(8, self.max_rows)
        out, acc, paths = [], [], []
        for s, p, t, par in segs:
            assert len(par) == len(t)
            assert p + len(t) - 1 < self.SequenceLength - 1, "a slot past the last position the plain loop feeds"
            depth = [0]
            for j in range(1, len(t)):
                assert 0 <= par[j] < j
                depth.append(depth[par[j]] + 1)
            kids = [(par[j], t[j]) for j in range(1, len(t))]
            assert len(set(kids)) == len(kids)
            nxt = [self.tok(s, p + 1 + depth[j]) for j in range(len(t))]
            u, path = 0, [0]
            while True:
                c = [j for j in range(1, len(t)) if par[j] == u and t[j] == nxt[u]]
                if not c:
                    break
                u = c[0]
                path.append(u)
            out += nxt
            acc.append(len(path) - 1)
            paths.append(path)
        self.calls.append([(s, p, list(t), list(par)) for s, p, t, par in segs])
        return np.array(out, np.int32), np.array(acc, np.int32), paths, None


def _engine(L, stop_id=999):
    class M:
        Vocabulary = L.model.Vocabulary(StopTokenIds=(stop_id,))
    return L.inference.InferenceEngine(M, L.model.InferenceArgs(0))


def _plain(i, start, seq_len, tok, stop_id=999):
    out = []
    for pos in range(start, seq_len):
        out.append(tok(i, pos))
        if out[-1] == stop_id:
            break
    return out


@pytest.mark.parametrize("branches", [2, 4])
@pytest.mark.parametrize("max_draft", [1, 3, 7])
def test_tree_loop_emits_the_plain_streams(L, branches, max_draft):
    """three sequences: one whose history repeats "a b" with two continuations (the second branch is the right one), one
    that stops on the stop id inside an accepted path, one of random tokens; every stream equals the plain one, each call is
    the drafter's tree and the emitted tokens follow the accepted path"""
    rng = np.random.default_rng(max_draft * 10 + branches)
    rnd = rng.integers(0, 900, size=200)
    seq_len = 60

    def tok(i, p):
        if i == 0:
            return [40, 41, 43][p % 3]
        if i == 1:
            return 999 if p == 33 else 20 + p % 3
        return int(rnd[p])

    prompts = [[40, 41, 42, 7, 40, 41, 43, 40, 41], [20, 21, 22, 20, 21, 22, 20], [int(t) for t in rnd[:6]]]
    eng = _engine(L)
    ctx = FakeTreeContext(seq_len, 8, tok)
    hists = [p + [tok(i, len(p))] for i, p in enumerate(prompts)]
    stats, times = [], []
    spec = L.inference.SpeculativeArgs(max_draft, Branches=branches)
    out = list(eng._generate_speculative(ctx, hists, [0, 1, 2], spec, times, stats))
    streams = {i: [] for i in range(3)}
    last = {}
    for i, state, t in out:
        assert last.get(i, L.inference.GSInProgress) == L.inference.GSInProgress
        streams[i].append(t)
        last[i] = state
    for i, p in enumerate(prompts):
        assert [hists[i][len(p)]] + streams[i] == _plain(i, len(p), seq_len, tok), i
    assert last[1] == L.inference.GSFinishedByReachingEOS
    assert last[0] == last[2] == L.inference.GSFinishedByReachingSeqLen
    assert len(stats) == len(times) == len(ctx.calls)
    pos = {i: len(p) for i, p in enumerate(prompts)}
    for call in ctx.calls:
        left = 8 - len(call)
        for s, p, t, par in call:
            assert p == pos[s] and t[0] == hists[s][p]
            want = L.inference.prompt_lookup_tree(hists[s][:p + 1], min(max_draft, left, seq_len - 2 - p), branches)
            assert (t[1:], par[1:]) == want
            left -= len(want[0])
            a = 0
            u = 0
            while True:
                c = [j for j in range(1, len(t)) if par[j] == u and t[j] == tok(s, p + 1 + a)]
                if not c:
                    break
                u, a = c[0], a + 1
            pos[s] = p + a + 1
    if max_draft >= 3:
        assert max(a for _, a in stats) >= 2, "the repeating sequence must accept a path through its second branch"


def test_tree_loop_stops_inside_an_accepted_path(L):
    """the stop id sits in the middle of an accepted path: the tokens after it are not emitted"""
    eng = _engine(L)
    tok = lambda i, p: 999 if p == 12 else 5 + p % 2   # noqa: E731
    ctx = FakeTreeContext(40, 8, tok)
    hists = [[5 + p % 2 for p in range(10)]]          # fed next: position 9; positions 10, 11, 12 (stop) follow
    out = list(eng._generate_speculative(ctx, hists, [0], L.inference.SpeculativeArgs(7, Branches=2)))
    assert [t for _, _, t in out] == [tok(0, p) for p in range(10, 13)]
    assert out[-1][1] == L.inference.GSFinishedByReachingEOS
    assert len(ctx.calls) == 1


def test_branches_one_issues_chain_calls(L):
    """Branches = 1 keeps today's calls: forward_speculative with prompt_lookup_drafts"""
    from tests.test_speculative_cpu import FakeSpecContext
    eng = _engine(L)
    ctx = FakeSpecContext(30, 8, lambda i, p: 1 + p % 3)
    list(eng._generate_speculative(ctx, [[1 + p % 3 for p in range(9)]], [0], L.inference.SpeculativeArgs(5, Branches=1)))
    assert ctx.calls and all(len(seg) == 3 for c in ctx.calls for seg in c)


def test_tree_argument_errors(L):
    class M:
        Vocabulary = L.model.Vocabulary()
    eng = L.inference.InferenceEngine(M, L.model.InferenceArgs(16))
    tree = L.inference.SpeculativeArgs(4, Branches=2)
    with pytest.raises(L.ml.MlError):
        list(eng.GenerateTokens([1], speculative=L.inference.SpeculativeArgs(4, Branches=0)))
    for kw in (dict(penalties=L.model.PenaltyArgs(RepetitionPenalty=1.3)), dict(logprobs=2), dict(grammar=object())):
        with pytest.raises(L.ml.MlError, match="not built"):
            list(eng.GenerateTokens([1], speculative=tree, **kw))
        with pytest.raises(L.ml.MlError, match="not built"):
            list(eng.GenerateTokensBatch([[1], [2]], speculative=tree, **kw))


def test_forward_speculative_tree_symbol_is_declared_and_bound(L):
    c = L._capi
    hdr = open(os.path.join(os.path.dirname(__file__), "..", "include", "lnb.h")).read()
    assert re.search(r"int lnb_forward_speculative_tree\(lnb_session\* s, int n_segs, const int32_t\* seq, const int32_t\* start_pos, "
                     r"const int32_t\* n_nodes,\s+const int32_t\* parent, const int32_t\* tokens, float\* logits, int32_t\* next_out, "
                     r"int32_t\* n_accepted,\s+int32_t\* path_out\);", hdr)
    assert "lnb_forward_speculative_tree" in c.SIGNATURES
    z = np.zeros(1, np.int32)
    p = c.ptr(z, c.i32p)
    assert c.lib.lnb_forward_speculative_tree(None, 1, p, p, p, p, p, None, None, None, None) == -1
    assert b"NULL" in c.lib.lnb_last_error()
