"""Regex-constrained generation without a GPU (DESIGN.md §9g): the regex compiler (lnb_regex_dfa, csrc/regex.cpp) against
Python's re.fullmatch(p, s, re.ASCII) over UTF-8 encodings, on hand-written and random patterns; the DFA's shape (start
state, trimmed, minimal by a brute-force Moore minimisation); unsupported syntax and the state cap; and the grammar's C
statement (orc_grammar_masks, orc_grammar_history in oracle_sampling/lnb_sample_ref.c) against a Python restatement of
the contract of include/lnb.h on random DFAs and token tables."""
import random
import re
import zlib

import numpy as np
import pytest

from oracle_sampling import sample_ref as SR


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


# characters the strings are drawn from: ASCII (with \n, \t, space, metacharacters) and 2-, 3- and 4-byte code points at
# the UTF-8 length boundaries
POOL = (list("abcxyzAZ09_-.*+?()[]{}|^$\\/ \n\t\r\x0b\x0c\x00\x7f") +
        ["\x80", "é", "ß", "߿", "ࠀ", "中", "€", "퟿", "", "￿", "\U00010000", "😀", "\U0010ffff"])

HAND = [
    "", "a", "abc", "a|b|", "(yes|no|maybe)", "[0-9]{4}-[0-9]{2}-[0-9]{2}", r"\d+(\.\d+)?", r"-?\d{1,3}(,\d{3})*",
    "[a-c]+x?", "[^a-c]*", "[^\n]", ".", ".*", ".+é", "(é|ß)+", "中文{2,3}", "😀|\U0010ffff", r"\w+@\w+\.(com|org)",
    r"\s*\S+\s*", r"\D\W", r"[\d_x-z]+", r"[\s\w]", r"[^\W\d]+", "a{0}", "a{3}", "a{2,}", "a{1,4}b", "(ab|a)(bc|c)",
    "((a|b)c)*d", "(?:ab)+", "a*?b+?c??d{2,3}?", r"\.\*\+\?\(\)\[\]\{\}\|\\\^\$\-\/\ ", r"\x41é中", r"[\x00-\x1f]",
    r"[ࠀ-￿]", "[]a]", "[a-]", "[-a]", "x[^]]y", r"\n\t\r\f\v", "(a|)+", "()", "(a*)*", "(a|b)*a(a|b){3}",
    "[é-ü]+", "[😀-😂]", "[^😀]", "(x+x+)+y",
]


class _Gen:
    """random patterns of the supported grammar with a sampler of strings of their language"""

    ATOMS = ["a", "b", "x", r"\.", r"\-", "é", "中", "😀", r"\n", ".", r"\d", r"\w", r"\s", r"\D", r"\S", r"\W", "[a-c]",
             "[^ab]", r"[\d_x-z]", "[é中]", r"[^\w]", r"\x41", r"é"]

    def __init__(self, rng):
        self.rng = rng

    def atom(self):
        a = self.rng.choice(self.ATOMS)
        ok = [c for c in POOL if re.fullmatch(a, c, re.ASCII)]
        return a, (lambda: self.rng.choice(ok))

    def node(self, depth):
        r = self.rng.random()
        if depth <= 0 or r < 0.35:
            return self.atom()
        if r < 0.55:
            parts = [self.node(depth - 1) for _ in range(self.rng.randint(2, 3))]
            return "".join(p for p, _ in parts), (lambda: "".join(g() for _, g in parts))
        if r < 0.75:
            parts = [self.node(depth - 1) for _ in range(self.rng.randint(2, 3))]
            return "(" + "|".join(p for p, _ in parts) + ")", (lambda: self.rng.choice(parts)[1]())
        p, g = self.node(depth - 1)
        q = self.rng.choice(["*", "+", "?", "{2}", "{0,2}", "{1,}", "{1,3}"])
        lo, hi = {"*": (0, 3), "+": (1, 3), "?": (0, 1), "{2}": (2, 2), "{0,2}": (0, 2), "{1,}": (1, 3), "{1,3}": (1, 3)}[q]
        lazy = "?" if self.rng.random() < 0.2 else ""
        return "(?:" + p + ")" + q + lazy, (lambda: "".join(g() for _ in range(self.rng.randint(lo, hi))))


def _accepts(trans, accept, data: bytes) -> bool:
    q = 0
    for b in data:
        q = trans[q, b]
        if q < 0:
            return False
    return bool(accept[q])


def _random_unicode(rng, n):
    return "".join(rng.choice(POOL) for _ in range(n))


def _mutations(rng, s, k):
    out = []
    for _ in range(k):
        i = rng.randint(0, len(s))
        op = rng.randint(0, 2)
        if op == 0:
            out.append(s[:i] + rng.choice(POOL) + s[i:])
        elif s:
            i = min(i, len(s) - 1)
            out.append(s[:i] + (rng.choice(POOL) if op == 1 else "") + s[i + 1:])
    return out


def _check_language(L, pattern, samples, rng):
    trans, accept = L.model.regex_dfa(pattern)
    strings = list(samples)
    for s in samples:
        strings += _mutations(rng, s, 4)
    strings += [_random_unicode(rng, rng.randint(0, 6)) for _ in range(60)]
    for s in strings:
        exp = re.fullmatch(pattern, s, re.ASCII) is not None
        assert _accepts(trans, accept, s.encode("utf-8")) == exp, (pattern, s)
    return trans, accept


def _moore_states(trans, accept) -> int:
    """the number of states of the minimal DFA of (trans, accept), by brute-force Moore refinement with ⊥ as a sink"""
    Q = trans.shape[0]
    t = np.where(trans < 0, Q, trans)
    t = np.vstack([t, np.full((1, 256), Q, t.dtype)])
    cls = np.append(accept.astype(np.int64), 2)
    while True:
        sig = {}
        new = np.array([sig.setdefault((cls[q],) + tuple(cls[t[q]]), len(sig)) for q in range(Q + 1)])
        if len(sig) == len(set(cls.tolist())):
            return len(sig) - 1   # (without the sink)
        cls = new


def _check_shape(trans, accept):
    Q = trans.shape[0]
    assert accept.shape == (Q,) and Q >= 1
    assert ((trans >= -1) & (trans < Q)).all()
    seen, todo = {0}, [0]   # every state is reachable from state 0
    while todo:
        q = todo.pop()
        for r in set(trans[q].tolist()) - {-1} - seen:
            seen.add(r)
            todo.append(r)
    assert len(seen) == Q
    live = set(np.flatnonzero(accept).tolist())   # every state reaches F
    changed = True
    while changed:
        changed = False
        for q in range(Q):
            if q not in live and any(r in live for r in trans[q].tolist() if r >= 0):
                live.add(q)
                changed = True
    assert len(live) == Q
    assert _moore_states(trans, accept) == Q


@pytest.mark.parametrize("pattern", HAND)
def test_hand_patterns_match_python_re(L, pattern):
    rng = random.Random(zlib.crc32(pattern.encode()))
    samples = [s for s in (_random_unicode(rng, rng.randint(0, 4)) for _ in range(2000)) if re.fullmatch(pattern, s, re.ASCII)]
    samples += ["", "a", "ab", "abc", "yes", "no", "maybe", "2024-01-31", "1,234", "3.14", "x@y.org", "中文文", "😀", "\U0010ffff"]
    trans, accept = _check_language(L, pattern, samples, rng)
    _check_shape(trans, accept)


@pytest.mark.parametrize("seed", range(40))
def test_random_patterns_match_python_re(L, seed):
    rng = random.Random(seed)
    pattern, gen = _Gen(rng).node(3)
    samples = [gen() for _ in range(30)]
    for s in samples:
        assert re.fullmatch(pattern, s, re.ASCII), (pattern, s)   # the sampler draws from the language
    trans, accept = _check_language(L, pattern, samples, rng)
    _check_shape(trans, accept)


def test_invalid_utf8_is_never_accepted(L):
    bad = [b"\x80", b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xf0\x80\x80\x80",
           b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xff", b"\xc3", b"\xe4\xb8", b"\xf0\x9f\x98", b"a\x80b", b"\xc3\xa9\xa9"]
    for pattern in [".", ".*", "[^a]*", r"\D*", r"\W+", r"\S*", "(.|\n)*", "[\u0000-\U0010ffff]*"]:
        trans, accept = L.model.regex_dfa(pattern)
        for b in bad:
            assert not _accepts(trans, accept, b), (pattern, b)
        assert _accepts(trans, accept, "é中😀".encode()) == (re.fullmatch(pattern, "é中😀", re.ASCII) is not None)


# (pattern, byte offset the error names)
UNSUPPORTED = [("^a", 0), ("a$", 1), (r"a\b", 1), (r"\B", 0), (r"\Aa", 0), (r"a\Z", 1), (r"(a)\1", 3), (r"\0", 0),
               ("a(?=b)", 1), ("a(?!b)", 1), ("(?<=a)b", 0), ("(?i)a", 0), ("(?P<n>a)", 0), ("a**", 2), ("a*+", 2),
               ("a{2}{3}", 4), ("*a", 0), ("a|+", 2), ("(a", 0), ("a)", 1), ("[ab", 0), ("a{", 1), ("a{,3}", 1),
               ("a{3,2}", 1), ("a{x}", 1), (r"[\d-z]", 1), ("[z-a]", 1), (r"\q", 0), (r"\é", 0), (r"\x4", 0),
               (r"\u12", 0), ("\\", 0), (r"\N{DIGIT ONE}", 0), (r"\U0001F600", 0), (r"\a", 0)]


@pytest.mark.parametrize("pattern,offset", UNSUPPORTED)
def test_unsupported_syntax_is_einval_with_offset(L, pattern, offset):
    with pytest.raises(L._capi.LnbError) as ei:
        L.model.regex_dfa(pattern)
    assert ei.value.code == -1
    assert f"at byte offset {offset}" in str(ei.value), str(ei.value)


def test_invalid_utf8_pattern_and_empty_language(L):
    with pytest.raises(L._capi.LnbError, match="invalid UTF-8 at byte offset 1"):
        L.model.regex_dfa(b"a\xffb")
    with pytest.raises(L._capi.LnbError, match="matches no string"):
        L.model.regex_dfa(r"[^\x00-\U0010ffff]".encode().replace(b"\\U0010ffff", "\U0010ffff".encode()))


def test_nesting_limit(L):
    trans, accept = L.model.regex_dfa("(" * 1000 + "a" + ")" * 1000)
    assert trans.shape[0] == 2
    with pytest.raises(L._capi.LnbError, match="groups nested deeper than 1000 at byte offset 1000"):
        L.model.regex_dfa("(" * 200000 + "a" + ")" * 200000)
    with pytest.raises(L._capi.LnbError, match="nested deeper than 1000 at byte offset 3000"):
        L.model.regex_dfa("(?:" * 1001 + "a" + ")" * 1001)


def test_state_cap(L):
    trans, accept = L.model.regex_dfa("(a|b)*a(a|b){10}")
    assert trans.shape[0] == 2048
    with pytest.raises(L._capi.LnbError, match="8192 states, more than 4096") as ei:
        L.model.regex_dfa("(a|b)*a(a|b){12}")
    assert ei.value.code == -1
    with pytest.raises(L._capi.LnbError, match="repeat count above 100000"):
        L.model.regex_dfa("a{100001}")
    with pytest.raises(L._capi.LnbError, match="NFA states"):
        L.model.regex_dfa("(a{1000}){2000}")


# ---- the grammar's C statement against a Python restatement of the contract -------------------------------------------
def _py_walk(trans, q, b):
    for x in b:
        if q < 0:
            return -1
        q = int(trans[q, x])
    return q


def _py_mask(trans, accept, tok, stop, q):
    V = len(tok)
    m = np.zeros(V, bool)
    if q >= 0:
        for t in range(V):
            if t in stop:
                m[t] = bool(accept[q])
            else:
                m[t] = len(tok[t]) >= 1 and _py_walk(trans, q, tok[t]) >= 0
    if not m.any():
        m[list(stop)] = True
    return m


def _random_grammar(rng, Q, V):
    trans = np.full((Q, 256), -1, np.int32)
    alphabet = [ord(c) for c in "abcd"] + [0xC3, 0xA9]
    for q in range(Q):
        for b in alphabet:
            if rng.random() < 0.5:
                trans[q, b] = rng.randrange(Q)
    accept = np.array([rng.random() < 0.3 for _ in range(Q)], np.uint8)
    if rng.random() < 0.5:
        trans[Q - 1, :] = -1   # a dead end: stuck unless it accepts
        accept[Q - 1] = 0
    tok = []
    for t in range(V):
        n = rng.choice([0, 1, 1, 2, 3])
        tok.append(bytes(rng.choice(alphabet + [ord("z")]) for _ in range(n)))
    stop = sorted(rng.sample(range(V), rng.randint(1, min(3, V))))
    return trans, accept, tok, stop


@pytest.mark.parametrize("seed", range(12))
def test_statement_masks_and_history_match_restatement(seed):
    rng = random.Random(1000 + seed)
    Q, V = rng.randint(1, 9), rng.choice([1, 31, 32, 33, 70])
    trans, accept, tok, stop = _random_grammar(rng, Q, V)
    g = SR.GrammarTables(trans, accept, tok, stop)
    masks, stuck = SR.grammar_masks(g)
    W = (V + 31) // 32
    exp_stuck = 0
    for q in list(range(Q)) + [-1]:
        m = _py_mask(trans, accept, tok, set(stop), q)
        words = np.zeros(W, np.uint32)
        for t in np.flatnonzero(m):
            words[t >> 5] |= np.uint32(1 << (t & 31))
        assert (masks[q if q >= 0 else Q] == words).all(), (q, masks[q], words)
        if q >= 0 and not accept[q] and not any(m[t] and t not in stop for t in range(V)):
            exp_stuck += 1
    assert stuck == exp_stuck
    # histories: tokens drawn mostly from the mask (a generated stream), some forced from anywhere (an out-of-grammar
    # prompt or caller token), first_pos anywhere, including the middle of the tokens
    for _ in range(6):
        n = rng.randint(0, 12)
        first_pos = rng.randint(0, n + 1)
        toks, q = [], None
        for p in range(n):
            if p == first_pos:
                q = 0
            allowed = np.flatnonzero(_py_mask(trans, accept, tok, set(stop), q)) if q is not None else range(V)
            t = rng.choice(list(allowed)) if rng.random() < 0.8 else rng.randrange(V)
            toks.append(t)
            if q is not None:
                ok = t not in stop and len(tok[t]) >= 1 and _py_walk(trans, q, tok[t]) >= 0
                q = _py_walk(trans, q, tok[t]) if ok and q >= 0 else -1
        hist = SR.grammar_history(g, toks, first_pos)
        exp = [-1] * (n + 1)
        if first_pos <= n:
            exp[first_pos] = 0
            for p in range(first_pos, n):
                qq, t = exp[p], toks[p]
                ok = qq >= 0 and t not in stop and len(tok[t]) >= 1 and _py_walk(trans, qq, tok[t]) >= 0
                exp[p + 1] = _py_walk(trans, qq, tok[t]) if ok else -1
        assert hist.tolist() == exp, (toks, first_pos)
