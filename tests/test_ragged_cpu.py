"""Continuous batching without a GPU: the scheduler of InferenceEngine.GenerateTokensContinuous against a fake context that
records its calls, and the C-ABI entry's NULL check."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


class FakeContext:
    """records every call; the 'model' emits token (7 * position + sequence-independent salt) % 1000, the stop id at
    positions listed in `stop_at` of a prompt"""

    def __init__(self, seq_len, max_rows, slots, prompts, stop_at, stop_id):
        self.SequenceLength, self.max_rows, self.slots = seq_len, max_rows, slots
        self.prompts, self.stop_at, self.stop_id = prompts, stop_at, stop_id
        self.calls = []          # ("ragged", [(slot, start, tokens)], owners) / ("batch", tokens, positions, owners)
        self.cache = [[] for _ in range(slots)]   # tokens each slot's cache holds, by position

    def _token(self, slot, pos):
        pi = self.owner[slot]
        return self.stop_id if pos in self.stop_at.get(pi, ()) else (7 * pos + 3 * pi + 1) % 1000

    def _write(self, slot, start, toks):
        c = self.cache[slot]
        if start == 0:
            c.clear()
            self.owner[slot] = next(i for i, p in enumerate(self.prompts) if i not in self.started and list(p[:len(toks)]) == list(toks))
            self.started.add(self.owner[slot])
        assert len(c) == start, "positions must continue the cache"
        c.extend(int(t) for t in toks)

    def forward_ragged(self, segs):
        out = []
        for s, p, t in segs:
            self._write(s, p, t)
            out.append(self._token(s, p + len(t)))
        self.calls.append(("ragged", [(s, p, list(t)) for s, p, t in segs], dict(self.owner)))
        return np.array(out, np.int32), None

    def forward_batch(self, tokens, positions):
        self.calls.append(("batch", list(tokens), list(positions), dict(self.owner)))
        for k, (t, p) in enumerate(zip(tokens, positions)):
            if p > 0 and p == len(self.cache[k]):     # a decoding row (free slots are fed token 0 at position 0)
                self.cache[k].append(int(t))
        return np.array([self._token(k, positions[k] + 1) if k in self.owner else 0 for k in range(len(tokens))], np.int32), None


def _run(L, prompts, slots, budget, seq_len, stop_at, stop_id=999):
    class M:   # the engine only reads model.Vocabulary
        Vocabulary = L.model.Vocabulary(StopTokenIds=(stop_id,))
    eng = L.inference.InferenceEngine(M, L.model.InferenceArgs(seq_len))
    ctx = FakeContext(seq_len, budget, slots, prompts, stop_at, stop_id)
    ctx.owner, ctx.started = {}, set()
    out = list(eng._generate_continuous(ctx, prompts, slots, budget))
    return ctx, out


@pytest.mark.parametrize("slots,budget", [(4, 48), (2, 8), (1, 5), (8, 64)])
def test_continuous_scheduler_policy(L, slots, budget):
    rng = np.random.default_rng(slots * budget)
    lens = [1, 70, 7, 33, 2, 48, 15, 64, 5, 29, 11]
    seq_len = 96
    prompts = [list(rng.integers(0, 900, size=n)) for n in lens]
    stop_at = {2: {10}, 6: {15}}     # prompt 2 stops on the EOS id at position 10, prompt 6 on its first token
    ctx, out = _run(L, prompts, slots, budget, seq_len, stop_at)
    GS = L.inference
    # all prompts finished, nothing after the end, each stream is what the single-prompt loop would emit
    streams = {i: [] for i in range(len(prompts))}
    states = {}
    for i, state, tok in out:
        assert states.get(i, GS.GSInProgress) == GS.GSInProgress
        streams[i].append(tok)
        states[i] = state
    for i, p in enumerate(prompts):
        exp = []
        for pos in range(len(p), seq_len):
            tok = 999 if pos in stop_at.get(i, ()) else (7 * pos + 3 * i + 1) % 1000
            exp.append(tok)
            if tok == 999:
                break
        assert streams[i] == exp, i
        assert states[i] == (GS.GSFinishedByReachingEOS if exp[-1] == 999 else GS.GSFinishedByReachingSeqLen)
    # call by call: within budget, at most one segment per slot, every decoding sequence in every step, chunks in order
    decoding = {}    # slot -> next position it decodes at
    fed = {}         # slot -> prompt tokens fed so far
    for call in ctx.calls:
        if call[0] == "batch":
            _, toks, poss, owner = call
            assert len(toks) <= slots
            assert all(poss[k] == decoding[k] for k in decoding)   # no decoding sequence skipped
            assert not fed, "a step with prompt rows waiting must not be decode-only"
            for k in list(decoding):
                decoding[k] += 1
        else:
            segs, owner = call[1], call[2]
            slots_in = [s for s, _, _ in segs]
            assert len(set(slots_in)) == len(slots_in) and all(0 <= s < slots for s in slots_in)
            assert sum(len(t) for _, _, t in segs) <= budget
            assert set(decoding) <= set(slots_in), "a decoding sequence was skipped"
            for s, p, t in segs:
                if s in decoding:
                    assert p == decoding[s] and len(t) == 1
                    decoding[s] += 1
                else:
                    assert p == fed.get(s, 0), "chunks at contiguous positions; a refilled slot starts at 0"
                    fed[s] = p + len(t)
        # retire finished slots / promote prefilled ones, as the scheduler does after the step
        for s in list(fed):
            pi = owner[s]
            if fed[s] == len(prompts[pi]):
                del fed[s]
                decoding[s] = len(prompts[pi])
        for s in list(decoding):
            last = decoding[s]       # position of the token just produced
            if last in stop_at.get(owner[s], ()) or last + 1 == seq_len:
                del decoding[s]
    assert not decoding and not fed


def test_continuous_scheduler_fifo_and_refill(L):
    """prompt chunks are served first in, first out, and a finished slot is refilled at position 0 by the next prompt"""
    prompts = [[1] * 30, [2] * 30, [3] * 4]
    ctx, _ = _run(L, prompts, slots=2, budget=16, seq_len=40, stop_at={})
    first = ctx.calls[0][1]
    assert [(s, p, len(t)) for s, p, t in first] == [(0, 0, 16)]           # prompt 0 takes the whole budget
    second = ctx.calls[1][1]
    assert [(s, p, len(t)) for s, p, t in second] == [(0, 16, 14), (1, 0, 2)]
    refills = [c for c in ctx.calls if c[0] == "ragged" and any(t[:1] == [3] and p == 0 for _, p, t in c[1])]
    assert len(refills) == 1


def test_continuous_rejects_bad_arguments(L):
    class M:
        Vocabulary = L.model.Vocabulary()
    eng = L.inference.InferenceEngine(M, L.model.InferenceArgs(16))
    with pytest.raises(L.ml.MlError):
        list(eng.GenerateTokensContinuous([[1]], slots=9))
    with pytest.raises(L.ml.MlError):
        list(eng.GenerateTokensContinuous([[1]], slots=4, step_tokens=3))
    ctx = FakeContext(16, 8, 2, [], {}, 999)
    with pytest.raises(L.ml.MlError):
        list(eng._generate_continuous(ctx, [list(range(16))], 2, 8))
    with pytest.raises(L.ml.MlError):
        list(eng._generate_continuous(ctx, [[]], 2, 8))


def test_forward_ragged_null_session_is_einval(L):
    c = L._capi
    seq = np.zeros(1, np.int32)
    assert c.lib.lnb_forward_ragged(None, 1, c.ptr(seq, c.i32p), c.ptr(seq, c.i32p), c.ptr(seq + 1, c.i32p), c.ptr(seq, c.i32p),
                                    None, None) == -1
    assert b"NULL" in c.lib.lnb_last_error()
