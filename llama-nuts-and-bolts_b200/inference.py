"""Host mirror of the reference's generate loop, src/inference/inference.go:173-254
(`generateTokensInternal`): prefill the prompt at position 0, then one token per Forward,
greedy argmax of the last row, stop on EOS / SequenceLength.  The loop stays on the host like
the Go original; each iteration is one call through the C-ABI.
"""
from __future__ import annotations

import collections
import math
import time
from dataclasses import dataclass

import numpy as np

from . import ml, model as model_mod

GSInProgress, GSFinishedByReachingEOS, GSFinishedByReachingSeqLen = 0, 1, 2
SamplingArgs = model_mod.SamplingArgs
PenaltyArgs = model_mod.PenaltyArgs


@dataclass
class SpeculativeArgs:
    """EXTENSION: speculative decoding (lnb_forward_speculative).  Each call feeds a sequence's last token plus up to MaxDraft
    tokens drafted by prompt lookup (prompt_lookup_drafts, n-grams of NgramMax down to NgramMin tokens) and keeps the drafts
    the model agrees with.  Every verified row has the bits of the plain step, so the generated stream is the plain one.
    Branches > 1: each call verifies a tree of up to MaxDraft nodes holding the top Branches distinct continuations
    (prompt_lookup_tree, lnb_forward_speculative_tree) and keeps its longest path the model agrees with; not with
    penalties, a grammar or logprobs.  Branches = 1 issues exactly the chain calls."""
    MaxDraft: int
    NgramMax: int = 3
    NgramMin: int = 1
    Branches: int = 1


@dataclass
class BeamSearchArgs:
    """EXTENSION: beam search (DESIGN.md §9f).  NumBeams B in [1, 8] hypotheses advance together, one lnb_forward_batch
    per step; a hypothesis of raw score s (the f64 sum of its tokens' logprobs) and n generated tokens ranks by
    h = s / n ** LengthPenalty.  EarlyStopping ends the search as soon as B hypotheses have finished; otherwise it ends when
    no live beam can beat the worst finished one.  GenerateBeams returns the NumReturn (1 .. B) best."""
    NumBeams: int
    LengthPenalty: float = 1.0
    EarlyStopping: bool = False
    NumReturn: int = 1


@dataclass
class BeamHypothesis:
    """one result of GenerateBeams: the generated tokens, their raw score s, h = s / len(Tokens) ** LengthPenalty, each
    token's logprob, and the state that ended it (GSFinishedByReachingEOS or GSFinishedByReachingSeqLen)"""
    Tokens: list
    Score: float
    NormalizedScore: float
    Logprobs: list
    State: int


def beam_order(x: float) -> tuple:
    """sort key of a score, best first: descending, -inf after every finite score, NaN last"""
    return (1, 0.0) if math.isnan(x) else (0, -x)


def beam_normalized(s: float, n: int, alpha: float) -> float:
    """h = s / n ** alpha (libm pow)"""
    return s / math.pow(float(n), alpha)


def beam_select(cands, B: int, stop) -> tuple[list, list]:
    """The selection of one beam step.  cands: (score, beam, rank, token).  Sorted by score (beam_order), then beam, then
    rank; walking the list with index i, a stop token goes to `finished` when i < B (skipped otherwise), any other token
    becomes the next new beam until B exist.  Returns (new beams, finished), each a list of candidates in walk order."""
    order = sorted(cands, key=lambda c: (beam_order(c[0]), c[1], c[2]))
    new, finished = [], []
    for i, c in enumerate(order):
        if len(new) == B:
            break
        if c[3] in stop:
            if i < B:
                finished.append(c)
        else:
            new.append(c)
    return new, finished


class BeamPool:
    """the finished hypotheses: the best B by h, ties won by the earlier insertion"""

    def __init__(self, B: int):
        self.B, self.items, self.n_ins = B, [], 0

    def _worst(self) -> int:
        return max(range(len(self.items)), key=lambda j: (beam_order(self.items[j][0].NormalizedScore), self.items[j][1]))

    def add(self, hyp: BeamHypothesis):
        entry = (hyp, self.n_ins)
        self.n_ins += 1
        if len(self.items) < self.B:
            self.items.append(entry)
            return
        w = self._worst()
        if beam_order(hyp.NormalizedScore) < beam_order(self.items[w][0].NormalizedScore):
            self.items[w] = entry

    def full(self) -> bool:
        return len(self.items) == self.B

    def worst_h(self) -> float:
        return self.items[self._worst()][0].NormalizedScore

    def result(self) -> list:
        return [h for h, _ in sorted(self.items, key=lambda e: (beam_order(e[0].NormalizedScore), e[1]))]


# Rows of one speculative call (the batch engine serves at most 8 rows per launch).
SPEC_MAX_ROWS = 8


def prompt_lookup_drafts(history, max_draft: int, ngram_max: int = 3, ngram_min: int = 1) -> list[int]:
    """Prompt-lookup drafter, a pure function of the token history h[0..L) (h[L-1] is the token about to be fed): for
    n = ngram_max down to ngram_min, the largest j with j + n < L and h[j..j+n) == h[L-n..L); the first n that matches gives
    the drafts h[j+n .. min(j+n+max_draft, L)).  No match (or max_draft <= 0) gives no drafts."""
    h = np.asarray(history, np.int64).reshape(-1)
    L = h.shape[0]
    if max_draft <= 0:
        return []
    for n in range(ngram_max, max(ngram_min, 1) - 1, -1):
        if L < n + 1:
            continue
        # windows h[j..j+n) for j = 0 .. L-n-1 (j + n < L keeps the suffix itself out and leaves at least one draft)
        win = np.lib.stride_tricks.sliding_window_view(h[:L - 1], n)
        hit = np.flatnonzero(np.all(win == h[L - n:], axis=1))
        if hit.size:
            j = int(hit[-1])
            return [int(t) for t in h[j + n:min(j + n + max_draft, L)]]
    return []


def prompt_lookup_tree(history, max_nodes: int, branches: int = 1, ngram_max: int = 3,
                       ngram_min: int = 1) -> tuple[list[int], list[int]]:
    """Tree drafter, a pure function of the token history h[0..L) (h[L-1] is the token about to be fed): up to `branches`
    distinct continuations, for n = ngram_max down to ngram_min and within one n the matches j (j + n < L,
    h[j..j+n) == h[L-n..L)) from the most recent, each h[j+n .. min(j+n+max_nodes, L)).  They are merged into a trie under
    the root (row 0, the fed token); its nodes are numbered breadth first, a depth's nodes in the order of the first
    continuation that reaches them, so every parent precedes its children, and the first max_nodes nodes are kept.
    Returns (tokens, parents) of the kept nodes: node i is row i + 1, under row parents[i].  branches = 1 gives
    prompt_lookup_drafts as a chain."""
    h = [int(t) for t in np.asarray(history, np.int64).reshape(-1)]
    L = len(h)
    if max_nodes <= 0 or branches <= 0:
        return [], []
    conts = []
    for n in range(ngram_max, max(ngram_min, 1) - 1, -1):
        if L < n + 1:
            continue
        suffix = h[L - n:]
        for j in range(L - n - 1, -1, -1):
            if h[j:j + n] == suffix:
                c = h[j + n:min(j + n + max_nodes, L)]
                if c not in conts:
                    conts.append(c)
                    if len(conts) == branches:
                        break
        if len(conts) == branches:
            break
    # the trie: key = the token path from the root; a node's rank = the first continuation that reaches it
    nodes = {}
    for rank, c in enumerate(conts):
        for d in range(1, len(c) + 1):
            nodes.setdefault(tuple(c[:d]), rank)
    order = sorted(nodes, key=lambda k: (len(k), nodes[k]))[:max_nodes]
    row = {(): 0}
    tokens, parents = [], []
    for k in order:
        row[k] = len(tokens) + 1
        tokens.append(k[-1])
        parents.append(row[k[:-1]])
    return tokens, parents


def _sampling_for(sampling, i: int):
    """prompt i of a batch or continuous run samples with Seed + i: its stream is GenerateTokens(prompts[i]) with that seed"""
    if sampling is None or sampling.Temperature == 0:
        return None
    return SamplingArgs(sampling.Temperature, sampling.TopK, sampling.TopP, (sampling.Seed + i) & (2**64 - 1))


def _logprob_lists(infContext, seqs, logprobs: int | None, logprobs_out: list | None, n_lists: int | None = None):
    """Turns logprobs on for the context's sequences `seqs` (logprobs: top_n, None: off) and returns the lists the records
    of emitted tokens go to: logprobs_out itself wrapped per sequence (n_lists None: logprobs_out is [the one list]), or
    n_lists new lists appended to logprobs_out.  None when there is nothing to collect."""
    if logprobs is None:
        return None
    for q in seqs:
        infContext.set_logprobs(q, logprobs)
    if n_lists is None:
        return None if logprobs_out[0] is None else logprobs_out
    if logprobs_out is None:
        return None
    lists = [[] for _ in range(n_lists)]
    logprobs_out.extend(lists)
    return lists


def _set_grammar(infContext, seq: int, grammar, i: int, prompt_len: int):
    """sequence `seq` of the context is constrained by `grammar` (one model.Grammar, or one per prompt: the i-th; None:
    left off; a None entry of the list turns it off) from the end of its prompt of prompt_len tokens on"""
    if grammar is not None:
        infContext.set_grammar(seq, grammar[i] if isinstance(grammar, (list, tuple)) else grammar, prompt_len)


def _set_penalties(infContext, seq: int, penalties: "PenaltyArgs | None", prompt_len: int):
    """sequence `seq` of the context is penalized with `penalties` for a prompt of prompt_len tokens (None: left off)"""
    if penalties is not None:
        infContext.set_penalties(seq, penalties, prompt_len)


def _check_speculative(speculative, use_reference_api: bool = False, keyed: bool = False):
    """keyed: the run has penalties, a grammar or logprobs on, whose records are keyed by position (no trees)"""
    if speculative is None:
        return
    if use_reference_api:
        raise ml.MlError("use_reference_api=True runs the reference's Forward -> Slice -> ml.Argmax calls; it cannot verify drafts")
    if speculative.MaxDraft < 0 or not 1 <= speculative.NgramMin <= speculative.NgramMax or speculative.Branches < 1:
        raise ml.MlError(f"SpeculativeArgs {speculative}: MaxDraft must be >= 0, 1 <= NgramMin <= NgramMax and Branches >= 1")
    if speculative.Branches > 1 and keyed:
        raise ml.MlError("speculative trees (Branches > 1) with penalties, a grammar or logprobs are not built: their records "
                         "are keyed by position, which sibling drafts share")

# Row budget of one GenerateTokensContinuous step.  FAST ragged steps of >= 32 rows run on the tensor cores (one pass over
# the weights); steps of 9..31 rows run the GEMV chain, which streams the weights once per 8 rows (up to 4 passes), and
# STRICT steps always do.  64 leaves 56 prompt rows beside 8 decode rows, so a step that admits prompt tokens is normally
# above the 32-row cliff.  tools/continuous_bench.py (8B, 32 prompts of 8..512 tokens, SequenceLength 1024, 8 slots, FAST,
# H100 80GB HBM3 at 700 W) measured 460 / 462 / 469 tokens/s at step_tokens 32 / 64 / 256: within run-to-run spread, so the
# budget was chosen from the cliff above, and kept small so that a long prompt delays decoding sequences by short steps.
DEFAULT_STEP_TOKENS = 64


class InferenceEngine:
    def __init__(self, model: "model_mod.Model", inferenceArgs: "model_mod.InferenceArgs", logFn=None,
                 acc_mode: int = model_mod.LNB_ACC_FAST, max_rows: int = 8, kv_format: str = "bf16"):
        """kv_format: the cache format of every context the engine creates ("bf16" or "mxfp8", DESIGN §9j)"""
        self.model = model
        self.kv_format = kv_format
        self.inferenceArgs = inferenceArgs
        self.logFn = logFn
        self.acc_mode = acc_mode
        self.max_rows = max_rows
        self.context_hook = None  # optional callable(InferenceContext), e.g. to enable the peer all-reduce

    def CreateInferenceContext(self) -> "model_mod.InferenceContext":  # inference.go:256-258
        ctx = model_mod.InferenceContext(self.model.Transformer, self.inferenceArgs, self.logFn,
                                         max_rows=self.max_rows, acc_mode=self.acc_mode, kv_format=self.kv_format)
        if self.context_hook is not None:
            self.context_hook(ctx)
        return ctx

    # --- tokenizer half of the engine (src/inference/tokenize.go), served by model.Vocabulary when it is a loaded one
    def _vocab(self):
        v = self.model.Vocabulary
        if not hasattr(v, "TokenizeString"):
            raise ml.MlError("the model was loaded without tokenizer.model (ids only)")
        return v

    def Tokenize(self, promptParts):                 # tokenize.go:27-95
        return self._vocab().Tokenize(promptParts)

    def TokenizeBatch(self, prompts):                # :97-107
        return self._vocab().TokenizeBatch(prompts)

    def TokenizeString(self, text, addBeginOfSentence: bool = False):   # :175-193 (the flag is unused there too)
        return self._vocab().TokenizeString(text)

    def TokenToString(self, tokenId, decodingContext):                  # :195-237
        return self._vocab().TokenToString(tokenId, decodingContext)

    def TokenBatchToString(self, tokenIdBatch):      # :239-258
        return self._vocab().TokenBatchToString(tokenIdBatch)

    # --- text streaming (generateStringInternal, inference.go:91-170) ------------------------------------------
    def GenerateString(self, promptTokens, **kw):
        """GenerateString (inference.go:56-58): GeneratedPart stream for the tokens the model generates"""
        return self.GenerateStringGeneric(self.GenerateTokens(promptTokens, **kw))

    def GenerateStringFromOutputTokens(self, outputTokens):
        """GenerateStringFromOutputTokens (inference.go:60-69): replays given ids through the detokenizer (the
        reference's own tests drive the streaming decoder this way)"""
        return self.GenerateStringGeneric((GSInProgress, int(t)) for t in outputTokens)

    def GenerateStringGeneric(self, tokenStream):
        """yields dict(DecodedString, TokenId, AddedToWaiting, IsResendOfWaiting, GenerationState) per token.  Tokens
        that end inside a UTF-8 sequence are reported with AddedToWaiting and, if the stream ends before they
        complete, re-sent at the end with their raw bytes (IsResendOfWaiting), the last one carrying the final
        state -- inference.go:104-170.  WaitingRunesExtraStr (emoji alias annotation) is not produced."""
        from .vocabulary import GenerationDecodingContext
        vocab = self._vocab()
        ctx = GenerationDecodingContext()
        waiting, last_state = [], GSInProgress
        for state, tok in tokenStream:
            text, added = vocab.TokenToString(tok, ctx)
            part = dict(DecodedString=text, TokenId=tok, AddedToWaiting=added, IsResendOfWaiting=False, GenerationState=GSInProgress)
            if state != GSInProgress and not waiting:
                part["GenerationState"] = state
            last_state = state
            if added:
                waiting.append(part)
            elif waiting:
                waiting = []
            yield part
        for i, w in enumerate(waiting):
            yield dict(DecodedString=vocab.IdToToken(w["TokenId"]).decode("utf-8", "replace"), TokenId=w["TokenId"], AddedToWaiting=False,
                       IsResendOfWaiting=True, GenerationState=last_state if i + 1 == len(waiting) else GSInProgress)

    def GenerateTokens(self, promptTokens, use_reference_api: bool = False, step_times: list | None = None,
                       prefill_chunk: int = 0, sampling: "SamplingArgs | None" = None,
                       speculative: "SpeculativeArgs | None" = None, spec_stats: list | None = None,
                       logprobs: int | None = None, logprobs_out: list | None = None,
                       penalties: "PenaltyArgs | None" = None, grammar: "model_mod.Grammar | None" = None):
        """Generator over (state, token id) exactly like generatedTokensCh.

        use_reference_api=True goes through the reference-shaped calls of every iteration
        (Transformer.Forward -> logits tensor -> Slice last row -> ml.Argmax); False uses the
        fused forward+argmax entry (same kernels, 4-byte read-back).

        prefill_chunk > 0 (EXTENSION, SURVEY 8f-4): the prompt is fed in chunks of that many tokens (Forward at
        startPos > 0 with S > 1, lnb_session_set_chunked_prefill) instead of one call; prompts longer than the context's
        max_rows become possible, and the generated stream is the same.

        sampling (EXTENSION): SamplingArgs of a seeded sampler in place of the greedy argmax (None / Temperature 0: greedy).
        The reference call sequence ends in ml.Argmax, so use_reference_api=True with a sampler is an error.

        speculative (EXTENSION): SpeculativeArgs.  After the prompt, every call verifies the last token plus prompt-lookup
        drafts in one pass over the weights (lnb_forward_speculative) and emits the accepted tokens one at a time through
        the same stop logic, so the stream (tokens, length, final state) is the plain loop's, greedy or sampled.  step_times
        then gets one entry per call, and spec_stats (optional) one (rows, accepted drafts) pair per call.  It also needs
        the fused entry: use_reference_api=True with speculative is an error.

        logprobs (EXTENSION): 0..20 turns on token log-probabilities (lnb_session_set_logprobs); logprobs_out then gets one
        model.TokenLogprob per emitted token, in order, with the top `logprobs` alternatives.  The stream is unchanged.

        penalties (EXTENSION): PenaltyArgs, applied on the device to every emitted token's logits before the sampler (or
        the greedy pick); CountPrompt False starts the counted history at the prompt's length.  The records of logprobs
        stay those of the raw distribution.  use_reference_api=True with penalties is an error.

        grammar (EXTENSION): a model.Grammar; every emitted token is masked on the device to those the grammar allows
        after the tokens emitted so far (DESIGN.md §9g), after the penalties and before the sampler.  The generated bytes
        are then always a prefix of a string of the grammar's language, and a stop token ends them only after a complete
        match.  use_reference_api=True with a grammar is an error."""
        sampling = _sampling_for(sampling, 0)
        if sampling is not None and use_reference_api:
            raise ml.MlError("use_reference_api=True ends in the greedy ml.Argmax (inference.go:207-216); it cannot sample")
        if penalties is not None and use_reference_api:
            raise ml.MlError("use_reference_api=True ends in the greedy ml.Argmax of the raw logits; it cannot apply penalties")
        if grammar is not None and use_reference_api:
            raise ml.MlError("use_reference_api=True ends in the greedy ml.Argmax of the raw logits; it cannot apply a grammar")
        _check_speculative(speculative, use_reference_api, penalties is not None or grammar is not None or logprobs is not None)
        infContext = self.CreateInferenceContext()
        try:
            if sampling is not None:
                infContext.set_sampling(0, sampling)
            lp_out = _logprob_lists(infContext, [0], logprobs, [logprobs_out])
            promptLength = len(promptTokens)
            _set_penalties(infContext, 0, penalties, promptLength)
            _set_grammar(infContext, 0, grammar, 0, promptLength)
            if prefill_chunk > 0:
                infContext.allow_chunked_prefill(True)
                if prefill_chunk > infContext.max_rows:
                    raise ml.MlError(f"prefill_chunk {prefill_chunk} exceeds the context's max_rows {infContext.max_rows}")
            if promptLength >= infContext.SequenceLength:  # :176-179
                raise ml.MlError(f"context SequenceLength {infContext.SequenceLength} must be higher than prompt "
                                 f"tokens length {promptLength}")
            if promptLength > infContext.max_rows and prefill_chunk <= 0:
                raise ml.MlError(f"prompt length {promptLength} exceeds the context's max_rows {infContext.max_rows}")
            pad = self.model.Vocabulary.PadId
            tokens = ml.Full([infContext.SequenceLength], ml.DT_INT32, pad)  # :181
            tokens.RawData[:promptLength] = np.asarray(promptTokens, np.int32)
            prevPos = 0
            if prefill_chunk > 0:      # all but the last chunk: Forward calls whose logits nobody needs
                while promptLength - prevPos > prefill_chunk:
                    self.model.Transformer.forward_argmax(infContext, tokens.RawData[prevPos:prevPos + prefill_chunk], prevPos)
                    prevPos += prefill_chunk
            for curPos in range(promptLength, infContext.SequenceLength):  # :194
                t0 = time.perf_counter()
                inputTokensSlice = tokens.Slice([prevPos], [curPos])
                if use_reference_api:
                    logits = self.model.Transformer.Forward(infContext, inputTokensSlice, prevPos)  # :202
                    logits = logits.Slice([logits.Size[0] - 1], [logits.Size[0]])                   # :207
                    nextTokenId = int(ml.Argmax(logits, len(logits.Size) - 1).Item())              # :211
                else:
                    nextTokenId, _ = self.model.Transformer.forward_argmax(infContext, inputTokensSlice.RawData, prevPos)
                existing = int(tokens.RawData[curPos])
                if existing != pad:  # :218-226 only replace token if prompt has already been generated
                    nextTokenId = existing
                tokens.RawData[curPos] = nextTokenId
                if step_times is not None:
                    step_times.append(time.perf_counter() - t0)
                if lp_out is not None:   # after the step's time: step_times measures the same with logprobs on or off
                    lp_out[0].append(infContext.read_logprobs(0, curPos, 1)[0])
                eos = nextTokenId in self.model.Vocabulary.StopTokenIds
                prevPos = curPos
                if eos:
                    yield GSFinishedByReachingEOS, nextTokenId
                    break
                if curPos + 1 == infContext.SequenceLength:
                    yield GSFinishedByReachingSeqLen, nextTokenId
                    break
                yield GSInProgress, nextTokenId
                if speculative is not None:   # the prompt is in the cache: from here on, verify drafts
                    hist = [[int(t) for t in tokens.RawData[:curPos + 1]]]
                    for _, state, tok in self._generate_speculative(infContext, hist, [0], speculative, step_times, spec_stats,
                                                                    lp_out):
                        yield state, tok
                    break
        finally:
            infContext.close()

    def GenerateBeams(self, promptTokens, beams: BeamSearchArgs, step_times: list | None = None,
                      sampling: "SamplingArgs | None" = None, penalties: "PenaltyArgs | None" = None,
                      speculative: "SpeculativeArgs | None" = None, grammar: "model_mod.Grammar | None" = None) -> list:
        """EXTENSION: beam search (DESIGN.md §9f) over a session of NumBeams sequences.  The prompt is prefilled once on
        sequence 0 and forked to the other beams (lnb_session_copy_sequences); each step is one lnb_forward_batch, whose
        logprob records give every beam's top 2B candidates, and one copy moves each surviving beam's parent rows.  Returns
        the NumReturn best BeamHypothesis, best first.  Beam search is deterministic on the raw distribution: it takes no
        sampling, penalties, grammar or speculation.  step_times gets the time of the prefill and of every step."""
        if _sampling_for(sampling, 0) is not None or penalties is not None or speculative is not None or grammar is not None:
            raise ml.MlError("beam search ranks the raw distribution deterministically: it takes no sampling, penalties, "
                             "grammar or speculative decoding")
        B = int(beams.NumBeams)
        if not 1 <= B <= 8:
            raise ml.MlError(f"NumBeams {B} must be in [1, 8]")
        if not math.isfinite(beams.LengthPenalty):
            raise ml.MlError(f"LengthPenalty {beams.LengthPenalty} must be finite")
        if not 1 <= beams.NumReturn <= B:
            raise ml.MlError(f"NumReturn {beams.NumReturn} must be in [1, NumBeams = {B}]")
        prompt = [int(t) for t in promptTokens]
        infContext = model_mod.InferenceContext(self.model.Transformer, self.inferenceArgs, self.logFn,
                                                max_rows=max(self.max_rows, B), acc_mode=self.acc_mode, n_seq=B,
                                                kv_format=self.kv_format)
        if self.context_hook is not None:
            self.context_hook(infContext)
        try:
            if len(prompt) >= infContext.SequenceLength:  # :176-179
                raise ml.MlError(f"context SequenceLength {infContext.SequenceLength} must be higher than prompt "
                                 f"tokens length {len(prompt)}")
            if len(prompt) < 1 or len(prompt) > infContext.max_rows:
                raise ml.MlError(f"prompt length {len(prompt)} must be in [1, {infContext.max_rows}]")
            return self._generate_beams(infContext, prompt, beams, step_times)[:beams.NumReturn]
        finally:
            infContext.close()

    def _generate_beams(self, infContext, prompt, beams: BeamSearchArgs, step_times: list | None = None) -> list:
        """the search of GenerateBeams on a given context (anything with SequenceLength, set_logprobs, read_logprobs,
        forward_batch and copy_sequences, whose sequence 0 the Transformer's forward_argmax prefills); returns the whole
        pool, best first"""
        B, alpha = int(beams.NumBeams), float(beams.LengthPenalty)
        seqLen, L = infContext.SequenceLength, len(prompt)
        stop = self.model.Vocabulary.StopTokenIds
        for b in range(B):
            infContext.set_logprobs(b, 2 * B)
        pool = BeamPool(B)
        # live beams: (tokens, raw score, logprobs)
        live = [([], 0.0, [])]
        for k in range(seqLen - L):
            t0 = time.perf_counter()
            if k == 0:
                self.model.Transformer.forward_argmax(infContext, np.asarray(prompt, np.int32), 0)
            else:
                infContext.forward_batch([g[-1] for g, _, _ in live], [L + k - 1] * len(live))
            if step_times is not None:
                step_times.append(time.perf_counter() - t0)
            cands = []
            for b, (_, sb, _) in enumerate(live):
                rec = infContext.read_logprobs(b, L + k, 1)[0]
                for j, (tok, lp) in enumerate(rec.Top):
                    cands.append((sb + lp, b, j, tok, lp))
            new, finished = beam_select(cands, B, stop)
            for sc, b, _, tok, lp in finished:
                g, _, lps = live[b]
                pool.add(BeamHypothesis(g + [tok], sc, beam_normalized(sc, len(g) + 1, alpha), lps + [lp], GSFinishedByReachingEOS))
            if len(new) < B:      # the search ends with the pool it has
                break
            parents = [c[1] for c in new]
            live = [(live[b][0] + [tok], sc, live[b][2] + [lp]) for sc, b, _, tok, lp in new]
            if L + k == seqLen - 1:   # the new tokens sit at the last position: every live beam finishes
                for g, sb, lps in live:
                    pool.add(BeamHypothesis(g, sb, beam_normalized(sb, len(g), alpha), lps, GSFinishedByReachingSeqLen))
                break
            if pool.full():
                best = min(beam_order(beam_normalized(sb, len(g), alpha)) for g, sb, _ in live)
                if beams.EarlyStopping or best >= beam_order(pool.worst_h()):
                    break
            moved = [i for i in range(B) if parents[i] != i]
            if moved:   # each new beam takes its parent's rows: the prompt after the prefill, the generated rows later
                infContext.copy_sequences([parents[i] for i in moved], moved, 0 if k == 0 else L, L + k)
        return pool.result()

    def _generate_speculative(self, infContext, hists, live, speculative: "SpeculativeArgs", step_times: list | None = None,
                              spec_stats: list | None = None, lp_out: list | None = None):
        """The speculative loop on a given context (anything with SequenceLength, max_rows and forward_speculative, or
        forward_speculative_tree when Branches > 1).  hists[i]: the tokens of sequence i so far, its last one emitted and not
        yet fed (it is fed at position len(hists[i]) - 1); live: the sequences still generating, each gets a row in every
        call.  The rows left of the budget min(8, max_rows) go to drafts (tree nodes) in sequence order, clamped so that no
        row passes position (tree: slot) SequenceLength - 2 (the last position the plain loop feeds).  Yields (sequence,
        state, token) per emitted token, a segment's accepted tokens in order; hists grow with them.  lp_out (or None): per
        sequence, the list that gets the logprob record of each emitted token (the records of the accepted positions)."""
        seqLen = infContext.SequenceLength
        stop = self.model.Vocabulary.StopTokenIds
        budget = min(SPEC_MAX_ROWS, infContext.max_rows)
        tree = speculative.Branches > 1
        live = list(live)
        if len(live) > budget:
            raise ml.MlError(f"{len(live)} sequences do not fit the row budget {budget} of a speculative call")
        while live:
            left = budget - len(live)
            segs = []
            for i in live:
                h = hists[i]
                pos = len(h) - 1
                k = min(speculative.MaxDraft, left, seqLen - 2 - pos)
                if tree:
                    drafts, parents = prompt_lookup_tree(h, k, speculative.Branches, speculative.NgramMax, speculative.NgramMin)
                    segs.append((i, pos, [h[-1]] + drafts, [-1] + parents))
                else:
                    drafts = prompt_lookup_drafts(h, k, speculative.NgramMax, speculative.NgramMin)
                    segs.append((i, pos, [h[-1]] + drafts))
                left -= len(drafts)
            t0 = time.perf_counter()
            if tree:
                nxt, acc, paths, _ = infContext.forward_speculative_tree(segs)
            else:
                nxt, acc, _ = infContext.forward_speculative(segs)
                paths = [list(range(int(a) + 1)) for a in acc]
            if step_times is not None:
                step_times.append(time.perf_counter() - t0)
            if spec_stats is not None:
                spec_stats.append((sum(len(sg[2]) for sg in segs), int(sum(int(a) for a in acc))))
            still, r0 = [], 0
            for sg, a, path in zip(segs, acc, paths):
                i, pos, toks = sg[0], sg[1], sg[2]
                finished = False
                recs = infContext.read_logprobs(i, pos + 1, int(a) + 1) if lp_out is not None else None
                for j in range(int(a) + 1):            # the next tokens of the path's rows, one at a time (:218-248)
                    tok, curPos = int(nxt[r0 + path[j]]), pos + 1 + j
                    hists[i].append(tok)
                    if recs is not None:
                        lp_out[i].append(recs[j])
                    if tok in stop:
                        state = GSFinishedByReachingEOS
                    elif curPos + 1 == seqLen:
                        state = GSFinishedByReachingSeqLen
                    else:
                        state = GSInProgress
                    yield i, state, tok
                    if state != GSInProgress:
                        finished = True
                        break
                r0 += len(toks)
                if not finished:
                    still.append(i)
            live = still

    def GenerateTokensContinuous(self, prompts, slots: int = 8, step_tokens: int | None = None,
                                 step_times: list | None = None, sampling: "SamplingArgs | None" = None,
                                 logprobs: int | None = None, logprobs_out: list | None = None,
                                 penalties: "PenaltyArgs | None" = None, grammar=None):
        """Continuous batching (EXTENSION, lnb_forward_ragged): any number of prompts through at most `slots` live
        sequences.  Every step is ONE forward whose rows may belong to different sequences: each decoding sequence gets
        its one row, the rest of the step's row budget (min(step_tokens, max_rows)) goes to prompt chunks, first in first
        out; a prompt whose last chunk is in the step emits its first token from that step; a finished sequence's slot
        is refilled at position 0 by the next waiting prompt.  Steps without prompt rows run lnb_forward_batch (the
        batch engine: one launch per step).  Yields (prompt index, state, token id); per prompt the stream is exactly
        what GenerateTokens(prompts[i]) yields (the bookkeeping of generateTokensInternal, inference.go:173-254).
        sampling: prompt i samples with Seed + i (the stream of GenerateTokens(prompts[i]) with that seed).
        logprobs / logprobs_out as in GenerateTokens: logprobs_out gets one list per prompt.  penalties as in GenerateTokens,
        for every prompt (set again at each admission: its first_pos follows the admitted prompt).  grammar: one
        model.Grammar for every prompt or one per prompt (None entries: unconstrained), set at each admission."""
        if step_tokens is None:
            step_tokens = DEFAULT_STEP_TOKENS
        if not 1 <= slots <= 8:
            raise ml.MlError(f"slots {slots} must be in [1, 8]")
        if step_tokens < slots:
            raise ml.MlError(f"step_tokens {step_tokens} must be at least slots {slots} (every decoding sequence gets a row)")
        prompts = [[int(t) for t in p] for p in prompts]
        infContext = model_mod.InferenceContext(self.model.Transformer, self.inferenceArgs, self.logFn,
                                                max_rows=max(self.max_rows, step_tokens), acc_mode=self.acc_mode, n_seq=slots,
                                                kv_format=self.kv_format)
        if self.context_hook is not None:
            self.context_hook(infContext)
        try:
            yield from self._generate_continuous(infContext, prompts, slots, min(step_tokens, infContext.max_rows), step_times,
                                                 sampling, logprobs, logprobs_out, penalties, grammar)
        finally:
            infContext.close()

    def _generate_continuous(self, infContext, prompts, slots: int, budget: int, step_times: list | None = None,
                             sampling: "SamplingArgs | None" = None, logprobs: int | None = None, logprobs_out: list | None = None,
                             penalties: "PenaltyArgs | None" = None, grammar=None):
        """the scheduler of GenerateTokensContinuous on a given context (anything with SequenceLength, forward_ragged and
        forward_batch, set_sampling when `sampling` samples, set_logprobs and read_logprobs when `logprobs` is set,
        set_penalties when `penalties` is set)"""
        seqLen = infContext.SequenceLength
        stop = self.model.Vocabulary.StopTokenIds
        for p in prompts:
            if len(p) >= seqLen:  # :176-179
                raise ml.MlError(f"context SequenceLength {seqLen} must be higher than prompt tokens length {len(p)}")
            if len(p) < 1:
                raise ml.MlError("empty prompt")
        lp_out = _logprob_lists(infContext, range(slots), logprobs, logprobs_out, len(prompts))
        waiting = collections.deque(range(len(prompts)))
        # per slot: prompt index, prompt tokens already in the cache, token fed next and its position (cur None: prefilling),
        # admission number (first in, first out among the prefilling slots)
        slot: list[dict | None] = [None] * slots
        admitted = 0
        while waiting or any(sl is not None for sl in slot):
            for k in range(slots):
                if slot[k] is None and waiting:
                    slot[k] = dict(i=waiting.popleft(), fed=0, cur=None, pos=0, order=admitted)
                    admitted += 1
                    sp = _sampling_for(sampling, slot[k]["i"])
                    if sp is not None:   # before the prompt's first segment (the slot's previous prompt had another seed)
                        infContext.set_sampling(k, sp)
                    _set_penalties(infContext, k, penalties, len(prompts[slot[k]["i"]]))
                    _set_grammar(infContext, k, grammar, slot[k]["i"], len(prompts[slot[k]["i"]]))
            decoding = [k for k in range(slots) if slot[k] is not None and slot[k]["cur"] is not None]
            prefilling = sorted((k for k in range(slots) if slot[k] is not None and slot[k]["cur"] is None),
                                key=lambda k: slot[k]["order"])
            segs = [(k, slot[k]["pos"], [slot[k]["cur"]]) for k in decoding]
            left = budget - len(decoding)
            for k in prefilling:
                if left <= 0:
                    break
                sl = slot[k]
                n = min(left, len(prompts[sl["i"]]) - sl["fed"])
                segs.append((k, sl["fed"], prompts[sl["i"]][sl["fed"]:sl["fed"] + n]))
                left -= n
            t0 = time.perf_counter()
            if not prefilling:
                # decode rows only: one batch-engine launch; row k = slot k (free slots below the last decoding one are
                # fed token 0 at position 0 of their own cache -- they hold no sequence, and a refill overwrites it)
                n = max(decoding) + 1
                toks = [slot[k]["cur"] if slot[k] is not None else 0 for k in range(n)]
                poss = [slot[k]["pos"] if slot[k] is not None else 0 for k in range(n)]
                nxt, _ = infContext.forward_batch(toks, poss)
                out = {k: int(nxt[k]) for k in decoding}
            else:
                nxt, _ = infContext.forward_ragged(segs)
                out = {k: int(nxt[j]) for j, (k, _, _) in enumerate(segs)}
            if step_times is not None:
                step_times.append(time.perf_counter() - t0)
            for k, _, chunk in segs:
                sl = slot[k]
                if sl["cur"] is None:
                    sl["fed"] += len(chunk)
                    if sl["fed"] < len(prompts[sl["i"]]):
                        continue
                    curPos = sl["fed"]                    # first generated token (:194-216)
                else:
                    curPos = sl["pos"] + 1
                tok = out[k]
                sl["cur"], sl["pos"] = tok, curPos
                if tok in stop:
                    state = GSFinishedByReachingEOS
                elif curPos + 1 == seqLen:
                    state = GSFinishedByReachingSeqLen
                else:
                    state = GSInProgress
                if state != GSInProgress:
                    slot[k] = None
                if lp_out is not None:
                    lp_out[sl["i"]].append(infContext.read_logprobs(k, curPos, 1)[0])
                yield sl["i"], state, tok

    def GenerateTokensBatch(self, prompts, step_times: list | None = None, sampling: "SamplingArgs | None" = None,
                            speculative: "SpeculativeArgs | None" = None, spec_stats: list | None = None,
                            logprobs: int | None = None, logprobs_out: list | None = None,
                            penalties: "PenaltyArgs | None" = None, grammar=None):
        """The consumer `InferenceEngine.TokenizeBatch` (src/inference/tokenize.go:97-107) never got in the
        reference (SURVEY 8f-4): every prompt runs the loop of generateTokensInternal (:173-254) -- own
        InferenceContext / KV cache, own positions, own stop condition -- but all sequences advance together,
        one pass over the weights per step (lnb_forward_batch).  Yields (sequence index, state, token id);
        per sequence the stream is exactly what GenerateTokens(prompts[i]) yields.  sampling: sequence i samples with
        Seed + i (the stream of GenerateTokens(prompts[i]) with that seed).
        speculative (EXTENSION): after the prompts, every call is one lnb_forward_speculative in which each unfinished
        sequence gets its row and the rest of the 8-row budget goes to prompt-lookup drafts in sequence order; the streams
        are the same.  spec_stats as in GenerateTokens; logprobs / logprobs_out as in GenerateTokens, logprobs_out gets one
        list per prompt; penalties as in GenerateTokens, for every sequence; grammar: one model.Grammar for every
        sequence or one per prompt (None entries: unconstrained)."""
        _check_speculative(speculative, False, penalties is not None or grammar is not None or logprobs is not None)
        n = len(prompts)
        if n < 1:
            raise ml.MlError("empty prompt batch")
        if n == 1:
            lp0 = None
            if logprobs is not None and logprobs_out is not None:
                lp0 = []
                logprobs_out.append(lp0)
            for state, tok in self.GenerateTokens(prompts[0], sampling=sampling, speculative=speculative, spec_stats=spec_stats,
                                                  logprobs=logprobs, logprobs_out=lp0, penalties=penalties,
                                                  grammar=grammar[0] if isinstance(grammar, (list, tuple)) else grammar):
                yield 0, state, tok
            return
        infContext = model_mod.InferenceContext(self.model.Transformer, self.inferenceArgs, self.logFn,
                                                max_rows=max(self.max_rows, n), acc_mode=self.acc_mode, n_seq=n,
                                                kv_format=self.kv_format)
        if self.context_hook is not None:
            self.context_hook(infContext)
        try:
            seqLen = infContext.SequenceLength
            stop = self.model.Vocabulary.StopTokenIds
            for p in prompts:
                if len(p) >= seqLen:  # :176-179
                    raise ml.MlError(f"context SequenceLength {seqLen} must be higher than prompt tokens length {len(p)}")
                if len(p) < 1 or len(p) > infContext.max_rows:
                    raise ml.MlError(f"prompt length {len(p)} must be in [1, {infContext.max_rows}]")
            for i in range(n):
                sp = _sampling_for(sampling, i)
                if sp is not None:
                    infContext.set_sampling(i, sp)
                _set_penalties(infContext, i, penalties, len(prompts[i]))
                _set_grammar(infContext, i, grammar, i, len(prompts[i]))
            lp_out = _logprob_lists(infContext, range(n), logprobs, logprobs_out, n)
            cur = [0] * n                                  # token fed next / position it is fed at
            pos = [0] * n
            done = [False] * n

            def emit(i, tok, curPos):
                """bookkeeping of one generated token at curPos (:218-248); returns the state to yield"""
                cur[i], pos[i] = tok, curPos
                if lp_out is not None:
                    lp_out[i].append(infContext.read_logprobs(i, curPos, 1)[0])
                if tok in stop:
                    done[i] = True
                    return GSFinishedByReachingEOS
                if curPos + 1 == seqLen:
                    done[i] = True
                    return GSFinishedByReachingSeqLen
                return GSInProgress

            t0 = time.perf_counter()
            for i, p in enumerate(prompts):                # prefill: the ordinary Forward on sequence i's cache
                infContext.set_active_sequence(i)
                nxt, _ = self.model.Transformer.forward_argmax(infContext, np.asarray(p, np.int32), 0)
                yield i, emit(i, int(nxt), len(p)), int(nxt)
            if step_times is not None:
                step_times.append(time.perf_counter() - t0)
            if speculative is not None:
                hists = [[int(t) for t in p] + [cur[i]] for i, p in enumerate(prompts)]
                live = [i for i in range(n) if not done[i]]
                yield from self._generate_speculative(infContext, hists, live, speculative, step_times, spec_stats, lp_out)
                return
            while not all(done):
                t0 = time.perf_counter()
                # finished sequences are stepped again at their last position (same token, same cache row: a no-op
                # for their state); the weights are read once per step regardless
                nxt, _ = infContext.forward_batch(cur, pos)
                if step_times is not None:
                    step_times.append(time.perf_counter() - t0)
                for i in range(n):
                    if not done[i]:
                        yield i, emit(i, int(nxt[i]), pos[i] + 1), int(nxt[i])
        finally:
            infContext.close()
