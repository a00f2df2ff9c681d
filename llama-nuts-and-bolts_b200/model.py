"""Host mirror of the reference's src/model package for the forward path:
ModelArgs (modelargs.go), Model / LlamaTransformer (llamatransformer.go:16-113,145-180) and
InferenceContext (inferencecontext.go).  The transformer's weights, KV cache and activations
live in HBM behind liblnb.so; `LlamaTransformer.Forward` is ONE call through the C-ABI.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _capi, ml, synth
from ._capi import LNB_ACC_FAST, LNB_ACC_STRICT, check, lib, ptr


@dataclass
class ModelArgs:  # src/model/modelargs.go:10-44 (+ derived HeadDim / FFN width)
    Dim: int = 4096
    N_Layers: int = 32
    N_Heads: int = 32
    N_KVHeads: int = 8
    VocabSize: int = 128256
    MultipleOf: int = 1024
    FFNDimMultiplier: float = 1.3
    NormEpsilon: float = 1e-5
    RopeTheta: float = 500000.0
    UseScaledRope: bool = True
    MaxSequenceLength: int = 2048
    HeadDim: int = field(default=0)
    FFNDim: int = field(default=0)

    def __post_init__(self):
        if not self.HeadDim:
            self.HeadDim = self.Dim // self.N_Heads  # llamatransformer.go:73
        if not self.FFNDim:  # llamatransformer.go:569-577
            hidden = int(2 * (4 * self.Dim) / 3)
            hidden = int(self.FFNDimMultiplier * hidden)
            self.FFNDim = self.MultipleOf * ((hidden + self.MultipleOf - 1) // self.MultipleOf)

    def to_c_dict(self) -> dict:
        return dict(dim=self.Dim, n_layers=self.N_Layers, n_heads=self.N_Heads, n_kv_heads=self.N_KVHeads,
                    head_dim=self.HeadDim, ffn_dim=self.FFNDim, vocab_size=self.VocabSize,
                    max_seq_len=self.MaxSequenceLength, norm_eps=self.NormEpsilon, rope_theta=self.RopeTheta,
                    use_scaled_rope=int(self.UseScaledRope))

    @classmethod
    def from_c_dict(cls, d: dict) -> "ModelArgs":
        return cls(Dim=d["dim"], N_Layers=d["n_layers"], N_Heads=d["n_heads"], N_KVHeads=d["n_kv_heads"],
                   VocabSize=d["vocab_size"], NormEpsilon=d["norm_eps"], RopeTheta=d["rope_theta"],
                   UseScaledRope=bool(d["use_scaled_rope"]), MaxSequenceLength=d["max_seq_len"],
                   HeadDim=d["head_dim"], FFNDim=d["ffn_dim"])


@dataclass
class Vocabulary:  # src/model/vocabulary.go (ids only; the tokenizer is out of scope)
    PadId: int = synth.PAD_ID
    StopTokenIds: tuple = synth.STOP_IDS


WEIGHT_FORMATS = {"bf16": _capi.LNB_WEIGHTS_BF16, "mxfp8": _capi.LNB_WEIGHTS_MXFP8, "mxfp4": _capi.LNB_WEIGHTS_MXFP4}


class LlamaTransformer:
    """model.LlamaTransformer: owns the device-side weights of one tensor-parallel rank."""

    def __init__(self, args: ModelArgs, device: int = 0, tp_rank: int = 0, tp_size: int = 1, nccl_id: bytes | None = None,
                 weight_format: str = "bf16"):
        """weight_format: "bf16", or "mxfp8" / "mxfp4": finalize quantizes the linear weights (DESIGN.md §9h, §9i)"""
        self.args = args
        self.device, self.tp_rank, self.tp_size = device, tp_rank, tp_size
        self._cargs = _capi.ModelArgsC(**args.to_c_dict())
        fmt = WEIGHT_FORMATS.get(weight_format)
        if fmt is None:
            raise ValueError(f"unknown weight_format {weight_format!r} (known: {', '.join(WEIGHT_FORMATS)})")
        h = C.c_void_p()
        idbuf = C.create_string_buffer(nccl_id, 128) if nccl_id is not None else None
        check(lib.lnb_model_create(C.byref(self._cargs), device, tp_rank, tp_size, idbuf, C.byref(h)))
        self.h = h
        self.finalized = False
        try:
            check(lib.lnb_model_set_weight_format(h, fmt))
        except Exception:
            self.close()
            raise
        self.weight_format = weight_format

    # --- weights -----------------------------------------------------------------------------
    def upload_tensor(self, name: str, data: np.ndarray):
        """getTensor + device upload (src/model/loader.go:183-197): `data` is the full bf16 tensor."""
        data = np.ascontiguousarray(data, np.uint16)
        shape = (C.c_int64 * data.ndim)(*data.shape)
        check(lib.lnb_model_upload_tensor(self.h, name.encode(), ptr(data, _capi.u16p), shape, data.ndim))

    def init_synthetic(self, seed: int = synth.SEED):
        check(lib.lnb_model_init_synthetic(self.h, seed))

    def load_pth(self, path: str) -> int:
        """every tensor the architecture names, from the checkpoint mapping straight to HBM (lnb_model_load_pth);
        returns how many were uploaded"""
        n = C.c_int(0)
        check(lib.lnb_model_load_pth(self.h, path.encode(), C.byref(n)))
        return n.value

    def finalize(self):
        check(lib.lnb_model_finalize(self.h))
        self.finalized = True

    def mxfp8_read(self, name: str) -> tuple[np.ndarray, np.ndarray]:
        """the E4M3 codes [rows, cols] and E8M0 scales [rows, ceil(cols / 32)] of a linear checkpoint tensor of a finalized
        MXFP8 model, in the checkpoint's row order"""
        shape = synth.tensor_shapes(self.args.to_c_dict()).get(name, (0,))
        rows, cols = shape if len(shape) == 2 else (shape[0], 1)   # the library names what is wrong with other names
        codes = np.empty((rows, cols), np.uint8)
        scales = np.empty((rows, (cols + 31) // 32), np.uint8)
        check(lib.lnb_model_mxfp8_read(self.h, name.encode(), codes.ctypes.data, scales.ctypes.data))
        return codes, scales

    def mxfp4_read(self, name: str) -> tuple[np.ndarray, np.ndarray]:
        """the E2M1 codes [rows, cols / 2] (two a byte, the even column in the low nibble) and E8M0 scales
        [rows, ceil(cols / 32)] of a linear checkpoint tensor of a finalized MXFP4 model, in the checkpoint's row order"""
        shape = synth.tensor_shapes(self.args.to_c_dict()).get(name, (0,))
        rows, cols = shape if len(shape) == 2 else (shape[0], 2)   # the library names what is wrong with other names
        codes = np.empty((rows, cols // 2), np.uint8)
        scales = np.empty((rows, (cols + 31) // 32), np.uint8)
        check(lib.lnb_model_mxfp4_read(self.h, name.encode(), codes.ctypes.data, scales.ctypes.data))
        return codes, scales

    def weight_info(self) -> dict:
        """{"format": "bf16" | "mxfp8" | "mxfp4", "device_bytes": weight bytes in HBM, "step_bytes": weight bytes one S = 1 step reads}"""
        fmt, dev, step = C.c_int(0), C.c_int64(0), C.c_int64(0)
        check(lib.lnb_model_weight_info(self.h, C.byref(fmt), C.byref(dev), C.byref(step)))
        names = {v: k for k, v in WEIGHT_FORMATS.items()}
        return {"format": names[fmt.value], "device_bytes": dev.value, "step_bytes": step.value}

    def rope_table(self, rows: int | None = None) -> np.ndarray:
        rows = rows or self.args.MaxSequenceLength * 2
        out = np.empty((rows, self.args.HeadDim // 2, 2), np.float32)
        check(lib.lnb_model_get_rope_table(self.h, ptr(out, _capi.f32p), rows))
        return out

    def silu_table(self) -> np.ndarray:
        out = np.empty(65536, np.uint16)
        check(lib.lnb_model_get_silu_table(self.h, ptr(out, _capi.u16p)))
        return out

    # --- forward -----------------------------------------------------------------------------
    def Forward(self, infContext: "InferenceContext", inputTokens: ml.Tensor, startPos: int) -> ml.Tensor:
        """LlamaTransformer.Forward (llamatransformer.go:145-180): returns f32 logits [S, vocab]."""
        if inputTokens.DataType is not ml.DT_INT32 or inputTokens.RawData.ndim != 1:
            raise ml.MlError("inputTokens must be a 1-D Int32 tensor")
        S = inputTokens.RawData.shape[0]
        if S == 0:
            raise ml.MlError("empty token array")
        # the [S, vocab] f32 result stays in HBM behind a handle; reading it (RawData) copies it to the host
        gen = C.c_int64(0)
        check(lib.lnb_forward_device(infContext.h, ptr(inputTokens.RawData, _capi.i32p), S, startPos, S, None, C.byref(gen)))
        infContext.generation = gen.value
        return ml.DeviceLogits(infContext, gen.value, 0, S, self.args.VocabSize)

    def forward_argmax(self, infContext: "InferenceContext", tokens, startPos: int, want_logits: str = "none"):
        """Fast path of the generate loop: forward + last-row argmax in one call.
        want_logits: "none" | "last" | "all"."""
        tokens = np.ascontiguousarray(tokens, np.int32)
        S = tokens.shape[0]
        nxt = C.c_int32(-1)
        logits = None
        if want_logits != "none":
            logits = np.empty((S if want_logits == "all" else 1, self.args.VocabSize), np.float32)
        check(lib.lnb_forward(infContext.h, ptr(tokens, _capi.i32p), S, startPos,
                              ptr(logits, _capi.f32p) if logits is not None else None,
                              1 if want_logits == "all" else 0, C.byref(nxt)))
        return nxt.value, logits

    def score(self, infContext: "InferenceContext", tokens, startPos: int = 0) -> list:
        """EXTENSION (lnb_score): the log-probability of tokens[1:] given what precedes them, one forward over tokens[:-1] at
        startPos.  Returns a TokenLogprob per token of tokens[1:] (positions startPos + 1 ..).  Chunks overlap by one token:
        the next call starts at startPos + len(tokens) - 1 with tokens[-1].  The active sequence must have logprobs on."""
        tokens = np.ascontiguousarray(tokens, np.int32)
        n = tokens.shape[0]
        check(lib.lnb_score(infContext.h, ptr(tokens, _capi.i32p), n, startPos))
        return infContext.read_logprobs(infContext.active_seq, startPos + 1, n - 1)

    def close(self):
        if self.h:
            lib.lnb_model_destroy(self.h)
            self.h = None


@dataclass
class InferenceArgs:  # src/common/inferenceargs.go:3-11
    SequenceLength: int = 0


@dataclass
class SamplingArgs:
    """EXTENSION (the reference only has the greedy ml.Argmax): seeded sampling of the next token, lnb_session_set_sampling.
    Temperature 0 is greedy; TopK 0 is the whole vocabulary; TopP in (0, 1], 1 is no top-p cut.  The draw for the token at
    position p uses splitmix64(Seed, p), so a stream depends only on the model, the prompt and these values."""
    Temperature: float = 0.0
    TopK: int = 0
    TopP: float = 1.0
    Seed: int = 0

    def c(self) -> "_capi.SamplingC":
        return _capi.SamplingC(float(self.Temperature), int(self.TopK), float(self.TopP), int(self.Seed) & (2**64 - 1))


@dataclass
class PenaltyArgs:
    """EXTENSION: repetition, frequency and presence penalties and a logit bias over the sequence's token history,
    lnb_session_set_penalties (DESIGN.md §9e).  For the token at position p, a token fed c >= 1 times among the last Window
    positions (0: all) has its logit l divided (l > 0) or multiplied (l <= 0) by RepetitionPenalty, then lowered by
    c * FrequencyPenalty + PresencePenalty; LogitBias {token: bias} adds bias (-inf: the token is never emitted).  The
    sampler (greedy at Temperature 0) then draws from those logits.  CountPrompt False counts generated tokens only (the
    OpenAI semantics): the prompt's positions are never counted.  The defaults are neutral (penalties off)."""
    RepetitionPenalty: float = 1.0
    FrequencyPenalty: float = 0.0
    PresencePenalty: float = 0.0
    Window: int = 0
    CountPrompt: bool = False
    LogitBias: dict = field(default_factory=dict)

    def first_pos(self, prompt_len: int) -> int:
        return 0 if self.CountPrompt else int(prompt_len)

    def c(self, prompt_len: int = 0) -> "_capi.PenaltiesC":
        """the lnb_penalties of a sequence whose prompt has prompt_len tokens"""
        if len(self.LogitBias) > _capi.LNB_LOGIT_BIAS_MAX:
            raise ml.MlError(f"LogitBias has {len(self.LogitBias)} entries, at most {_capi.LNB_LOGIT_BIAS_MAX}")
        p = _capi.PenaltiesC()
        p.repetition_penalty = float(self.RepetitionPenalty)
        p.frequency_penalty = float(self.FrequencyPenalty)
        p.presence_penalty = float(self.PresencePenalty)
        p.window = int(self.Window)
        p.first_pos = self.first_pos(prompt_len)
        p.n_bias = len(self.LogitBias)
        for j, (t, b) in enumerate(self.LogitBias.items()):
            p.bias_token[j] = int(t)
            p.bias[j] = float(b)
        return p


@dataclass
class TokenLogprob:
    """EXTENSION: one record of lnb_session_logprobs_read.  Logprob is the raw model distribution's (temperature 1, no
    top-k / top-p); Rank 1 is the greedy token; Top holds (token, logprob) of the top_n first tokens in rank order."""
    Token: int
    Logprob: float
    Rank: int
    Top: list


def regex_dfa(pattern: str | bytes):
    """EXTENSION: lnb_regex_dfa -> (trans int32 [Q, 256], -1: no string of the language continues; accept uint8 [Q]).
    The language is re.fullmatch(pattern, s, re.ASCII) over the UTF-8 encodings of s; state 0 is the start, and the DFA
    is minimal and trimmed.  Unsupported syntax raises _capi.LnbError (LNB_EINVAL, the message gives the byte offset)."""
    b = pattern.encode("utf-8") if isinstance(pattern, str) else bytes(pattern)
    cap = _capi.LNB_GRAMMAR_MAX_STATES
    trans = np.empty((cap, 256), np.int32)
    accept = np.empty(cap, np.uint8)
    q = C.c_int(0)
    check(lib.lnb_regex_dfa(b, len(b), ptr(trans, _capi.i32p), accept.ctypes.data_as(C.POINTER(C.c_uint8)), cap, C.byref(q)))
    return trans[:q.value].copy(), accept[:q.value].copy()


def token_bytes_table(token_bytes) -> tuple:
    """[bytes of token t] -> (uint8 concatenation, int64 offsets [V + 1]) as lnb_grammar_create takes them"""
    off = np.zeros(len(token_bytes) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in token_bytes])
    data = np.frombuffer(b"".join(token_bytes), np.uint8).copy() if off[-1] else np.zeros(1, np.uint8)
    return data, off


def vocabulary_token_bytes(vocabulary, n: int) -> list:
    """the bytes of tokens 0 .. n-1 of a loaded vocabulary.Vocabulary: special tokens (the 256 after the mergeable ones)
    and ids past the vocabulary are empty, so a grammar never emits them as text"""
    n_merge = len(vocabulary) - 256
    return [vocabulary.IdToToken(t) if t < n_merge else b"" for t in range(n)]


class Grammar:
    """EXTENSION: regex-constrained generation, lnb_grammar_create (DESIGN.md §9g).  Tokens a sequence emits after its
    grammar's first position spell a prefix of a string of re.fullmatch(regex, s, re.ASCII), and a stop token can only
    follow a complete match; once a stop token (or a token the caller feeds outside the grammar) is fed, only stop tokens
    may follow.  The token bytes come from `vocabulary` (a loaded vocabulary.Vocabulary; Z = its StopTokenIds) or from
    token_bytes / stop_ids directly.  The masks of every DFA state are built on the model's device, once."""

    def __init__(self, model, regex: str | bytes, vocabulary=None, token_bytes=None, stop_ids=None):
        transformer = getattr(model, "Transformer", model)
        V = transformer.args.VocabSize
        if vocabulary is not None:
            token_bytes = vocabulary_token_bytes(vocabulary, V)
            stop_ids = vocabulary.StopTokenIds
        if token_bytes is None or stop_ids is None or len(token_bytes) != V:
            raise ml.MlError(f"a grammar needs the bytes of all {V} tokens and the stop ids")
        self.transformer = transformer
        self.regex = regex
        b = regex.encode("utf-8") if isinstance(regex, str) else bytes(regex)
        data, off = token_bytes_table(token_bytes)
        stop = np.ascontiguousarray(stop_ids, np.int32)
        h = C.c_void_p()
        check(lib.lnb_grammar_create(transformer.h, b, len(b), data.ctypes.data_as(C.POINTER(C.c_uint8)), ptr(off, _capi.i64p),
                                     ptr(stop, _capi.i32p), int(stop.shape[0]), C.byref(h)))
        self.h = h
        info = self.info()
        self.NumStates, self.W = info["states"], (V + 31) // 32

    def info(self) -> dict:
        """states Q, stuck (states whose mask is the stop set), device bytes, the mask build's device time in ns"""
        out = np.zeros(4, np.int64)
        check(lib.lnb_grammar_info(self.h, ptr(out, _capi.i64p)))
        return dict(states=int(out[0]), stuck=int(out[1]), bytes=int(out[2]), build_ns=int(out[3]))

    def read_mask(self, state: int) -> np.ndarray:
        """mask(state) as uint32 words (bit t & 31 of word t >> 5); state -1: ⊥ (the stop set)"""
        out = np.zeros(self.W, np.uint32)
        check(lib.lnb_grammar_read_mask(self.h, state, out.ctypes.data_as(C.POINTER(C.c_uint32))))
        return out

    def close(self):
        """LnbError (LNB_ESTATE) while a session's sequence still uses the grammar"""
        if self.h:
            check(lib.lnb_grammar_destroy(self.h))
            self.h = None


def _token_logprobs(recs) -> list:
    return [TokenLogprob(int(r.token), float(r.logprob), int(r.rank),
                         [(int(r.top_token[j]), float(r.top_logprob[j])) for j in range(r.n_top)]) for r in recs]


class InferenceContext:
    """model.InferenceContext (inferencecontext.go:8-46): the KV cache (here: in HBM)."""

    KV_FORMATS = {"bf16": _capi.LNB_KV_BF16, "mxfp8": _capi.LNB_KV_MXFP8}

    def __init__(self, transformer: LlamaTransformer, inferenceArgs: InferenceArgs, logFn=None,
                 max_rows: int = 8, acc_mode: int = LNB_ACC_FAST, n_seq: int = 1, kv_format: str = "bf16"):
        """kv_format: "bf16", or "mxfp8" for the MXFP8 KV cache (lnb_session_create_kv, DESIGN §9j)"""
        if kv_format not in self.KV_FORMATS:
            raise ValueError(f"kv_format must be one of {sorted(self.KV_FORMATS)}, not {kv_format!r}")
        self.transformer = transformer
        self.SequenceLength = inferenceArgs.SequenceLength if inferenceArgs.SequenceLength > 0 \
            else transformer.args.MaxSequenceLength
        self.logFn = logFn
        self.acc_mode = acc_mode
        self.max_rows = max_rows
        self.n_seq = n_seq
        self.kv_format = kv_format
        h = C.c_void_p()
        if kv_format != "bf16":
            check(lib.lnb_session_create_kv(transformer.h, self.SequenceLength, n_seq, max_rows, acc_mode,
                                            self.KV_FORMATS[kv_format], C.byref(h)))
        elif n_seq > 1:   # n_seq reference InferenceContexts that share the weights (batched decode)
            check(lib.lnb_session_create_batch(transformer.h, self.SequenceLength, n_seq, max_rows, acc_mode, C.byref(h)))
        else:
            check(lib.lnb_session_create(transformer.h, self.SequenceLength, max_rows, acc_mode, C.byref(h)))
        self.h = h
        self.active_seq = 0
        self.generation = 0        # forward calls made through lnb_forward_device (validity of ml.DeviceLogits handles)
        self.pre_close_hook = None  # tensor-parallel sessions: barrier before the peer-mapped region is freed

    def Logf(self, fmt, *v):
        if self.logFn:
            self.logFn(fmt, *v)

    # CacheK / CacheV of the reference are host tensors; here they are read back on demand
    def CacheK(self, layer: int) -> ml.Tensor:
        return self._cache(_capi.LNB_BUF_CACHE_K, layer)

    def CacheV(self, layer: int) -> ml.Tensor:
        return self._cache(_capi.LNB_BUF_CACHE_V, layer)

    def _cache(self, which, layer):
        a = self.transformer.args
        kv_l = a.N_KVHeads // self.transformer.tp_size
        out = np.empty((self.SequenceLength, kv_l, a.HeadDim), np.uint16)
        check(lib.lnb_session_read(self.h, which, layer, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return ml.Tensor(out, ml.DT_BF16)

    def kv_info(self) -> tuple[str, int]:
        """(the cache format, the bytes its K and V caches hold in HBM)"""
        fmt, nbytes = C.c_int(), C.c_int64()
        check(lib.lnb_session_kv_info(self.h, C.byref(fmt), C.byref(nbytes)))
        return {v: k for k, v in self.KV_FORMATS.items()}[fmt.value], nbytes.value

    def kv_read(self, seq: int, layer: int, which: str, pos0: int, n: int) -> tuple[np.ndarray, np.ndarray]:
        """the raw MXFP8 blocks of positions [pos0, pos0 + n) of K (which="k") or V ("v"): (codes [n, kv_l] u8, scales
        [n, n_kv, ceil(head_dim / 32)] u8), heads in checkpoint order"""
        a, tp = self.transformer.args, self.transformer.tp_size
        n_kv = a.N_KVHeads // tp
        codes = np.empty((n, n_kv * a.HeadDim), np.uint8)
        scales = np.empty((n, n_kv, (a.HeadDim + 31) // 32), np.uint8)
        w = {"k": _capi.LNB_BUF_CACHE_K, "v": _capi.LNB_BUF_CACHE_V}[which]
        check(lib.lnb_session_kv_read(self.h, seq, layer, w, pos0, n, codes.ctypes.data_as(C.c_void_p),
                                      scales.ctypes.data_as(C.c_void_p)))
        return codes, scales

    def residual(self, rows: int) -> np.ndarray:
        out = np.empty((rows, self.transformer.args.Dim), np.uint16)
        check(lib.lnb_session_read(self.h, _capi.LNB_BUF_RESIDUAL, 0, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    _STAGES = {"q": (_capi.LNB_BUF_Q, "q"), "attn": (_capi.LNB_BUF_ATTN, "q"), "post_attn": (_capi.LNB_BUF_POST_ATTN, "dim"),
               "normed": (_capi.LNB_BUF_NORMED, "dim"), "ffn": (_capi.LNB_BUF_FFN, "ffn")}

    def stage(self, name: str, rows: int) -> np.ndarray:
        """the first `rows` rows of a stage buffer of the last forward's last layer (lnb_session_read): "q" (rotated
        queries), "attn" (attention output), "post_attn" (x + Wo), "normed" (the rows the last normalising GEMM read) or
        "ffn" (SiLU(gate) * up), as [rows, width] bf16 bits"""
        which, w = self._STAGES[name]
        a, tp = self.transformer.args, self.transformer.tp_size
        width = {"q": a.N_Heads * a.HeadDim // tp, "dim": a.Dim, "ffn": a.FFNDim // tp}[w]
        out = np.empty((rows, width), np.uint16)
        check(lib.lnb_session_read(self.h, which, 0, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def set_active_sequence(self, seq: int):
        check(lib.lnb_session_set_active_sequence(self.h, seq))
        self.active_seq = seq

    def forward_batch(self, tokens, positions, want_logits: bool = False):
        """one decode step for len(tokens) independent sequences: (greedy tokens [n], logits [n, vocab] or None)"""
        tokens = np.ascontiguousarray(tokens, np.int32)
        positions = np.ascontiguousarray(positions, np.int32)
        n = tokens.shape[0]
        nxt = np.empty(n, np.int32)
        logits = np.empty((n, self.transformer.args.VocabSize), np.float32) if want_logits else None
        check(lib.lnb_forward_batch(self.h, ptr(tokens, _capi.i32p), ptr(positions, _capi.i32p), n,
                                    ptr(logits, _capi.f32p) if want_logits else None, ptr(nxt, _capi.i32p)))
        return nxt, logits

    def forward_ragged(self, segments, want_logits: bool = False):
        """EXTENSION (continuous batching, lnb_forward_ragged): ONE forward over segments (seq, start_pos, tokens) of
        different sequences -- prompts, prompt chunks and decode rows -- each with the arithmetic of its own Forward.
        Returns (greedy token of each segment's last row [n_segs], logits [n_segs, vocab] of those rows or None)."""
        n = len(segments)
        seq = np.array([s for s, _, _ in segments], np.int32)
        start = np.array([p for _, p, _ in segments], np.int32)
        toks = [np.asarray(t, np.int32).reshape(-1) for _, _, t in segments]
        lens = np.array([len(t) for t in toks], np.int32)
        flat = np.ascontiguousarray(np.concatenate(toks) if toks else np.zeros(0, np.int32), np.int32)
        nxt = np.empty(n, np.int32)
        logits = np.empty((n, self.transformer.args.VocabSize), np.float32) if want_logits else None
        check(lib.lnb_forward_ragged(self.h, n, ptr(seq, _capi.i32p), ptr(start, _capi.i32p), ptr(lens, _capi.i32p),
                                     ptr(flat, _capi.i32p), ptr(logits, _capi.f32p) if want_logits else None,
                                     ptr(nxt, _capi.i32p)))
        return nxt, logits

    def forward_speculative(self, segments, want_logits: bool = False):
        """EXTENSION (speculative verification, lnb_forward_speculative): ONE forward over segments (seq, start_pos, tokens)
        whose tokens are the sequence's last emitted token followed by drafted tokens, row j at position start_pos + j.
        Returns (next token of every row [rows], accepted drafts of every segment [n_segs], logits [rows, vocab] or None);
        segment i emits the next tokens of its rows 0 .. accepted[i]."""
        n = len(segments)
        seq = np.array([s for s, _, _ in segments], np.int32)
        start = np.array([p for _, p, _ in segments], np.int32)
        toks = [np.asarray(t, np.int32).reshape(-1) for _, _, t in segments]
        n_draft = np.array([len(t) - 1 for t in toks], np.int32)
        flat = np.ascontiguousarray(np.concatenate(toks) if toks else np.zeros(0, np.int32), np.int32)
        rows = flat.shape[0]
        nxt = np.empty(rows, np.int32)
        acc = np.empty(n, np.int32)
        logits = np.empty((rows, self.transformer.args.VocabSize), np.float32) if want_logits else None
        check(lib.lnb_forward_speculative(self.h, n, ptr(seq, _capi.i32p), ptr(start, _capi.i32p), ptr(n_draft, _capi.i32p),
                                          ptr(flat, _capi.i32p), ptr(logits, _capi.f32p) if want_logits else None,
                                          ptr(nxt, _capi.i32p), ptr(acc, _capi.i32p)))
        return nxt, acc, logits

    def forward_speculative_tree(self, segments, want_logits: bool = False):
        """EXTENSION (tree speculative verification, lnb_forward_speculative_tree): ONE forward over segments
        (seq, start_pos, tokens, parent): tokens[0] is the sequence's last emitted token (the root, parent[0] is not read),
        node j > 0 carries tokens[j] under parent[j] in [0, j), at position start_pos + its depth.  Returns (next token of
        every row [rows], accepted depth of every segment [n_segs], the accepted path of every segment as segment-local
        rows, root first, logits [rows, vocab] or None); segment i emits the next tokens of its path's rows."""
        n = len(segments)
        seq = np.array([s for s, _, _, _ in segments], np.int32)
        start = np.array([p for _, p, _, _ in segments], np.int32)
        toks = [np.asarray(t, np.int32).reshape(-1) for _, _, t, _ in segments]
        n_nodes = np.array([len(t) - 1 for t in toks], np.int32)
        flat = np.ascontiguousarray(np.concatenate(toks) if toks else np.zeros(0, np.int32), np.int32)
        par = np.ascontiguousarray(np.concatenate([np.asarray(q, np.int32).reshape(-1) for _, _, _, q in segments])
                                   if segments else np.zeros(0, np.int32), np.int32)
        rows = flat.shape[0]
        if par.shape[0] != rows:
            raise ml.MlError(f"forward_speculative_tree: {par.shape[0]} parent entries for {rows} rows")
        nxt = np.empty(rows, np.int32)
        acc = np.empty(n, np.int32)
        path = np.empty(rows, np.int32)
        logits = np.empty((rows, self.transformer.args.VocabSize), np.float32) if want_logits else None
        check(lib.lnb_forward_speculative_tree(self.h, n, ptr(seq, _capi.i32p), ptr(start, _capi.i32p),
                                               ptr(n_nodes, _capi.i32p), ptr(par, _capi.i32p), ptr(flat, _capi.i32p),
                                               ptr(logits, _capi.f32p) if want_logits else None, ptr(nxt, _capi.i32p),
                                               ptr(acc, _capi.i32p), ptr(path, _capi.i32p)))
        paths, w, r0 = [], 0, 0
        for i in range(n):
            paths.append([int(r) - r0 for r in path[w:w + acc[i] + 1]])
            w += int(acc[i]) + 1
            r0 += len(toks[i])
        return nxt, acc, paths, logits

    def set_sampling(self, seq: int, args: "SamplingArgs | None"):
        """EXTENSION: sequence `seq` samples its next tokens with `args` (None or Temperature 0: greedy) from its next
        forward on; every token output of forward_argmax / forward_batch / forward_ragged / decode_run then carries the
        sampled token for it"""
        if args is None:
            check(lib.lnb_session_set_sampling(self.h, seq, None))
        else:
            c = args.c()
            check(lib.lnb_session_set_sampling(self.h, seq, C.byref(c)))

    def set_penalties(self, seq: int, args: "PenaltyArgs | None", prompt_len: int = 0):
        """EXTENSION: sequence `seq` is penalized with `args` (None or neutral values: off) from its next forward on.
        Turning them on clears the sequence's token history; prompt_len gives first_pos when args.CountPrompt is False."""
        if args is None:
            check(lib.lnb_session_set_penalties(self.h, seq, None))
        else:
            c = args.c(prompt_len)
            check(lib.lnb_session_set_penalties(self.h, seq, C.byref(c)))

    def set_grammar(self, seq: int, grammar: "Grammar | None", first_pos: int = 0):
        """EXTENSION: sequence `seq` is constrained by `grammar` (None: off) from its next forward on; the grammar's start
        state is the state before position first_pos (typically the prompt's length)"""
        check(lib.lnb_session_set_grammar(self.h, seq, None if grammar is None else grammar.h, int(first_pos)))

    def set_logprobs(self, seq: int, top_n: int | None):
        """EXTENSION: from its next forward on, every token sequence `seq` emits writes its logprob record (the raw model
        distribution, its rank and the top_n first tokens, 0..20) at the position it occupies; None turns them off"""
        check(lib.lnb_session_set_logprobs(self.h, seq, -1 if top_n is None else int(top_n)))

    def read_logprobs(self, seq: int, pos0: int, n: int) -> list:
        """the records of positions pos0 .. pos0 + n - 1 of sequence `seq` (TokenLogprob; Token -1: never written)"""
        recs = (_capi.LogprobC * n)()
        check(lib.lnb_session_logprobs_read(self.h, seq, pos0, n, recs))
        return _token_logprobs(recs)

    def copy_sequences(self, src, dst, pos0: int, pos1: int):
        """EXTENSION (lnb_session_copy_sequences): positions [pos0, pos1) of sequence dst[i] get what sequence src[i] held
        there before the call -- K and V of every layer, the penalty history and the logprob records.  The sources are read
        as a snapshot (swaps, cycles and forks are legal in one call); one launch, stream-ordered."""
        src = np.ascontiguousarray(src, np.int32).reshape(-1)
        dst = np.ascontiguousarray(dst, np.int32).reshape(-1)
        if src.shape != dst.shape:
            raise ml.MlError(f"{src.shape[0]} sources for {dst.shape[0]} destinations")
        check(lib.lnb_session_copy_sequences(self.h, int(src.shape[0]), ptr(src, _capi.i32p), ptr(dst, _capi.i32p), int(pos0),
                                             int(pos1)))

    def allow_chunked_prefill(self, on: bool = True):
        """EXTENSION (not in the reference): accept S > 1 at startPos > 0 with the [S,T] causal mask"""
        check(lib.lnb_session_set_chunked_prefill(self.h, int(on)))

    def set_layer_limit(self, n: int):
        check(lib.lnb_session_set_layer_limit(self.h, n))

    def launch_count(self) -> int:
        return int(lib.lnb_session_launch_count(self.h))

    def decode_run(self, first_token: int, start_pos: int, n_steps: int, use_graph: bool = True):
        """device-resident decode (lnb_decode_run; greedy unless the active sequence samples): returns (tokens, ms,
        used_graph)"""
        toks = np.empty(n_steps, np.int32)
        ms = C.c_float(0)
        rc = check(lib.lnb_decode_run(self.h, first_token, start_pos, n_steps, int(use_graph),
                                      ptr(toks, _capi.i32p), C.byref(ms)))
        return toks, ms.value, bool(rc)

    def enable_peer_allreduce(self, all_gather_bytes):
        """Switch this session from NCCL to the fused peer-memory all-reduce.  `all_gather_bytes(b: bytes) ->
        list[bytes]` must return every rank's contribution ordered by rank (e.g. torch.distributed)."""
        buf = C.create_string_buffer(64)
        check(lib.lnb_session_p2p_export(self.h, buf))
        handles = all_gather_bytes(buf.raw)
        blob = b"".join(handles)
        check(lib.lnb_session_p2p_import(self.h, C.create_string_buffer(blob, len(blob)), len(handles)))

    def bench_kernel(self, kind: int, reps: int = 3):
        """(ms per launch, algorithmic weight bytes per launch, launches timed) -- bench.py roofline"""
        ms, nb, nl = C.c_float(0), C.c_int64(0), C.c_int32(0)
        check(lib.lnb_session_bench_kernel(self.h, kind, reps, C.byref(ms), C.byref(nb), C.byref(nl)))
        return ms.value, nb.value, nl.value

    def close(self):
        if self.h:
            if self.pre_close_hook is not None:
                self.pre_close_hook(self)   # peers may still be storing into this session's all-reduce region
            lib.lnb_session_destroy(self.h)
            self.h = None

    def uses_engine(self) -> bool:
        """True: S=1 steps of this context run as the persistent decode engine (one launch per decode_run / Forward)"""
        return bool(check(lib.lnb_session_decode_engine(self.h)))

    def engine_profile(self, batch=False):
        """LNB_ENGINE_PROF=1: {section: (mean cycles, max cycles)} of the decode engine's consumer thread 0 since the last call
        (batch=True: the sections of the batch engine, engine_batch.cuh BatchParams.prof)"""
        out = (C.c_double * 24)()
        check(lib.lnb_session_engine_profile(self.h, out))
        names = ["grid_barrier", "prologue", "main_loop", "epilogue", "attention", "peer_reduce", "input_wait", "scan_maps", "scan_scans",
                 "scan_walk", "scan_count"]
        if batch:
            names = ["grid_barrier", "setup", "x_tile|mma:acc_wait", "stage_wait", "fma|mma:w_wait", "epilogue", "scale", "attention", "other",
                     "tiles", "mma:x_wait", "mma:issue"]
        return {n: (out[2 * i], out[2 * i + 1]) for i, n in enumerate(names)}

    def disable_peer_allreduce(self):
        """back to ncclAllReduce (e.g. after LNB_ETIMEOUT); every rank must do the same"""
        check(lib.lnb_session_p2p_disable(self.h))


class Model:
    """model.Model (src/model/model.go:43-107): args + vocabulary + transformer."""

    def __init__(self, args: ModelArgs, device: int = 0, tp_rank: int = 0, tp_size: int = 1, nccl_id=None,
                 weight_format: str = "bf16"):
        self.ModelArgs = args
        self.Vocabulary = Vocabulary()
        self.Transformer = LlamaTransformer(args, device, tp_rank, tp_size, nccl_id, weight_format)

    def Free(self):
        self.Transformer.close()


def LoadSyntheticModel(args_dict: dict | None = None, seed: int = synth.SEED, device: int = 0, tp_rank: int = 0,
                       tp_size: int = 1, nccl_id=None, weight_format: str = "bf16") -> Model:
    """Stand-in for model.LoadModel (src/model/loader.go:18-70) when no checkpoint exists:
    random-init weights of the given architecture, generated directly in HBM."""
    args = ModelArgs.from_c_dict(args_dict or synth.LLAMA31_8B)
    m = Model(args, device, tp_rank, tp_size, nccl_id, weight_format)
    m.Transformer.init_synthetic(seed)
    m.Transformer.finalize()
    return m


def LoadModelFromTensors(args_dict: dict, tensors: dict[str, np.ndarray], device: int = 0, tp_rank: int = 0,
                         tp_size: int = 1, nccl_id=None, weight_format: str = "bf16") -> Model:
    """The reference's flow (loader.go:22-70): tensors come from host memory (the checkpoint mmap)
    and are bound by name + shape."""
    args = ModelArgs.from_c_dict(args_dict)
    m = Model(args, device, tp_rank, tp_size, nccl_id, weight_format)
    for name, arr in tensors.items():
        m.Transformer.upload_tensor(name, arr)
    m.Transformer.finalize()
    return m


def load_model_args(modelDir: str, max_seq_len: int = 2048) -> dict:
    """loadModelArgs (src/model/loader.go:72-82): params.json -> model args incl. the derived widths"""
    import os
    c = _capi.ModelArgsC()
    check(lib.lnb_model_args_from_params_json(os.path.join(modelDir, "params.json").encode(), max_seq_len, C.byref(c)))
    return {f: getattr(c, f) for f, _ in _capi.ModelArgsC._fields_}


def LoadModel(modelDir: str, device: int = 0, tp_rank: int = 0, tp_size: int = 1, nccl_id=None, max_seq_len: int = 2048,
              weight_format: str = "bf16") -> Model:
    """model.LoadModel (src/model/loader.go:18-70): <modelDir>/consolidated.00.pth + params.json.
    tokenizer.model is optional here: when present it becomes model.Vocabulary and supplies / checks VocabSize like
    the reference (loader.go:84-120); when absent VocabSize falls back to the rows of tok_embeddings.weight."""
    import os
    from .torch_reader import TorchModelReader
    path = os.path.join(modelDir, "consolidated.00.pth")
    d = load_model_args(modelDir, max_seq_len)
    vocab = None
    vocab_path = os.path.join(modelDir, "tokenizer.model")
    if os.path.exists(vocab_path):                      # loadVocab + checkModelArgs (loader.go:84-120)
        from . import vocabulary
        vocab = vocabulary.Load(vocab_path)
        if d["vocab_size"] < 1:
            d["vocab_size"] = len(vocab)
        elif d["vocab_size"] != len(vocab):
            raise _capi.LnbError(-1, f"error while checking config and model: [VocabSize={d['vocab_size']} and vocabulary model "
                                     f"length={len(vocab)} aren't equal]")
    if d["vocab_size"] < 1:
        with TorchModelReader(path) as r:
            t = r.Load().get("tok_embeddings.weight")
        if t is None:
            raise _capi.LnbError(-1, 'tensor "tok_embeddings.weight" not found')
        d["vocab_size"] = t.Size[0]
    m = Model(ModelArgs.from_c_dict(d), device, tp_rank, tp_size, nccl_id, weight_format)
    if vocab is not None:
        m.Vocabulary = vocab
    try:
        m.Transformer.load_pth(path)
        m.Transformer.finalize()
    except Exception:
        m.Free()
        raise
    return m


def applyScaling(freqs: ml.Tensor) -> ml.Tensor:
    """applyScaling (src/model/llamatransformer.go:662-692): the Llama-3.1 inverse-frequency remap, evaluated in
    float32 per element on a bf16 vector"""
    scaleFactor, lowFreqFactor, highFreqFactor, oldContextLen = np.float32(8), np.float32(1), np.float32(4), np.float32(8192)
    lowFreqWavelen, highFreqWavelen = oldContextLen / lowFreqFactor, oldContextLen / highFreqFactor
    twoPi = np.float32(2.0 * np.pi)
    out = []
    for freq in freqs.to_f32_array():
        freq = np.float32(freq)
        wavelen = twoPi / freq
        if wavelen < highFreqWavelen:
            new = freq
        elif wavelen > lowFreqWavelen:
            new = freq / scaleFactor
        else:
            smooth = (oldContextLen / wavelen - lowFreqFactor) / (highFreqFactor - lowFreqFactor)
            new = np.float32((np.float32(1) - smooth) * freq) / scaleFactor + np.float32(smooth * freq)
        out.append(np.float32(new))
    return ml.Tensor.from_f32(np.array(out, np.float32), ml.DT_BF16)


def precomputeFreqsCis(dim: int, end: int, theta: float, useScaled: bool) -> ml.Tensor:
    """precomputeFreqsCis (llamatransformer.go:694-751) from the ml builders, exactly as the Go host does it; the
    result ([end, dim/2] complex64) can be handed to lnb_model_set_rope_table, which otherwise builds the same bits"""
    freqs = ml.ARange(0, dim, 2, ml.DT_BF16)
    val = freqs.to_f32_array()
    freqs = ml.Tensor.from_f32((1.0 / np.power(theta, (val / np.float32(dim)).astype(np.float64))).astype(np.float32), ml.DT_BF16)
    t = ml.ARange(0, end, 1, ml.DT_BF16)
    if useScaled:
        freqs = applyScaling(freqs)
    freqs = ml.Outer(t, freqs)
    return ml.Polar(ml.OnesLike(freqs), freqs)
