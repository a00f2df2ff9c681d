"""A catalogue of small model shapes with the traits of published Llama shapes (GQA ratios 1..16, head_dim 48..256, widths
off the 128-wide tiles, unscaled RoPE), and a host restatement of what the library does with a shape, so a test can say
which route each call takes before it compares bits:

- lnb_model_create (api.cu:264-281): positive dimensions, n_heads % n_kv_heads == 0, head_dim % 8 == 0 (every attention
  kernel reads a K/V row as 16-byte vectors), dim / q_l / kv_l multiples of 32, ffn_l / vocab_l multiples of 16;
- session creation (api.cu:1216-1218): sdpa_kernel keeps a row's seq_len scores in shared memory; past that every row streams
  (stream_attn), which ss_shape_ok (api.cu:889: head_dim % 8 == 0, head_dim <= 128, n_rep 1..8) must admit;
- sdpa_smem_decode (api.cu:1231-1237): the whole K/V history of one KV head fits sdpa_decode_kernel's shared memory;
- engine_probe (api.cu:1500-1523): the decode engine, and with it the batch engine (batch_engine_usable, api.cu:1832), or
  the first no(...) reason that applies; STRICT also needs dim to fit the binade scan (eng_scan_shape, engine.cuh:325);
- forward_tc_ok (api.cu:2122): a FAST prompt of >= 32 rows runs on the tensor cores only when every projection is
  tc_eligible (api.cu:1032: N and K multiples of 128);
- launch_attention (api.cu:2054-2092): which attention kernel a call's rows run."""
from __future__ import annotations

from tests.engine_shapes import ENG_WORK, eng_sdpa_smem

ENG_XMAX = 56 * 1024        # engine.cuh:103
ENG_NCONS = 256             # engine.cuh:99
SMEM_200K = 200 * 1024      # sdpa_kernel / sdpa_decode_kernel dynamic shared memory
TC_BN = TC_KT = 128         # gemm_tc.cuh:41
SP_HD = 128                 # kernels.cuh:312: sdpa_tc_kernel / sdpa_prefill_kernel serve this head_dim only
BATCH_NORM_BYTES = 16 * 1024   # batch_engine_usable: norm weights as f32 in 16 KB of shared memory


def _args(dim, n_heads, n_kv_heads, ffn_dim, vocab_size, n_layers=2, max_seq_len=1024, rope_theta=500000.0, use_scaled_rope=1):
    return dict(dim=dim, n_layers=n_layers, n_heads=n_heads, n_kv_heads=n_kv_heads, head_dim=dim // n_heads, ffn_dim=ffn_dim,
                vocab_size=vocab_size, max_seq_len=max_seq_len, norm_eps=1e-5, rope_theta=rope_theta,
                use_scaled_rope=use_scaled_rope)


# Miniatures of published shapes: each keeps the traits named beside it, not the size.  head_dim = dim / n_heads throughout,
# so every entry can be written as a Meta params.json.
CATALOGUE = {
    # Llama 2 7B: MHA, unscaled RoPE at theta 10000; ffn and vocab off the 128-wide tiles (FAST prompts stay on the chain)
    "mha": _args(768, 12, 12, 1376, 1040, rope_theta=10000.0, use_scaled_rope=0),
    # Llama 3.2 3B: 24 / 8 heads of 128 -- sdpa_tc_kernel's GQA head mapping at n_rep 3
    "gqa3": _args(1536, 12, 4, 4096, 2048),
    # Llama 3.1 70B / TinyLlama: n_rep 8
    "gqa8": _args(1024, 16, 2, 2816, 2048),
    # head_dim 96, not a power of two, n_rep 2
    "hd96": _args(768, 8, 4, 2048, 1024),
    # llama2.c stories15M's widths: dim 288 (no tensor-core GEMM, no STRICT engine scan), 6 heads of 48, MHA
    "stories": _args(288, 6, 6, 768, 1008, rope_theta=10000.0, use_scaled_rope=0),
    # head_dim 256: accepted, single-sequence calls on the kernel chain only.  max_seq_len reaches past sdpa_kernel's limit
    "hd256": _args(1024, 4, 2, 1024, 1024, max_seq_len=17100),
    # n_rep 16: accepted, single-sequence calls on the kernel chain only
    "rep16": _args(1024, 32, 2, 2048, 1024, max_seq_len=17100),
    # the shortest phase list
    "one_layer": _args(256, 8, 2, 512, 1024, n_layers=1, max_seq_len=64),
}

# shapes lnb_model_create must refuse: name -> (args, a fragment of lnb_last_error)
_T = CATALOGUE["one_layer"]
REFUSED = {
    "hd36": (dict(_T, dim=576, n_heads=16, n_kv_heads=16, head_dim=36), "multiple of 8"),
    "hd44": (dict(_T, dim=704, n_heads=16, n_kv_heads=16, head_dim=44), "multiple of 8"),
    "hd33": (dict(_T, dim=1056, n_heads=32, n_kv_heads=32, head_dim=33), "multiple of 8"),
    "heads_7_2": (dict(_T, n_heads=7), "not a multiple of n_kv_heads"),
    "heads_8_3": (dict(_T, n_kv_heads=3), "not a multiple of n_kv_heads"),
    "dim_272": (dict(_T, dim=272), "not tileable"),
    "q_l_24": (dict(_T, n_heads=3, n_kv_heads=1, head_dim=8), "not tileable"),
    "kv_l_16": (dict(_T, n_heads=8, n_kv_heads=1, head_dim=16), "not tileable"),
    "ffn_520": (dict(_T, ffn_dim=520), "not tileable"),
    "vocab_1032": (dict(_T, vocab_size=1032), "not tileable"),
}


def n_rep(args: dict) -> int:
    return args["n_heads"] // args["n_kv_heads"]


def widths(args: dict) -> dict:
    hd = args["head_dim"]
    return dict(q_l=args["n_heads"] * hd, kv_l=args["n_kv_heads"] * hd, ffn_l=args["ffn_dim"], vocab_l=args["vocab_size"])


def create_error(args: dict) -> str | None:
    """the fragment of lnb_last_error lnb_model_create fails with (single GPU), or None: accepted"""
    a = args
    if min(a["dim"], a["n_layers"], a["n_heads"], a["n_kv_heads"], a["head_dim"], a["ffn_dim"], a["vocab_size"], a["max_seq_len"]) <= 0:
        return "non-positive model dimension"
    if a["n_heads"] % a["n_kv_heads"]:
        return "not a multiple of n_kv_heads"
    if a["head_dim"] % 8:
        return "multiple of 8"
    w = widths(a)
    if a["dim"] % 32 or w["q_l"] % 32 or w["kv_l"] % 32 or w["ffn_l"] % 16 or w["vocab_l"] % 16:
        return "not tileable"
    return None


def ss_shape_ok(args: dict) -> bool:
    """the streamed attention kernels serve this head shape (api.cu:889)"""
    hd, r = args["head_dim"], n_rep(args)
    return hd % 8 == 0 and hd <= 128 and 1 <= r <= 8


def stream_attn(args: dict, seq_len: int) -> bool:
    """every row of a session of this SequenceLength streams: sdpa_kernel cannot hold seq_len scores (api.cu:1216)"""
    return seq_len * 12 + args["head_dim"] * 4 > SMEM_200K


def session_error(args: dict, seq_len: int) -> str | None:
    if seq_len > args["max_seq_len"]:
        return "exceeds the RoPE table"
    if stream_attn(args, seq_len) and not ss_shape_ok(args):
        return "needs the streamed attention kernel"
    return None


def sdpa_decode_smem(args: dict, T: int) -> int:
    hd, r = args["head_dim"], n_rep(args)
    return T * ((hd + 8) + hd) * 2 + r * (hd * 4 + T * 12 + 5 * 8) + 256


def sdpa_smem_decode(args: dict, seq_len: int) -> bool:
    """sdpa_decode_kernel serves S = 1 and batched rows of a session of this SequenceLength (api.cu:1231-1237)"""
    hd, r = args["head_dim"], n_rep(args)
    return sdpa_decode_smem(args, seq_len) <= SMEM_200K and r <= 8 and hd <= 128 and hd % 8 == 0


def sdpa_decode_fit(args: dict) -> int:
    """the longest SequenceLength sdpa_decode_kernel holds (0: none)"""
    if not sdpa_smem_decode(args, 1):
        return 0
    T = 1
    while sdpa_smem_decode(args, T + 1):
        T += 1
    return T


def engine_max_seq_len(args: dict) -> int:
    """the longest SequenceLength whose in-engine attention fits the work area (engine_shapes.max_seq_len for any shape)"""
    T = 0
    while eng_sdpa_smem(T + 1, args["head_dim"], n_rep(args)) <= ENG_WORK:
        T += 1
    return T


def eng_scan_shape(D: int) -> tuple[int, int] | None:
    for c in (16, 8, 4, 2):
        if D % c == 0 and (D // c) % 32 == 0 and 32 <= D // c <= ENG_NCONS:
            return c, D // c
    return None


def engine_refusal(args: dict, seq_len: int, strict: bool, sms: int = 132, env: str | None = None) -> str | None:
    """the reason engine_probe gives (lnb_last_error after lnb_session_decode_engine), or None: the decode engine and the
    batch engine can run this session.  env: LNB_ENGINE"""
    if env == "0":
        return "LNB_ENGINE=0"
    w = widths(args)
    d, hd = args["dim"], args["head_dim"]
    if max(d, w["q_l"], w["ffn_l"]) * 4 > ENG_XMAX:
        return "activation vector exceeds the engine's shared-memory work area"
    if d % 8 or w["q_l"] % 8 or w["ffn_l"] % 8:
        return "widths must be multiples of 8"
    if d * 8 > ENG_XMAX:
        return "dim too wide for the engine's RMSNorm prologue"
    if hd > 128 or hd % 8 or n_rep(args) > 8:
        return "head shape"
    if eng_sdpa_smem(seq_len, hd, n_rep(args)) > ENG_WORK:
        return "SequenceLength too long for the in-engine attention phase"
    if strict and eng_scan_shape(d) is None:
        return "dim does not fit the engine's binade scan"
    if w["q_l"] // hd > sms:
        return "more query heads than SMs"
    return None


def uses_engine(args: dict, seq_len: int, strict: bool, sms: int = 132, env: str | None = None) -> bool:
    """single-sequence S = 1 steps run the decode engine: probe passes, and the session is not single-GPU FAST unless
    LNB_ENGINE=1 (api.cu:1503)"""
    return engine_refusal(args, seq_len, strict, sms, env) is None and (strict or env == "1")


def batch_engine(args: dict, seq_len: int, strict: bool, sms: int = 132, env: str | None = None, batch_env: str | None = None) -> bool:
    """batched steps and speculative calls of >= 2 rows run the batch engine (batch_engine_usable, api.cu:1832)"""
    return (engine_refusal(args, seq_len, strict, sms, env) is None and args["dim"] * 4 <= BATCH_NORM_BYTES
            and batch_env != "0")


def tc_eligible(M: int, N: int, K: int) -> bool:
    return M >= 32 and N % TC_BN == 0 and K % TC_KT == 0


def projections_tc(args: dict, S: int) -> dict[str, bool]:
    w = widths(args)
    d, f = args["dim"], w["ffn_l"]
    return {"wqkv": tc_eligible(S, w["q_l"] + 2 * w["kv_l"], d), "wo": tc_eligible(S, d, w["q_l"]),
            "w13": tc_eligible(S, 2 * f, d), "w2": tc_eligible(S, d, f)}


def forward_tc(args: dict, S: int, strict: bool, max_rows: int) -> bool:
    """this forward runs on the tensor cores (forward_tc_ok, api.cu:2122): FAST, a session of >= 32 rows, S >= 32 and every
    projection tc_eligible"""
    return not strict and max_rows >= 32 and S >= 32 and all(projections_tc(args, S).values())


def attention_kernel(args: dict, seq_len: int, kind: str, S: int = 1, strict: bool = True, max_rows: int = 8,
                     sdpa_tc: bool = True) -> str:
    """the kernel launch_attention runs for a call (kind: "single", "batched", "speculative" or "ragged"; S rows), once
    the decode engines are ruled out; "refused" where the call fails with LNB_EINVAL before anything is enqueued"""
    decode_fit = sdpa_smem_decode(args, seq_len)
    if kind == "ragged":
        return "stream" if ss_shape_ok(args) else "refused"
    batched = kind in ("batched", "speculative")
    if batched and not decode_fit and not (ss_shape_ok(args) or stream_attn(args, seq_len)):
        return "refused"
    out_x8 = forward_tc(args, S, strict, max_rows)
    if not out_x8 and (S == 1 or batched) and decode_fit:
        return "sdpa_decode"
    if out_x8 and args["head_dim"] == SP_HD:
        return "sdpa_tc" if sdpa_tc else "sdpa_prefill"
    if batched or stream_attn(args, seq_len):
        return "stream"
    return "sdpa_kernel"


def traits(name: str) -> dict:
    """what a catalogue entry reaches, for the default route of each call kind (132 SMs)"""
    a = CATALOGUE[name]
    fit = sdpa_decode_fit(a)
    return dict(
        n_rep=n_rep(a), head_dim=a["head_dim"], n_layers=a["n_layers"], scaled_rope=bool(a["use_scaled_rope"]),
        rope_theta=a["rope_theta"], ffn_on_tiles=a["ffn_dim"] % 128 == 0, vocab_on_tiles=a["vocab_size"] % 128 == 0,
        strict_engine=engine_refusal(a, 64, True) is None, fast_engine=engine_refusal(a, 64, False) is None,
        batch_engine=batch_engine(a, 64, True), prompt_tc=forward_tc(a, 40, False, 40),
        prompt_attention=attention_kernel(a, 64, "single", 40, strict=False, max_rows=40), decode_fit=fit,
        streamed_batched=ss_shape_ok(a) and fit + 1 <= a["max_seq_len"],
        batched=attention_kernel(a, 64, "batched", 3), ragged=attention_kernel(a, 64, "ragged", 4),
        speculative=attention_kernel(a, 64, "speculative", 4))


def params_json(args: dict) -> dict:
    """a Meta params.json that lnb_model_args_from_params_json turns into `args` (head_dim = dim / n_heads; the FFN width
    from 4 * dim * 2 / 3 scaled by ffn_dim_multiplier and rounded up to multiple_of, llamatransformer.go:569-577)"""
    hidden = int(2 * (4 * args["dim"]) / 3)
    assert args["dim"] % args["n_heads"] == 0 and args["dim"] // args["n_heads"] == args["head_dim"]
    out = {"dim": args["dim"], "n_layers": args["n_layers"], "n_heads": args["n_heads"], "n_kv_heads": args["n_kv_heads"],
           "vocab_size": args["vocab_size"], "multiple_of": 16, "ffn_dim_multiplier": (args["ffn_dim"] + 0.5) / hidden,
           "norm_eps": args["norm_eps"], "rope_theta": args["rope_theta"], "use_scaled_rope": bool(args["use_scaled_rope"])}
    assert 16 * ((int(out["ffn_dim_multiplier"] * hidden) + 15) // 16) == args["ffn_dim"]
    return out
