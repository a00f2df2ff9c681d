"""Models and shapes for the MXFP8 KV cache's edge tests (DESIGN.md §9j), shared by the CPU and GPU suites.

- extreme_kv_tensors: a synthetic checkpoint whose K and V heads are scaled by powers of two (exact in bf16) so that the
  blocks a forward stores reach the ends of the E8M0 range -- X = -117 with subnormal and flushed codes, K blocks at
  X >= 100 and V blocks at X = 119 (values >= 2^127) -- beside ordinary heads in the same row.  The query rows of each
  scaled head's group and the output-projection columns of that head carry the inverse power, so the residual stream and
  the logits stay ordinary, and a decode that is wrong only at the range's ends changes the logits.
- nonfinite_kv_tensors: one V head of layer 0 that stores +inf and -inf at the position of one chosen token.
- decode: the block rule's decode restated from the codes and scales, with switches for four broken decodes.
- SHAPES: head shapes the streamed kernels admit beyond tests/model_shapes.CATALOGUE -- tail blocks of 8 and 24 columns,
  STRICT d-ranges whose scale block spans two CTAs, n_rep 5..7 and the largest shared-memory configuration."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O
from oracle_sampling import sample_ref as SR
from tests.helpers import host_tensors
from tests.model_shapes import _args

# X of the blocks the extreme heads are aimed at: layer 0 head 0 K (>= 100) and V (119), layer 1 head 0 K and V (-117)
K_HIGH, V_HIGH, LOW = 106, 119, -119


def _times_pow2(w: np.ndarray, e: int) -> np.ndarray:
    """bf16 bits w * 2^e (in f64: 2^e itself may lie outside f32)"""
    return O.bf16_bits((O.bf16_to_f32(w).astype(np.float64) * 2.0 ** e).astype(np.float32))


def _scale_rows(w: np.ndarray, rows: slice, e: int) -> None:
    w[rows] = _times_pow2(w[rows], e).reshape(w[rows].shape)


def _scale_cols(w: np.ndarray, cols: slice, e: int) -> None:
    w[:, cols] = _times_pow2(w[:, cols], e).reshape(w[:, cols].shape)


def _layer0_rows(args: dict, t: dict, name: str, head: int) -> np.ndarray:
    """K (before RoPE) or V rows of layer 0, KV head `head`, for every token of the vocabulary: [vocab, head_dim] f32,
    in the STRICT order and in the FAST GEMV order (layer 0 depends on the token alone)"""
    hd = args["head_dim"]
    xn = O.rmsnorm(np.ascontiguousarray(t["tok_embeddings.weight"]), t["layers.0.attention_norm.weight"], args["norm_eps"])
    w = np.ascontiguousarray(t[f"layers.0.attention.{name}.weight"][head * hd:(head + 1) * hd])
    return [O.bf16_to_f32(O.linear_order_bf16(xn, w, ks)) for ks in (1, O.ORDER_FAST_STREAM[0])]


def _sigma(args: dict, t: dict, l: int, name: str, head: int) -> float:
    """the typical magnitude of an element of KV head `head` of layer l's K or V rows: the rows read RMSNorm's output,
    whose elements are the norm weights times values of unit RMS"""
    hd = args["head_dim"]
    w = O.bf16_to_f32(t[f"layers.{l}.attention.{name}.weight"][head * hd:(head + 1) * hd]).astype(np.float64)
    g = O.bf16_to_f32(t[f"layers.{l}.attention_norm.weight"]).astype(np.float64)
    return float(np.sqrt(((w * g[None, :]) ** 2).sum(1).mean()))


def _scale_head(args: dict, t: dict, l: int, head: int, ek: int, ev: int) -> None:
    """K rows of KV head `head` times 2^ek and its group's query rows times 2^-ek; V rows times 2^ev and the head's
    output-projection columns times 2^-ev"""
    hd, rep = args["head_dim"], args["n_heads"] // args["n_kv_heads"]
    p = f"layers.{l}."
    h = slice(head * hd, (head + 1) * hd)
    q = slice(head * rep * hd, (head + 1) * rep * hd)
    _scale_rows(t[p + "attention.wk.weight"], h, ek)
    _scale_rows(t[p + "attention.wq.weight"], q, -ek)
    _scale_rows(t[p + "attention.wv.weight"], h, ev)
    _scale_cols(t[p + "attention.wo.weight"], q, -ev)


def _copy(tensors: dict) -> dict:
    return {k: np.array(v, copy=True) for k, v in tensors.items()}


def extreme_kv_tensors(args: dict, seed: int) -> tuple[dict, list]:
    """(tensors, hot): host_tensors(args, seed) with KV head 0 of layer 0 aimed at K blocks of X ~ K_HIGH and V blocks of
    X = 119, and KV head 0 of the last layer at blocks clamped to X = -117 (amax ~ 2^LOW: subnormal and flushed codes);
    every other head ordinary.  hot: the tokens whose layer-0 V rows reach X = 119 (a prompt holding one stores such a
    block).  The V exponent is the largest whose rows stay finite for every token in the STRICT and the FAST GEMV order."""
    assert args["n_layers"] >= 2 and args["n_kv_heads"] >= 2
    t = _copy(host_tensors(args, seed))
    k0 = max(float(np.abs(r).max()) for r in _layer0_rows(args, t, "wk", 0))
    ek = K_HIGH + 8 - int(np.floor(np.log2(k0)))        # the largest block of any token at X = K_HIGH
    v0 = max(float(np.abs(r).max()) for r in _layer0_rows(args, t, "wv", 0))
    ev = 127 - int(np.floor(np.log2(v0)))               # the largest V element in [2^127, 2^128)
    while True:
        u = _copy({k: t[k] for k in ("tok_embeddings.weight", "layers.0.attention_norm.weight", "layers.0.attention.wv.weight")})
        _scale_rows(u["layers.0.attention.wv.weight"], slice(0, args["head_dim"]), ev)
        rows = _layer0_rows(args, u, "wv", 0)
        if all(np.isfinite(r).all() for r in rows):
            break
        ev -= 1
    amax = np.abs(rows[0]).reshape(len(rows[0]), -1, min(32, args["head_dim"])).max(2).max(1)
    hot = [int(i) for i in np.flatnonzero(amax >= 2.0 ** 127)]
    _scale_head(args, t, 0, 0, ek, ev)
    l1 = args["n_layers"] - 1
    lk = LOW - int(np.round(np.log2(2.5 * _sigma(args, t, l1, "wk", 0))))
    lv = LOW - int(np.round(np.log2(2.5 * _sigma(args, t, l1, "wv", 0))))
    _scale_head(args, t, l1, 0, lk, lv)
    return t, hot


def extreme_prompt(args: dict, hot: list, n: int, seed: int) -> np.ndarray:
    """n random tokens with hot tokens at every fifth position from 0"""
    rng = np.random.default_rng(seed)
    p = rng.integers(0, args["vocab_size"], n).astype(np.int32)
    for i in range(0, n, 5):
        p[i] = hot[rng.integers(0, len(hot))]
    return p


def nonfinite_kv_tensors(args: dict, seed: int, token: int) -> tuple[dict, tuple]:
    """(tensors, (j_pinf, j_ninf)): host_tensors(args, seed) in which the embedding of `token` is a spike (column i0, which
    every other token's embedding has zeroed) and two V rows of layer 0, KV head 0, read that column with weights
    +-2^127: at a position holding `token` that head's V elements j_pinf and j_ninf overflow to +inf and -inf in any
    summation order; at every other position the spike meets zeros and adds nothing.  (No NaN: inf - inf of two
    overflowing products is NaN only where the products are rounded before the sum, and the fused multiply-adds of the
    STRICT projections keep them exact, so the two forwards would store different values, not different blocks.)"""
    t = _copy(host_tensors(args, seed))
    g = O.bf16_to_f32(t["layers.0.attention_norm.weight"])
    i0 = int(np.argmax(np.abs(g)))
    emb = t["tok_embeddings.weight"]
    emb[:, i0] = 0
    emb[token] = 0
    emb[token, i0] = O.bf16_bits(np.float32([1.0]))[0]
    xn = O.bf16_to_f32(O.rmsnorm(np.ascontiguousarray(emb[token:token + 1]), t["layers.0.attention_norm.weight"], args["norm_eps"]))[0]
    assert abs(xn[i0]) >= 2.0, "the spike does not overflow the products"
    s0 = float(np.sign(xn[i0]))
    wv = t["layers.0.attention.wv.weight"]
    j = (1, 6)                                               # elements of the head's first block
    wv[j[0], i0] = O.bf16_bits(np.float32([s0 * 2.0 ** 127]))[0]
    wv[j[1], i0] = O.bf16_bits(np.float32([-s0 * 2.0 ** 127]))[0]
    return t, j


# ---- the block rule's decode, restated -------------------------------------------------------------------------------
def _e4m3_value(c: np.ndarray) -> np.ndarray:
    c = c.astype(np.int64)
    e, m = (c >> 3) & 0xF, c & 7
    mag = np.where(e == 0, m * 2.0 ** -9, (1 + m / 8.0) * 2.0 ** (e - 7.0))
    return np.where(c & 0x80, -mag, mag)


def decode(codes, scales, head_dim: int, flush_subnormal=False, high_from=None, high_at=None, sat_as_7d=False) -> np.ndarray:
    """bf16 bits [n, n_kv * head_dim] of e4m3(code) * 2^X (NaN codes -> 0x7fc0).  The switches break it: subnormal codes
    read as 0; X read one binade high when X >= high_from, or when X == high_at; code 0x7e read as 0x7d"""
    codes = np.asarray(codes, np.uint8)
    n, kv = codes.shape
    nb = (head_dim + 31) // 32
    col = np.arange(kv)
    X = np.asarray(scales, np.int64).reshape(n, -1, nb)[:, col // head_dim, (col % head_dim) // 32] - 127
    if high_from is not None:
        X = np.where(X >= high_from, X + 1, X)
    if high_at is not None:
        X = np.where(X == high_at, X + 1, X)
    c = codes.astype(np.int64)
    if sat_as_7d:
        c = np.where((c & 0x7F) == 0x7E, c - 1, c)
    v = _e4m3_value(c)
    if flush_subnormal:
        v = np.where((c & 0x78) == 0, 0.0, v)
    with np.errstate(over="ignore"):        # a broken decode may read 448 * 2^120: inf
        out = O.bf16_bits((v * np.exp2(X.astype(np.float64))).astype(np.float32))
    return np.where((c & 0x7F) == 0x7F, np.uint16(0x7FC0), out).astype(np.uint16)


def c_decode(rows, head_dim: int) -> np.ndarray:
    """the C statement's decoded rows"""
    return SR.kv_mxfp8_quantize(rows, head_dim)[2]


# ---- head shapes beyond the catalogue ----------------------------------------------------------------------------------
SHAPES = {
    "hd40": _args(320, 8, 4, 640, 1024),         # tail block of 8 columns
    "hd56": _args(448, 8, 4, 896, 1024),         # tail block of 24 columns
    "hd80": _args(640, 8, 2, 1280, 1024, max_seq_len=2048),     # STRICT d-range of 40 columns: a block spans two CTAs
    "hd112": _args(896, 8, 2, 1792, 1024, max_seq_len=2048),    # STRICT d-range of 56 columns
    "rep5": _args(320, 10, 2, 640, 1024),
    "rep6": _args(384, 12, 2, 768, 1024),
    "rep7": _args(448, 14, 2, 896, 1024),
    "hd128_rep8": _args(2048, 16, 2, 2048, 1024, max_seq_len=2048),   # the largest shared memory ss_shape_ok admits (FAST)
}
LONG_SHAPES = ("hd80", "hd112", "hd128_rep8")
