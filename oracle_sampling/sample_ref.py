"""ctypes binding of the sampler's sequential C statement (TEST INFRASTRUCTURE, NOT PRODUCT CODE; DESIGN.md §9b, §9e, §9g).

Only tests/ and tools/ may import this module.  See lnb_sample_ref.c.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SO = os.path.join(_HERE, "liblnb_sample_ref.so")
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from oracle import oracle as _oracle  # noqa: E402

_f32p, _i32p, _i64p, _u64p, _f64p = (C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_double))
_lib = None

LOGIT_BIAS_MAX = 64


class Penalties(C.Structure):   # lnb_penalties (include/lnb.h)
    _fields_ = [("repetition_penalty", C.c_float), ("frequency_penalty", C.c_float), ("presence_penalty", C.c_float),
                ("window", C.c_int32), ("first_pos", C.c_int32), ("n_bias", C.c_int32),
                ("bias_token", C.c_int32 * LOGIT_BIAS_MAX), ("bias", C.c_float * LOGIT_BIAS_MAX)]


def penalties(rp: float = 1.0, fp: float = 0.0, pp: float = 0.0, window: int = 0, first_pos: int = 0, bias=None) -> Penalties:
    """an lnb_penalties; bias: {token: bias}"""
    p = Penalties(float(rp), float(fp), float(pp), int(window), int(first_pos), 0)
    for j, (t, b) in enumerate((bias or {}).items()):
        p.bias_token[j] = int(t)
        p.bias[j] = float(b)
        p.n_bias = j + 1
    return p


def build(force: bool = False) -> str:
    _oracle.build()
    src = [os.path.join(_HERE, f) for f in ("lnb_sample_ref.c", "Makefile")] + \
          [os.path.join(_ROOT, "llama-nuts-and-bolts_b200", "csrc", f) for f in ("sample_det.h", "penalty_det.h")] + \
          [os.path.join(_ROOT, "include", "lnb.h")]
    stale = (not os.path.exists(_SO)) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in src)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _oracle.lib()
        L = C.CDLL(_SO)
        L.orc_exp_det.restype, L.orc_exp_det.argtypes = C.c_double, [C.c_double]
        L.orc_exp_det_n.restype, L.orc_exp_det_n.argtypes = None, [_f64p, _f64p, C.c_int64]
        L.orc_exp_det_max_ulp_f32.restype, L.orc_exp_det_max_ulp_f32.argtypes = C.c_int64, [C.c_uint32, C.c_uint32]
        L.orc_sample_weight.restype, L.orc_sample_weight.argtypes = C.c_uint64, [C.c_float, C.c_float, C.c_float]
        L.orc_sample_row.restype = C.c_int32
        L.orc_sample_row.argtypes = [_f32p, C.c_int, C.c_float, C.c_int32, C.c_float, C.c_uint64, C.c_int64]
        L.orc_sample_rows.restype = None
        L.orc_sample_rows.argtypes = [_f32p, C.c_int, C.c_int, _f32p, _i32p, _f32p, _u64p, _i64p, _i32p]
        L.orc_logprob_rows.restype = None
        L.orc_logprob_rows.argtypes = [_f32p, C.c_int, C.c_int, _i32p, C.c_int, C.c_void_p]
        L.orc_penalize_rows.restype = None
        L.orc_penalize_rows.argtypes = [_f32p, C.c_int, C.c_int, C.POINTER(Penalties), _i32p, C.c_int, _i32p, _f32p]
        L.orc_generate_processed.restype = C.c_int
        L.orc_generate_processed.argtypes = [C.c_void_p, C.c_int, _i32p, C.c_int, C.c_int, _i32p, C.c_int, C.c_float, C.c_int32,
                                             C.c_float, C.c_uint64, C.POINTER(Penalties), _i32p]
        _u8p = C.POINTER(C.c_uint8)
        L.orc_grammar_masks.restype = C.c_int
        L.orc_grammar_masks.argtypes = [_i32p, _u8p, C.c_int, _u8p, _i64p, C.c_int, _i32p, C.c_int, C.POINTER(C.c_uint32)]
        L.orc_grammar_history.restype = None
        L.orc_grammar_history.argtypes = [_i32p, _u8p, C.c_int, _u8p, _i64p, C.c_int, _i32p, C.c_int, _i32p, C.c_int, C.c_int, _i32p]
        L.orc_generate_constrained.restype = C.c_int
        L.orc_generate_constrained.argtypes = [C.c_void_p, C.c_int, _i32p, C.c_int, C.c_int, _i32p, C.c_int, C.c_float, C.c_int32,
                                               C.c_float, C.c_uint64, C.POINTER(Penalties), _i32p, _u8p, C.c_int, _u8p, _i64p,
                                               _i32p, C.c_int, C.c_int, _i32p]
        _u16p = C.POINTER(C.c_uint16)
        L.orc_mxfp8_quantize.restype = C.c_int64
        L.orc_mxfp8_quantize.argtypes = [_u16p, C.c_int, C.c_int, _u8p, _u8p]
        L.orc_mxfp8_dequantize.restype = None
        L.orc_mxfp8_dequantize.argtypes = [_u8p, _u8p, C.c_int, C.c_int, _u16p]
        L.orc_kv_mxfp8_quantize.restype = None
        L.orc_kv_mxfp8_quantize.argtypes = [_u16p, C.c_int, C.c_int, C.c_int, _u8p, _u8p, _u16p]
        L.orc_mxfp4_quantize.restype = C.c_int64
        L.orc_mxfp4_quantize.argtypes = [_u16p, C.c_int, C.c_int, _u8p, _u8p]
        L.orc_mxfp4_dequantize.restype = None
        L.orc_mxfp4_dequantize.argtypes = [_u8p, _u8p, C.c_int, C.c_int, _u16p]
        L.orc_generate_sampled.restype = C.c_int
        L.orc_generate_sampled.argtypes = [C.c_void_p, C.c_int, _i32p, C.c_int, C.c_int, _i32p, C.c_int, C.c_float, C.c_int32,
                                           C.c_float, C.c_uint64, _i32p]
        _lib = L
    return _lib


def exp_det(z) -> np.ndarray | float:
    """lnb_exp_det (csrc/sample_det.h) of a float or an f64 array"""
    if np.isscalar(z):
        return lib().orc_exp_det(float(z))
    z = np.ascontiguousarray(z, np.float64)
    out = np.empty_like(z)
    lib().orc_exp_det_n(z.ctypes.data_as(_f64p), out.ctypes.data_as(_f64p), z.size)
    return out


def exp_det_max_ulp_f32(lo_bits: int, hi_bits: int) -> int:
    return int(lib().orc_exp_det_max_ulp_f32(lo_bits, hi_bits))


def sample_weight(l: float, m: float, T: float) -> int:
    return int(lib().orc_sample_weight(l, m, T))


def sample_row(logits, T: float, K: int, P: float, seed: int, p_next: int) -> int:
    row = np.ascontiguousarray(logits, np.float32).reshape(-1)
    return int(lib().orc_sample_row(row.ctypes.data_as(_f32p), row.size, T, K, P, seed & (2**64 - 1), p_next))


# lnb_logprob (include/lnb.h) as a numpy record
LOGPROB_DTYPE = np.dtype([("token", "<i4"), ("rank", "<i4"), ("logprob", "<f8"), ("n_top", "<i4"), ("top_token", "<i4", (20,)),
                          ("top_logprob", "<f8", (20,))], align=True)
assert LOGPROB_DTYPE.itemsize == 264


def logprob_rows(logits, targets, top_n: int) -> np.ndarray:
    """orc_logprob_row of every row of logits [rows, V] with its target: LOGPROB_DTYPE [rows]"""
    l = np.ascontiguousarray(logits, np.float32)
    l = l.reshape(-1, l.shape[-1])
    t = np.ascontiguousarray(targets, np.int32).reshape(-1)
    assert t.shape[0] == l.shape[0]
    out = np.zeros(l.shape[0], LOGPROB_DTYPE)
    lib().orc_logprob_rows(l.ctypes.data_as(_f32p), l.shape[0], l.shape[1], t.ctypes.data_as(_i32p), top_n, out.ctypes.data)
    return out


def generate_sampled(om, prompt, seq_len: int, T: float, K: int, P: float, seed: int, stop_ids=(128008, 128009)) -> np.ndarray:
    """orc_generate with the sampler in place of the argmax (om: oracle.OracleModel)"""
    prompt = np.ascontiguousarray(prompt, np.int32)
    stop = np.ascontiguousarray(stop_ids, np.int32)
    out = np.empty(seq_len, np.int32)
    n = lib().orc_generate_sampled(om.h, om.args.vocab, prompt.ctypes.data_as(_i32p), len(prompt), seq_len,
                                   stop.ctypes.data_as(_i32p), len(stop), T, K, P, seed & (2**64 - 1), out.ctypes.data_as(_i32p))
    if n < 0:
        raise RuntimeError("orc_generate_sampled failed")
    return out[:n].copy()


def penalize_rows(logits, params, hist, p_next) -> np.ndarray:
    """orc_penalize_row of every row of logits [rows, V] with params[r] (Penalties), history hist[r] (a row of a
    [rows, hist_len] int array, -1: not counted) and p_next[r]: l' [rows, V] f32"""
    l = np.ascontiguousarray(logits, np.float32)
    l = l.reshape(-1, l.shape[-1])
    rows = l.shape[0]
    h = np.ascontiguousarray(hist, np.int32).reshape(rows, -1)
    pn = np.ascontiguousarray(p_next, np.int32).reshape(-1)
    assert pn.shape[0] == rows and len(params) == rows
    assert all(0 <= int(x) <= h.shape[1] for x in pn)
    par = (Penalties * rows)(*params)
    out = np.empty_like(l)
    lib().orc_penalize_rows(l.ctypes.data_as(_f32p), rows, l.shape[1], par, h.ctypes.data_as(_i32p), h.shape[1],
                            pn.ctypes.data_as(_i32p), out.ctypes.data_as(_f32p))
    return out


def generate_processed(om, prompt, seq_len: int, T: float, K: int, P: float, seed: int, pen: "Penalties | None",
                       stop_ids=(128008, 128009)) -> np.ndarray:
    """orc_generate with the penalties, then the sampler (greedy at T = 0), in place of the argmax (om: oracle.OracleModel)"""
    prompt = np.ascontiguousarray(prompt, np.int32)
    stop = np.ascontiguousarray(stop_ids, np.int32)
    out = np.empty(seq_len, np.int32)
    n = lib().orc_generate_processed(om.h, om.args.vocab, prompt.ctypes.data_as(_i32p), len(prompt), seq_len,
                                     stop.ctypes.data_as(_i32p), len(stop), T, K, P, seed & (2**64 - 1),
                                     C.byref(pen) if pen is not None else None, out.ctypes.data_as(_i32p))
    if n < 0:
        raise RuntimeError("orc_generate_processed failed")
    return out[:n].copy()


# ---- grammars (DESIGN.md §9g) -----------------------------------------------------------------------------------------------
class GrammarTables:
    """a grammar as the C statement takes it: trans int32 [Q, 256] (-1: ⊥), accept [Q], the bytes of each of the V tokens,
    the stop set"""

    def __init__(self, trans, accept, token_bytes, stop_ids):
        self.trans = np.ascontiguousarray(trans, np.int32)
        self.accept = np.ascontiguousarray(accept, np.uint8)
        self.Q = int(self.accept.shape[0])
        self.V = len(token_bytes)
        self.off = np.zeros(self.V + 1, np.int64)
        self.off[1:] = np.cumsum([len(b) for b in token_bytes])
        self.bytes = np.frombuffer(b"".join(token_bytes) + b"\0", np.uint8).copy()
        self.stop = np.ascontiguousarray(stop_ids, np.int32)

    def args(self):
        u8 = C.POINTER(C.c_uint8)
        return (self.trans.ctypes.data_as(_i32p), self.accept.ctypes.data_as(u8), self.Q, self.bytes.ctypes.data_as(u8),
                self.off.ctypes.data_as(_i64p), self.V, self.stop.ctypes.data_as(_i32p), int(self.stop.shape[0]))


def grammar_masks(g: GrammarTables) -> tuple:
    """orc_grammar_masks: (uint32 [Q + 1, ceil(V / 32)], row Q = ⊥; the number of states whose mask is Z)"""
    out = np.zeros((g.Q + 1, (g.V + 31) // 32), np.uint32)
    stuck = lib().orc_grammar_masks(*g.args(), out.ctypes.data_as(C.POINTER(C.c_uint32)))
    return out, int(stuck)


def grammar_history(g: GrammarTables, tokens, first_pos: int) -> np.ndarray:
    """orc_grammar_history: the state before each position 0 .. n of tokens fed at 0 .. n-1 (-1: ⊥)"""
    t = np.ascontiguousarray(tokens, np.int32)
    out = np.empty(t.shape[0] + 1, np.int32)
    lib().orc_grammar_history(*g.args(), t.ctypes.data_as(_i32p), int(t.shape[0]), int(first_pos), out.ctypes.data_as(_i32p))
    return out


def generate_constrained(om, prompt, seq_len: int, T: float, K: int, P: float, seed: int, pen: "Penalties | None",
                         g: GrammarTables, first_pos: int, stop_ids=(128008, 128009)) -> np.ndarray:
    """orc_generate_processed with the grammar's mask between the penalties and the sampler (om: oracle.OracleModel)"""
    prompt = np.ascontiguousarray(prompt, np.int32)
    stop = np.ascontiguousarray(stop_ids, np.int32)
    out = np.empty(seq_len, np.int32)
    a = g.args()
    n = lib().orc_generate_constrained(om.h, om.args.vocab, prompt.ctypes.data_as(_i32p), len(prompt), seq_len,
                                       stop.ctypes.data_as(_i32p), len(stop), T, K, P, seed & (2**64 - 1),
                                       C.byref(pen) if pen is not None else None, a[0], a[1], a[2], a[3], a[4], a[6], a[7],
                                       int(first_pos), out.ctypes.data_as(_i32p))
    if n < 0:
        raise RuntimeError("orc_generate_constrained failed")
    return out[:n].copy()


# ---- beam search (DESIGN.md §9f) -----------------------------------------------------------------------------------------
_STEP_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, _i32p, _i32p, _f64p, _i32p)
_REORDER_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, _i32p, _i32p, C.c_int, C.c_int)


class _BeamIO(C.Structure):   # orc_beam_io
    _fields_ = [("ctx", C.c_void_p), ("step", _STEP_CB), ("reorder", _REORDER_CB)]


def _beam_lib():
    L = lib()
    if not getattr(L, "_beam_bound", False):
        L.orc_beam_select.restype = None
        L.orc_beam_select.argtypes = [_f64p, _i32p, _i32p, _i32p, C.c_int, C.c_int, _i32p, C.c_int, _i32p, _i32p, _i32p, _i32p]
        L.orc_beam_pool_run.restype = C.c_int
        L.orc_beam_pool_run.argtypes = [_f64p, C.c_int, C.c_int, _i32p]
        out = [_i32p, _f64p, _i32p, _f64p, _f64p, _i32p]
        L.orc_beam_search_io.restype = C.c_int
        L.orc_beam_search_io.argtypes = [C.POINTER(_BeamIO), C.c_int, C.c_int, _i32p, C.c_int, C.c_int, C.c_double, C.c_int] + out
        L.orc_beam_search.restype = C.c_int
        L.orc_beam_search.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _i32p, C.c_int, C.c_int, _i32p, C.c_int, C.c_int,
                                      C.c_double, C.c_int] + out + [_i64p]
        L._beam_bound = True
    return L


def beam_select(cands, B: int, stop):
    """orc_beam_select: cands (score, beam, rank, token) -> (new beams, finished) as lists of candidate tuples in walk order"""
    n = len(cands)
    sc = np.array([c[0] for c in cands], np.float64)
    bm = np.array([c[1] for c in cands], np.int32)
    rk = np.array([c[2] for c in cands], np.int32)
    tk = np.array([c[3] for c in cands], np.int32)
    st = np.ascontiguousarray(list(stop) or [-1], np.int32)
    ni, fi = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
    nn, nf = C.c_int32(0), C.c_int32(0)
    _beam_lib().orc_beam_select(sc.ctypes.data_as(_f64p), bm.ctypes.data_as(_i32p), rk.ctypes.data_as(_i32p), tk.ctypes.data_as(_i32p),
                                n, B, st.ctypes.data_as(_i32p), len(list(stop)), ni.ctypes.data_as(_i32p), C.byref(nn),
                                fi.ctypes.data_as(_i32p), C.byref(nf))
    row = lambda i: (float(sc[i]), int(bm[i]), int(rk[i]), int(tk[i]))   # noqa: E731
    return [row(i) for i in ni[:nn.value]], [row(i) for i in fi[:nf.value]]


def beam_pool_run(h, B: int) -> list:
    """orc_beam_pool_run: the insertion indices a pool of B keeps after inserting h[0..n) in order, best first"""
    hh = np.ascontiguousarray(h, np.float64)
    kept = np.zeros(B, np.int32)
    m = _beam_lib().orc_beam_pool_run(hh.ctypes.data_as(_f64p), hh.shape[0], B, kept.ctypes.data_as(_i32p))
    if m < 0:
        raise ValueError(f"pool size {B} outside [1, 8]")
    return [int(x) for x in kept[:m]]


def _beam_out(n, tok, lp, ln, s, h, state):
    return [dict(tokens=[int(t) for t in tok[i, :ln[i]]], logprobs=[float(x) for x in lp[i, :ln[i]]], s=float(s[i]), h=float(h[i]),
                 state=int(state[i])) for i in range(n)]


def beam_search_io(step, reorder, n_prompt: int, seq_len: int, stop, B: int, alpha: float, early: bool) -> list:
    """orc_beam_search_io with Python callbacks: step(k, last[n]) -> per live beam a list of (token, logprob) in rank order;
    reorder(src, dst, pos0, pos1).  Returns the hypotheses (dicts: tokens, logprobs, s, h, state), best first."""
    def _step(ctx, k, n, last, top_tok, top_lp, n_top):
        rows = step(k, [int(last[b]) for b in range(n)])
        for b, r in enumerate(rows):
            n_top[b] = len(r)
            for j, (t, x) in enumerate(r):
                top_tok[b * 20 + j] = int(t)
                top_lp[b * 20 + j] = float(x)
        return 0

    def _reorder(ctx, n, src, dst, pos0, pos1):
        reorder([int(src[i]) for i in range(n)], [int(dst[i]) for i in range(n)], int(pos0), int(pos1))
        return 0

    io = _BeamIO(None, _STEP_CB(_step), _REORDER_CB(_reorder))
    st = np.ascontiguousarray(list(stop) or [-1], np.int32)
    tok, lp = np.zeros((B, seq_len), np.int32), np.zeros((B, seq_len), np.float64)
    ln, state = np.zeros(B, np.int32), np.zeros(B, np.int32)
    s, h = np.zeros(B, np.float64), np.zeros(B, np.float64)
    n = _beam_lib().orc_beam_search_io(C.byref(io), n_prompt, seq_len, st.ctypes.data_as(_i32p), len(list(stop)), B, alpha, int(early),
                                       tok.ctypes.data_as(_i32p), lp.ctypes.data_as(_f64p), ln.ctypes.data_as(_i32p),
                                       s.ctypes.data_as(_f64p), h.ctypes.data_as(_f64p), state.ctypes.data_as(_i32p))
    if n < 0:
        raise RuntimeError("orc_beam_search_io failed")
    return _beam_out(n, tok, lp, ln, s, h, state)


def beam_search(om, prompt, seq_len: int, B: int, alpha: float = 1.0, early: bool = False, stop_ids=(128008, 128009)):
    """orc_beam_search on the oracle model (om: oracle.OracleModel): (hypotheses best first, number of reorders)"""
    a = om.args
    prompt = np.ascontiguousarray(prompt, np.int32)
    st = np.ascontiguousarray(list(stop_ids) or [-1], np.int32)
    tok, lp = np.zeros((B, seq_len), np.int32), np.zeros((B, seq_len), np.float64)
    ln, state = np.zeros(B, np.int32), np.zeros(B, np.int32)
    s, h = np.zeros(B, np.float64), np.zeros(B, np.float64)
    moves = C.c_int64(0)
    n = _beam_lib().orc_beam_search(om.h, a.vocab, a.n_layers, a.n_kv_heads * a.head_dim, prompt.ctypes.data_as(_i32p), len(prompt),
                                    seq_len, st.ctypes.data_as(_i32p), len(list(stop_ids)), B, alpha, int(early),
                                    tok.ctypes.data_as(_i32p), lp.ctypes.data_as(_f64p), ln.ctypes.data_as(_i32p),
                                    s.ctypes.data_as(_f64p), h.ctypes.data_as(_f64p), state.ctypes.data_as(_i32p), C.byref(moves))
    if n < 0:
        raise RuntimeError("orc_beam_search failed")
    return _beam_out(n, tok, lp, ln, s, h, state), int(moves.value)


def mxfp8_quantize(w) -> tuple[np.ndarray, np.ndarray]:
    """orc_mxfp8_quantize of a bf16 matrix (uint16 bits [rows, cols]): (codes [rows, cols] u8, scales [rows, ceil(cols/32)]
    u8).  A non-finite weight raises ValueError naming its row and column."""
    w = np.ascontiguousarray(w, np.uint16)
    rows, cols = w.shape
    codes = np.empty((rows, cols), np.uint8)
    scales = np.empty((rows, (cols + 31) // 32), np.uint8)
    u8 = C.POINTER(C.c_uint8)
    bad = lib().orc_mxfp8_quantize(w.ctypes.data_as(C.POINTER(C.c_uint16)), rows, cols, codes.ctypes.data_as(u8),
                                   scales.ctypes.data_as(u8))
    if bad >= 0:
        raise ValueError(f"non-finite weight at row {bad // cols}, column {bad % cols}")
    return codes, scales


def mxfp8_dequantize(codes, scales) -> np.ndarray:
    """orc_mxfp8_dequantize: the bf16 bits [rows, cols] of e4m3(code) * 2^X"""
    codes = np.ascontiguousarray(codes, np.uint8)
    scales = np.ascontiguousarray(scales, np.uint8)
    rows, cols = codes.shape
    assert scales.shape == (rows, (cols + 31) // 32)
    out = np.empty((rows, cols), np.uint16)
    u8 = C.POINTER(C.c_uint8)
    lib().orc_mxfp8_dequantize(codes.ctypes.data_as(u8), scales.ctypes.data_as(u8), rows, cols,
                               out.ctypes.data_as(C.POINTER(C.c_uint16)))
    return out


def kv_mxfp8_quantize(rows, head_dim: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """orc_kv_mxfp8_quantize of K or V rows (uint16 bits [n, n_kv * head_dim]): (codes [n, n_kv * head_dim] u8, scales
    [n, n_kv, ceil(head_dim / 32)] u8, decoded rows [n, n_kv * head_dim] bf16 bits)"""
    rows = np.ascontiguousarray(rows, np.uint16)
    n, kv = rows.shape
    n_kv = kv // head_dim
    codes = np.empty((n, kv), np.uint8)
    scales = np.empty((n, n_kv, (head_dim + 31) // 32), np.uint8)
    deq = np.empty((n, kv), np.uint16)
    u8 = C.POINTER(C.c_uint8)
    lib().orc_kv_mxfp8_quantize(rows.ctypes.data_as(C.POINTER(C.c_uint16)), n, head_dim, n_kv, codes.ctypes.data_as(u8),
                                scales.ctypes.data_as(u8), deq.ctypes.data_as(C.POINTER(C.c_uint16)))
    return codes, scales, deq


def mxfp4_quantize(w) -> tuple[np.ndarray, np.ndarray]:
    """orc_mxfp4_quantize of a bf16 matrix (uint16 bits [rows, cols], cols even): (codes [rows, cols / 2] u8, two a byte
    with the even column in the low nibble, scales [rows, ceil(cols/32)] u8).  A non-finite weight raises ValueError
    naming its row and column."""
    w = np.ascontiguousarray(w, np.uint16)
    rows, cols = w.shape
    assert cols % 2 == 0
    codes = np.empty((rows, cols // 2), np.uint8)
    scales = np.empty((rows, (cols + 31) // 32), np.uint8)
    u8 = C.POINTER(C.c_uint8)
    bad = lib().orc_mxfp4_quantize(w.ctypes.data_as(C.POINTER(C.c_uint16)), rows, cols, codes.ctypes.data_as(u8),
                                   scales.ctypes.data_as(u8))
    if bad >= 0:
        raise ValueError(f"non-finite weight at row {bad // cols}, column {bad % cols}")
    return codes, scales


def mxfp4_dequantize(codes, scales) -> np.ndarray:
    """orc_mxfp4_dequantize: the bf16 bits [rows, 2 * codes.shape[1]] of e2m1(code) * 2^X"""
    codes = np.ascontiguousarray(codes, np.uint8)
    scales = np.ascontiguousarray(scales, np.uint8)
    rows, cols = codes.shape[0], 2 * codes.shape[1]
    assert scales.shape == (rows, (cols + 31) // 32)
    out = np.empty((rows, cols), np.uint16)
    u8 = C.POINTER(C.c_uint8)
    lib().orc_mxfp4_dequantize(codes.ctypes.data_as(u8), scales.ctypes.data_as(u8), rows, cols,
                               out.ctypes.data_as(C.POINTER(C.c_uint16)))
    return out
