"""ctypes binding of the CPU oracle (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.  See oracle/lnb_oracle.h for what each function restates
(reference file:line) and for the parity status.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liblnb_oracle.so")


def build(force: bool = False) -> str:
    src = [os.path.join(_HERE, f) for f in ("lnb_oracle.c", "lnb_oracle.h", "Makefile")]
    stale = (not os.path.exists(_SO)) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in src)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_lib = None


def usable_cpus() -> int:
    """CPUs this process may really use: affinity mask, capped by the cgroup CPU quota (containers often
    expose all host cores in nproc while granting only a few; an OpenMP team larger than that spends its
    time spinning at barriers)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except Exception:
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                n = min(n, max(1, q // per))
        except Exception:
            pass
    return max(1, n)


def lib():
    global _lib
    if _lib is None:
        build()
        os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")   # idle team members sleep instead of spinning
        _lib = C.CDLL(_SO)
        _declare(_lib)
        want = int(os.environ.get("LNB_ORACLE_THREADS", "0")) or min(usable_cpus(), 64)
        _lib.orc_set_num_threads(want)
    return _lib


class OrcArgs(C.Structure):
    _fields_ = [
        ("dim", C.c_int), ("n_layers", C.c_int), ("n_heads", C.c_int), ("n_kv_heads", C.c_int),
        ("head_dim", C.c_int), ("ffn_dim", C.c_int), ("vocab", C.c_int), ("max_seq_len", C.c_int),
        ("norm_eps", C.c_float), ("rope_theta", C.c_double), ("use_scaled_rope", C.c_int),
    ]


class OrcOrder(C.Structure):
    _fields_ = [("ks", C.c_int), ("rms_parts", C.c_int), ("attn", C.c_int)]


# summation orders (lnb_oracle.h): (ks, rms_parts, attn).  ATTN_REF is the reference's order; FAST / FAST_STREAM state the
# order of LNB_ACC_FAST on the FMA pipe with the shared-memory attention kernels / the streamed attention kernels
ATTN_REF, ATTN_TREE, ATTN_STREAM = 0, 1, 2
ORDER_REF = (1, 1, ATTN_REF)
ORDER_FAST = (8, 256, ATTN_TREE)
ORDER_FAST_STREAM = (8, 256, ATTN_STREAM)


def _order(order):
    return C.byref(OrcOrder(*order)) if order is not None else None


_u16p = C.POINTER(C.c_uint16)
_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
_f64p = C.POINTER(C.c_double)


def _declare(L):
    L.orc_f32_to_bf16.restype = C.c_uint16
    L.orc_f32_to_bf16.argtypes = [C.c_float]
    L.orc_bf16_to_f32.restype = C.c_float
    L.orc_bf16_to_f32.argtypes = [C.c_uint16]
    L.orc_linear_bf16.argtypes = [_u16p, _u16p, _u16p, C.c_int, C.c_int, C.c_int]
    L.orc_linear_bf16_f32out.argtypes = [_u16p, _u16p, _f32p, C.c_int, C.c_int, C.c_int]
    L.orc_linear_f32.argtypes = [_f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int]
    L.orc_matmul_bf16.argtypes = [_u16p, _u16p, _u16p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.orc_pow2_bf16.argtypes = [_u16p, _f32p, C.c_int64]
    L.orc_mean_f32.argtypes = [_f32p, _f32p, C.c_int, C.c_int]
    L.orc_add_bf16.argtypes = [_u16p, _u16p, _u16p, C.c_int64]
    L.orc_mul_bf16.argtypes = [_u16p, _u16p, _u16p, C.c_int64]
    L.orc_div_scalar_bf16.argtypes = [_u16p, C.c_uint16, _u16p, C.c_int64]
    L.orc_softmax_f32.argtypes = [_f32p, _f32p, C.c_int, C.c_int]
    L.orc_argmax_f32.restype = C.c_int32
    L.orc_argmax_f32.argtypes = [_f32p, C.c_int]
    L.orc_silu_bf16.argtypes = [_u16p, _u16p, C.c_int64]
    L.orc_silu_table_bf16.argtypes = [_u16p]
    L.orc_get_rows_bf16.argtypes = [_u16p, _i32p, _u16p, C.c_int, C.c_int]
    L.orc_rms_scale.argtypes = [_u16p, _f32p, C.c_int, C.c_int, C.c_float]
    L.orc_rmsnorm_stage1.argtypes = [_u16p, _u16p, C.c_int, C.c_int, C.c_float]
    L.orc_rmsnorm.argtypes = [_u16p, _u16p, _u16p, C.c_int, C.c_int, C.c_float]
    L.orc_rope_table.argtypes = [C.c_int, C.c_int, C.c_double, C.c_int, _u16p, _f32p]
    L.orc_rope_apply.argtypes = [_u16p, _f32p, _u16p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.orc_attention.argtypes = [_u16p, _u16p, _u16p, _u16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    L.orc_attention_pos.argtypes = [_u16p, _u16p, _u16p, _u16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    L.orc_model_new.restype = C.c_void_p
    L.orc_model_new.argtypes = [C.POINTER(OrcArgs)]
    L.orc_model_free.argtypes = [C.c_void_p]
    L.orc_model_bind.restype = C.c_int
    L.orc_model_bind.argtypes = [C.c_void_p, C.c_char_p, _u16p]
    L.orc_session_new.restype = C.c_void_p
    L.orc_session_new.argtypes = [C.c_void_p, C.c_int]
    L.orc_session_free.argtypes = [C.c_void_p]
    L.orc_session_cache_k.restype = _u16p
    L.orc_session_cache_k.argtypes = [C.c_void_p, C.c_int]
    L.orc_session_cache_v.restype = _u16p
    L.orc_session_cache_v.argtypes = [C.c_void_p, C.c_int]
    L.orc_forward.restype = C.c_int
    L.orc_forward.argtypes = [C.c_void_p, C.c_void_p, _i32p, C.c_int, C.c_int, _f32p, C.c_int, _u16p]
    L.orc_forward_chunk.restype = C.c_int
    L.orc_forward_chunk.argtypes = [C.c_void_p, C.c_void_p, _i32p, C.c_int, C.c_int, _f32p, C.c_int]
    L.orc_forward_tp.restype = C.c_int
    L.orc_forward_tp.argtypes = [C.c_void_p, C.c_void_p, _i32p, C.c_int, C.c_int, _f32p, C.c_int, C.c_int]
    L.orc_forward_order.restype = C.c_int
    L.orc_forward_order.argtypes = [C.c_void_p, C.c_void_p, _i32p, C.c_int, C.c_int, _f32p, C.c_int, _u16p, C.POINTER(OrcOrder)]
    L.orc_forward_chunk_order.restype = C.c_int
    L.orc_forward_chunk_order.argtypes = [C.c_void_p, C.c_void_p, _i32p, C.c_int, C.c_int, _f32p, C.c_int, C.POINTER(OrcOrder)]
    L.orc_linear_order_bf16.restype = C.c_int
    L.orc_linear_order_bf16.argtypes = [_u16p, _u16p, _u16p, C.c_int, C.c_int, C.c_int, C.c_int]
    L.orc_rms_scale_order.restype = C.c_int
    L.orc_rms_scale_order.argtypes = [_u16p, _f32p, C.c_int, C.c_int, C.c_float, C.c_int]
    L.orc_attention_order.restype = C.c_int
    L.orc_attention_order.argtypes = [_u16p, _u16p, _u16p, _u16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int]
    L.orc_attention_z.restype = C.c_double
    L.orc_attention_z.argtypes = [_f64p, C.c_int, C.c_int]
    L.orc_generate.restype = C.c_int
    L.orc_generate.argtypes = [C.c_void_p, _i32p, C.c_int, C.c_int, _i32p, C.c_int, _i32p, _f64p]
    L.orc_synth_fill.argtypes = [C.c_uint64, C.c_char_p, C.c_float, C.c_float, C.c_int64, _u16p]
    L.orc_num_threads.restype = C.c_int
    L.orc_set_num_threads.argtypes = [C.c_int]


# ----------------------------------------------------------------- numpy helpers

def _p(a: np.ndarray, ty):
    assert a.flags["C_CONTIGUOUS"], "oracle arrays must be C-contiguous"
    return a.ctypes.data_as(ty)


def u16(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.uint16)


def bf16_bits(x) -> np.ndarray:
    """f32 -> bf16 bit pattern by truncation (src/dtype/bfloat16.go:59-61)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    return (x.view(np.uint32) >> 16).astype(np.uint16)


def bf16_to_f32(b) -> np.ndarray:
    b = np.ascontiguousarray(b, dtype=np.uint16)
    return (b.astype(np.uint32) << 16).view(np.float32)


def linear_bf16(x: np.ndarray, w: np.ndarray) -> np.ndarray:
    S, K = x.shape
    N, K2 = w.shape
    assert K == K2
    out = np.empty((S, N), np.uint16)
    lib().orc_linear_bf16(_p(x, _u16p), _p(w, _u16p), _p(out, _u16p), S, K, N)
    return out


def linear_bf16_f32out(x, w):
    S, K = x.shape
    N, _ = w.shape
    out = np.empty((S, N), np.float32)
    lib().orc_linear_bf16_f32out(_p(x, _u16p), _p(w, _u16p), _p(out, _f32p), S, K, N)
    return out


def linear_f32(x, w):
    S, K = x.shape
    N, _ = w.shape
    out = np.empty((S, N), np.float32)
    lib().orc_linear_f32(_p(x, _f32p), _p(w, _f32p), _p(out, _f32p), S, K, N)
    return out


def matmul_bf16(a, b):
    *lead, M, K = a.shape
    N = b.shape[-1]
    B = int(np.prod(lead)) if lead else 1
    out = np.empty((*lead, M, N), np.uint16)
    lib().orc_matmul_bf16(_p(a, _u16p), _p(b, _u16p), _p(out, _u16p), B, M, K, N)
    return out


def pow2_bf16(x):
    out = np.empty(x.shape, np.float32)
    lib().orc_pow2_bf16(_p(x, _u16p), _p(out, _f32p), x.size)
    return out


def mean_f32(x):
    rows = int(np.prod(x.shape[:-1]))
    out = np.empty(x.shape[:-1] + (1,), np.float32)
    lib().orc_mean_f32(_p(x, _f32p), _p(out, _f32p), rows, x.shape[-1])
    return out


def add_bf16(a, b):
    out = np.empty(a.shape, np.uint16)
    lib().orc_add_bf16(_p(a, _u16p), _p(b, _u16p), _p(out, _u16p), a.size)
    return out


def mul_bf16(a, b):
    out = np.empty(a.shape, np.uint16)
    lib().orc_mul_bf16(_p(a, _u16p), _p(b, _u16p), _p(out, _u16p), a.size)
    return out


def div_scalar_bf16(a, scalar_bits: int):
    out = np.empty(a.shape, np.uint16)
    lib().orc_div_scalar_bf16(_p(a, _u16p), scalar_bits, _p(out, _u16p), a.size)
    return out


def softmax_f32(x):
    rows = int(np.prod(x.shape[:-1]))
    out = np.empty(x.shape, np.float32)
    lib().orc_softmax_f32(_p(x, _f32p), _p(out, _f32p), rows, x.shape[-1])
    return out


def argmax_f32(x) -> int:
    return int(lib().orc_argmax_f32(_p(x, _f32p), x.size))


def silu_bf16(x):
    out = np.empty(x.shape, np.uint16)
    lib().orc_silu_bf16(_p(x, _u16p), _p(out, _u16p), x.size)
    return out


def silu_table_bf16():
    out = np.empty(65536, np.uint16)
    lib().orc_silu_table_bf16(_p(out, _u16p))
    return out


def rms_scale(x, eps=1e-5):
    """r[s] of RMSNorm.Forward (llamatransformer.go:641-656) for x[S, D] bf16 bits"""
    x = np.ascontiguousarray(x, np.uint16)
    S, D = x.shape
    r = np.empty(S, np.float32)
    lib().orc_rms_scale(_p(x, _u16p), _p(r, _f32p), S, D, eps)
    return r


def rmsnorm_stage1(x, eps=1e-5):
    S, D = x.shape
    out = np.empty((S, D), np.uint16)
    lib().orc_rmsnorm_stage1(_p(x, _u16p), _p(out, _u16p), S, D, eps)
    return out


def rmsnorm(x, w, eps=1e-5):
    S, D = x.shape
    out = np.empty((S, D), np.uint16)
    lib().orc_rmsnorm(_p(x, _u16p), _p(w, _u16p), _p(out, _u16p), S, D, eps)
    return out


def rope_table(dim=128, end=4096, theta=500000.0, use_scaled=True):
    freqs = np.empty(dim // 2, np.uint16)
    cis = np.empty((end, dim // 2, 2), np.float32)
    lib().orc_rope_table(dim, end, theta, int(use_scaled), _p(freqs, _u16p), _p(cis, _f32p))
    return freqs, cis


def rope_apply(x, cis, start_pos):
    S, H, hd = x.shape
    out = np.empty(x.shape, np.uint16)
    lib().orc_rope_apply(_p(x, _u16p), _p(cis, _f32p), _p(out, _u16p), S, H, hd, start_pos)
    return out


def attention(q, cache_k, cache_v, T, causal_mask, q_pos0=0):
    """q_pos0 > 0 (EXTENSION, beyond the reference): query row s sits at position q_pos0 + s, so a causal row sees the
    keys t <= q_pos0 + s -- the [S,T] mask of a chunked prefill"""
    S, nh, hd = q.shape
    nkv = cache_k.shape[1]
    out = np.empty((S, nh * hd), np.uint16)
    if q_pos0:
        lib().orc_attention_pos(_p(q, _u16p), _p(cache_k, _u16p), _p(cache_v, _u16p), _p(out, _u16p),
                                S, T, nh, nkv, hd, int(causal_mask), int(q_pos0))
    else:
        lib().orc_attention(_p(q, _u16p), _p(cache_k, _u16p), _p(cache_v, _u16p), _p(out, _u16p),
                            S, T, nh, nkv, hd, int(causal_mask))
    return out


def linear_order_bf16(x, w, ks):
    """linear with k-streams of 8-element chunks (ks = 1: orc_linear_bf16's order)"""
    S, K = x.shape
    N = w.shape[0]
    out = np.empty((S, N), np.uint16)
    if lib().orc_linear_order_bf16(_p(x, _u16p), _p(w, _u16p), _p(out, _u16p), S, K, N, int(ks)) != 0:
        raise ValueError(f"no linear order ks={ks} at K={K}")
    return out


def rms_scale_order(x, eps=1e-5, parts=1):
    """rms_scale with the sum of squares in `parts` interleaved partials, butterfly and groups of 32 in order"""
    x = np.ascontiguousarray(x, np.uint16)
    S, D = x.shape
    r = np.empty(S, np.float32)
    if lib().orc_rms_scale_order(_p(x, _u16p), _p(r, _f32p), S, D, eps, int(parts)) != 0:
        raise ValueError(f"no RMS order with {parts} partials")
    return r


def attention_order(q, cache_k, cache_v, T, causal_mask, q_pos0=0, attn=ATTN_REF):
    """attention with the softmax denominator and the output chains in the order attn (ATTN_REF: attention's bits)"""
    S, nh, hd = q.shape
    nkv = cache_k.shape[1]
    out = np.empty((S, nh * hd), np.uint16)
    rc = lib().orc_attention_order(_p(q, _u16p), _p(cache_k, _u16p), _p(cache_v, _u16p), _p(out, _u16p), S, T, nh, nkv, hd,
                                   int(causal_mask), int(q_pos0), int(attn))
    if rc != 0:
        raise ValueError(f"no attention order {attn}")
    return out


def attention_z(e, attn):
    """the softmax denominator alone: the f64 sum of e in the order attn"""
    e = np.ascontiguousarray(e, np.float64)
    return float(lib().orc_attention_z(_p(e, _f64p), e.size, int(attn)))


def synth_fill(seed: int, name: str, scale: float, offset: float, n: int, out: np.ndarray | None = None):
    if out is None:
        out = np.empty(n, np.uint16)
    lib().orc_synth_fill(seed, name.encode(), scale, offset, n, _p(out, _u16p))
    return out


class OracleModel:
    """Owns an orc_model plus the numpy arrays its tensors alias."""

    def __init__(self, args: dict, tensors: dict[str, np.ndarray]):
        self.args = OrcArgs(**args)
        self.h = lib().orc_model_new(C.byref(self.args))
        self.tensors = tensors
        for name, arr in tensors.items():
            rc = lib().orc_model_bind(self.h, name.encode(), _p(arr, _u16p))
            if rc != 0:
                raise KeyError(name)

    def close(self):
        if self.h:
            lib().orc_model_free(self.h)
            self.h = None

    def new_session(self, seq_len: int) -> "OracleSession":
        return OracleSession(self, seq_len)

    def generate(self, prompt, seq_len, stop_ids=(128008, 128009), want_times=False):
        prompt = np.ascontiguousarray(prompt, np.int32)
        stop = np.ascontiguousarray(stop_ids, np.int32)
        out = np.empty(seq_len, np.int32)
        times = np.zeros(seq_len, np.float64)
        n = lib().orc_generate(self.h, _p(prompt, _i32p), len(prompt), seq_len, _p(stop, _i32p), len(stop),
                               _p(out, _i32p), _p(times, _f64p))
        if n < 0:
            raise RuntimeError("orc_generate failed")
        return (out[:n].copy(), times[:n].copy()) if want_times else out[:n].copy()


class OracleSession:
    def __init__(self, model: OracleModel, seq_len: int):
        self.model = model
        self.seq_len = seq_len
        self.h = lib().orc_session_new(model.h, seq_len)

    def close(self):
        if self.h:
            lib().orc_session_free(self.h)
            self.h = None

    def forward_chunk(self, tokens, start_pos, all_rows=True, order=None):
        """EXTENSION (beyond the reference): a prompt chunk of S > 1 tokens at start_pos > 0 with the [S,T] causal mask.
        order (ks, rms_parts, attn): sum in that order (None: the reference's)"""
        tokens = np.ascontiguousarray(tokens, np.int32)
        S = len(tokens)
        logits = np.empty((S if all_rows else 1, self.model.args.vocab), np.float32)
        if order is not None:
            rc = lib().orc_forward_chunk_order(self.model.h, self.h, _p(tokens, _i32p), S, start_pos, _p(logits, _f32p),
                                               int(all_rows), _order(order))
        else:
            rc = lib().orc_forward_chunk(self.model.h, self.h, _p(tokens, _i32p), S, start_pos, _p(logits, _f32p), int(all_rows))
        if rc != 0:
            raise RuntimeError("orc_forward_chunk failed (bad tokens / positions)")
        return logits

    def forward(self, tokens, start_pos, all_rows=True, trace=False, tp=1, order=None):
        """order (ks, rms_parts, attn), e.g. ORDER_FAST: every sum in that order (None: the reference's)"""
        tokens = np.ascontiguousarray(tokens, np.int32)
        S = len(tokens)
        V, D, L = self.model.args.vocab, self.model.args.dim, self.model.args.n_layers
        logits = np.empty((S if all_rows else 1, V), np.float32)
        tr = np.empty((L + 1, S, D), np.uint16) if trace else None
        if order is not None:
            if tp > 1:
                raise ValueError("a summation order and a tensor-parallel split do not combine")
            rc = lib().orc_forward_order(self.model.h, self.h, _p(tokens, _i32p), S, start_pos, _p(logits, _f32p), int(all_rows),
                                         _p(tr, _u16p) if trace else None, _order(order))
        elif tp > 1:
            rc = lib().orc_forward_tp(self.model.h, self.h, _p(tokens, _i32p), S, start_pos, _p(logits, _f32p),
                                      int(all_rows), tp)
        else:
            rc = lib().orc_forward(self.model.h, self.h, _p(tokens, _i32p), S, start_pos, _p(logits, _f32p),
                                   int(all_rows), _p(tr, _u16p) if trace else None)
        if rc != 0:
            raise RuntimeError("orc_forward failed (bad tokens / positions)")
        return (logits, tr) if trace else logits

    def cache(self, layer):
        a = self.model.args
        n = self.seq_len * a.n_kv_heads * a.head_dim
        k = np.ctypeslib.as_array(lib().orc_session_cache_k(self.h, layer), shape=(n,))
        v = np.ctypeslib.as_array(lib().orc_session_cache_v(self.h, layer), shape=(n,))
        shp = (self.seq_len, a.n_kv_heads, a.head_dim)
        return k.reshape(shp), v.reshape(shp)


# ---------------------------------------------------------------------------------------------------------
# Building blocks of the RoPE table and the causal mask (init-time ops of src/ml), restated in NumPy.  The C
# oracle computes precomputeFreqsCis in one piece (orc_rope_table); these blocks are pinned to the reference's own
# literals (TestARange*, TestOuter, TestPolar, TestTriangularUpper*) and then composed the way
# precomputeFreqsCis composes them (src/model/llamatransformer.go:694-751) to cross-check the C table bit for bit.

def arange_bf16(start: int, end: int, step: int) -> np.ndarray:
    """ml.ARange(start, end, step, DT_BF16) (src/ml/operations_impl.go:11-24): float32(val) truncated to bf16"""
    if start >= end:
        raise ValueError(f"start value {start} must be less than end value {end} in ARange")
    return bf16_bits(np.arange(start, end, step, dtype=np.int64).astype(np.float32))


def outer_bf16(vec1: np.ndarray, vec2: np.ndarray) -> np.ndarray:
    """ml.Outer for BF16 vectors (operations_impl.go:26-52): float32 product, truncated to bf16"""
    a, b = bf16_to_f32(vec1), bf16_to_f32(vec2)
    return bf16_bits((a[:, None] * b[None, :]).astype(np.float32))


def polar(abs_f32: np.ndarray, angle_f32: np.ndarray) -> np.ndarray:
    """ml.Polar (operations_impl.go:100-140): complex64(complex(abs * cos(angle), abs * sin(angle))) in float64"""
    a, t = np.asarray(abs_f32, np.float64), np.asarray(angle_f32, np.float64)
    return ((a * np.cos(t)) + 1j * (a * np.sin(t))).astype(np.complex64)


def full_f32(size, value) -> np.ndarray:
    """ml.Full(size, DT_F32, value) (operations_impl.go:55-64)"""
    return np.full(size, np.float32(value), np.float32)


def triangular_upper(x: np.ndarray, diagonal: int) -> np.ndarray:
    """ml.TriangularUpper (operations_impl.go:175-195): keeps x[i, j] where j - i >= diagonal, zero elsewhere"""
    i, j = np.indices(x.shape)
    return np.where(j - i >= diagonal, x, np.zeros_like(x))


def rope_table_from_blocks(dim: int, end: int, theta: float, inv_freqs_bf16: np.ndarray) -> np.ndarray:
    """the tail of precomputeFreqsCis (llamatransformer.go:728-750): t = ARange(0, end) in bf16, Outer(t, freqs) in
    bf16, Polar(ones, .) -> [end, dim/2] complex64, returned as [end, dim/2, 2] float32 (cos, sin)"""
    t = arange_bf16(0, end, 1)
    ang = outer_bf16(t, inv_freqs_bf16)
    c = polar(np.ones(ang.shape, np.float32), bf16_to_f32(ang))
    return np.stack([c.real, c.imag], -1).astype(np.float32)
