"""Synthetic Llama-3.1-8B checkpoint description (SURVEY.md 8d / Appendix B).

No real checkpoint exists in the build or bench environment, so weights are random-init
tensors of the 8B architecture produced by a counter-based generator
(value(i) = t((2u-1)*scale + offset), u = top 24 bits of splitmix64(seed ^ fnv1a(name), i)).
The same generator exists on the device (lnb_model_init_synthetic), on the host
(lnb_synth_fill_host) and inside the test oracle; all three produce identical bits.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi

SEED = 0x4C4E42  # "LNB"

# docs/04-LOADING-MODEL-ARGS.md:27-41 ; FFN width: src/model/llamatransformer.go:569-577
LLAMA31_8B = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=8, head_dim=128, ffn_dim=14336,
                  vocab_size=128256, max_seq_len=2048, norm_eps=1e-5, rope_theta=500000.0, use_scaled_rope=1)

# a structurally identical miniature for fast tests (all tiling constraints hold)
TINY = dict(dim=256, n_layers=2, n_heads=8, n_kv_heads=2, head_dim=32, ffn_dim=512,
            vocab_size=1024, max_seq_len=64, norm_eps=1e-5, rope_theta=500000.0, use_scaled_rope=1)

# the same with the 8B model's head_dim of 128: FAST prompts of >= 32 tokens run the tensor-core prefill with its
# wgmma attention kernel (sdpa_tc_kernel), which only serves head_dim 128
TINY128 = dict(dim=1024, n_layers=2, n_heads=8, n_kv_heads=2, head_dim=128, ffn_dim=1024,
               vocab_size=2048, max_seq_len=512, norm_eps=1e-5, rope_theta=500000.0, use_scaled_rope=1)

# 8 fixed prompt ids (first = <|begin_of_text|>) and the reference's stop ids
# (src/tiktoken/tiktokenreader.go:81)
PROMPT_8 = [128000, 9906, 11, 856, 836, 374, 220, 16]
STOP_IDS = (128008, 128009)
PAD_ID = -1

_LAYER_TENSORS = ["attention_norm.weight", "attention.wq.weight", "attention.wk.weight", "attention.wv.weight",
                  "attention.wo.weight", "ffn_norm.weight", "feed_forward.w1.weight", "feed_forward.w2.weight",
                  "feed_forward.w3.weight"]


def tensor_shapes(args: dict) -> dict[str, tuple[int, ...]]:
    """name -> checkpoint shape, exactly the 291-tensor inventory the reference binds
    (llamatransformer.go:84-105,191,202,273-282,580-586)."""
    d, q, kv, f, v = args["dim"], args["n_heads"] * args["head_dim"], args["n_kv_heads"] * args["head_dim"], \
        args["ffn_dim"], args["vocab_size"]
    per_layer = {"attention_norm.weight": (d,), "attention.wq.weight": (q, d), "attention.wk.weight": (kv, d),
                 "attention.wv.weight": (kv, d), "attention.wo.weight": (d, q), "ffn_norm.weight": (d,),
                 "feed_forward.w1.weight": (f, d), "feed_forward.w2.weight": (d, f), "feed_forward.w3.weight": (f, d)}
    out = {"tok_embeddings.weight": (v, d), "norm.weight": (d,), "output.weight": (v, d)}
    for l in range(args["n_layers"]):
        for n in _LAYER_TENSORS:
            out[f"layers.{l}.{n}"] = per_layer[n]
    return out


def args_c(args: dict) -> _capi.ModelArgsC:
    return _capi.ModelArgsC(**args)


def spec(args: dict, name: str) -> tuple[float, float]:
    sc, off = C.c_float(), C.c_float()
    _capi.check(_capi.lib.lnb_synth_spec(C.byref(args_c(args)), name.encode(), C.byref(sc), C.byref(off)))
    return sc.value, off.value


def fill_host(args: dict, name: str, seed: int = SEED) -> np.ndarray:
    """Host copy of one synthetic tensor (single-threaded; meant for small tensors)."""
    shape = tensor_shapes(args)[name]
    n = int(np.prod(shape))
    sc, off = spec(args, name)
    out = np.empty(n, np.uint16)
    _capi.check(_capi.lib.lnb_synth_fill_host(seed, name.encode(), sc, off, n, _capi.ptr(out, _capi.u16p)))
    return out.reshape(shape)


def batch_prompt(b: int) -> list[int]:
    """prompt of concurrent sequence b (SURVEY.md 8d)"""
    return [PROMPT_8[0]] + [(t + 977 * b) % 128000 for t in PROMPT_8[1:]]


def shard_window(args: dict, name: str, tp_rank: int, tp_size: int) -> tuple[int, int, int, int]:
    """(row0, col0, rows, cols) of the window of tensor `name` owned by a tensor-parallel rank"""
    r0, c0, r, c = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
    _capi.check(_capi.lib.lnb_tp_shard_window(C.byref(args_c(args)), name.encode(), tp_rank, tp_size,
                                              C.byref(r0), C.byref(c0), C.byref(r), C.byref(c)))
    return r0.value, c0.value, r.value, c.value
