"""ctypes binding of liblnb.so (include/lnb.h).  No fallbacks: a missing library is an error."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblnb.so")

LNB_ACC_STRICT, LNB_ACC_FAST = 0, 1
LNB_BUF_RESIDUAL, LNB_BUF_CACHE_K, LNB_BUF_CACHE_V, LNB_BUF_LOGITS = 0, 1, 2, 3
LNB_BUF_Q, LNB_BUF_ATTN, LNB_BUF_POST_ATTN, LNB_BUF_NORMED, LNB_BUF_FFN = 4, 5, 6, 7, 8
LNB_WEIGHTS_BF16, LNB_WEIGHTS_MXFP8, LNB_WEIGHTS_MXFP4 = 0, 1, 2
LNB_KV_BF16, LNB_KV_MXFP8 = 0, 1


class LnbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"lnb error {code}: {msg}")
        self.code = code


class ModelArgsC(C.Structure):
    _fields_ = [
        ("dim", C.c_int32), ("n_layers", C.c_int32), ("n_heads", C.c_int32), ("n_kv_heads", C.c_int32),
        ("head_dim", C.c_int32), ("ffn_dim", C.c_int32), ("vocab_size", C.c_int32), ("max_seq_len", C.c_int32),
        ("norm_eps", C.c_float), ("rope_theta", C.c_double), ("use_scaled_rope", C.c_int32),
    ]


class SamplingC(C.Structure):   # lnb_sampling
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float), ("seed", C.c_uint64)]


LNB_LOGPROBS_TOP_MAX = 20


LNB_LOGIT_BIAS_MAX = 64
LNB_GRAMMAR_MAX_STATES = 4096


class PenaltiesC(C.Structure):   # lnb_penalties
    _fields_ = [("repetition_penalty", C.c_float), ("frequency_penalty", C.c_float), ("presence_penalty", C.c_float),
                ("window", C.c_int32), ("first_pos", C.c_int32), ("n_bias", C.c_int32),
                ("bias_token", C.c_int32 * LNB_LOGIT_BIAS_MAX), ("bias", C.c_float * LNB_LOGIT_BIAS_MAX)]


class LogprobC(C.Structure):   # lnb_logprob
    _fields_ = [("token", C.c_int32), ("rank", C.c_int32), ("logprob", C.c_double), ("n_top", C.c_int32),
                ("top_token", C.c_int32 * LNB_LOGPROBS_TOP_MAX), ("top_logprob", C.c_double * LNB_LOGPROBS_TOP_MAX)]


u16p = C.POINTER(C.c_uint16)
f32p = C.POINTER(C.c_float)
i32p = C.POINTER(C.c_int32)
i64p = C.POINTER(C.c_int64)
vp = C.c_void_p

# name -> (restype, argtypes); also the list tests check against include/lnb.h
SIGNATURES = {
    "lnb_last_error": (C.c_char_p, []),
    "lnb_version": (C.c_int, []),
    "lnb_device_count": (C.c_int, []),
    "lnb_model_create": (C.c_int, [C.POINTER(ModelArgsC), C.c_int, C.c_int, C.c_int, vp, C.POINTER(vp)]),
    "lnb_nccl_unique_id": (C.c_int, [vp]),
    "lnb_tp_shard_window": (C.c_int, [C.POINTER(ModelArgsC), C.c_char_p, C.c_int, C.c_int, i64p, i64p, i64p, i64p]),
    "lnb_model_upload_tensor": (C.c_int, [vp, C.c_char_p, u16p, i64p, C.c_int]),
    "lnb_model_init_synthetic": (C.c_int, [vp, C.c_uint64]),
    "lnb_synth_fill_host": (C.c_int, [C.c_uint64, C.c_char_p, C.c_float, C.c_float, C.c_int64, u16p]),
    "lnb_synth_spec": (C.c_int, [C.POINTER(ModelArgsC), C.c_char_p, f32p, f32p]),
    "lnb_model_set_rope_table": (C.c_int, [vp, f32p, C.c_int]),
    "lnb_model_set_silu_table": (C.c_int, [vp, u16p]),
    "lnb_model_get_rope_table": (C.c_int, [vp, f32p, C.c_int]),
    "lnb_model_get_silu_table": (C.c_int, [vp, u16p]),
    "lnb_model_finalize": (C.c_int, [vp]),
    "lnb_model_destroy": (C.c_int, [vp]),
    "lnb_model_wpack_read": (C.c_int, [vp, C.c_int, vp, vp, u16p, i64p]),
    "lnb_model_set_weight_format": (C.c_int, [vp, C.c_int]),
    "lnb_model_mxfp8_read": (C.c_int, [vp, C.c_char_p, vp, vp]),
    "lnb_model_mxfp4_read": (C.c_int, [vp, C.c_char_p, vp, vp]),
    "lnb_model_weight_info": (C.c_int, [vp, C.POINTER(C.c_int), i64p, i64p]),
    "lnb_session_create": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "lnb_session_destroy": (C.c_int, [vp]),
    "lnb_forward": (C.c_int, [vp, i32p, C.c_int, C.c_int, f32p, C.c_int, i32p]),
    "lnb_forward_device": (C.c_int, [vp, i32p, C.c_int, C.c_int, C.c_int, i32p, i64p]),
    "lnb_session_logits_read": (C.c_int, [vp, C.c_int64, C.c_int, C.c_int, f32p]),
    "lnb_session_logits_argmax": (C.c_int, [vp, C.c_int64, C.c_int, C.c_int, i32p]),
    "lnb_decode_run": (C.c_int, [vp, C.c_int32, C.c_int, C.c_int, C.c_int, i32p, f32p]),
    "lnb_session_create_batch": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "lnb_session_set_active_sequence": (C.c_int, [vp, C.c_int]),
    "lnb_session_create_kv": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "lnb_session_kv_info": (C.c_int, [vp, C.POINTER(C.c_int), i64p]),
    "lnb_session_kv_read": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]),
    "lnb_forward_batch": (C.c_int, [vp, i32p, i32p, C.c_int, f32p, i32p]),
    "lnb_session_p2p_export": (C.c_int, [vp, vp]),
    "lnb_session_p2p_import": (C.c_int, [vp, vp, C.c_int]),
    "lnb_session_p2p_disable": (C.c_int, [vp]),
    "lnb_session_engine_profile": (C.c_int, [vp, C.POINTER(C.c_double)]),
    "lnb_session_decode_engine": (C.c_int, [vp]),
    "lnb_session_set_chunked_prefill": (C.c_int, [vp, C.c_int]),
    "lnb_forward_ragged": (C.c_int, [vp, C.c_int, i32p, i32p, i32p, i32p, f32p, i32p]),
    "lnb_forward_speculative": (C.c_int, [vp, C.c_int, i32p, i32p, i32p, i32p, f32p, i32p, i32p]),
    "lnb_forward_speculative_tree": (C.c_int, [vp, C.c_int, i32p, i32p, i32p, i32p, i32p, f32p, i32p, i32p, i32p]),
    "lnb_session_set_sampling": (C.c_int, [vp, C.c_int, C.POINTER(SamplingC)]),
    "lnb_session_set_logprobs": (C.c_int, [vp, C.c_int, C.c_int]),
    "lnb_session_set_penalties": (C.c_int, [vp, C.c_int, C.POINTER(PenaltiesC)]),
    "lnb_regex_dfa": (C.c_int, [C.c_char_p, C.c_int64, i32p, C.POINTER(C.c_uint8), C.c_int, C.POINTER(C.c_int)]),
    "lnb_grammar_create": (C.c_int, [vp, C.c_char_p, C.c_int64, C.POINTER(C.c_uint8), i64p, i32p, C.c_int, C.POINTER(vp)]),
    "lnb_grammar_info": (C.c_int, [vp, i64p]),
    "lnb_grammar_read_mask": (C.c_int, [vp, C.c_int, C.POINTER(C.c_uint32)]),
    "lnb_grammar_destroy": (C.c_int, [vp]),
    "lnb_session_set_grammar": (C.c_int, [vp, C.c_int, vp, C.c_int]),
    "lnb_session_logprobs_read": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, vp]),
    "lnb_score": (C.c_int, [vp, i32p, C.c_int, C.c_int]),
    "lnb_session_copy_sequences": (C.c_int, [vp, C.c_int, i32p, i32p, C.c_int, C.c_int]),
    "lnb_session_read": (C.c_int, [vp, C.c_int, C.c_int, vp, C.c_int64]),
    "lnb_session_set_layer_limit": (C.c_int, [vp, C.c_int]),
    "lnb_session_launch_count": (C.c_int64, [vp]),
    "lnb_session_sync": (C.c_int, [vp]),
    "lnb_session_bench_kernel": (C.c_int, [vp, C.c_int, C.c_int, f32p, i64p, i32p]),
    "lnb_pth_open": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "lnb_pth_close": (C.c_int, [C.c_void_p]),
    "lnb_pth_tensor_count": (C.c_int, [C.c_void_p]),
    "lnb_pth_tensor_info": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                      C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "lnb_pth_tensor_data": (C.c_void_p, [C.c_void_p, C.c_int]),
    "lnb_model_load_pth": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]),
    "lnb_model_args_from_params_json": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(ModelArgsC)]),
    "lnb_pth_writer_create": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "lnb_pth_writer_add": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.POINTER(C.c_int64), C.c_int]),
    "lnb_pth_writer_finish": (C.c_int, [C.c_void_p]),
    "lnb_pth_write_synthetic": (C.c_int, [C.c_char_p, C.POINTER(ModelArgsC), C.c_uint64]),
    "lnb_vocab_load": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "lnb_vocab_write_synthetic": (C.c_int, [C.c_char_p, C.c_int]),
    "lnb_vocab_destroy": (C.c_int, [C.c_void_p]),
    "lnb_vocab_size": (C.c_int, [C.c_void_p]),
    "lnb_vocab_token_id": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, i32p]),
    "lnb_vocab_token_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "lnb_vocab_special_ids": (C.c_int, [C.c_void_p, i32p, i32p, i32p, i32p]),
    "lnb_split_pieces": (C.c_int, [C.c_char_p, C.c_int64, i64p, C.c_int, C.POINTER(C.c_int)]),
    "lnb_tokenize_string": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64, i32p, C.c_int, C.POINTER(C.c_int)]),
    "lnb_tokenize_prompt": (C.c_int, [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_int, i32p, C.c_int, C.POINTER(C.c_int)]),
    "lnb_detokenize": (C.c_int, [C.c_void_p, i32p, C.c_int, C.c_char_p, C.c_int64, C.POINTER(C.c_int64)]),
    "lnb_op_linear_bf16": (C.c_int, [u16p, u16p, u16p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "lnb_op_matmul_bf16": (C.c_int, [u16p, u16p, u16p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "lnb_op_rmsnorm_bf16": (C.c_int, [u16p, u16p, u16p, C.c_int, C.c_int, C.c_float, C.c_int]),
    "lnb_op_rms_scale_f32": (C.c_int, [u16p, f32p, C.c_int, C.c_int, C.c_float, C.c_int]),
    "lnb_op_rope_bf16": (C.c_int, [u16p, f32p, u16p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "lnb_op_attention_bf16": (C.c_int, [u16p, u16p, u16p, u16p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "lnb_op_silu_bf16": (C.c_int, [u16p, u16p, C.c_int64]),
    "lnb_op_add_bf16": (C.c_int, [u16p, u16p, u16p, C.c_int64]),
    "lnb_op_mul_bf16": (C.c_int, [u16p, u16p, u16p, C.c_int64]),
    "lnb_op_softmax_f32": (C.c_int, [f32p, f32p, C.c_int, C.c_int]),
    "lnb_op_argmax_f32": (C.c_int, [f32p, C.c_int, C.c_int, i32p]),
    "lnb_op_sample_f32": (C.c_int, [f32p, C.c_int, C.c_int, C.POINTER(SamplingC), i32p, i32p]),
    "lnb_op_logprobs_f32": (C.c_int, [f32p, C.c_int, C.c_int, i32p, C.c_int, vp]),
    "lnb_op_penalize_f32": (C.c_int, [f32p, C.c_int, C.c_int, C.POINTER(PenaltiesC), i32p, C.c_int, i32p, f32p]),
    "lnb_op_get_rows_bf16": (C.c_int, [u16p, i32p, u16p, C.c_int, C.c_int, C.c_int]),
    "lnb_op_kv_quantize_bf16": (C.c_int, [u16p, C.c_int, C.c_int, C.c_int, vp, vp, u16p]),
}

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
        "There is no CPU fallback.")

lib = C.CDLL(LIB_PATH)
for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)  # AttributeError if the library does not export a declared symbol
    _fn.restype = _res
    _fn.argtypes = _args


def check(rc: int) -> int:
    if rc < 0:
        raise LnbError(rc, lib.lnb_last_error().decode(errors="replace"))
    return rc


def ptr(arr, ty):
    """numpy array -> typed pointer (array must be C-contiguous)."""
    if arr is None:
        return None
    assert arr.flags["C_CONTIGUOUS"]
    return arr.ctypes.data_as(ty)
