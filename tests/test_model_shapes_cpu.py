"""The model-shape catalogue (tests/model_shapes.py) without a GPU: each entry has the traits its row claims and together
they cover the GQA ratios and head dims of published checkpoints; the restatement agrees with engine_shapes.py and with the
library's own argument checks; the oracle runs every accepted shape; and Meta params.json files give the published shapes."""
import ctypes as C
import json

import numpy as np
import pytest

import lnb_b200 as L
from oracle import oracle as O
from tests import engine_shapes as ES
from tests import model_shapes as M
from tests.helpers import host_tensors, oracle_model

# what each catalogue row claims (model_shapes.traits, 132 SMs)
EXPECTED = {
    "mha": dict(n_rep=1, head_dim=64, scaled_rope=False, rope_theta=10000.0, ffn_on_tiles=False, vocab_on_tiles=False,
                strict_engine=True, batch_engine=True, prompt_tc=False, prompt_attention="sdpa_kernel", decode_fit=719),
    "gqa3": dict(n_rep=3, head_dim=128, strict_engine=True, batch_engine=True, prompt_tc=True, prompt_attention="sdpa_tc",
                 decode_fit=359),
    "gqa8": dict(n_rep=8, head_dim=64, strict_engine=True, batch_engine=True, prompt_tc=True, prompt_attention="sdpa_kernel",
                 decode_fit=549),
    "hd96": dict(n_rep=2, head_dim=96, strict_engine=True, batch_engine=True, prompt_tc=True, decode_fit=480),
    "stories": dict(n_rep=1, head_dim=48, scaled_rope=False, strict_engine=False, fast_engine=True, batch_engine=False,
                    prompt_tc=False, prompt_attention="sdpa_kernel", decode_fit=928),
    "hd256": dict(n_rep=2, head_dim=256, strict_engine=False, fast_engine=False, batch_engine=False, prompt_tc=True,
                  prompt_attention="sdpa_kernel", decode_fit=0, streamed_batched=False, batched="refused", ragged="refused",
                  speculative="refused"),
    "rep16": dict(n_rep=16, head_dim=32, strict_engine=False, fast_engine=False, batch_engine=False, prompt_tc=True,
                  decode_fit=0, streamed_batched=False, batched="refused", ragged="refused", speculative="refused"),
    "one_layer": dict(n_rep=4, head_dim=32, n_layers=1, strict_engine=True, batch_engine=True),
}


@pytest.mark.parametrize("name", list(M.CATALOGUE))
def test_each_entry_hits_the_traits_of_its_row(name):
    a, t = M.CATALOGUE[name], M.traits(name)
    for k, v in EXPECTED[name].items():
        assert t[k] == v, (name, k, t[k], v)
    assert M.create_error(a) is None
    if name not in ("hd256", "rep16"):
        assert t["batched"] == "sdpa_decode" and t["ragged"] == "stream" and t["speculative"] == "sdpa_decode"
    if name != "one_layer":
        assert a["n_layers"] == 2
    # every shape with the streamed kernels has a SequenceLength just past sdpa_decode_kernel's fit within its RoPE table,
    # except TINY's one-layer copy (its fit is past max_seq_len 64)
    assert t["streamed_batched"] == (name not in ("hd256", "rep16", "one_layer"))


def test_catalogue_covers_the_published_ratios_and_head_dims():
    ts = {n: M.traits(n) for n in M.CATALOGUE}
    assert {t["n_rep"] for t in ts.values()} >= {1, 2, 3, 4, 8, 16}
    assert {t["head_dim"] for t in ts.values()} >= {48, 64, 96, 128, 256}
    # the engines at n_rep 1, 2, 3 and 8; the streamed batched kernels at the same ratios
    assert {t["n_rep"] for t in ts.values() if t["strict_engine"]} >= {1, 2, 3, 8}
    assert {t["n_rep"] for t in ts.values() if t["streamed_batched"]} >= {1, 2, 3, 8}
    # sdpa_tc_kernel at a ratio no other model test runs; unscaled RoPE; a STRICT engine refusal by the scan shape
    assert ts["gqa3"]["prompt_attention"] == "sdpa_tc" and ts["gqa3"]["n_rep"] == 3
    assert {n for n, t in ts.items() if not t["scaled_rope"]} == {"mha", "stories"}
    assert M.engine_refusal(M.CATALOGUE["stories"], 64, True) == "dim does not fit the engine's binade scan"
    # stories: no projection of a prompt is tensor-core eligible; the FAST engine's K = 288 is one short k-tile
    assert not any(M.projections_tc(M.CATALOGUE["stories"], 40).values())
    assert ES.eng_kt(False, 2 * 768, 288, 132) == 288
    # mha: the FFN and vocabulary are off the 128-wide tiles, so only some projections are eligible and the prompt stays on
    # the kernel chain
    pt = M.projections_tc(M.CATALOGUE["mha"], 40)
    assert pt["wqkv"] and pt["wo"] and not pt["w13"] and not pt["w2"]


def test_refusals_of_the_restatement():
    for name in ("hd256", "rep16"):
        a = M.CATALOGUE[name]
        for strict in (True, False):
            assert M.engine_refusal(a, 64, strict) == "head shape"
            assert not M.uses_engine(a, 64, strict, env="1")
        assert M.attention_kernel(a, 64, "single", 1) == "sdpa_kernel"
        # sdpa_kernel holds seq_len scores up to 16981 (head_dim 256) / 17056 (head_dim 32) positions; past that the session
        # would stream, which these head shapes cannot
        last = (M.SMEM_200K - a["head_dim"] * 4) // 12
        assert M.session_error(a, last) is None and M.session_error(a, last + 1) == "needs the streamed attention kernel"
        assert last + 1 <= a["max_seq_len"]
    # an engine-served shape loses the engines past their attention limit, and the streamed kernels take its batched rows
    a = M.CATALOGUE["gqa8"]
    assert M.engine_refusal(a, 227, True) is None
    assert M.engine_refusal(a, 228, True) == "SequenceLength too long for the in-engine attention phase"
    assert M.attention_kernel(a, 549, "batched", 3) == "sdpa_decode" and M.attention_kernel(a, 550, "batched", 3) == "stream"
    # FAST single-GPU S = 1 stays on the chain unless LNB_ENGINE=1; LNB_ENGINE=0 forces the chain everywhere
    assert not M.uses_engine(a, 64, False) and M.uses_engine(a, 64, False, env="1") and not M.uses_engine(a, 64, True, env="0")


def test_restatement_agrees_with_engine_shapes():
    from lnb_b200 import synth
    for args in (ES.wide_args(132), ES.deep_args(), dict(synth.TINY128), dict(synth.TINY), *M.CATALOGUE.values()):
        if M.engine_refusal(args, 1, False) == "head shape":
            continue
        assert M.engine_max_seq_len(args) == ES.max_seq_len(args)
    # the published fits: 351 positions of sdpa_decode_kernel at head_dim 128 / n_rep 4 (include/lnb.h), 549 at 64 / 8
    assert M.sdpa_decode_fit(dict(synth.TINY128)) == 351
    assert M.sdpa_decode_fit(M.CATALOGUE["gqa8"]) == 549
    assert (ES.max_seq_len(ES.wide_args(132)), ES.max_seq_len(dict(synth.TINY128))) == (264, 145)


@pytest.mark.parametrize("name", list(M.CATALOGUE) + list(M.REFUSED))
def test_model_create_agrees_with_the_restatement(name):
    """lnb_model_create validates its arguments before touching a device: a refused shape fails with LNB_EINVAL and the
    restatement's message on any machine; an accepted one passes validation (then needs a GPU)"""
    lib = L._capi.lib
    args, frag = M.REFUSED[name] if name in M.REFUSED else (M.CATALOGUE[name], None)
    assert M.create_error(args) == frag
    h = C.c_void_p()
    rc = lib.lnb_model_create(C.byref(L.synth.args_c(args)), 0, 0, 1, None, C.byref(h))
    if frag is not None:
        assert rc == -1 and frag.encode() in lib.lnb_last_error(), (rc, lib.lnb_last_error())
        return
    if rc == 0:
        lib.lnb_model_destroy(h)
    else:
        assert lib.lnb_device_count() <= 0 and rc == -2, (rc, lib.lnb_last_error())      # LNB_ECUDA: no device here


def test_head_dim_36_is_refused_with_the_constraint():
    """dim 576 over 16 heads: head_dim 36 passed the old `head_dim % 2` check, but sdpa_kernel reads K/V rows 8 elements at a
    time from h * 36, past the head and misaligned for odd h"""
    lib = L._capi.lib
    args = dict(M.CATALOGUE["one_layer"], dim=576, n_heads=16, n_kv_heads=16, head_dim=36)
    h = C.c_void_p()
    assert lib.lnb_model_create(C.byref(L.synth.args_c(args)), 0, 0, 1, None, C.byref(h)) == -1
    assert lib.lnb_last_error() == b"head_dim 36 must be a multiple of 8 (the attention kernels read K/V rows 8 elements at a time)"


def test_load_model_surfaces_the_refusal(tmp_path):
    """LoadModel of a params.json with head_dim 36 fails in model creation with the library's message, before any
    checkpoint is read"""
    a = dict(M.CATALOGUE["one_layer"], dim=576, n_heads=16, n_kv_heads=16, head_dim=36)
    (tmp_path / "params.json").write_text(json.dumps(M.params_json(a)))
    assert L.model.load_model_args(str(tmp_path), 64)["head_dim"] == 36
    with pytest.raises(L._capi.LnbError, match="head_dim 36 must be a multiple of 8"):
        L.model.LoadModel(str(tmp_path), max_seq_len=64)


@pytest.mark.parametrize("name", list(M.CATALOGUE))
def test_params_json_of_each_entry_gives_its_args(tmp_path, name):
    a = M.CATALOGUE[name]
    (tmp_path / "params.json").write_text(json.dumps(M.params_json(a)))
    d = L.model.load_model_args(str(tmp_path), a["max_seq_len"])
    for k in ("dim", "n_layers", "n_heads", "n_kv_heads", "head_dim", "ffn_dim", "vocab_size", "max_seq_len", "use_scaled_rope"):
        assert d[k] == a[k], (k, d[k], a[k])
    assert d["rope_theta"] == a["rope_theta"] and abs(d["norm_eps"] - a["norm_eps"]) < 1e-12


# published params.json texts: (file, the shape it must give)
PUBLISHED = {
    # Llama 2 7B: no n_kv_heads (MHA), no multiplier, no RoPE fields (theta falls back to the loader's default)
    "llama2_7b": ({"dim": 4096, "multiple_of": 256, "n_heads": 32, "n_layers": 32, "norm_eps": 1e-05, "vocab_size": -1},
                  dict(n_kv_heads=32, head_dim=128, ffn_dim=11008, vocab_size=-1, use_scaled_rope=0)),
    "llama32_1b": ({"dim": 2048, "n_layers": 16, "n_heads": 32, "n_kv_heads": 8, "vocab_size": 128256, "ffn_dim_multiplier": 1.5,
                    "multiple_of": 256, "norm_eps": 1e-05, "rope_theta": 500000.0, "use_scaled_rope": True},
                   dict(n_kv_heads=8, head_dim=64, ffn_dim=8192, vocab_size=128256, use_scaled_rope=1)),
    "llama32_3b": ({"dim": 3072, "n_layers": 28, "n_heads": 24, "n_kv_heads": 8, "vocab_size": 128256, "ffn_dim_multiplier": 1.0,
                    "multiple_of": 256, "norm_eps": 1e-05, "rope_theta": 500000.0, "use_scaled_rope": True},
                   dict(n_kv_heads=8, head_dim=128, ffn_dim=8192, vocab_size=128256, use_scaled_rope=1)),
    # TinyLlama 1.1B written as a Meta params.json: 32 heads over 4 KV heads of 64, FFN 5632
    "tinyllama": ({"dim": 2048, "n_layers": 22, "n_heads": 32, "n_kv_heads": 4, "vocab_size": 32000, "ffn_dim_multiplier": 1.03125,
                   "multiple_of": 256, "norm_eps": 1e-05, "rope_theta": 10000.0},
                  dict(n_kv_heads=4, head_dim=64, ffn_dim=5632, vocab_size=32000, use_scaled_rope=0)),
    "llama31_70b": ({"dim": 8192, "n_layers": 80, "n_heads": 64, "n_kv_heads": 8, "vocab_size": 128256, "ffn_dim_multiplier": 1.3,
                     "multiple_of": 4096, "norm_eps": 1e-05, "rope_theta": 500000.0, "use_scaled_rope": True},
                    dict(n_kv_heads=8, head_dim=128, ffn_dim=28672, vocab_size=128256, use_scaled_rope=1)),
    # llama2.c stories15M: dim 288, 6 heads of 48
    "stories15m": ({"dim": 288, "n_layers": 6, "n_heads": 6, "n_kv_heads": 6, "vocab_size": 32000, "multiple_of": 32,
                    "norm_eps": 1e-05},
                   dict(n_kv_heads=6, head_dim=48, ffn_dim=768, vocab_size=32000, use_scaled_rope=0)),
}


@pytest.mark.parametrize("name", list(PUBLISHED))
def test_published_params_json_give_the_published_shapes(tmp_path, name):
    text, want = PUBLISHED[name]
    (tmp_path / "params.json").write_text(json.dumps(text))
    d = L.model.load_model_args(str(tmp_path), 4096)
    for k, v in want.items():
        assert d[k] == v, (k, d[k], v)
    assert d["dim"] == text["dim"] and d["n_layers"] == text["n_layers"] and d["n_heads"] == text["n_heads"]
    # every published shape is one the library accepts (the tokenizer supplies Llama 2's vocabulary size: 32000)
    assert M.create_error(dict(d, vocab_size=d["vocab_size"] if d["vocab_size"] > 0 else 32000)) is None


@pytest.mark.parametrize("name", list(M.CATALOGUE))
def test_oracle_orders_run_and_agree_on_every_shape(name):
    """the oracle's reference-order and FAST-order forwards of every accepted shape stay within 1e-2 of each other (max
    abs logits): a sanity floor for the bit-for-bit statements the GPU tests rely on"""
    a = M.CATALOGUE[name]
    om = oracle_model(a, host_tensors(a, 31))
    toks = np.random.default_rng(len(name)).integers(0, a["vocab_size"], size=9).astype(np.int32)
    ref, fast = om.new_session(16), om.new_session(16)
    try:
        lr = np.concatenate([ref.forward(toks[:8], 0, all_rows=True), ref.forward(toks[8:], 8)])
        lf = np.concatenate([fast.forward(toks[:8], 0, all_rows=True, order=O.ORDER_FAST),
                             fast.forward(toks[8:], 8, order=O.ORDER_FAST)])
        assert np.isfinite(lr).all() and np.abs(lr).max() > 0
        assert np.abs(lr - lf).max() <= 1e-2, np.abs(lr - lf).max()
    finally:
        ref.close(); fast.close(); om.close()
