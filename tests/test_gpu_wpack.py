"""The packed copies of w1|w3 and the LM head that the STRICT decode engine streams (csrc/wpack.cuh, DESIGN §4):
- the device encoder writes exactly the bytes and unit table of the host restatement (tests/wpack.py), on random weights and
  on weights with inf, NaN, zeros, subnormals and 15 / 16-binade spreads, and the restated decoder gives back every bf16;
- with weights that mix raw and packed units inside one row tile and one stage, the STRICT engine still equals the kernel
  chain (which never reads the packed copy) and the oracle bit for bit, at TINY, `wide` and `tiny128`;
- the synthetic 8B model packs at least 90 % of its units, so the benchmark runs the packed path."""
import ctypes as C

import numpy as np
import pytest

from tests import engine_shapes as ES
from tests import wpack as WP
from tests.helpers import host_tensors
from tests.test_gpu_engine import _load, check_engine_equals_kernel_chain_and_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    import lnb_b200
    return lnb_b200


def read_pack(L, gm, layer):
    """(info, data, units, src) of the packed copy of layer `layer`'s w1|w3 (-1: the LM head)"""
    lib, h = L._capi.lib, gm.Transformer.h
    info = np.zeros(5, np.int64)
    rc = L._capi.check(lib.lnb_model_wpack_read(h, layer, None, None, None, info.ctypes.data_as(L._capi.i64p)))
    assert rc == 1, lib.lnb_last_error().decode()
    kt, n_units, _, _, N = (int(v) for v in info)
    K = gm.Transformer.args.Dim
    data = np.zeros((N // 8, 12 * K), np.uint8)
    units = np.zeros((N // 8, n_units // (N // 8)), np.uint8)
    src = np.zeros((N // 8, K // 8, 8, 8), np.uint16)
    L._capi.check(lib.lnb_model_wpack_read(h, layer, data.ctypes.data_as(C.c_void_p), units.ctypes.data_as(C.c_void_p),
                                           src.ctypes.data_as(L._capi.u16p), info.ctypes.data_as(L._capi.i64p)))
    return info, data, units, src


def check_pack(L, gm, layer):
    info, data, units, src = read_pack(L, gm, layer)
    kt = int(info[0])
    hd, hu = WP.encode(src, kt)
    assert np.array_equal(units, hu), f"layer {layer}: unit table"
    assert np.array_equal(data, hd), f"layer {layer}: packed bytes"
    assert np.array_equal(WP.decode(data, units, src, kt), src)
    assert int(info[2]) == int((units != WP.RAW).sum())
    assert int(info[3]) == WP.read_bytes(units, src.shape[1] * 8, kt)
    return units


def _deepen(t: np.ndarray, rows, cols, by: int = 20) -> np.ndarray:
    """lower the exponent field of t[rows, cols] by `by` binades (normal values stay normal): their units turn raw"""
    t = t.copy()
    v = t[np.ix_(rows, cols)].astype(np.int32)
    e = (v >> 7) & 0xFF
    ok = e > by + 1
    v = np.where(ok, (v & 0x807F) | ((e - by) << 7), v)
    t[np.ix_(rows, cols)] = v.astype(np.uint16)
    return t


def mixed_tensors(args, seed=4321):
    """weights whose packed copies mix raw and packed units: in every third panel the first column sinks 20 binades, and in
    every fifth panel (offset 1) the last column does -- so one row tile, and one stage, holds both kinds"""
    t = dict(host_tensors(args, seed))
    for name in ["output.weight"] + [f"layers.{l}.feed_forward.w{i}.weight" for l in range(args["n_layers"]) for i in (1, 3)]:
        w = t[name]
        R, K = w.shape
        rows = np.arange(R)
        t[name] = _deepen(w, rows[(rows // 8) % 3 == 0], [0])
        t[name] = _deepen(t[name], rows[(rows // 8) % 5 == 1], [K - 1])
    return t


def test_encoder_equals_host_restatement_on_adversarial_weights(L):
    args = dict(L.synth.TINY)
    t = mixed_tensors(args)
    rng = np.random.default_rng(5)
    w1 = t["layers.0.feed_forward.w1.weight"].copy()
    R, K = w1.shape
    specials = np.array([0x7F80, 0xFF80, 0x7FC1, 0xFFFF, 0x0000, 0x8000, 0x0001, 0x807F], np.uint16)
    w1[8:16, :] = specials[rng.integers(0, len(specials), size=(8, K))]            # a panel of specials only
    w1[16, 3] = 0x7FC0                                                             # one NaN in an otherwise normal panel
    top = rng.integers(100, 120)
    for p, spread in ((3, 14), (4, 15)):                                           # 15 binades pack, 16 do not
        e = rng.integers(top - spread, top + 1, size=(8, K))
        e[0, 0], e[1, 1] = top, top - spread
        w1[8 * p:8 * p + 8] = ((rng.integers(0, 2, size=(8, K)) << 15) | (e << 7) | rng.integers(0, 128, size=(8, K))).astype(np.uint16)
    t["layers.0.feed_forward.w1.weight"] = w1
    t["output.weight"] = rng.integers(0, 65536, size=t["output.weight"].shape).astype(np.uint16)   # random bit patterns
    gm = L.model.LoadModelFromTensors(args, t)
    try:
        assert (check_pack(L, gm, -1) == WP.RAW).all()           # random bit patterns span far more than 15 binades
        for layer in range(args["n_layers"]):
            units = check_pack(L, gm, layer)
            assert (units == WP.RAW).any() and (units != WP.RAW).any()
    finally:
        gm.Free()


def _mixed_model(L, args):
    args, om, gm = _load(L, args, mixed_tensors(args))
    units = check_pack(L, gm, 0)
    assert (units == WP.RAW).any() and (units != WP.RAW).any()
    # one 16-panel row tile (and so one stage) of w1|w3 holds both kinds
    assert any(len(set((units[r:r + 16, 0] == WP.RAW).tolist())) == 2 for r in range(0, units.shape[0], 16))
    return args, om, gm


@pytest.mark.parametrize("shape", ["tiny", "wide", "tiny128"])
def test_strict_engine_with_mixed_units_equals_chain_and_oracle(L, shape):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    args = {"tiny": dict(L.synth.TINY), "wide": ES.wide_args(sms), "tiny128": dict(L.synth.TINY128)}[shape]
    model = _mixed_model(L, args)
    try:
        check_engine_equals_kernel_chain_and_oracle(L, model, "strict")
    finally:
        model[2].Free()
        model[1].close()


def test_8b_synthetic_weights_pack_at_least_90_percent(L):
    args = dict(L.synth.LLAMA31_8B)
    gm = L.model.LoadSyntheticModel(args, seed=L.synth.SEED)
    try:
        shares = {}
        for layer in (-1, 0, args["n_layers"] - 1):
            info = np.zeros(5, np.int64)
            assert L._capi.check(L._capi.lib.lnb_model_wpack_read(gm.Transformer.h, layer, None, None, None,
                                                                  info.ctypes.data_as(L._capi.i64p))) == 1
            shares[layer] = int(info[2]) / int(info[1])
            assert int(info[0]) == 128
        print("8B packed-unit shares:", shares)
        assert min(shares.values()) >= 0.9, shares
    finally:
        gm.Free()
