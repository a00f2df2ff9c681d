"""The packed weight format of the STRICT decode engine (csrc/wpack.cuh), restated on the host (tests/wpack.py): every bf16
pattern decodes to itself, units switch to raw exactly at a spread of 16 binades or at inf / NaN, and short last units
keep the layout arithmetic."""
import numpy as np
import pytest

from tests import wpack as WP


def _panels(vals: np.ndarray, P: int) -> np.ndarray:
    """values in column order per row, row-major [P * 8][K] -> panel-major [P][K/8][8][8]"""
    m = vals.astype(np.uint16).reshape(P, 8, -1, 8)
    return np.ascontiguousarray(m.transpose(0, 2, 1, 3))


def _roundtrip(W: np.ndarray, kt: int):
    data, units = WP.encode(W, kt)
    assert np.array_equal(WP.decode(data, units, W, kt), W)
    return data, units


@pytest.mark.parametrize("kt", [64, 128, 256])
def test_every_bf16_pattern_in_column_order(kt):
    W = _panels(np.arange(65536, dtype=np.uint32), 8)          # 8 panels x K = 1024
    _roundtrip(W, kt)


def test_every_finite_pattern_lands_in_a_packed_unit():
    """patterns sorted by exponent field: each 1024-weight unit spans 4 binades, so every unit without inf / NaN is packed"""
    pats = np.arange(65536, dtype=np.uint32)
    order = np.argsort(((pats >> 7) & 0xFF) * 65536 + pats, kind="stable")
    W = np.ascontiguousarray(pats[order].astype(np.uint16).reshape(8, 128, 8, 8))   # unit (p, t) = 1024 consecutive patterns
    data, units = _roundtrip(W, 128)
    e = (W.astype(np.uint32) >> 7) & 0xFF
    for p in range(8):
        for t in range(8):
            has_inf_nan = (e[p, t * 16:(t + 1) * 16] == 255).any()
            assert (units[p, t] == WP.RAW) == has_inf_nan


@pytest.mark.parametrize("spread,raw", [(14, False), (15, True), (0, False)])
@pytest.mark.parametrize("top", [254, 127, 15, 9])
def test_raw_boundary_at_sixteen_binades(spread, raw, top):
    """nonzero exponent fields [top - spread, top]: 15 binades pack, 16 do not; tops below 15 exercise E - 15 < 0"""
    lo = max(1, top - spread)
    rng = np.random.default_rng(top * 100 + spread)
    K = 128
    exps = rng.integers(lo, top + 1, size=(8, K))
    exps[0, 0], exps[1, 1] = top, lo
    vals = (rng.integers(0, 2, size=(8, K)) << 15) | (exps << 7) | rng.integers(0, 128, size=(8, K))
    vals[2, 5] = 0x0000
    vals[3, 6] = 0x8000                        # -0
    vals[4, 7] = 0x0001                        # smallest subnormal
    vals[5, 8] = 0x807F                        # negative subnormal
    W = _panels(vals, 1)
    data, units = _roundtrip(W, 128)
    expect_raw = raw and top - spread >= 1
    assert units[0, 0] == (WP.RAW if expect_raw else top)
    if expect_raw:
        assert not data.any()


@pytest.mark.parametrize("special", [0x7F80, 0xFF80, 0x7FC0, 0x7F81, 0xFFFF])
def test_inf_and_nan_units_are_raw(special):
    rng = np.random.default_rng(special)
    vals = (120 << 7) | rng.integers(0, 128, size=(16, 256))
    vals[9, 200] = special                     # panel 1, second unit at kt = 128
    W = _panels(vals, 2)
    _, units = _roundtrip(W, 128)
    assert units[1, 1] == WP.RAW
    assert (units[0] == 120).all() and units[1, 0] == 120


def test_zero_and_subnormal_only_unit():
    vals = np.zeros((8, 64), np.uint32)
    vals[:, ::3] = 0x0005
    vals[:, 1::5] = 0x8000
    W = _panels(vals, 1)
    data, units = _roundtrip(W, 64)
    assert units[0, 0] == 0


@pytest.mark.parametrize("K,kt", [(160, 128), (96, 64), (4096 + 32, 512), (1536, 512)])
def test_short_last_units(K, kt):
    rng = np.random.default_rng(K)
    P = 3
    s = rng.uniform(-0.02, 0.02, size=(P * 8, K)).astype(np.float32)
    vals = (s.view(np.uint32) >> 16)
    vals[5, K - 1] = 0x0001                     # a subnormal in the last unit of panel 0
    W = _panels(vals, P)
    data, units = _roundtrip(W, kt)
    n_tiles = (K + kt - 1) // kt
    assert units.shape == (P, n_tiles)
    last = K - (n_tiles - 1) * kt
    assert data.shape == (P, 12 * K)
    lens = [kt] * (n_tiles - 1) + [last]
    assert WP.read_bytes(units, K, kt) == sum((16 if units[p, t] == WP.RAW else 12) * lens[t]
                                              for p in range(P) for t in range(n_tiles)) + P * n_tiles


def test_uniform_weights_pack_almost_everywhere():
    """weights uniform in [-s, s] (the synthetic model's): half sit in the top binade, and 15 binades hold all but ~2^-14 of
    them, so nearly every 1024-weight unit packs"""
    rng = np.random.default_rng(0)
    s = rng.uniform(-0.0156, 0.0156, size=(64 * 8, 1024)).astype(np.float32)
    W = _panels(s.view(np.uint32) >> 16, 64)
    _, units = _roundtrip(W, 128)
    assert (units != WP.RAW).mean() >= 0.9
