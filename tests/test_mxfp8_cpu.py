"""MXFP8 weights without a GPU (DESIGN.md §9h): the C statement (orc_mxfp8_quantize / orc_mxfp8_dequantize in
oracle_sampling/lnb_sample_ref.c) against an independent numpy restatement that uses integer arithmetic on the bf16 bit
fields only, against torch's float8_e4m3fn cast where that cast is defined, and the exactness claim the identity rests
on: every (code, X) dequantizes to a bf16 value."""
import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import mx_cases as MC


# ---- the integer restatement -----------------------------------------------------------------------------------------
def _block_x(w_block, clamp_lo=-117):
    mag = int((np.asarray(w_block, np.uint16) & 0x7FFF).max()) if len(w_block) else 0
    E = mag >> 7
    if E == 0:
        return clamp_lo
    return max(clamp_lo, min(119, E - 127 - 8))


def _e4m3(bits: int, X: int, half_up: bool = False) -> int:
    """E4M3 code of bf16 `bits` * 2^-X: round to nearest even, saturated to 448, from integers alone"""
    sign = 0x80 if bits & 0x8000 else 0
    E, M = (bits >> 7) & 0xFF, bits & 0x7F
    sig = (128 + M) if E else M
    if sig == 0:
        return sign
    e2 = (E if E else 1) - 127 - 7 - X            # |v| = sig * 2^e2
    if (sig << max(e2, 0)) >= (448 << max(-e2, 0)):
        return sign | 0x7E
    fl = sig.bit_length() - 1 + e2                # floor(log2 |v|)
    q = max(-9, fl - 3)                           # the quantum of |v|'s E4M3 binade (2^-9 below 2^-6)
    k = q - e2                                    # |v| / 2^q = sig / 2^k
    if k <= 0:
        n = sig << -k
    else:
        n, rem, half = sig >> k, sig & ((1 << k) - 1), 1 << (k - 1)
        if rem > half or (rem == half and (half_up or n & 1)):
            n += 1
    if q == -9:
        return sign | n                           # subnormal codes; n == 8 is 2^-6 = 0x08
    return sign | (((q + 3 + 7) << 3) + n - 8)    # n == 16 carries into the next binade


def restate_quantize(w, clamp_lo=-117, half_up=False):
    w = np.asarray(w, np.uint16)
    rows, cols = w.shape
    nb = (cols + 31) // 32
    codes = np.zeros((rows, cols), np.uint8)
    scales = np.zeros((rows, nb), np.uint8)
    for r in range(rows):
        for b in range(nb):
            blk = w[r, 32 * b:32 * b + 32]
            X = _block_x(blk, clamp_lo)
            scales[r, b] = (X + 127) & 0xFF
            for i, v in enumerate(blk):
                codes[r, 32 * b + i] = _e4m3(int(v), X, half_up)
    return codes, scales


def restate_dequant(code: int, X: int) -> int:
    """bf16 bits of e4m3(code) * 2^X, from integers alone"""
    sign = (code & 0x80) << 8
    e, m = (code >> 3) & 15, code & 7
    if e == 0 and m == 0:
        return sign
    if e == 0:
        msb = m.bit_length() - 1
        E, mant = X - 9 + msb + 127, (m - (1 << msb)) << (7 - msb)
    else:
        E, mant = e - 7 + X + 127, m << 4
    assert 1 <= E <= 254, (code, X)
    return sign | (E << 7) | mant


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _bf16(x):
    return (np.asarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16)


def _random_rows(rng, rows, cols):
    # finite bf16 patterns over the whole exponent range, blocks of one scale and of mixed scales
    w = rng.integers(0, 0x7F80, (rows, cols), dtype=np.uint16) | (rng.integers(0, 2, (rows, cols), dtype=np.uint16) << 15)
    narrow = _bf16(rng.standard_normal((rows, cols)).astype(np.float32) * np.float32(0.02))
    return np.where(rng.random((rows, 1)) < 0.5, w, narrow).astype(np.uint16)


def _cases():
    rng = np.random.default_rng(9)
    return {
        "random": _random_rows(rng, 24, 96),
        "random_tail16": _random_rows(rng, 16, 80),      # cols % 32 == 16: a 16-wide last block
        "ties": MC.mxfp8_tie_rows(),
        "edges": MC.mxfp8_edge_rows(),
        "edges_tail16": np.ascontiguousarray(MC.mxfp8_edge_rows()[:, :48]),
        "extremes": np.vstack(MC.mxfp8_extreme_blocks()),
        "case_matrix_tail16": MC.matrix("mxfp8", 40, 208, shift=3),
    }


@pytest.mark.parametrize("name", list(_cases()))
def test_c_statement_matches_integer_restatement(name):
    w = _cases()[name]
    codes, scales = SR.mxfp8_quantize(w)
    rc, rs = restate_quantize(w)
    assert np.array_equal(scales, rs)
    assert np.array_equal(codes, rc), np.argwhere(codes != rc)[:8]
    d = SR.mxfp8_dequantize(codes, scales)
    nb = scales.shape[1]
    exp = np.array([[restate_dequant(int(codes[r, c]), int(scales[r, c // 32]) - 127) for c in range(w.shape[1])]
                    for r in range(w.shape[0])], np.uint16)
    assert nb == (w.shape[1] + 31) // 32
    assert np.array_equal(d, exp)


def test_edge_cases_cover_what_they_claim():
    codes, scales = SR.mxfp8_quantize(MC.mxfp8_edge_rows())
    X = scales.astype(int) - 127
    assert (codes[0] & 0x7F == 0x7E).sum() >= 20                     # saturation to 448
    assert ((codes[1] & 0x7F) < 8).sum() > 10 and (codes[1] & 0x7F == 0).sum() > 0   # E4M3 subnormals and underflow
    assert X[2, 0] == -117                                           # the clamp
    assert X[3, 0] == 119                                            # the largest finite bf16
    assert (codes[4] == 0).all() and X[4, 0] == -117                 # zero block
    assert (codes[5, :16] == 0x80).all()                             # -0 stays -0
    tc, _ = SR.mxfp8_quantize(MC.mxfp8_tie_rows())
    assert ((tc[:, 1:] & 1) == 0).all()                              # every midpoint went to the even neighbour
    assert len(set((tc & 0x7F).ravel().tolist())) > 50               # ... over the whole code space


def test_torch_cast_agrees_in_range():
    torch = pytest.importorskip("torch")
    c = _cases()
    w = np.concatenate([c["random"][:, :32], c["ties"], c["edges"]], axis=0)
    codes, scales = SR.mxfp8_quantize(w)
    X = np.repeat(scales.astype(np.int32) - 127, 32, axis=1)[:, :w.shape[1]]
    v = (w.astype(np.uint32) << 16).view(np.float32).astype(np.float64) * np.exp2(-X.astype(np.float64))
    v32 = v.astype(np.float32)
    ok = np.abs(v) < 448                                          # torch does not promise saturation: in-range values only
    t = torch.from_numpy(v32).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    assert ok.sum() > 1000
    assert np.array_equal(t[ok], codes[ok])


def test_every_code_and_scale_dequantizes_to_an_exact_bf16():
    codes = np.array([c for c in range(256) if c & 0x7F != 0x7F], np.uint8)
    xs = np.arange(-117, 120)
    c2 = np.tile(codes, (len(xs), 1))
    s2 = np.repeat((xs + 127).astype(np.uint8)[:, None], (len(codes) + 31) // 32, axis=1)
    d = SR.mxfp8_dequantize(c2, s2)
    val = (d.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    mag = codes & 0x7F
    e, m = mag >> 3, (mag & 7).astype(np.float64)
    e4 = np.where(e == 0, m * 2.0 ** -9, (8 + m) * np.exp2(e.astype(np.float64) - 10))
    e4 = np.where(codes & 0x80, -e4, e4)
    assert np.array_equal(val, e4[None, :] * np.exp2(xs.astype(np.float64))[:, None])
    E = (d >> 7) & 0xFF
    assert ((E >= 1) | ((d & 0x7FFF) == 0)).all()                 # never a bf16 subnormal, never inf
    assert (E <= 254).all()
    for X in (-117, -60, 0, 119):
        for c in (0x01, 0x07, 0x08, 0x7E, 0x85, 0xFE):
            assert restate_dequant(c, X) == int(SR.mxfp8_dequantize(np.array([[c]], np.uint8), np.array([[X + 127]], np.uint8))[0, 0])


@pytest.mark.parametrize("bad", [0x7F80, 0xFF80, 0x7FC0, 0x7F81])
def test_non_finite_weights_are_refused(bad):
    w = _random_rows(np.random.default_rng(1), 4, 64)
    w[2, 37] = bad
    with pytest.raises(ValueError, match="row 2, column 37"):
        SR.mxfp8_quantize(w)


def test_broken_rules_are_caught():
    ties, edges = MC.mxfp8_tie_rows(), MC.mxfp8_edge_rows()
    c, _ = SR.mxfp8_quantize(ties)
    bc, _ = restate_quantize(ties, half_up=True)
    assert not np.array_equal(c, bc)
    _, s = SR.mxfp8_quantize(edges)
    _, bs = restate_quantize(edges, clamp_lo=-127)
    assert not np.array_equal(s, bs)
