"""MXFP4 weights without a GPU (DESIGN.md §9i): the C statement (orc_mxfp4_quantize / orc_mxfp4_dequantize in
oracle_sampling/lnb_sample_ref.c) against an independent numpy restatement that uses integer arithmetic on the bf16 bit
fields only, and the exactness claim the identity rests on: every (code, X) dequantizes to a bf16 value.  Restatements
that round ties away from zero, take the OCP floor scale or swap the nibbles disagree with the statement on these inputs."""
import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import mx_cases as MC

MIDS4 = (1, 3, 5, 7, 10, 14, 20)     # 4 x the midpoints 0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5 of the E2M1 grid


# ---- the integer restatement -----------------------------------------------------------------------------------------
def _block_x(w_block, ocp=False):
    mag = int((np.asarray(w_block, np.uint16) & 0x7FFF).max()) if len(w_block) else 0
    E, f = mag >> 7, mag & 0x7F
    if E == 0:
        return -125
    X = E - 127 - 2 if (ocp or f <= 64) else E - 127 - 1
    return max(-125, min(125, X))


def _e2m1(bits: int, X: int, ties_away: bool = False) -> int:
    """E2M1 code of bf16 `bits` * 2^-X: nearest grid value, ties to the even code, saturated at 6, from integers alone"""
    sign = 8 if bits & 0x8000 else 0
    E, M = (bits >> 7) & 0xFF, bits & 0x7F
    sig = (128 + M) if E else M
    s = (E if E else 1) - 127 - 7 - X + 2           # 4 |w| 2^-X = sig * 2^s
    k = 0
    for i, t in enumerate(MIDS4):
        lhs, rhs = sig << max(s, 0), t << max(-s, 0)
        up_on_tie = ties_away or (i & 1) == 1       # the tie's upper neighbour i + 1 is even when i is odd
        k += lhs > rhs or (lhs == rhs and up_on_tie)
    return sign | k


def restate_quantize(w, ocp=False, ties_away=False, swap_nibbles=False):
    w = np.asarray(w, np.uint16)
    rows, cols = w.shape
    nb = (cols + 31) // 32
    codes = np.zeros((rows, cols // 2), np.uint8)
    scales = np.zeros((rows, nb), np.uint8)
    for r in range(rows):
        for b in range(nb):
            blk = w[r, 32 * b:32 * b + 32]
            X = _block_x(blk, ocp)
            scales[r, b] = X + 127
            for i, v in enumerate(blk):
                c = 32 * b + i
                lo_nibble = (c & 1) == (1 if swap_nibbles else 0)
                codes[r, c // 2] |= _e2m1(int(v), X, ties_away) << (0 if lo_nibble else 4)
    return codes, scales


def restate_dequant(code: int, X: int) -> int:
    """bf16 bits of e2m1(code) * 2^X"""
    sign = 0x8000 if code & 8 else 0
    e, m = (code >> 1) & 3, code & 1
    if e == 0 and m == 0:
        return sign
    if e == 0:
        return sign | ((X - 1 + 127) << 7)          # 0.5 * 2^X
    return sign | ((e - 1 + X + 127) << 7) | (m << 6)


bf16 = MC.bf16


def bf16_matrix(rng, rows, cols, scale=1.0):
    return (rng.standard_normal((rows, cols)).astype(np.float32) * scale).view(np.uint32).__rshift__(16).astype(np.uint16)


def _check(w):
    got = SR.mxfp4_quantize(w)
    exp = restate_quantize(w)
    assert np.array_equal(got[1], exp[1]), "scales"
    assert np.array_equal(got[0], exp[0]), "codes"
    return got


# ---- quantization ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [32, 48, 64, 96, 208])   # 48, 208: a 16-wide last block
def test_random_blocks_match_restatement(cols):
    rng = np.random.default_rng(cols)
    w = bf16_matrix(rng, 8, cols)
    w[1] = bf16_matrix(rng, 1, cols, 1e-30)[0]            # small binades
    w[2] = bf16_matrix(rng, 1, cols, 1e30)[0]             # large binades
    w[3, ::3] = 0                                         # zeros inside blocks
    _check(w)


@pytest.mark.parametrize("e", [-120, -40, -3, 0, 1, 7, 60, 120])
def test_scale_on_both_sides_of_f_64(e):
    for f, dx in ((63, 2), (64, 2), (65, 1), (127, 1), (0, 2)):
        amax = (1 + f / 128) * 2.0 ** e
        w = np.array([MC.mxfp4_f64_row(e, f)], np.uint16)
        codes, scales = _check(w)
        assert int(scales[0, 0]) - 127 == e - dx, (e, f)
        assert amax <= 6.0 * 2.0 ** (e - dx) < 2 * amax  # the smallest X that does not clip the block maximum


def test_every_tie_rounds_to_the_even_code():
    ties = MC.TIES4
    for X in MC.TIE4_X:
        w = np.array([MC.mxfp4_tie_row(X)], np.uint16)  # amax = 6 * 2^X: f = 64, so X = e - 2 exactly
        codes, scales = _check(w)
        assert int(scales[0, 0]) - 127 == X
        nib = [(codes[0, c // 2] >> (4 * (c & 1))) & 15 for c in range(32)]
        assert nib[0] == 7
        for i, (t, k) in enumerate(ties.items()):
            assert nib[1 + 2 * i] == k and nib[2 + 2 * i] == 8 | k, (X, t)


def test_upper_clamp_saturates_to_six():
    w = np.array([MC.mxfp4_upper_clamp_row()], np.uint16)   # +-max bf16, 2^127, 2^125
    codes, scales = _check(w)
    assert int(scales[0, 0]) - 127 == 125
    assert codes[0, 0] == 0xF7                          # +6 (low nibble), -6 (high nibble)
    assert codes[0, 1] == 0x26                          # 2^127 and 2^125: 4 and 1 times 2^125


def test_lower_clamp_subnormal_zero_and_negative_zero():
    # amax 2^-125 (E = 2): X = -127 -> -125; a subnormal amax: -125; a zero block with -0; a negative weight that rounds
    # to 0 keeps its sign
    w = np.array(MC.mxfp4_lower_rows(), np.uint16)
    codes, scales = _check(w)
    assert list(scales[:3, 0].astype(int) - 127) == [-125, -125, -125]
    assert codes[2, 0] == 0x80                          # +0, -0
    assert codes[3, 0] & 15 == 0x8


@pytest.mark.parametrize("cols", [208, 256])
def test_case_blocks_match_restatement(cols):
    _check(MC.matrix("mxfp4", 48, cols, shift=5))
    _check(np.vstack(MC.mxfp4_extreme_blocks()))


def test_non_finite_weights_are_refused():
    for bad in (0x7F80, 0xFF80, 0x7FC1):
        w = np.full((3, 64), bf16(1.0), np.uint16)
        w[2, 37] = bad
        with pytest.raises(ValueError, match="row 2, column 37"):
            SR.mxfp4_quantize(w)


# ---- dequantization --------------------------------------------------------------------------------------------------
def test_every_code_and_scale_dequantizes_to_an_exact_bf16():
    Xs = np.arange(-125, 126)
    codes = np.array([[(c | (c << 4)) for c in range(16)] * 2] * len(Xs), np.uint8)      # 64 columns: 2 blocks
    scales = np.repeat((Xs + 127)[:, None], 2, axis=1).astype(np.uint8)
    out = SR.mxfp4_dequantize(codes, scales)
    grid = (0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0)
    for i, X in enumerate(Xs):
        for c in range(64):
            code = c // 2 % 16
            assert out[i, c] == restate_dequant(code, int(X)), (code, X)
            v = np.array([int(out[i, c]) << 16], np.uint32).view(np.float32)[0]
            exact = grid[code & 7] * 2.0 ** int(X) * (-1 if code & 8 else 1)
            assert float(v) == exact and (v == 0 or np.isfinite(v) and abs(v) >= 2.0 ** -126), (code, X)


def test_quantize_then_dequantize_is_within_half_a_step():
    rng = np.random.default_rng(5)
    w = bf16_matrix(rng, 16, 96)
    codes, scales = SR.mxfp4_quantize(w)
    d = SR.mxfp4_dequantize(codes, scales)
    wf = (w.astype(np.uint32) << 16).view(np.float32)
    df = (d.astype(np.uint32) << 16).view(np.float32)
    step = 2.0 ** (np.repeat(scales.astype(np.int32) - 127, 32, axis=1)[:, :96])    # the widest grid gap is 2 * 2^X
    assert np.all(np.abs(wf - df) <= step)


# ---- the statement is the one documented -----------------------------------------------------------------------------
def _variant_inputs():
    rng = np.random.default_rng(11)
    ties = [bf16(t) for t in (0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0)]
    tie_row = [bf16(6.0)] + ties + [0] * (32 - 1 - len(ties))
    wide = [bf16(7.0)] + [bf16(x) for x in (1.0, 3.0, 6.5)] + [0] * 28     # f > 64: the OCP scale clips 7 to 6 * 2^(X)
    return np.vstack([np.array([tie_row, wide], np.uint16), bf16_matrix(rng, 2, 32)])


@pytest.mark.parametrize("variant", ["ties_away", "ocp", "swap_nibbles"])
def test_other_statements_are_caught(variant):
    w = _variant_inputs()
    got = SR.mxfp4_quantize(w)
    assert all(np.array_equal(a, b) for a, b in zip(got, restate_quantize(w)))
    wrong = restate_quantize(w, **{variant: True})
    assert not all(np.array_equal(a, b) for a, b in zip(got, wrong))
