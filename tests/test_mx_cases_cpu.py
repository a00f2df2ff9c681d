"""tests/mx_cases.py without a GPU: its matrices hold every case they claim, at both block widths, and the extreme LM head
(mx_cases.extreme_head) is sharp -- the oracle's logits of its D(W) are finite and change under each broken dequantization
the GPU suites must catch."""
import numpy as np
import pytest

from oracle_sampling import sample_ref as SR
from tests import mx_cases as MC

QUANT = {"mxfp8": SR.mxfp8_quantize, "mxfp4": SR.mxfp4_quantize}
DEQUANT = {"mxfp8": SR.mxfp8_dequantize, "mxfp4": SR.mxfp4_dequantize}


def _nibbles(codes):
    return np.stack([codes & 15, codes >> 4], axis=-1).reshape(codes.shape[0], -1)


def _X(scales):
    return scales.astype(int) - 127


@pytest.mark.parametrize("K", [256, 528, 1024])       # 528: a 16-wide last block
@pytest.mark.parametrize("shift", [0, 11])
def test_mxfp8_matrices_hold_every_case(K, shift):
    N = 64
    w = MC.matrix("mxfp8", N, K, shift)
    assert w.shape == (N, K)
    codes, scales = SR.mxfp8_quantize(w)
    X = _X(scales)
    for cols in (slice(0, 32), slice(32 * (X.shape[1] - 1), K)):       # first block, last block (16 wide when K = 528)
        Xb, cb = X[:, cols.start // 32], codes[:, cols]
        assert Xb.min() == MC.MX8_X[0] and Xb.max() == MC.MX8_X[1]
        assert {0, 118}.issubset(set(Xb.tolist()))
        assert ((cb & 0x7F) == 0x7E).any(), "saturation to 448"
        assert (((cb & 0x7F) > 0) & ((cb & 0x7F) < 8)).any(), "E4M3 subnormal codes"
        assert (cb == 0x80).any() and (cb == 0).any(), "-0 and +0"
    for rows in (slice(0, 8), slice(N - 8, N)):                          # the first and last panel: both clamps
        assert X[rows].min() == MC.MX8_X[0] and X[rows].max() == MC.MX8_X[1]
    # every tie at each of its X, with both signs, somewhere in a full block
    f = (w.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    for Xt in MC.TIE8_X:
        full = (X == Xt)[:, :K // 32].repeat(32, axis=1)
        have = set(np.abs(f[:, :K // 32 * 32][full]).tolist())
        assert all(v * 2.0 ** Xt in have for v in MC.mxfp8_tie_values()), Xt
    assert (w[:, :K // 32 * 32] == 0x7F7F).any() and (w[:, :K // 32 * 32] == 0xFF7F).any()
    if K % 32:
        last = w[:, K - 16:]
        assert (last == 0x7F7F).any() and _X(scales[:, -1]).min() == MC.MX8_X[0]


@pytest.mark.parametrize("K", [256, 528, 1024])
@pytest.mark.parametrize("shift", [0, 11])
def test_mxfp4_matrices_hold_every_case(K, shift):
    N = 64
    w = MC.matrix("mxfp4", N, K, shift)
    codes, scales = SR.mxfp4_quantize(w)
    X, nib = _X(scales), _nibbles(codes)
    for b in (0, X.shape[1] - 1):
        cb = nib[:, 32 * b:32 * b + 32]
        assert X[:, b].min() == MC.MX4_X[0] and X[:, b].max() == MC.MX4_X[1]
        assert 124 in X[:, b].tolist()
        wb = w[:, 32 * b:32 * b + 32]
        sat = (wb & 0x7FFF) > MC.bf16(6.0 * 2.0 ** 125)
        assert sat.any() and ((cb[:, :wb.shape[1]][sat] & 7) == 7).all(), "saturation at 6"
        assert (cb == 8).any() and (cb == 0).any(), "-0 and +0"
        assert ((wb & 0x7F80) == 0).any() and (wb & 0x7F).any(), "subnormal weights"
    for rows in (slice(0, 8), slice(N - 8, N)):
        assert X[rows].min() == MC.MX4_X[0] and X[rows].max() == MC.MX4_X[1]
    # every tie with both signs at each X of TIE4_X (a tie row's 15 entries fit a 16-wide last block too)
    for Xt in MC.TIE4_X:
        want = {MC.bf16(s * t * 2.0 ** Xt) for t in MC.TIES4 for s in (1, -1)}
        assert any(want <= set(w[r, 32 * b:32 * b + 32].tolist()) for r, b in np.argwhere(X == Xt)), Xt
    # both sides of f = 64
    amax = (w.reshape(N, -1, 16)[:, :, 0] & 0x7FFF)
    assert ((amax & 0x7F) == 64).any() and ((amax & 0x7F) == 65).any()


# ---- the extreme LM head -----------------------------------------------------------------------------------------------
def _head_model(fmt):
    import lnb_b200
    from tests.helpers import host_tensors
    args = dict(lnb_b200.synth.TINY128, vocab_size=4096)
    return args, MC.extreme_head(fmt, host_tensors(args, 2718))


def _dequantized(fmt, args, tensors, how=None):
    from tests.test_gpu_mxfp8 import linear_names
    out = dict(tensors)
    for name in linear_names(args):
        codes, scales = QUANT[fmt](tensors[name])
        out[name] = DEQUANT[fmt](codes, scales) if how is None else MC.broken_dequant(fmt, codes, scales, how)
    return out


@pytest.mark.parametrize("fmt", ["mxfp8", "mxfp4"])
def test_extreme_head_is_finite_and_sharp(fmt):
    from tests.helpers import oracle_model
    args, t = _head_model(fmt)
    codes, scales = QUANT[fmt](t["output.weight"])
    X = _X(scales)
    lo, hi = MC.MX8_X if fmt == "mxfp8" else MC.MX4_X
    for cls in range(MC.HEAD_CLASSES):                          # every class in every panel
        rows = np.arange(cls, args["vocab_size"], MC.HEAD_CLASSES)
        assert len(np.unique(rows // 8)) == args["vocab_size"] // 8
    assert (X[0::4].max(axis=1) == hi).all() and (X[1::4].min(axis=1) == lo).all()
    prompt = np.array([1, 50, 999, 7], np.int32)

    def logits(tensors):
        om = oracle_model(args, tensors)
        try:
            s = om.new_session(16)
            lg = s.forward(prompt, 0)
            s.close()
            return lg
        finally:
            om.close()

    base = logits(_dequantized(fmt, args, t))
    assert np.isfinite(base).all()
    huge, tiny = np.abs(base[:, 0::4]), np.abs(base[:, 1::4])
    assert (huge > 2.0 ** 90).mean() > 0.9 and huge.max() < 2.0 ** 120, "huge rows: large but finite"
    assert (tiny > 0).mean() > 0.9 and tiny.max() < 2.0 ** -100, "tiny rows: nonzero, far below the others"
    for how in ("flush", "sat", "lo", "hi"):
        broken = logits(_dequantized(fmt, args, t, how))
        assert not np.array_equal(broken, base), how
