"""The edge and tie blocks of the MXFP8 and MXFP4 weight formats (DESIGN.md §9h, §9i), and bf16 matrices of any [N, K]
built from them.  Shared by the CPU suites, which pin the C statement (orc_mxfp{8,4}_quantize) on these blocks, and the GPU
suites, which load the matrices as weights so that the device quantizers and decoders meet every clamp, tie and saturation.

Every block is 32 bf16 bit patterns whose interesting entries come first, so that a block cut to the 16-wide last block of a
row (K % 32 == 16) still holds a case: the block maximum, which sets X, is always in its first 16 entries."""
import numpy as np

MX8_X = (-117, 119)          # MXFP8's scale clamps
MX4_X = (-125, 125)          # MXFP4's
TIES4 = {0.25: 0, 0.75: 2, 1.25: 2, 1.75: 4, 2.5: 4, 3.5: 6, 5.0: 6}   # E2M1 midpoint -> the even code it rounds to
TIE4_X = (-125, -100, -6, -1, 0, 3, 90, 125)                           # MXFP4 tie rows: X of each
TIE8_X = (-117, 0, 119)                                                # MXFP8 tie rows: X of each


def bf16(x: float) -> int:
    """the bf16 bits of x, which must be a bf16 value"""
    b = int(np.array([x], np.float32).view(np.uint32)[0])
    assert b & 0xFFFF == 0, x
    return b >> 16


def bf16_trunc(x):
    """bf16 bits of x truncated toward zero (the f32's top half)"""
    return (np.asarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16)


def _row(vals, n=32):
    assert len(vals) <= n
    return list(vals) + [0] * (n - len(vals))


# ---- MXFP8 ------------------------------------------------------------------------------------------------------------
def mxfp8_tie_values():
    """the midpoints between neighbouring E4M3 codes, at X = 0: of every binade, and of the subnormals"""
    vals = []
    for e in range(-6, 9):
        for n in range(8, 15 if e == 8 else 16):
            vals.append((n + 0.5) * 2.0 ** (e - 3))
    vals += [(n + 0.5) * 2.0 ** -9 for n in range(0, 8)]
    return [v for v in vals if v < 448]


def mxfp8_tie_rows():
    """rows of 256 * 2^X (the block maximum: X exactly) and 31 midpoints times 2^X, for X in TIE8_X, and their negations"""
    vals = mxfp8_tie_values()
    rows = []
    for X in TIE8_X:
        for i in range(0, len(vals), 31):
            row = _row([bf16(256.0 * 2.0 ** X)] + [bf16(v * 2.0 ** X) for v in vals[i:i + 31]])
            rows.append(row)
            rows.append([x | 0x8000 for x in row])
    return np.array(rows, np.uint16)


def mxfp8_edge_rows():
    """saturation to 448, E4M3 subnormals and underflow, the lower clamp, the largest finite bf16, a zero and a -0 block"""
    f = lambda xs: list(bf16_trunc(np.array(xs, np.float32)))   # noqa: E731
    sat = f([511.0, 448.0, 449.0, 455.0, 456.0, 460.0, 464.0, 472.0, 480.0, 500.0, 447.0, 440.0, 432.0, 416.0, 444.0, 452.0])
    sat += [x | 0x8000 for x in sat]
    small = f([1.0] + [2.0 ** -k for k in range(6, 17)] + [3 * 2.0 ** -12, 5 * 2.0 ** -13, 7 * 2.0 ** -12, 2.0 ** -15 * 1.5] +
              [9 * 2.0 ** -13, 1.0 / 3, 0.1, 2.0 ** -14 * 1.75] + [0.0] * 12)
    clamp = [0x0001, 0x0002, 0x007F, 0x0080, 0x0081, 0x00FF, 0x0100, 0x0180, 0x0200, 0x0280, 0x0300, 0x0301,
             0x8001, 0x807F, 0x8080, 0x8300] + [0x0000] * 14 + [0x0380, 0x03FF]     # amax < 2^-109: X = -117
    big = [0x7F7F, 0xFF7F, 0x7F00, 0x7E80, 0x3F80, 0x0001, 0x8001, 0x0080] + [0x7F7F - i for i in range(24)]
    zero = [0x0000] * 32
    negz = [0x8000] * 16 + [0x0000] * 16
    return np.array([sat, small, clamp, big, zero, negz], np.uint16)


def mxfp8_extreme_blocks():
    """(upper-clamp blocks, lower-clamp blocks): X = 119 or 118, and X = -117 with normal, subnormal or no amax"""
    upper = [_row([0x7F7F, 0xFF7F, 0x7F00, 0x7E80, 0xFF00, 0x7F40, 0x7F10, 0x7C00, 0x3F80]),
             _row([0x7F00, 0xFEC0, 0x7E80, 0x7E40, 0x7E00]),                     # 2^127 and its binade's quarters
             _row([0x7EC0, 0xFE80, 0x7E40, 0x7D80, 0x7D00])]                     # 1.5 * 2^126: X = 118
    lower = [mxfp8_edge_rows()[2].tolist(),
             _row([0x0480, 0x8400, 0x0300, 0x0181, 0x0100, 0x00C0, 0x0080, 0x8041]),  # amax 2^-118
             _row([0x007F, 0x8041, 0x0040, 0x003F, 0x0021, 0x0001, 0x8000]),     # subnormal amax
             [0x0000] * 32, [0x8000] * 16 + [0x0000] * 16]
    return np.array(upper, np.uint16), np.array(lower, np.uint16)


# ---- MXFP4 ------------------------------------------------------------------------------------------------------------
def mxfp4_f64_row(e: int, f: int):
    """amax = (1 + f/128) * 2^e, then 31 quarters of it: X = e - 2 when f <= 64, else e - 1"""
    amax = (1 + f / 128) * 2.0 ** e
    return [bf16(amax)] + [bf16(amax / 4)] * 31


def mxfp4_tie_row(X: int):
    """6 * 2^X (f = 64, so X exactly), then every midpoint of the grid times 2^X and its negation"""
    row = [bf16(6.0 * 2.0 ** X)]
    for t in TIES4:
        row += [bf16(t * 2.0 ** X), bf16(-t * 2.0 ** X)]
    return _row(row)


def mxfp4_upper_clamp_row():
    """+-max bf16, 2^127, 2^125: X = 125, the first two saturated to +-6"""
    return [0x7F7F, 0xFF7F, 0x7F00, 0x7E00] + [0x3F80] * 28


def mxfp4_lower_rows():
    """amax 2^-125 (X = -127 clamped to -125), a subnormal amax, a zero block with -0, a negative weight rounding to -0"""
    tiny = [0x0080, 0x8100, 0x00C0] + [0x0080] * 29
    sub = [0x0040, 0x8001, 0x0020, 0x0000] + [0x0001] * 28
    zero = [0x0000, 0x8000] * 16
    neg = [0x8000 | bf16(0.125)] + [bf16(4.0)] * 31
    return [tiny, sub, zero, neg]


def mxfp4_edge_rows():
    """every tie at each X of TIE4_X, both sides of f = 64 at both ends of the range, both clamps"""
    rows = [mxfp4_tie_row(X) for X in TIE4_X]
    rows += [mxfp4_f64_row(e, f) for e in (-123, 0, 127) for f in (0, 63, 64, 65, 127)]
    rows += [mxfp4_upper_clamp_row()] + mxfp4_lower_rows()
    return np.array(rows, np.uint16)


def mxfp4_extreme_blocks():
    """(upper-clamp blocks, lower-clamp blocks): X = 125 or 124, and X = -125 with normal, subnormal or no amax"""
    upper = [mxfp4_upper_clamp_row(),
             _row([0x7F00, 0xFEC0, 0x7EA0, 0x7E80, 0x7E40, 0x7E00, 0xFD80]),     # 2^127: X = 125, codes 4 down to 0.5
             _row([0x7EC0, 0xFE80, 0x7E40, 0x7E00, 0x7DC0])]                     # 1.5 * 2^126: f = 64, X = 124
    lower = [mxfp4_lower_rows()[0],
             _row([0x00C0, 0x8080, 0x0060, 0x0041, 0x8040, 0x0020]),             # amax 1.5 * 2^-126: X = -125
             _row([0x007F, 0x8060, 0x0041, 0x0040, 0x0001]),                     # subnormal amax
             [0x0000] * 32, mxfp4_lower_rows()[2]]
    return np.array(upper, np.uint16), np.array(lower, np.uint16)


# ---- matrices ---------------------------------------------------------------------------------------------------------
def _interleave(groups):
    """the rows of the groups taken in turn, shorter groups repeated: every run of len(groups) rows holds every group"""
    n = max(len(g) for g in groups)
    return np.array([g[i % len(g)] for i in range(n) for g in groups], np.uint16)


def blocks(fmt: str) -> np.ndarray:
    """every case block of a format, [n, 32], its groups interleaved: ties, edges, upper clamp, lower clamp"""
    if fmt == "mxfp8":
        ties, edges = mxfp8_tie_rows(), mxfp8_edge_rows()
        m = len(ties) // len(TIE8_X)
        return _interleave([ties[:m], ties[m:2 * m], ties[2 * m:], edges, *mxfp8_extreme_blocks()])
    e = mxfp4_edge_rows()
    n = len(TIE4_X)
    return _interleave([e[:n], e[n:n + 15], e[n + 15:], *mxfp4_extreme_blocks()])


def matrix(fmt: str, N: int, K: int, shift: int = 0) -> np.ndarray:
    """a bf16 [N, K] matrix whose block b of row r is case (r + b + shift) mod n, cut to 16 columns in a 16-wide last
    block: every case starts some row's first block and ends some row's last block, and the last n rows hold them all"""
    assert K % 16 == 0
    B = blocks(fmt)
    nb = (K + 31) // 32
    idx = (np.arange(N)[:, None] + np.arange(nb)[None, :] + shift) % len(B)
    return np.ascontiguousarray(B[idx].reshape(N, nb * 32)[:, :K])


def extreme_blocks(fmt: str):
    return mxfp8_extreme_blocks() if fmt == "mxfp8" else mxfp4_extreme_blocks()


def ordinary_blocks(fmt: str) -> np.ndarray:
    """the ties and saturating blocks of a format at ordinary scale (|X| <= 8): the LM head's third row class"""
    if fmt == "mxfp8":
        ties = mxfp8_tie_rows()
        return np.vstack([ties[:len(ties) // len(TIE8_X)], mxfp8_edge_rows()[:2]])
    return np.array([mxfp4_tie_row(X) for X in TIE4_X if abs(X) <= 8] + [mxfp4_f64_row(0, f) for f in (63, 64, 65)], np.uint16)


HEAD_CLASSES = 4    # LM-head row r belongs to class r % 4: huge, tiny, ordinary, synthetic (every class in every panel)


def extreme_head(fmt: str, tensors: dict) -> dict:
    """a checkpoint whose LM head decodes every extreme scale into finite logits that depend on every extreme block.
    norm.weight is 2^-24 on the even 32-column blocks and 1 on the odd ones.  Rows of class 0 (huge) hold upper-clamp
    blocks in the even blocks and zeros in the odd ones: their products with the down-weighted activations stay near 2^106.
    Rows of class 1 (tiny) hold lower-clamp, subnormal-amax, zero and -0 blocks in the odd blocks and zeros in the even
    ones.  Rows of class 2 hold the ordinary-scale ties and saturating blocks in every block; class 3 keeps its synthetic
    weights."""
    out = dict(tensors)
    W = tensors["output.weight"].copy()
    V, dim = W.shape
    nb = dim // 32
    assert dim % 32 == 0 and V % (8 * HEAD_CLASSES) == 0
    even = np.arange(nb) % 2 == 0
    out["norm.weight"] = np.where(np.repeat(even, 32), bf16(2.0 ** -24), bf16(1.0)).astype(np.uint16)
    upper, lower = extreme_blocks(fmt)
    ordinary = ordinary_blocks(fmt)
    zero = np.zeros((1, 32), np.uint16)
    for cls, (src, mask) in enumerate(((upper, even), (lower, ~even), (ordinary, np.ones(nb, bool)))):
        rows = np.arange(cls, V, HEAD_CLASSES)
        idx = (rows[:, None] // HEAD_CLASSES + np.arange(nb)[None, :]) % len(src)
        blk = np.where(mask[None, :, None], src[idx], zero[None])
        W[rows] = blk.reshape(len(rows), dim)
    out["output.weight"] = W
    return out


def broken_dequant(fmt: str, codes: np.ndarray, scales: np.ndarray, how: str) -> np.ndarray:
    """the C statement's dequantization with one deliberate mistake (the sharpness check of extreme_head):
    "flush" -- blocks at the lower clamp decode as 0;  "sat" -- the largest magnitude code (6, 448) decodes as the next
    one down (4, 416);  "lo" / "hi" -- X one step inside the lower / upper clamp"""
    import oracle_sampling.sample_ref as SR
    lo, hi = MX8_X if fmt == "mxfp8" else MX4_X
    deq = SR.mxfp8_dequantize if fmt == "mxfp8" else SR.mxfp4_dequantize
    codes, scales = codes.copy(), scales.copy()
    if how == "sat":
        if fmt == "mxfp8":
            codes[(codes & 0x7F) == 0x7E] -= 1
        else:
            lo_n, hi_n = codes & 15, codes >> 4
            lo_n[(lo_n & 7) == 7] -= 1
            hi_n[(hi_n & 7) == 7] -= 1
            codes = (lo_n | (hi_n << 4)).astype(np.uint8)
    elif how in ("lo", "hi"):
        scales = np.clip(scales, lo + 1 + 127 if how == "lo" else 0, hi - 1 + 127 if how == "hi" else 255).astype(np.uint8)
    d = deq(codes, scales)
    if how == "flush":
        cols = d.shape[1]
        d[np.repeat(scales == lo + 127, 32, axis=1)[:, :cols]] = 0
    return d
