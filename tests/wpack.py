"""A host restatement of the packed weight format (csrc/wpack.cuh): the encoder, and a decoder that repeats the device's
integer arithmetic (wp_pair) step for step, so a CPU test can pin both to the bf16 bits they must reproduce.

Matrices are panel-major bf16 as the model stores them: uint16 [P panels][K / 8 chunks][8 rows][8 columns]."""
from __future__ import annotations

import numpy as np

RAW = 0xFF
GROUP_BYTES = 384


def _tiles(K: int, kt: int):
    for k0 in range(0, K, kt):
        yield k0, min(kt, K - k0)


def encode(W: np.ndarray, kt: int) -> tuple[np.ndarray, np.ndarray]:
    """-> (data uint8 [P][12 * K], units uint8 [P][ceil(K / kt)])"""
    P, nc = W.shape[0], W.shape[1]
    K = nc * 8
    assert W.shape == (P, nc, 8, 8) and W.dtype == np.uint16
    data = np.zeros((P, 12 * K), np.uint8)
    units = np.zeros((P, (K + kt - 1) // kt), np.uint8)
    for t, (k0, n) in enumerate(_tiles(K, kt)):
        assert n % 32 == 0, "unit lengths are multiples of 32"
        blk = W[:, k0 // 8:(k0 + n) // 8].astype(np.uint32)            # [P][n/8][8][8]
        e = (blk >> 7) & 0xFF
        nz = e != 0
        emax = np.where(nz, e, 0).reshape(P, -1).max(axis=1)
        emin = np.where(nz, e, 255).reshape(P, -1).min(axis=1)
        raw = (emax == 255) | ((emax > 0) & (emin + 14 < emax))
        units[:, t] = np.where(raw, RAW, emax)
        sm = (((blk >> 8) & 0x80) | (blk & 0x7F)).astype(np.uint8)
        code = np.where(nz, e + 15 - emax[:, None, None, None], 0).astype(np.uint32)
        ng = n // 32
        sm = sm.reshape(P, ng, 4, 8, 8)                                   # [P][g][chunk][row][col]
        a = sm[:, :, 0:2].transpose(0, 1, 3, 2, 4).reshape(P, ng, 128)    # row r: chunks 0, 1
        b = sm[:, :, 2:4].transpose(0, 1, 3, 2, 4).reshape(P, ng, 128)    # row r: chunks 2, 3
        i = np.arange(8, dtype=np.uint32)
        shift = 16 * (i & 1) + 4 * (i >> 1)
        cw = (code.reshape(P, ng, 4, 8, 8) << shift).sum(axis=-1, dtype=np.uint64).astype(np.uint32)   # [P][g][chunk][row]
        c = np.ascontiguousarray(cw.transpose(0, 1, 3, 2)).view(np.uint8).reshape(P, ng, 128)
        unit = np.concatenate([a, b, c], axis=2).reshape(P, 12 * n)
        unit[raw] = 0
        data[:, 12 * k0:12 * (k0 + n)] = unit
    return data, units


def _pair(sm: np.ndarray, cw: np.ndarray, bb: np.ndarray, p: int) -> np.ndarray:
    """wp_pair<p> (wpack.cuh), in uint32 arithmetic modulo 2^32"""
    b_lo = (sm >> (16 * (p & 1))) & 0xFF
    b_hi = (sm >> (16 * (p & 1) + 8)) & 0xFF
    rep = b_lo | (b_lo << 8) | (b_hi << 16) | (b_hi << 24)
    sh = 7 - 4 * p
    t = ((cw << sh) if sh >= 0 else (cw >> -sh)) & 0x07800780
    nz = ((t + 0x7F807F80) >> 15) & 0x00010001
    e = (nz * bb + t) & 0xFFFFFFFF
    return (rep & 0x807F807F) | e


def decode(data: np.ndarray, units: np.ndarray, W: np.ndarray, kt: int) -> np.ndarray:
    """the bf16 matrix the engine's chains see: packed units decoded, raw units read from W"""
    P, nc = W.shape[0], W.shape[1]
    K = nc * 8
    out = W.copy()
    for t, (k0, n) in enumerate(_tiles(K, kt)):
        ng = n // 32
        u = np.ascontiguousarray(data[:, 12 * k0:12 * (k0 + n)]).view(np.uint32).reshape(P, ng, 3, 8, 4).astype(np.uint64)
        # u: [P][g][region][row][word]; region 0: chunks 0, 1 (2 words each), 1: chunks 2, 3, 2: one code word per chunk
        E = units[:, t].astype(np.uint64)
        bb = (((E - 15) & 0xFFFFFFFF) << 7) & 0xFFFFFFFF
        bb = bb[:, None, None]
        dec = np.zeros((P, ng, 4, 8, 8), np.uint16)
        for q in range(4):
            reg, w0 = divmod(q, 2)
            sm_lo, sm_hi = u[:, :, reg, :, 2 * w0], u[:, :, reg, :, 2 * w0 + 1]
            cw = u[:, :, 2, :, q]
            for p in range(4):
                word = _pair(sm_lo if p < 2 else sm_hi, cw, bb, p)
                dec[:, :, q, :, 2 * p] = (word & 0xFFFF).astype(np.uint16)
                dec[:, :, q, :, 2 * p + 1] = (word >> 16).astype(np.uint16)
        packed = units[:, t] != RAW
        blk = dec.reshape(P, n // 8, 8, 8)
        out[packed, k0 // 8:(k0 + n) // 8] = blk[packed]
    return out


def read_bytes(units: np.ndarray, K: int, kt: int) -> int:
    """bytes the engine streams for one pass over the matrix: 12 or 16 per column of a panel, plus the unit table"""
    lens = np.array([n for _, n in _tiles(K, kt)], np.int64)
    return int((np.where(units == RAW, 16, 12) * lens[None, :]).sum()) + units.size
