// wpack.cuh -- the lossless 12-bit packing of a panel-major bf16 matrix that the STRICT decode engine streams for w1|w3 and
// the LM head (DESIGN §4 "Packed copy"): the encoder kernel and the decoder the engine's chain warps run.
//
// Unit: one 8-row panel x one k-tile of `kt` elements (the engine's k-tile of the phase; the last unit of a panel holds the
// K % kt remaining elements).  Unit lengths are multiples of 32.
//   unit byte E: the largest exponent field among the unit's weights whose exponent field is nonzero (0 when there is none);
//                WP_RAW (0xFF) marks a raw unit, whose weights are read from the bf16 matrix itself.  A unit is raw when it
//                holds an exponent field of 255 (inf / NaN) or a nonzero exponent field below E - 14.
//   per weight:  one byte (sign << 7 | 7 mantissa bits) and a 4-bit code: 0 = exponent field 0 (zeros and subnormals),
//                c in 1..15 = exponent field E - 15 + c.  The decoded bf16 bits equal the original ones.
// Layout: unit (panel p, tile t) starts at byte p * 12 * K + t * 12 * kt (12 bytes per column of the panel, like the bf16
// panel's 16); inside it, group g of 32 columns (chunks 4g .. 4g+3 of 8 columns) takes 384 bytes:
//   [  0, 128)  row r at r * 16: the bytes of chunks 4g and 4g+1 (8 + 8, column order)
//   [128, 256)  row r at 128 + r * 16: the bytes of chunks 4g+2 and 4g+3
//   [256, 384)  row r at 256 + r * 16: four 32-bit code words, one per chunk; column i of the chunk sits at bit
//               16 * (i & 1) + 4 * (i >> 1), so the codes of the column pair (2p, 2p+1) are one shift and mask away from the
//               exponent positions of a bf16 pair word
// Every load of a lane (one row) is 16 bytes, and the 8 rows of a panel read 128 contiguous bytes: conflict-free like the
// bf16 tile.  Raw units leave their 12 * len bytes zero.
#pragma once
#include "common.cuh"

namespace lnb {

constexpr uint8_t WP_RAW = 0xFF;
constexpr int WP_GROUP_BYTES = 384;   // 8 rows x 32 columns x 12 bits

// the bf16 pair word (column 2p in the low half, 2p+1 in the high half) of chunk word `sm` (4 columns' sign|mantissa
// bytes: p even uses bytes 0, 1, p odd bytes 2, 3) and code word `cw`; bb = (E - 15) << 7 as u32
template <int P>
LNB_DEVINL uint32_t wp_pair(uint32_t sm, uint32_t cw, uint32_t bb) {
  const uint32_t rep = __byte_perm(sm, 0u, (P & 1) ? 0x3322 : 0x1100);            // [b, b] per half
  const uint32_t t = ((P == 0) ? (cw << 7) : (P == 1) ? (cw << 3) : (P == 2) ? (cw >> 1) : (cw >> 5)) & 0x07800780u;  // code << 7
  const uint32_t nz = ((t + 0x7F807F80u) >> 15) & 0x00010001u;                      // 1 per half with a nonzero code
  const uint32_t e = nz * bb + t;                                                   // (E - 15 + c) << 7, or 0
  return (rep & 0x807F807Fu) | e;                                                   // sign | exponent | mantissa
}
// one chunk (8 columns) of a packed row as the four bf16 pair words of the raw layout
LNB_DEVINL uint4 wp_chunk(uint32_t sm_lo, uint32_t sm_hi, uint32_t cw, uint32_t bb) {
  return make_uint4(wp_pair<0>(sm_lo, cw, bb), wp_pair<1>(sm_lo, cw, bb), wp_pair<2>(sm_hi, cw, bb), wp_pair<3>(sm_hi, cw, bb));
}

// Encoder: one warp per unit.  W = panel-major bf16 [n_panels][K/8][8][8]; out = packed bytes, units = [n_panels][n_tiles]
// unit bytes; counters[0] += bytes the engine reads for this matrix per pass (12 or 16 per weight column of a panel, plus
// the unit table), counters[1] += packed units.
__global__ void __launch_bounds__(256) wpack_encode_kernel(const uint16_t* __restrict__ W, int n_panels, int K, int kt,
                                                           uint8_t* __restrict__ out, uint8_t* __restrict__ units,
                                                           unsigned long long* __restrict__ counters) {
  const int lane = threadIdx.x & 31;
  const int n_tiles = (K + kt - 1) / kt;
  const long long n_units = (long long)n_panels * n_tiles;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long u = warp0; u < n_units; u += n_warps) {
    const int p = (int)(u / n_tiles), t = (int)(u % n_tiles);
    const int k0 = t * kt, len = min(kt, K - k0);
    const uint16_t* src = W + ((size_t)p * K + (size_t)k0) * 8;     // [len/8 chunks][8 rows][8]
    uint8_t* dst = out + (size_t)p * 12 * K + (size_t)k0 * 12;
    // pass 1: largest nonzero exponent field, smallest nonzero one, any 255
    uint32_t emax = 0, emin = 255;
    for (int i = lane; i < len; i += 32) {                           // 8-element words: len * 8 / 8
      const uint4 v = *reinterpret_cast<const uint4*>(src + (size_t)i * 8);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int h = 0; h < 8; h++) {
        const uint32_t e = ((h & 1) ? (w[h >> 1] >> 23) : (w[h >> 1] >> 7)) & 0xFFu;
        if (e) { emax = max(emax, e); emin = min(emin, e); }
      }
    }
    emax = __reduce_max_sync(0xffffffffu, emax);
    emin = __reduce_min_sync(0xffffffffu, emin);
    const bool raw = emax == 255u || (emax > 0u && emin + 14u < emax);
    // pass 2: one (group, row) per lane and iteration
    const int n_items = (len / 32) * 8;
    for (int it = lane; it < n_items; it += 32) {
      const int g = it >> 3, r = it & 7;
      uint32_t smw[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u}, cw[4] = {0u, 0u, 0u, 0u};
      if (!raw) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const uint4 v = *reinterpret_cast<const uint4*>(src + ((size_t)(g * 4 + q) * 8 + r) * 8);
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int i = 0; i < 8; i++) {
            const uint32_t b = (i & 1) ? (w[i >> 1] >> 16) : (w[i >> 1] & 0xFFFFu);
            const uint32_t e = (b >> 7) & 0xFFu;
            const uint32_t code = e ? e + 15u - emax : 0u;
            smw[q * 2 + (i >> 2)] |= (((b >> 8) & 0x80u) | (b & 0x7Fu)) << (8 * (i & 3));
            cw[q] |= code << (16 * (i & 1) + 4 * (i >> 1));
          }
        }
      }
      uint8_t* gd = dst + (size_t)g * WP_GROUP_BYTES + (size_t)r * 16;
      *reinterpret_cast<uint4*>(gd) = make_uint4(smw[0], smw[1], smw[2], smw[3]);
      *reinterpret_cast<uint4*>(gd + 128) = make_uint4(smw[4], smw[5], smw[6], smw[7]);
      *reinterpret_cast<uint4*>(gd + 256) = make_uint4(cw[0], cw[1], cw[2], cw[3]);
    }
    if (lane == 0) {
      units[u] = raw ? WP_RAW : (uint8_t)emax;
      atomicAdd(&counters[0], (unsigned long long)len * (raw ? 16u : 12u) + 1ull);
      if (!raw) atomicAdd(&counters[1], 1ull);
    }
  }
}

}  // namespace lnb
