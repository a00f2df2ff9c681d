// mxfp4.cuh -- MXFP4 linear weights (DESIGN.md §9i): the quantizer that runs once at lnb_model_finalize, the dequantizer
// that feeds the tensor-core prompt path, and the exact decode the GEMV consumers use (gemv.cuh, WF_MXFP4).
//
// Format (OCP Microscaling MXFP4 with a clip-free scale): the MXFP8 blocks and scale array (mxfp8.cuh: 32 columns of a row,
// the last one 16 wide when K % 32 == 16, one E8M0 byte X + 127 per block, mx_nbp layout) with one E2M1 code per weight,
// {0, 0.5, 1, 1.5, 2, 3, 4, 6} and a sign bit.  The rule, on the bf16 bit fields of amax = max |w| of the block:
//   e, f = its unbiased exponent and 7-bit mantissa field;  X = e - 2 if f <= 64 else e - 1 (the smallest X with
//   amax <= 6 * 2^X), clamped to [-125, 125];  a zero or subnormal amax: X = -125;
//   code = sign(w) | |w| * 2^-X rounded to the nearest grid value, ties to the even mantissa bit, saturated at 6.
// Every dequantized value d = e2m1(code) * 2^X is then zero or a normal number of at most 2 significant bits inside the
// bf16 range (2^-126 <= |d| <= 1.5 * 2^127), so an MXFP4 model computes exactly what the bf16 model with weights d computes.
//
// Device layout: the bf16 panel-major index map with 4-bit elements.  Codes: the 32-bit word of (panel p, 8-column chunk c,
// row r) is at byte ((p*K/8 + c)*8 + r)*4 and holds column 8c + e in bits 4e..4e+3 (the even column in a byte's low nibble,
// as torch.float4_e2m1fn_x2 packs).  Scales: the MXFP8 scale layout.
#pragma once
#include "mxfp8.cuh"

namespace lnb {

// bf16x2 {e2m1(code g) * 2^-126, e2m1(code g + 4) * 2^-126} of a word of eight codes (g = 0 or 1): the two nibbles are
// masked out, shifted to bits 6..9 / 22..25 and copied 6 bits up by one multiply (a * 65 = a | a << 6), so each code's
// sign lands on its half's sign bit and its magnitude bits on the low exponent bits and the top mantissa bit.  Magnitude 1
// (0.5) becomes the subnormal 2^-127, so the value is exact for every code.
template <int g>
LNB_DEVINL uint32_t e2m1x2_raw(uint32_t v) { return ((v & (0x000f000fu << (4 * g))) * (65u << (6 - 4 * g))) & 0x81c081c0u; }
LNB_DEVINL uint32_t bf16x2_mul(uint32_t a, uint32_t b) {
  uint32_t d;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
  return d;
}
// the 8 weights of a chunk row's code word as bf16x2 pairs P[g] = {d(column g), d(column g + 4)}, g = 0..3: times 2^126
// (the exact e2m1 values) and times the block's 2^X, both exact (scale2: 2^X in both halves, mx4_scale2)
LNB_DEVINL uint32_t mx4_scale2(uint32_t e8m0) { return e8m0 * 0x00800080u; }
LNB_DEVINL void mx4_decode8(uint32_t v, uint32_t scale2, uint32_t* P) {
  const uint32_t v8 = v >> 8, two126 = 0x7e807e80u;
  P[0] = bf16x2_mul(bf16x2_mul(e2m1x2_raw<0>(v), two126), scale2);
  P[1] = bf16x2_mul(bf16x2_mul(e2m1x2_raw<1>(v), two126), scale2);
  P[2] = bf16x2_mul(bf16x2_mul(e2m1x2_raw<0>(v8), two126), scale2);
  P[3] = bf16x2_mul(bf16x2_mul(e2m1x2_raw<1>(v8), two126), scale2);
}

// the E2M1 magnitude code of q = |w| * 2^-X >= 0: the midpoints between grid values, a tie going to the code whose
// mantissa bit is 0 (the even code)
LNB_DEVINL uint32_t e2m1_round(float q) {
  return (uint32_t)(q > 0.25f) + (uint32_t)(q >= 0.75f) + (uint32_t)(q > 1.25f) + (uint32_t)(q >= 1.75f) +
         (uint32_t)(q > 2.5f) + (uint32_t)(q >= 3.5f) + (uint32_t)(q > 5.0f);
}

// One pass over a bf16 panel-major matrix W[N, K]: one thread per (panel, block, row).  Writes the codes and scales
// above; a non-finite weight lowers *flag (preset to ~0) to row * K + col of the first one, in the matrix's row order.
__global__ void mxfp4_quantize_kernel(const uint16_t* __restrict__ W, int N, int K, uint8_t* __restrict__ codes,
                                      uint8_t* __restrict__ scales, unsigned long long* flag) {
  const int nb = (K + 31) / 32, nbp = mx_nbp(K), kc = K / 8;
  const int64_t total = (int64_t)(N / 8) * nb * 8;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(t & 7), b = (int)((t >> 3) % nb);
    const int64_t p = (t >> 3) / nb;
    const int c0 = b * 4, nc = min(4, kc - c0);
    uint4 v[4];
    uint32_t amax = 0;
    bool bad = false;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      if (q >= nc) break;
      v[q] = *reinterpret_cast<const uint4*>(W + ((p * kc + c0 + q) * 8 + r) * 8);
      const uint32_t u[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
      for (int h = 0; h < 4; h++)
        for (int s = 0; s < 32; s += 16) {
          const uint32_t mag = (u[h] >> s) & 0x7fffu;
          if (mag >= 0x7f80u && !bad) {
            bad = true;
            atomicMin(flag, (unsigned long long)(p * 8 + r) * (unsigned long long)K + (unsigned long long)(c0 * 8 + q * 8 + h * 2 + s / 16));
          }
          amax = max(amax, mag);
        }
    }
    const int E = (int)(amax >> 7);                                    // bf16 exponent field of amax (0: zero or subnormal)
    const int X = E == 0 ? -125 : max(-125, min(125, E - 127 - ((amax & 0x7fu) <= 64u ? 2 : 1)));
    scales[(p * nbp + b) * 8 + r] = (uint8_t)(X + 127);
    const float inv = __uint_as_float((uint32_t)(127 - X) << 23);      // 2^-X, X in [-125, 125]: a normal f32
#pragma unroll
    for (int q = 0; q < 4; q++) {
      if (q >= nc) break;
      const uint32_t u[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
      uint32_t o = 0;
#pragma unroll
      for (int e = 0; e < 8; e++) {
        const uint32_t bits = (u[e >> 1] >> (16 * (e & 1))) & 0xffffu;
        // |w| * 2^-X is exact unless it underflows, which only values far below the first midpoint do
        const uint32_t code = ((bits >> 12) & 8u) | e2m1_round(__fmul_rn(__uint_as_float((bits & 0x7fffu) << 16), inv));
        o |= code << (4 * e);
      }
      *reinterpret_cast<uint32_t*>(codes + ((p * kc + c0 + q) * 8 + r) * 4) = o;
    }
  }
}

// The bf16 panel-major form of rows [0, N) of an MXFP4 matrix (the tensor-core prompt path's operand).  One thread per
// 4-byte chunk row.  Waits for the previous kernel before writing: the GEMM before it may still read `out`.
__global__ void mxfp4_dequant_kernel(const uint8_t* __restrict__ codes, const uint8_t* __restrict__ scales, int N, int K,
                                     uint16_t* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int kc = K / 8, nbp = mx_nbp(K);
  const int64_t total = (int64_t)(N / 8) * kc * 8;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i & 7), c = (int)((i >> 3) % kc);
    const int64_t p = (i >> 3) / kc;
    uint32_t P[4];
    mx4_decode8(*reinterpret_cast<const uint32_t*>(codes + i * 4), mx4_scale2(scales[(p * nbp + c / 4) * 8 + r]), P);
    uint4 o;   // columns 0..7 in order: the low halves of P[0..3], then the high halves
    o.x = __byte_perm(P[0], P[1], 0x5410);
    o.y = __byte_perm(P[2], P[3], 0x5410);
    o.z = __byte_perm(P[0], P[1], 0x7632);
    o.w = __byte_perm(P[2], P[3], 0x7632);
    *reinterpret_cast<uint4*>(out + i * 8) = o;
  }
}

}  // namespace lnb
