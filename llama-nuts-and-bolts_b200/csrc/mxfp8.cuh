// mxfp8.cuh -- MXFP8 linear weights (DESIGN.md §9h): the quantizer that runs once at lnb_model_finalize, the dequantizer
// that feeds the tensor-core prompt path, and the exact decode the GEMV consumers use (gemv.cuh, WF_MXFP8).
//
// Format (OCP Microscaling MXFP8, scale exponent clamped at -117): each row of a weight matrix is cut into blocks of 32
// columns (the last one 16 wide when K % 32 == 16); a block holds one E8M0 scale byte (X + 127) and one E4M3 code per
// weight.  The rule:
//   amax = max |w| of the block;  X = floor(log2(amax)) - 8 clamped to [-117, 119] (a zero block: -117);
//   code = e4m3(w * 2^-X), round to nearest even, magnitude saturated to 448 (cvt.rn.satfinite.e4m3x2.f32); -0 stays -0.
// With X >= -117 every dequantized value d = e4m3(code) * 2^X is zero or a normal number of at most 4 significant bits
// inside the bf16 range, so d IS a bf16 value and x * d is exact in fp32: an MXFP8 model computes exactly what the bf16
// model with weights d computes.
//
// Device layout: the bf16 panel-major index map with 1-byte elements.  Codes: address(p, c, r, e) = ((p*K/8 + c)*8 + r)*8 + e
// (a (panel, 8-column chunk) is 64 contiguous bytes, a panel's k-range one contiguous byte range); scales: address(p, b, r) =
// (p * NBP + b) * 8 + r with NBP = ceil(K/32) rounded up to even, so the scales of a panel's k-tile are one 16-byte-aligned
// range too.  Element i of the codes and element i of the bf16 panel-major matrix are the same weight.
#pragma once
#include "common.cuh"

namespace lnb {

enum { WF_BF16 = 0, WF_MXFP8 = 1, WF_MXFP4 = 2 };   // = LNB_WEIGHTS_*; WF_MXFP4: mxfp4.cuh

// scale bytes per panel row of 8 rows: blocks of 32 columns, padded to an even count
__host__ __device__ inline int mx_nbp(int K) { return ((K + 31) / 32 + 1) & ~1; }

// f32 bits of e4m3(code) * 2^-120 from a word holding the code in its top byte: sign to bit 31, exponent and mantissa to
// the low bits of the f32 exponent field.  E4M3 subnormals land on f32 subnormals of the same scaled value, so the result
// is exact for every finite code.
LNB_DEVINL float e4m3_raw(uint32_t top) { return __uint_as_float(((uint32_t)((int32_t)top >> 4)) & 0x87f00000u); }
// 2^(X+8) from the E8M0 byte X + 127 (X + 8 is in [-109, 127]: a normal f32)
LNB_DEVINL float mx_scale(uint32_t e8m0) { return __uint_as_float((e8m0 + 8u) << 23); }
// d = e4m3(code) * 2^X exactly: (e4m3 * 2^-120) * 2^112 is e4m3 * 2^-8, a normal f32; times 2^(X+8)
LNB_DEVINL float mx_dequant(uint32_t top, float scale) { return __fmul_rn(__fmul_rn(e4m3_raw(top), 0x1p112f), scale); }
// the 8 weights of one 8-byte chunk (byte e = column e)
LNB_DEVINL void mx_decode8(uint2 v, float scale, float* w) {
  w[0] = mx_dequant(__byte_perm(v.x, 0u, 0x0444), scale);
  w[1] = mx_dequant(__byte_perm(v.x, 0u, 0x1444), scale);
  w[2] = mx_dequant(__byte_perm(v.x, 0u, 0x2444), scale);
  w[3] = mx_dequant(v.x & 0xff000000u, scale);
  w[4] = mx_dequant(__byte_perm(v.y, 0u, 0x0444), scale);
  w[5] = mx_dequant(__byte_perm(v.y, 0u, 0x1444), scale);
  w[6] = mx_dequant(__byte_perm(v.y, 0u, 0x2444), scale);
  w[7] = mx_dequant(v.y & 0xff000000u, scale);
}

LNB_DEVINL uint32_t e4m3x2(float hi, float lo) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// The block rule shared by the weight quantizer and the KV cache writer (kvcache.cuh): X from the largest bf16 magnitude
// field amax (bits & 0x7fff) of the block, and 2^-X, the factor each element is multiplied by before e4m3x2
LNB_DEVINL int mx_block_x(uint32_t amax) {
  const int E = (int)(amax >> 7);                                   // bf16 exponent field of amax (0: zero or subnormal)
  return E == 0 ? -117 : max(-117, min(119, E - 127 - 8));
}
LNB_DEVINL float mx_inv_scale(int X) { return __uint_as_float((uint32_t)(127 - X) << 23); }   // X in [-117, 119]: normal

// One pass over a bf16 panel-major matrix W[N, K]: one thread per (panel, block, row).  Writes the codes and scales
// above; a non-finite weight lowers *flag (preset to ~0) to row * K + col of the first one, in the matrix's row order.
__global__ void mxfp8_quantize_kernel(const uint16_t* __restrict__ W, int N, int K, uint8_t* __restrict__ codes,
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
    const int X = mx_block_x(amax);
    scales[(p * nbp + b) * 8 + r] = (uint8_t)(X + 127);
    const float inv = mx_inv_scale(X);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      if (q >= nc) break;
      const uint32_t u[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
      uint32_t o[2];
      for (int h = 0; h < 2; h++) {
        const uint32_t a = e4m3x2(__fmul_rn(bf_hi(u[2 * h]), inv), __fmul_rn(bf_lo(u[2 * h]), inv));
        const uint32_t c = e4m3x2(__fmul_rn(bf_hi(u[2 * h + 1]), inv), __fmul_rn(bf_lo(u[2 * h + 1]), inv));
        o[h] = a | (c << 16);
      }
      *reinterpret_cast<uint2*>(codes + ((p * kc + c0 + q) * 8 + r) * 8) = make_uint2(o[0], o[1]);
    }
  }
}

// The bf16 panel-major form of rows [0, N) of an MXFP8 matrix (the tensor-core prompt path's operand).  One thread per
// 8-byte chunk row.  Waits for the previous kernel before writing: the GEMM before it may still read `out`.
__global__ void mxfp8_dequant_kernel(const uint8_t* __restrict__ codes, const uint8_t* __restrict__ scales, int N, int K,
                                     uint16_t* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int kc = K / 8, nbp = mx_nbp(K);
  const int64_t total = (int64_t)(N / 8) * kc * 8;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i & 7), c = (int)((i >> 3) % kc);
    const int64_t p = (i >> 3) / kc;
    const uint2 v = *reinterpret_cast<const uint2*>(codes + i * 8);
    float w[8];
    mx_decode8(v, mx_scale(scales[(p * nbp + c / 4) * 8 + r]), w);
    uint4 o;
    o.x = f2bf(w[0]) | ((uint32_t)f2bf(w[1]) << 16);
    o.y = f2bf(w[2]) | ((uint32_t)f2bf(w[3]) << 16);
    o.z = f2bf(w[4]) | ((uint32_t)f2bf(w[5]) << 16);
    o.w = f2bf(w[6]) | ((uint32_t)f2bf(w[7]) << 16);
    *reinterpret_cast<uint4*>(out + i * 8) = o;
  }
}

}  // namespace lnb
