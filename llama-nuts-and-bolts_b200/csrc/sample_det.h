/* sample_det.h -- the arithmetic of the seeded sampler (DESIGN.md §9b), defined once for the sampler kernel
 * (sample.cuh, nvcc) and for its sequential C restatement (oracle_sampling/lnb_sample_ref.c, gcc -ffp-contract=off).
 *
 * Every floating-point step below is one separately rounded IEEE operation: on the device the _rn intrinsics (nvcc can
 * neither contract them to an FMA nor reorder them), on the host plain C operators under -ffp-contract=off.  After the
 * one exp a weight is a 64-bit integer, so every sum, threshold and draw of the sampler is integer arithmetic and any
 * reduction order gives the same bits. */
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define LNB_SD_FN __host__ __device__ __forceinline__
#else
#define LNB_SD_FN static inline
#endif

LNB_SD_FN double lnb_sd_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
LNB_SD_FN double lnb_sd_add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

/* exp(z) for z in [-28, 0]: z = k ln2 + r with |r| <= ln2 / 2 (Cody-Waite, ln2 split so that k * LN2_HI is exact), then
 * the Taylor polynomial of degree 13 in Horner form, then the exact scaling by 2^k.  Within 2 ulp of the correctly
 * rounded exp on [-28, 0] and exactly 1.0 at 0 (tests/test_sampling_cpu.py checks both). */
LNB_SD_FN double lnb_exp_det(double z) {
  const double kd = floor(lnb_sd_add(lnb_sd_mul(z, 0x1.71547652b82fep+0 /* log2(e) */), 0.5));
  const double r = lnb_sd_add(lnb_sd_add(z, -lnb_sd_mul(kd, 0x1.62e42fee00000p-1)), -lnb_sd_mul(kd, 0x1.a39ef35793c76p-33));
  double p = 0x1.6124613a86d09p-33;                 /* 1/13! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.1eed8eff8d898p-29);   /* 1/12! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.ae64567f544e4p-26);   /* 1/11! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.27e4fb7789f5cp-22);   /* 1/10! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.71de3a556c734p-19);   /* 1/9! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.a01a01a01a01ap-16);   /* 1/8! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.a01a01a01a01ap-13);   /* 1/7! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.6c16c16c16c17p-10);   /* 1/6! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.1111111111111p-7);    /* 1/5! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.5555555555555p-5);    /* 1/4! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0x1.5555555555555p-3);    /* 1/3! */
  p = lnb_sd_add(lnb_sd_mul(p, r), 0.5);
  p = lnb_sd_add(lnb_sd_mul(p, r), 1.0);
  p = lnb_sd_add(lnb_sd_mul(p, r), 1.0);
  return ldexp(p, (int)kd);
}

/* Integer weight of logit l in a row whose rank-0 logit is m, at temperature T > 0:
 * z = f32(f32(l - m) / T);  W = floor(exp(z) * 2^40) for z >= -28, else 0.  W(m) = 2^40, and a vocabulary's sum is < 2^57.
 * The cut at -28 is the contract's one truncation: a token more than 28 nats (after temperature) below the top is never
 * drawn. */
#define LNB_SAMPLE_ONE 1099511627776.0 /* 2^40 */
LNB_SD_FN uint64_t lnb_sample_weight(float l, float m, float T) {
#if defined(__CUDA_ARCH__)
  const float z = __fdiv_rn(__fsub_rn(l, m), T);
#else
  const float d = l - m;
  const float z = d / T;
#endif
  if (!(z >= -28.0f)) return 0;
  return (uint64_t)lnb_sd_mul(lnb_exp_det((double)z), LNB_SAMPLE_ONE);
}

/* rank order (logit descending, index ascending -- the greedy argmax's tie rule): order-preserving map of an f32 */
LNB_SD_FN uint32_t lnb_sample_ord(float l) {
  uint32_t u;
#if defined(__CUDA_ARCH__)
  u = __float_as_uint(l);
#else
  union { float f; uint32_t u; } c;
  c.f = l;
  u = c.u;
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
/* ---- token log-probabilities (DESIGN.md §9d) ----
 * key = ord(l) << 32 | (2^32 - 1 - i): rank order is key descending, and a key gives its logit and index back, so a record
 * of keys is enough to finish it on the host. */
LNB_SD_FN uint64_t lnb_logprob_key(float l, int32_t i) {
  return ((uint64_t)lnb_sample_ord(l) << 32) | (0xffffffffu - (uint32_t)i);
}
LNB_SD_FN int32_t lnb_logprob_key_index(uint64_t k) { return (int32_t)(0xffffffffu - (uint32_t)(k & 0xffffffffu)); }
LNB_SD_FN float lnb_logprob_key_logit(uint64_t k) {
  const uint32_t o = (uint32_t)(k >> 32);
  const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#if defined(__CUDA_ARCH__)
  return __uint_as_float(u);
#else
  union { uint32_t u; float f; } c;
  c.u = u;
  return c.f;
#endif
}
/* The host finish of a logprob: (f64(l) - f64(m)) - log(f64(sum) * 2^-40), every step one rounded f64 operation and the log
 * the host libm's.  sum is the row's whole-vocabulary mass at T = 1 (sum of lnb_sample_weight(l_i, m, 1)), m its rank-0
 * logit.  The device never evaluates a log: the record it writes holds integers and keys only. */
#if defined(__CUDACC__)
__host__
#endif
static inline double lnb_logprob_finish(float l, float m, uint64_t sum) {
  return ((double)l - (double)m) - log(ldexp((double)sum, -40));
}

/* top-p target mass: Q = clamp(ceil(f64(P) * f64(W_C)), 1, W_C) (f64(W_C) rounds to nearest) */
LNB_SD_FN uint64_t lnb_sample_top_p_mass(float P, uint64_t WC) {
#if defined(__CUDA_ARCH__)
  const double wc = __ull2double_rn(WC);
#else
  const double wc = (double)WC;
#endif
  uint64_t q = (uint64_t)ceil(lnb_sd_mul((double)P, wc));
  if (q < 1) q = 1;
  if (q > WC) q = WC;
  return q;
}

/* splitmix64 at index i: the generator of the synthetic weights (csrc/kernels.cuh) and of the draw's 64 random bits, which
 * are lnb_splitmix64_at(seed, p_next) */
LNB_SD_FN uint64_t lnb_splitmix64_at(uint64_t seed, uint64_t i) {
  uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
/* R = high 64 bits of r * W_kept, in [0, W_kept) */
LNB_SD_FN uint64_t lnb_sample_scale(uint64_t r, uint64_t W) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(r, W);
#else
  return (uint64_t)(((unsigned __int128)r * W) >> 64);
#endif
}
