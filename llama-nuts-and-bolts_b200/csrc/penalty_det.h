/* penalty_det.h -- the arithmetic of the repetition, frequency and presence penalties and the logit bias (DESIGN.md §9e),
 * defined once for the penalty kernels (penalty.cuh, nvcc) and for their sequential C restatement
 * (oracle_sampling/lnb_sample_ref.c, gcc -ffp-contract=off).
 *
 * Every floating-point step is one separately rounded IEEE operation: on the device the _rn intrinsics, on the host plain C
 * operators under -ffp-contract=off.  The counts are integers, so the order in which a history is counted does not matter.
 * A NaN that a step produces is made 0x7FFFFFFF, the NaN the device's arithmetic returns, because the host's arithmetic
 * keeps an input NaN's payload and sign instead: both sides then hold the same bits, and the sampler ranks them the same. */
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/lnb.h"
#include "sample_det.h"

LNB_SD_FN float lnb_pen_canon(float x) {
  if (x == x) return x;
#if defined(__CUDA_ARCH__)
  return __uint_as_float(0x7fffffffu);
#else
  union { uint32_t u; float f; } c;
  c.u = 0x7fffffffu;
  return c.f;
#endif
}

/* steps 2 and 3 for a token fed c >= 1 times in the window (c == 0: l itself) */
LNB_SD_FN float lnb_pen_apply(float l, uint32_t c, float rp, float fp, float pp) {
  if (c == 0) return l;
  float a = l;
#if defined(__CUDA_ARCH__)
  if (rp != 1.0f) a = lnb_pen_canon(l > 0.0f ? __fdiv_rn(l, rp) : __fmul_rn(l, rp));
  const float d = lnb_pen_canon(__fadd_rn(__fmul_rn(__uint2float_rn(c), fp), pp));
  return lnb_pen_canon(__fsub_rn(a, d));
#else
  if (rp != 1.0f) a = lnb_pen_canon(l > 0.0f ? l / rp : l * rp);
  const float cf = (float)c;
  const float cfp = cf * fp;
  const float d = lnb_pen_canon(cfp + pp);
  return lnb_pen_canon(a - d);
#endif
}

/* step 4: a -inf bias bans the token whatever b is (b + -inf would be NaN for b = +inf) */
LNB_SD_FN float lnb_pen_bias(float b, float bias) {
  if (bias == -INFINITY) return -INFINITY;
#if defined(__CUDA_ARCH__)
  return lnb_pen_canon(__fadd_rn(b, bias));
#else
  return lnb_pen_canon(b + bias);
#endif
}

/* the first position the window of the row emitting position p_next counts */
LNB_SD_FN int32_t lnb_pen_lo(const lnb_penalties* p, int32_t p_next) {
  int32_t lo = p->first_pos;
  if (p->window > 0 && p_next - p->window > lo) lo = p_next - p->window;
  return lo;
}

/* neutral parameters are "off": the sequence is not penalized at all */
LNB_SD_FN int lnb_pen_neutral(const lnb_penalties* p) {
  return p->repetition_penalty == 1.0f && p->frequency_penalty == 0.0f && p->presence_penalty == 0.0f && p->n_bias == 0;
}
