// sample.cuh -- seeded temperature / top-k / top-p sampling of logits rows (DESIGN.md §9b).
//
// The arithmetic is csrc/sample_det.h: after the one exp every weight is a 64-bit integer, so the sums below may run in any
// order and still give the bits of the sequential statement (oracle_sampling/lnb_sample_ref.c).  Two kernels, launched
// together; each row is served by exactly one of them, chosen on the device from the row's parameters:
//  - sample_split_kernel, rows whose candidate set is small (top_k <= 1024 and top_k * slices <= 2048, e.g. K <= 64 at the
//    8B vocabulary): the row is split over one CTA per 4096 logits; each sorts its slice's keys in shared memory and
//    publishes its top K; the last CTA of the row merges those (the row's top K is among them), then forms the weights,
//    the top-p cut and the draw on at most K candidates.
//  - sample_kernel, every other row (the whole vocabulary, large K, temperature 0): one CTA of 1024 threads; top-k and top-p
//    are thresholds in rank order (logit descending, index ascending), found by radix selects over the order-preserving
//    logit bits (counts for top-k, integer mass for top-p) plus one index-order search among the logits equal to the
//    threshold; the draw is one index-order prefix scan.
// A row whose weights are all 0 (its top logit is +inf or NaN) keeps its rank-0 token.
#pragma once
#include "../../include/lnb.h"
#include "common.cuh"
#include "sample_det.h"

namespace lnb {

#define SMP_THREADS 1024
#define SMP_MAX_ROWS 8
#define SMP_SLICE 4096   // logits per CTA of sample_split_kernel
#define SMP_MERGE 2048   // candidates its last CTA merges

// One launch samples up to 8 rows of a logits buffer.  Row b: logits row row[b], parameters params[slot[b]], the draw
// keyed on p_next[b] (< 0: *pos_ptr, the position a decode run's step has just advanced to), token to out[out_idx[b]]
// (out may be null).  st non-null (decode run, one row): the token also becomes st->next_token, the next step's input,
// and tok_out[st->step - 1].
struct SampleJob {
  const float* logits;
  long long ld;
  int V;
  int n;
  const lnb_sampling* params;
  unsigned long long* wbuf;   // [n][V] weights of the rows (scratch, sample_kernel)
  unsigned long long* cand;   // [n][SMP_MERGE] slice candidates (scratch, sample_split_kernel)
  unsigned int* cnt;          // [n] CTAs of a row that finished (zero between launches)
  const int32_t* pos_ptr;
  int32_t* out;
  LnbDevState* st;
  int32_t* tok_out;
  int32_t row[SMP_MAX_ROWS], slot[SMP_MAX_ROWS], p_next[SMP_MAX_ROWS], out_idx[SMP_MAX_ROWS];
};

__global__ void sample_set_params_kernel(lnb_sampling* slot, lnb_sampling p) {
  pdl_launch_dependents();
  pdl_wait();
  *slot = p;
}

LNB_DEVINL unsigned long long smp_block_max(unsigned long long v, unsigned long long* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
  for (int i = 1; i < SMP_THREADS / 32; i++) v = red[i] > v ? red[i] : v;
  return v;
}
// exclusive block scan of one u64 per thread; *total = the sum over the block
LNB_DEVINL unsigned long long smp_block_exscan(unsigned long long v, unsigned long long* red, unsigned long long* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
  if (lane == 31) red[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const unsigned long long s = red[lane];
    unsigned long long w = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    red[lane] = w - s;   // exclusive prefix of the warp totals
    if (lane == 31) red[32] = w;
  }
  __syncthreads();
  *total = red[32];
  return red[wid] + inc - v;
}

// The smallest index i whose index-order prefix sum of w(.) exceeds target(total) (total: the sum over the row).  Each
// warp owns a contiguous range of the row, read 32 consecutive elements at a time; the warp whose range holds the
// crossing walks it again with a warp scan per 32 elements.
template <class Wf, class Tf>
LNB_DEVINL int smp_find(int V, Wf w, Tf target_of_total, unsigned long long* red, int* res) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int span = ((V + SMP_THREADS / 32 - 1) / (SMP_THREADS / 32) + 31) & ~31;
  const int lo = min(V, wid * span), hi = min(V, lo + span);
  unsigned long long s = 0;
  for (int i = lo + lane; i < hi; i += 32) s += w(i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  unsigned long long total;
  const unsigned long long ex = smp_block_exscan(lane == 0 ? s : 0ull, red, &total);   // lane 0 carries its warp's sum
  const unsigned long long wex = __shfl_sync(0xffffffffu, ex, 0);
  const unsigned long long t = target_of_total(total);
  if (threadIdx.x == 0) *res = -1;
  __syncthreads();
  if (wex <= t && t < wex + s) {   // warp-uniform
    unsigned long long c = wex;
    for (int base = lo; base < hi; base += 32) {
      const int i = base + lane;
      const unsigned long long v = i < hi ? w(i) : 0ull;
      unsigned long long inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
      }
      const unsigned hit = __ballot_sync(0xffffffffu, c + inc > t);
      if (hit) {
        if (lane == __ffs(hit) - 1) *res = i;
        break;
      }
      c += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
  __syncthreads();
  return *res;
}

// Radix select over the order-preserving logit bits u(i), 8 bits per level from the top: the value v such that the
// elements with u > v carry less than `need` and those with u >= v at least `need`, where an element carries mass(i)
// (0 for elements outside the set).  Returns v; *rest = what the elements with u == v must still supply.
template <bool kCounts, class Mf>
LNB_DEVINL uint32_t smp_radix_select(const float* __restrict__ l, int V, Mf mass, unsigned long long need, unsigned long long* hist,
                                     unsigned long long* bc, unsigned long long* rest) {
  uint32_t prefix = 0, mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    if (threadIdx.x < 256) hist[threadIdx.x] = 0;
    __syncthreads();
    for (int base = 0; base < V; base += SMP_THREADS) {
      const int i = base + threadIdx.x;
      unsigned long long w = 0;
      uint32_t digit = 256;
      if (i < V) {
        const uint32_t u = lnb_sample_ord(l[i]);
        if ((u & mask) == prefix) {
          w = mass(i);
          if (w) digit = (u >> shift) & 255u;
        }
      }
      if (!__any_sync(0xffffffffu, digit < 256)) continue;   // warp-uniform: nothing of this warp is in the set
      // lanes with the same digit add their mass first (a row's logits share few top bytes: one atomic per digit and warp).
      // A mass is at most 2^40: its two halves summed over 32 lanes fit 32 bits each.
      const unsigned peers = __match_any_sync(0xffffffffu, digit);
      if (kCounts) {   // top-k: every element of the set weighs 1
        if (digit < 256 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[digit], (unsigned long long)__popc(peers));
        continue;
      }
      const unsigned lo_sum = __reduce_add_sync(peers, (unsigned)(w & 0xffffffu));
      const unsigned hi_sum = __reduce_add_sync(peers, (unsigned)(w >> 24));
      if (digit < 256 && (int)(threadIdx.x & 31) == __ffs(peers) - 1)
        atomicAdd(&hist[digit], ((unsigned long long)hi_sum << 24) + lo_sum);
    }
    __syncthreads();
    if (threadIdx.x < 32) {   // warp 0: lane L holds digits 255-8L .. 248-8L; find where the running mass reaches need
      const int lane = threadIdx.x;
      unsigned long long s = 0;
      for (int j = 0; j < 8; j++) s += hist[255 - 8 * lane - j];
      unsigned long long inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      const unsigned long long ex = inc - s;
      if (ex < need && need <= inc) {
        unsigned long long c = ex;
        for (int j = 0; j < 8; j++) {
          const int d = 255 - 8 * lane - j;
          if (c + hist[d] >= need) { bc[0] = (unsigned long long)d; bc[1] = need - c; break; }
          c += hist[d];
        }
      }
    }
    __syncthreads();
    prefix |= (uint32_t)bc[0] << shift;
    mask |= 255u << shift;
    need = bc[1];
    __syncthreads();
  }
  *rest = need;
  return prefix;
}

LNB_DEVINL int smp_slices(int V) { return (V + SMP_SLICE - 1) / SMP_SLICE; }
// the candidate count K of a row sample_split_kernel serves, 0 for the rows of sample_kernel
LNB_DEVINL int smp_split_k(const lnb_sampling& p, int V) {
  const int k = (p.top_k == 0 || p.top_k >= V) ? V : p.top_k;
  return (p.temperature > 0.0f && k <= SMP_THREADS && k * smp_slices(V) <= SMP_MERGE) ? k : 0;
}
LNB_DEVINL unsigned long long smp_key(float l, int i) {   // rank order = key descending
  return ((unsigned long long)lnb_sample_ord(l) << 32) | (0xffffffffu - (uint32_t)i);
}
LNB_DEVINL int smp_key_index(unsigned long long k) { return (int)(0xffffffffu - (uint32_t)(k & 0xffffffffull)); }
// bitonic sort of a[0..n) (n a power of two) into descending order, the whole CTA
LNB_DEVINL void smp_sort_desc(unsigned long long* a, int n) {
  for (int k = 2; k <= n; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < n / 2; t += SMP_THREADS) {
        const int i = 2 * t - (t & (j - 1)), p = i + j;
        const unsigned long long x = a[i], y = a[p];
        if (((i & k) == 0) ? x < y : x > y) { a[i] = y; a[p] = x; }
      }
      __syncthreads();
    }
}
LNB_DEVINL int smp_pow2(int n) {
  int p = 2;
  while (p < n) p <<= 1;
  return p;
}
LNB_DEVINL void smp_publish(const SampleJob& J, int b, int tok) {
  if (J.out) J.out[J.out_idx[b]] = tok;
  if (J.st) {
    J.st->next_token = tok;
    if (J.tok_out) J.tok_out[J.st->step - 1] = tok;
  }
}

// grid (smp_slices(V), n): CTA g of row b holds logits [g * 4096, (g + 1) * 4096)
__global__ void __launch_bounds__(SMP_THREADS, 1) sample_split_kernel(const SampleJob J) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned long long keys[SMP_SLICE];
  __shared__ unsigned long long wk[SMP_THREADS];
  __shared__ unsigned long long red[33];
  __shared__ int flag;
  const int b = blockIdx.y, g = blockIdx.x, G = gridDim.x, V = J.V;
  const lnb_sampling prm = J.params[J.slot[b]];
  const int K = smp_split_k(prm, V);
  if (K == 0) return;   // sample_kernel's row
  const float* __restrict__ l = J.logits + (size_t)J.row[b] * J.ld;
  unsigned long long* cand = J.cand + (size_t)b * SMP_MERGE;
  // this slice's top K, in rank order, to cand[g * K, (g + 1) * K) (0 = no candidate)
  const int lo = g * SMP_SLICE, n_loc = min(V - lo, SMP_SLICE), np = smp_pow2(n_loc);
  for (int t = threadIdx.x; t < np; t += SMP_THREADS) keys[t] = t < n_loc ? smp_key(l[lo + t], lo + t) : 0ull;
  __syncthreads();
  smp_sort_desc(keys, np);
  for (int t = threadIdx.x; t < K; t += SMP_THREADS) cand[g * K + t] = t < n_loc ? keys[t] : 0ull;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) flag = (atomicAdd(&J.cnt[b], 1u) == (unsigned)(G - 1));
  __syncthreads();
  if (!flag) return;
  // the last CTA of the row: the row's top K are the first K of the merged slice candidates
  __threadfence();
  const int nm = G * K, npm = smp_pow2(nm);
  for (int t = threadIdx.x; t < npm; t += SMP_THREADS) keys[t] = t < nm ? __ldcg(&cand[t]) : 0ull;
  if (threadIdx.x == 0) J.cnt[b] = 0;   // ready for the next launch (a graph replays this one)
  __syncthreads();
  smp_sort_desc(keys, npm);
  const int t = threadIdx.x;
  const int i_t = t < K ? smp_key_index(keys[t]) : 0;
  const float m = l[smp_key_index(keys[0])];
  const float T = prm.temperature, P = prm.top_p;
  const unsigned long long w = t < K ? lnb_sample_weight(l[i_t], m, T) : 0ull;
  unsigned long long WC;
  const unsigned long long ex = smp_block_exscan(w, red, &WC);   // rank-order prefix of C
  int tok = smp_key_index(keys[0]);
  if (WC != 0ull) {
    // top-p: rank t is kept when the mass before it is below Q; then the index-order prefix mass at each kept candidate
    const bool kept = t < K && (!(P < 1.0f) || ex < lnb_sample_top_p_mass(P, WC));
    wk[t] = kept ? w : 0ull;
    unsigned long long Wk;
    smp_block_exscan(kept ? w : 0ull, red, &Wk);   // (also publishes wk)
    const int pn = J.p_next[b] >= 0 ? J.p_next[b] : *J.pos_ptr;
    const unsigned long long R = lnb_sample_scale(lnb_splitmix64_at(prm.seed, (uint64_t)(int64_t)pn), Wk);
    if (threadIdx.x == 0) flag = 0x7fffffff;
    __syncthreads();
    if (kept) {
      unsigned long long S = 0;
      for (int s = 0; s < K; s++)
        if (smp_key_index(keys[s]) <= i_t) S += wk[s];
      if (S > R) atomicMin(&flag, i_t);   // the smallest index whose prefix mass exceeds R
    }
    __syncthreads();
    tok = flag;
  }
  if (threadIdx.x == 0) smp_publish(J, b, tok);
}

__global__ void __launch_bounds__(SMP_THREADS, 1) sample_kernel(const SampleJob J) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned long long hist[256];
  __shared__ unsigned long long red[33];
  __shared__ unsigned long long bc[2];
  __shared__ int res;
  const int b = blockIdx.x;
  const int V = J.V;
  const float* __restrict__ l = J.logits + (size_t)J.row[b] * J.ld;
  unsigned long long* __restrict__ wb = J.wbuf + (size_t)b * V;
  const lnb_sampling prm = J.params[J.slot[b]];
  if (smp_split_k(prm, V)) return;   // sample_split_kernel's row

  // rank 0: the greedy argmax key (logit bits, then the lower index)
  unsigned long long best = 0;
  for (int i = threadIdx.x; i < V; i += SMP_THREADS) {
    const unsigned long long k = ((unsigned long long)lnb_sample_ord(l[i]) << 32) | (0xffffffffu - (uint32_t)i);
    best = k > best ? k : best;
  }
  best = smp_block_max(best, red);
  int tok = (int)(0xffffffffu - (uint32_t)(best & 0xffffffffull));
  const float T = prm.temperature, P = prm.top_p;
  const int K = prm.top_k;
  if (T > 0.0f && K != 1) {
    const float m = l[tok];
    // candidates C: ranks < K, i.e. u > vk, or u == vk and i <= ik
    const bool all = (K == 0 || K >= V);
    uint32_t vk = 0;
    int ik = V;
    if (!all) {
      unsigned long long rest;
      vk = smp_radix_select<true>(l, V, [](int) { return 1ull; }, (unsigned long long)K, hist, bc, &rest);
      ik = smp_find(V, [=](int i) { return lnb_sample_ord(l[i]) == vk ? 1ull : 0ull; }, [=](unsigned long long) { return rest - 1; },
                    red, &res);
    }
    // integer weights of C (0 elsewhere) and their sum W_C
    unsigned long long wsum = 0;
    for (int i = threadIdx.x; i < V; i += SMP_THREADS) {
      const float li = l[i];
      const uint32_t u = lnb_sample_ord(li);
      const bool in_c = all || u > vk || (u == vk && i <= ik);
      const unsigned long long w = in_c ? lnb_sample_weight(li, m, T) : 0ull;
      wb[i] = w;
      wsum += w;
    }
    unsigned long long WC;
    smp_block_exscan(wsum, red, &WC);   // (also publishes wb to the whole block)
    if (WC == 0ull) goto publish;       // every weight 0 (top logit +inf or NaN): the rank-0 token
    {
    // top-p: the shortest rank prefix of C whose mass reaches Q; ends at u == vp, i <= ip
    const bool pall = !(P < 1.0f);
    uint32_t vp = 0;
    int ip = V;
    if (!pall) {
      const unsigned long long Q = lnb_sample_top_p_mass(P, WC);
      unsigned long long rest;
      vp = smp_radix_select<false>(l, V, [=](int i) { return wb[i]; }, Q, hist, bc, &rest);
      // the elements with u == vp in C all weigh the same: the last one kept is where their index-order mass reaches rest
      ip = smp_find(V, [=](int i) { return lnb_sample_ord(l[i]) == vp ? wb[i] : 0ull; }, [=](unsigned long long) { return rest - 1; },
                    red, &res);
    }
    // the draw: R = (r * W_kept) >> 64, the token is the first index whose index-order prefix mass exceeds R
    const int pn = J.p_next[b] >= 0 ? J.p_next[b] : *J.pos_ptr;
    const unsigned long long r = lnb_splitmix64_at(prm.seed, (uint64_t)(int64_t)pn);
    tok = smp_find(
        V,
        [=](int i) {
          const unsigned long long w = wb[i];
          if (pall || w == 0ull) return w;
          const uint32_t u = lnb_sample_ord(l[i]);
          return (u > vp || (u == vp && i <= ip)) ? w : 0ull;
        },
        [=](unsigned long long wk) { return lnb_sample_scale(r, wk); }, red, &res);
    }
  }
publish:
  if (threadIdx.x == 0) smp_publish(J, b, tok);
}

}  // namespace lnb
