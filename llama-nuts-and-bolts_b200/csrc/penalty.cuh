// penalty.cuh -- repetition, frequency and presence penalties and logit bias over each sequence's token history
// (DESIGN.md §9e).
//
// The arithmetic is csrc/penalty_det.h.  One job processes up to 8 logits rows into a [rows][V] f32 buffer, which the
// sampler (sample.cuh) then reads in place of the logits.  Two PDL launches:
//  - penalty_count_kernel, grid (PEN_COUNT_CTAS, rows): the row's window of its sequence's history, read once, adds each
//    token's occurrences into a [rows][V] u32 scratch (lanes of a warp holding the same token add once).  Counts are
//    integers: any order gives the same bits, and a window of any length needs no sorting.
//  - penalty_apply_kernel, grid (slices of 4096 logits, rows): reads a slice's logits and counts, writes l', resets the
//    counts it read to 0 (so a captured graph may replay the job), then adds the row's biases that fall in the slice.
// A row of a sequence without penalties (a sampled neighbour in the same call) is copied unchanged.
#pragma once
#include "../../include/lnb.h"
#include "common.cuh"
#include "penalty_det.h"

namespace lnb {

#define PEN_THREADS 256
#define PEN_MAX_ROWS 8
#define PEN_SLICE 4096        // logits per CTA of penalty_apply_kernel
#define PEN_COUNT_CTAS 32     // CTAs per row of penalty_count_kernel (a 131072-position window: 16 positions per thread)

// Row b of a job: logits row row[b] (leading dimension ld), sequence seq[b] with parameters params[slot[b]], emitting the
// token at position p_next[b] (< 0: *pos_ptr, the position a decode run's step has just advanced to); on[b] == 0: copied.
struct PenaltyJob {
  const float* logits;
  long long ld;
  int V;
  int n;
  const lnb_penalties* params;
  const int32_t* hist;     // [..][hist_len]: row b counts hist[seq[b] * hist_len + p]
  int hist_len;
  unsigned int* cnt;       // [n][V] counts (zero between launches)
  float* out;              // [n][V] l'
  const int32_t* pos_ptr;
  int32_t row[PEN_MAX_ROWS], slot[PEN_MAX_ROWS], seq[PEN_MAX_ROWS], p_next[PEN_MAX_ROWS], on[PEN_MAX_ROWS];
};

__global__ void penalty_set_params_kernel(lnb_penalties* slot, lnb_penalties p) {
  pdl_launch_dependents();
  pdl_wait();
  *slot = p;
}

// The history write of one forward: row r's token (tokens[r], else `token` if >= 0, else st->next_token) at its position
// (pos_arr[r], else (pos0 >= 0 ? pos0 : st->pos) + r) of its sequence (row_seq[r], else `seq`).
__global__ void penalty_record_kernel(int32_t* __restrict__ hist, int hist_len, const LnbDevState* st, const int32_t* tokens,
                                      const int32_t* pos_arr, const int32_t* row_seq, int seq, int token, int pos0, int S) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= S) return;
  const int32_t t = tokens ? tokens[r] : (token >= 0 ? token : st->next_token);
  const int32_t p = pos_arr ? pos_arr[r] : (pos0 >= 0 ? pos0 : st->pos) + r;
  const int32_t q = row_seq ? row_seq[r] : seq;
  if (p >= 0 && p < hist_len) hist[(size_t)q * hist_len + p] = t;
}

LNB_DEVINL int pen_p_next(const PenaltyJob& J, int b) { return J.p_next[b] >= 0 ? J.p_next[b] : *J.pos_ptr; }

__global__ void __launch_bounds__(PEN_THREADS) penalty_count_kernel(const PenaltyJob J) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  if (!J.on[b]) return;
  const lnb_penalties* prm = J.params + J.slot[b];
  const int pn = min(pen_p_next(J, b), J.hist_len);
  const int lo = max(0, lnb_pen_lo(prm, pn));
  const int32_t* __restrict__ h = J.hist + (size_t)J.seq[b] * J.hist_len;
  unsigned int* __restrict__ cnt = J.cnt + (size_t)b * J.V;
  const int lane = threadIdx.x & 31;
  const int stride = gridDim.x * PEN_THREADS;
  // the base is warp-uniform, so every lane of a warp takes part in each match
  for (int base = lo + blockIdx.x * PEN_THREADS + (threadIdx.x & ~31); base < pn; base += stride) {
    const int i = base + lane;
    int32_t t = i < pn ? h[i] : -1;
    if (t >= J.V) t = -1;
    const unsigned peers = __match_any_sync(0xffffffffu, t);
    if (t >= 0 && lane == __ffs(peers) - 1) atomicAdd(&cnt[t], (unsigned)__popc(peers));
  }
}

__global__ void __launch_bounds__(PEN_THREADS) penalty_apply_kernel(const PenaltyJob J) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y, V = J.V;
  const int lo = blockIdx.x * PEN_SLICE, hi = min(V, lo + PEN_SLICE);
  const float* __restrict__ l = J.logits + (size_t)J.row[b] * J.ld;
  float* __restrict__ out = J.out + (size_t)b * V;
  if (!J.on[b]) {
    for (int i = lo + threadIdx.x; i < hi; i += PEN_THREADS) out[i] = l[i];
    return;
  }
  const lnb_penalties* prm = J.params + J.slot[b];
  const float rp = prm->repetition_penalty, fp = prm->frequency_penalty, pp = prm->presence_penalty;
  unsigned int* __restrict__ cnt = J.cnt + (size_t)b * V;
  for (int i = lo + threadIdx.x; i < hi; i += PEN_THREADS) {
    const unsigned c = cnt[i];
    if (c) cnt[i] = 0u;
    out[i] = lnb_pen_apply(l[i], c, rp, fp, pp);
  }
  const int nb = prm->n_bias;
  if (nb == 0) return;
  __syncthreads();   // this CTA's l' of the slice are visible to all its threads
  if (threadIdx.x < nb) {
    const int t = prm->bias_token[threadIdx.x];
    if (t >= lo && t < hi) out[t] = lnb_pen_bias(out[t], prm->bias[threadIdx.x]);
  }
}

}  // namespace lnb
