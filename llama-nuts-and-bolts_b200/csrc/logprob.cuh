// logprob.cuh -- token log-probabilities of logits rows (DESIGN.md §9d).
//
// For one row l and a target t the device computes integers only, so any reduction order gives the bits of the sequential
// statement (oracle_sampling/lnb_sample_ref.c, orc_logprob_row): the rank-0 key (rank order = lnb_logprob_key descending,
// the sampler's and greedy's order), the number of keys above the target's, the top N keys, and the sampler's weight sum at
// temperature 1.  The host turns a record into logprobs with lnb_logprob_finish (sample_det.h).  Two launches over a grid
// of (4096-logit slices, rows), as sample_split_kernel:
//  - logprob_rank_kernel: each CTA finds its slice's top max(N, 1) keys and its keys above the target's; the last CTA of the
//    row merges them (the row's top N are among the slices' top N) and writes the record with sum = 0;
//  - logprob_mass_kernel: once the rank-0 logit m is known, each CTA adds its slice's weights to the record's sum (u64
//    atomics: integer, so order-free).
#pragma once
#include "../../include/lnb.h"
#include "common.cuh"
#include "sample_det.h"

namespace lnb {

#define LP_THREADS 512
#define LP_SLICE 4096                    // logits per CTA
#define LP_PER (LP_SLICE / LP_THREADS)   // keys per thread
#define LP_TOP LNB_LOGPROBS_TOP_MAX
#define LP_MAX_VOCAB (LP_SLICE * (LP_SLICE / LP_TOP))   // the merge holds every slice's top 20 in one CTA's registers

// The device record of one position; the host finishes it into an lnb_logprob.
struct LpRecord {
  unsigned long long sum;           // the row's weights at temperature 1 (lnb_sample_weight(l_i, m, 1))
  unsigned long long key[LP_TOP];   // the row's top max(N, 1) keys in rank order (key[0]: the rank-0 key, which gives m)
  float target_logit;
  int32_t target;                   // -1: never written
  int32_t rank;
  int32_t n_top;                    // min(N, V)
  unsigned long long pad;
};
static_assert(sizeof(LpRecord) == 192, "LpRecord is 192 bytes");

// One row of a job, in device memory (a job may have thousands of rows; a captured graph reads the table when it replays):
// logits row, target token (often computed earlier in the same call), record rec + (rec_pos ? *rec_pos : 0), and the
// sequence whose top_n the row uses.
struct LpRow {
  const float* logits;
  const int32_t* target;
  LpRecord* rec;
  const int32_t* rec_pos;
  int32_t seq;
  int32_t pad;
};

struct LogprobJob {
  const LpRow* rows;
  const int32_t* top_n;       // [seq] N of each sequence
  int V;
  unsigned long long* cand;   // [n][slices][LP_TOP] top keys of each slice
  unsigned int* above;        // [n][slices] keys above the target's, per slice
  unsigned int* done;         // [n] CTAs of a row that finished (zero between launches)
};

__global__ void logprob_set_top_n_kernel(int32_t* slot, int top_n) {
  pdl_launch_dependents();
  pdl_wait();
  *slot = top_n;
}

LNB_DEVINL unsigned long long lp_warp_max(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// The K (1..20) largest of the CTA's keys (LP_PER per thread, 0 = no key) in descending order, stored by warp 0 to
// out[0, K).  Keys are distinct (the index is part of the key), so "the largest below the previous one" walks them.  The
// first round takes any key: ~0 is a real key (logit bits 0x7FFFFFFF, the NaN the device's arithmetic makes, at index 0).
LNB_DEVINL void lp_block_topk(const unsigned long long (&k)[LP_PER], int K, unsigned long long (*wtop)[LP_TOP], unsigned long long* out) {
  constexpr int NW = LP_THREADS / 32, NC = (NW * LP_TOP + 31) / 32;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long prev = 0;
  for (int r = 0; r < K; r++) {   // each warp's top K
    unsigned long long v = 0;
#pragma unroll
    for (int j = 0; j < LP_PER; j++) v = ((r == 0 || k[j] < prev) && k[j] > v) ? k[j] : v;
    v = lp_warp_max(v);
    if (lane == 0) wtop[w][r] = v;
    prev = v;
  }
  __syncthreads();
  if (w != 0) return;
  unsigned long long c[NC];   // warp 0 merges the NW * K warp candidates
#pragma unroll
  for (int j = 0; j < NC; j++) {
    const int f = lane + 32 * j;
    c[j] = f < NW * K ? wtop[f / K][f % K] : 0ull;
  }
  prev = 0;
  for (int r = 0; r < K; r++) {
    unsigned long long v = 0;
#pragma unroll
    for (int j = 0; j < NC; j++) v = ((r == 0 || c[j] < prev) && c[j] > v) ? c[j] : v;
    v = lp_warp_max(v);
    if (lane == 0) out[r] = v;
    prev = v;
  }
}

// grid (ceil(V / 4096), n): CTA g of row b holds logits [g * 4096, (g + 1) * 4096)
__global__ void __launch_bounds__(LP_THREADS) logprob_rank_kernel(const LogprobJob J) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned long long wtop[LP_THREADS / 32][LP_TOP];
  __shared__ unsigned long long top[LP_TOP];
  __shared__ unsigned int above;
  __shared__ int last;
  const int b = blockIdx.y, g = blockIdx.x, G = gridDim.x, V = J.V;
  const int top_n = J.top_n[J.rows[b].seq];
  const int K = top_n > 1 ? top_n : 1;
  const float* __restrict__ l = J.rows[b].logits;
  const int t = *J.rows[b].target;
  const float lt = l[t];
  const unsigned long long kt = lnb_logprob_key(lt, t);
  if (threadIdx.x == 0) above = 0;
  unsigned long long k[LP_PER];
  unsigned int c = 0;
#pragma unroll
  for (int j = 0; j < LP_PER; j++) {
    const int i = g * LP_SLICE + j * LP_THREADS + threadIdx.x;
    k[j] = i < V ? lnb_logprob_key(l[i], i) : 0ull;
    c += k[j] > kt ? 1u : 0u;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  __syncthreads();
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&above, c);
  unsigned long long* cand = J.cand + (size_t)b * G * LP_TOP;
  lp_block_topk(k, K, wtop, cand + (size_t)g * LP_TOP);
  __syncthreads();
  if (threadIdx.x == 0) J.above[(size_t)b * G + g] = above;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = (atomicAdd(&J.done[b], 1u) == (unsigned)(G - 1));
  __syncthreads();
  if (!last) return;
  // the last CTA of the row: merge the slices' top K and their counts
  __threadfence();
#pragma unroll
  for (int j = 0; j < LP_PER; j++) {
    const int f = j * LP_THREADS + threadIdx.x;
    k[j] = f < G * K ? __ldcg(&cand[(size_t)(f / K) * LP_TOP + f % K]) : 0ull;
  }
  unsigned int a = 0;
  for (int s = threadIdx.x; s < G; s += LP_THREADS) a += __ldcg(&J.above[(size_t)b * G + s]);
  a = __reduce_add_sync(0xffffffffu, a);
  if (threadIdx.x == 0) { above = 0; J.done[b] = 0; }   // the counter is ready for the next launch (a graph replays this one)
  __syncthreads();
  if ((threadIdx.x & 31) == 0 && a) atomicAdd(&above, a);
  lp_block_topk(k, K, wtop, top);
  __syncthreads();
  const LpRow& R = J.rows[b];   // (read here, not kept live across the merge)
  LpRecord* rec = R.rec + (R.rec_pos ? *R.rec_pos : 0);
  if (threadIdx.x < LP_TOP) rec->key[threadIdx.x] = threadIdx.x < K ? top[threadIdx.x] : 0ull;
  if (threadIdx.x == 0) {
    rec->sum = 0;
    rec->target_logit = lt;
    rec->target = t;
    rec->rank = 1 + (int)above;
    rec->n_top = top_n < 0 ? 0 : (top_n < V ? top_n : V);
  }
}

// grid (ceil(V / 4096), n), after logprob_rank_kernel: the weights of CTA g's slice, added to the record's sum
__global__ void __launch_bounds__(LP_THREADS) logprob_mass_kernel(const LogprobJob J) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y, g = blockIdx.x, V = J.V;
  const LpRow R = J.rows[b];
  LpRecord* rec = R.rec + (R.rec_pos ? *R.rec_pos : 0);
  const float m = lnb_logprob_key_logit(rec->key[0]);
  const float* __restrict__ l = R.logits;
  unsigned long long s = 0;
#pragma unroll
  for (int j = 0; j < LP_PER; j++) {
    const int i = g * LP_SLICE + j * LP_THREADS + threadIdx.x;
    if (i < V) s += lnb_sample_weight(l[i], m, 1.0f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(&rec->sum, s);
}

}  // namespace lnb
