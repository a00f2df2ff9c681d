// grammar.cuh -- regex-constrained generation: token masks per DFA state, the state history of each sequence, and the
// mask applied to a logits row before the sampler (DESIGN.md §9g).
//
// A grammar is a byte-level DFA (csrc/regex.cpp: Q states, trans [Q][256], -1 = ⊥) with the bytes of every token and a
// stop set Z.  Its masks [Q + 1][W] (W = ⌈V/32⌉ words) are built once by grammar_mask_kernel; row Q is Z, the mask of ⊥.
// A session keeps, per sequence, g[seq][p] for p in [0, seq_len]: the grammar state before the token at position p.
// Three PDL launches, each starting with griddepcontrol.wait:
//  - grammar_mask_kernel, grid (⌈Q/GRM_BUILD_STATES⌉): every thread takes one token at a time, walks its bytes from each of
//    the CTA's states, and a warp's 32 consecutive tokens give one mask word per state by __ballot_sync.  A state whose
//    mask is empty (no token continues it and it does not accept) gets Z.
//  - grammar_record_kernel, one thread per row: the first row of each run of one sequence's rows walks the run in position
//    order, writing g[p + 1] from g[p] and the row's token.  Serial per sequence, since each state depends on the one before.
//  - grammar_apply_kernel, grid (⌈V/GRM_SLICE⌉, rows): l'_t = l_t where mask(g[p_next]) has t, else -inf.
#pragma once
#include "../../include/lnb.h"
#include "common.cuh"

namespace lnb {

#define GRM_MAX_STATES 4096
#define GRM_MAX_ROWS 8
#define GRM_THREADS 256
#define GRM_SLICE 4096          // logits per CTA of grammar_apply_kernel
#define GRM_BUILD_THREADS 512
#define GRM_BUILD_STATES 4      // states per CTA of grammar_mask_kernel

// a grammar's device tables
struct GrammarDev {
  const int32_t* trans;     // [Q][256], -1: ⊥
  const uint32_t* masks;    // [Q + 1][W]; row Q: Z
  const uint8_t* bytes;     // token t's bytes: bytes[off[t] .. off[t + 1])
  const int64_t* off;       // [V + 1]
  int Q, W, V;
};
// a sequence's grammar (trans NULL: none) and the position of its start state
struct GrammarSlot {
  GrammarDev g;
  int32_t first_pos;
};

LNB_DEVINL bool grm_bit(const uint32_t* row, int t) { return (row[t >> 5] >> (t & 31)) & 1u; }

// δ*(q, b(t)) when t is an allowed text token in q, else ⊥ (-1).  A state outside [0, Q) is ⊥ (it cannot arise from the
// history rules; the check keeps every table read inside this grammar's tables whatever the history holds).
LNB_DEVINL int grammar_step(const GrammarDev& G, int q, int t) {
  if (q < 0 || q >= G.Q || t < 0 || t >= G.V || grm_bit(G.masks + (size_t)G.Q * G.W, t)) return -1;
  const int64_t b0 = G.off[t], b1 = G.off[t + 1];
  if (b1 == b0) return -1;
  for (int64_t i = b0; i < b1 && q >= 0; i++) q = G.trans[(size_t)q * 256 + G.bytes[i]];
  return q;
}

// masks rows [0, Q) of G (row Q, Z, is uploaded first); n_stuck counts the states whose mask is Z
__global__ void __launch_bounds__(GRM_BUILD_THREADS) grammar_mask_kernel(GrammarDev G, const uint8_t* __restrict__ accept,
                                                                           uint32_t* __restrict__ masks, unsigned int* n_stuck) {
  pdl_launch_dependents();
  pdl_wait();
  const int q0 = blockIdx.x * GRM_BUILD_STATES, nq = min(GRM_BUILD_STATES, G.Q - q0);
  const uint32_t* __restrict__ Z = masks + (size_t)G.Q * G.W;
  const int lane = threadIdx.x & 31;
  bool any[GRM_BUILD_STATES];
#pragma unroll
  for (int k = 0; k < GRM_BUILD_STATES; k++) any[k] = false;
  // every thread runs the same number of iterations, so each ballot has the full warp
  for (int base = 0; base < G.V; base += GRM_BUILD_THREADS) {
    const int t = base + threadIdx.x, word = t >> 5;
    const bool have = t < G.V, word_ok = base + (int)(threadIdx.x & ~31u) < G.V;
    const bool stop = have && grm_bit(Z, t);
    const int64_t b0 = have ? G.off[t] : 0, b1 = have ? G.off[t + 1] : 0;
#pragma unroll
    for (int k = 0; k < GRM_BUILD_STATES; k++) {
      bool ok = false;
      if (have && k < nq) {
        if (stop) {
          ok = accept[q0 + k] != 0;
        } else if (b1 > b0) {
          int q = q0 + k;
          for (int64_t i = b0; i < b1 && q >= 0; i++) q = G.trans[(size_t)q * 256 + G.bytes[i]];
          ok = q >= 0;
        }
      }
      const unsigned w = __ballot_sync(0xffffffffu, ok);
      if (k < nq && lane == 0 && word_ok) masks[(size_t)(q0 + k) * G.W + word] = w;
      any[k] |= ok;
    }
  }
#pragma unroll
  for (int k = 0; k < GRM_BUILD_STATES; k++) {
    // (also the barrier that orders this CTA's mask words before the rewrite below)
    if (__syncthreads_or(any[k]) || k >= nq) continue;
    for (int w = threadIdx.x; w < G.W; w += GRM_BUILD_THREADS) masks[(size_t)(q0 + k) * G.W + w] = Z[w];
    if (threadIdx.x == 0) atomicAdd(n_stuck, 1u);
  }
}

__global__ void grammar_set_slot_kernel(GrammarSlot* slot, GrammarSlot v, int32_t* gst_first) {
  pdl_launch_dependents();
  pdl_wait();
  *slot = v;
  if (gst_first) *gst_first = 0;   // g[first_pos] = q0
}

// The state history write of one forward (rows as penalty_record_kernel reads them): row r holds token tokens[r] (else
// `token` if >= 0, else st->next_token) at position pos_arr[r] (else (pos0 >= 0 ? pos0 : st->pos) + r) of sequence
// row_seq[r] (else `seq`).  Rows of one sequence are consecutive positions, in order.
__global__ void grammar_record_kernel(int32_t* gst, int gst_len, const GrammarSlot* __restrict__ slots, const LnbDevState* st,
                                      const int32_t* tokens, const int32_t* pos_arr, const int32_t* row_seq, int seq, int token,
                                      int pos0, int S) {
  pdl_launch_dependents();
  pdl_wait();
  const int r0 = blockIdx.x * blockDim.x + threadIdx.x;
  if (r0 >= S) return;
  auto seq_of = [&](int r) { return row_seq ? row_seq[r] : seq; };
  const int q = seq_of(r0);
  if (r0 > 0 && seq_of(r0 - 1) == q) return;   // not the first row of its sequence's run
  const GrammarSlot& sl = slots[q];
  if (!sl.g.trans) return;
  int32_t* g = gst + (size_t)q * gst_len;
  for (int r = r0; r < S && seq_of(r) == q; r++) {
    const int t = tokens ? tokens[r] : (token >= 0 ? token : st->next_token);
    const int p = pos_arr ? pos_arr[r] : (pos0 >= 0 ? pos0 : st->pos) + r;
    if (p < sl.first_pos || p + 1 >= gst_len) continue;
    g[p + 1] = grammar_step(sl.g, g[p], t);
  }
}

// Row b of a job: logits row row[b] of `in` (leading dimension ld) of sequence seq[b], emitting the token at position
// p_next[b] (< 0: *pos_ptr, the position a decode run's step has just advanced to), to row b of `out` ([n][V]).  on[b] == 0,
// or p_next below the sequence's first_pos: copied (nothing to do when in == out).
struct GrammarJob {
  const float* in;
  long long ld;
  float* out;
  int V;
  int n;
  const GrammarSlot* slots;
  const int32_t* gst;       // [n_seq][gst_len]
  int gst_len;
  const int32_t* pos_ptr;
  int32_t row[GRM_MAX_ROWS], seq[GRM_MAX_ROWS], p_next[GRM_MAX_ROWS], on[GRM_MAX_ROWS];
};

__global__ void __launch_bounds__(GRM_THREADS) grammar_apply_kernel(const GrammarJob J) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y, V = J.V;
  const int lo = blockIdx.x * GRM_SLICE, hi = min(V, lo + GRM_SLICE);
  const float* l = J.in + (size_t)J.row[b] * J.ld;
  float* out = J.out + (size_t)b * V;
  const uint32_t* mrow = nullptr;
  if (J.on[b]) {
    const GrammarSlot& sl = J.slots[J.seq[b]];
    const int pn = J.p_next[b] >= 0 ? J.p_next[b] : *J.pos_ptr;
    if (sl.g.trans && pn >= sl.first_pos && pn < J.gst_len) {
      const int q = J.gst[(size_t)J.seq[b] * J.gst_len + pn];
      mrow = sl.g.masks + (size_t)((q < 0 || q >= sl.g.Q) ? sl.g.Q : q) * sl.g.W;   // (outside [0, Q): ⊥)
    }
  }
  if (!mrow) {
    if (l != out)
      for (int i = lo + threadIdx.x; i < hi; i += GRM_THREADS) out[i] = l[i];
    return;
  }
  for (int i = lo + threadIdx.x; i < hi; i += GRM_THREADS) {
    const bool keep = grm_bit(mrow, i);
    if (l != out) out[i] = keep ? l[i] : -INFINITY;
    else if (!keep) out[i] = -INFINITY;
  }
}

}  // namespace lnb
