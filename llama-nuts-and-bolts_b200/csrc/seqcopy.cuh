// seqcopy.cuh -- lnb_session_copy_sequences: fork and permute sequences' per-position state in place (DESIGN.md §9f).
//
// One launch copies, for positions [pos0, pos1) and every pair i < n, what sequence src[i] held there BEFORE the launch
// to sequence dst[i]: K and V of every layer, the penalty history and the logprob records (when allocated).  For one
// buffer, sequence q's rows [pos0, pos1) are one contiguous segment (caches [n_seq][seq_len][kv_l], history
// [n_seq][seq_len], records [n_seq][seq_len + 1]), at the same offset in every sequence.  The grid walks tiles of
// SC_TILE elements of that segment (16-byte vectors for caches and records, 4-byte words for the history); a thread owns
// element e of the tile for EVERY sequence at once.
//
// In-place invariant: element e of sequence q is read (when q is a source) and written (when q is a destination) by the
// one thread that owns e, and that thread loads all its sources into registers before it stores any destination.  No
// other thread touches e of any sequence, so swaps, cycles and one source fanned out to many destinations read the
// snapshot without a barrier and without scratch memory.
#pragma once
#include "common.cuh"

namespace lnb {

#define SC_THREADS 256
#define SC_PER 2                             // elements per thread and sequence
#define SC_TILE (SC_THREADS * SC_PER)        // elements per CTA tile
#define SC_MAX_PAIRS 8
#define SC_MAX_LAYERS 128

struct SeqCopyJob {
  int n;                                     // pairs
  int src[SC_MAX_PAIRS], dst[SC_MAX_PAIRS];  // a pair with src == dst moves nothing
  int n_kv;                                  // cache buffers: K of every layer, then V of every layer
  long long kv_stride, kv_len;               // in 16-byte vectors: one sequence's cache, the copied segment
  long long rec_stride, rec_len;             // records, 16-byte vectors (rec NULL: none)
  long long hist_stride, hist_len;           // history, 4-byte words (hist NULL: none)
  long long kv_tiles, rec_tiles;             // tiles of one cache buffer / of the records
  uint4* kv[2 * SC_MAX_LAYERS];              // each at its pos0 offset
  uint4* rec;
  int32_t* hist;
};

// one tile of one buffer: base points at sequence 0's pos0, stride elements between sequences, len elements in the segment
template <typename T>
LNB_DEVINL void sc_tile(const SeqCopyJob& J, T* base, long long stride, long long len, long long tile) {
  T v[SC_MAX_PAIRS][SC_PER];
  const long long e0 = tile * SC_TILE + threadIdx.x;
#pragma unroll
  for (int i = 0; i < SC_MAX_PAIRS; i++) {
    if (i >= J.n || J.src[i] == J.dst[i]) continue;
    const T* s = base + (long long)J.src[i] * stride;
#pragma unroll
    for (int k = 0; k < SC_PER; k++) {
      const long long e = e0 + k * SC_THREADS;
      if (e < len) v[i][k] = s[e];
    }
  }
  // every source element this thread will overwrite is in v[] now (the invariant above)
#pragma unroll
  for (int i = 0; i < SC_MAX_PAIRS; i++) {
    if (i >= J.n || J.src[i] == J.dst[i]) continue;
    T* d = base + (long long)J.dst[i] * stride;
#pragma unroll
    for (int k = 0; k < SC_PER; k++) {
      const long long e = e0 + k * SC_THREADS;
      if (e < len) d[e] = v[i][k];
    }
  }
}

// grid: n_kv * kv_tiles cache tiles, then rec_tiles record tiles, then the history tiles
__global__ void __launch_bounds__(SC_THREADS) seqcopy_kernel(const SeqCopyJob J) {
  pdl_wait();   // the caches may still be written by the forward before this launch
  pdl_launch_dependents();
  long long b = blockIdx.x;
  const long long n_kv_tiles = (long long)J.n_kv * J.kv_tiles;
  if (b < n_kv_tiles) {
    sc_tile<uint4>(J, J.kv[b / J.kv_tiles], J.kv_stride, J.kv_len, b % J.kv_tiles);
    return;
  }
  b -= n_kv_tiles;
  if (b < J.rec_tiles) {
    sc_tile<uint4>(J, J.rec, J.rec_stride, J.rec_len, b);
    return;
  }
  b -= J.rec_tiles;
  sc_tile<int32_t>(J, J.hist, J.hist_stride, J.hist_len, b);
}

}  // namespace lnb
