// kvcache.cuh -- the MXFP8 KV cache (DESIGN.md §9j): the writer that rotates, quantizes and stores a call's K and V rows,
// and the exact decode the streamed attention kernels (sdpa_stream.cuh) apply to every key they read.
//
// Rule: §9h's block rule (mxfp8.cuh: mx_block_x, mx_inv_scale, e4m3x2) on blocks of 32 consecutive elements of one KV
// head's row (the last block of a head is head_dim % 32 wide when that is nonzero).  amax is taken over the block's
// FINITE elements; a NaN element stores the NaN code and decodes to NaN, a +-inf element saturates to +-448 * 2^X.
// Every finite decoded value e4m3(code) * 2^X is a bf16 value, so attention over the decoded rows computes what the bf16
// kernels compute over those rows.
//
// Layout: a layer's K (and V) cache is [n_seq][seq_len] records of kv_row_bytes(kv_l, n_kv) bytes: the kv_l codes of the
// position in checkpoint head order, then one 4-byte scale slot per KV head (blocks 0..nb-1 of the head, E8M0 bytes
// X + 127; head_dim <= 128 so nb <= 4; unused bytes 0), padded to 16 bytes.  So a record is a whole number of 16-byte
// vectors (seqcopy_kernel moves it unchanged), a head's scales are one aligned 4-byte copy, and its codes are 8-byte
// aligned (head_dim % 8 == 0): the attention kernels copy codes in 8-byte pieces.  An unwritten record is zero, which
// decodes to 0.
#pragma once
#include "gemm_tc.cuh"
#include "mxfp8.cuh"

namespace lnb {

enum { KVF_BF16 = 0, KVF_MXFP8 = 1 };   // = LNB_KV_*

LNB_HDINL int kv_scale_bytes(int n_kv) { return (4 * n_kv + 15) & ~15; }
LNB_HDINL int kv_row_bytes(int kv_l, int n_kv) { return kv_l + kv_scale_bytes(n_kv); }

// the bf16 bits of e4m3(code) * 2^X for the E8M0 byte e8m0 = X + 127; the NaN codes (0x7f, 0xff) decode to NaN
LNB_DEVINL uint32_t kv_dec1(uint32_t code, float scale) {
  if ((code & 0x7fu) == 0x7fu) return 0x7fc0u | ((code & 0x80u) << 8);
  return f2bf(mx_dequant(code << 24, scale));
}
// 8 codes (byte e = element e) of one block with scale mx_scale(e8m0) -> 8 bf16, element 0 in the low half of .x
LNB_DEVINL uint4 kv_decode8(uint2 c, float scale) {
  uint4 o;
  o.x = kv_dec1(c.x & 0xffu, scale) | (kv_dec1((c.x >> 8) & 0xffu, scale) << 16);
  o.y = kv_dec1((c.x >> 16) & 0xffu, scale) | (kv_dec1(c.x >> 24, scale) << 16);
  o.z = kv_dec1(c.y & 0xffu, scale) | (kv_dec1((c.y >> 8) & 0xffu, scale) << 16);
  o.w = kv_dec1((c.y >> 16) & 0xffu, scale) | (kv_dec1(c.y >> 24, scale) << 16);
  return o;
}

// One block, by one warp: lane j holds element j of the block (valid: j < the block's width) as bf16 bits v.  Writes
// the lane's code to code[j] and the block's E8M0 byte to *scale; returns the E8M0 byte.
LNB_DEVINL uint32_t kvq_block(uint32_t v, bool valid, uint8_t* code, uint8_t* scale, int lane) {
  const uint32_t mag = v & 0x7fffu;
  uint32_t amax = valid && mag < 0x7f80u ? mag : 0u;   // finite elements only
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = max(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const int X = mx_block_x(amax);
  const uint32_t c = e4m3x2(0.f, __fmul_rn(bf2f((uint16_t)v), mx_inv_scale(X))) & 0xffu;
  if (valid) code[lane] = (uint8_t)c;
  if (lane == 0) *scale = (uint8_t)(X + 127);
  return (uint32_t)(X + 127);
}

// The cache writer of a quantized session, after the wq|wk|wv projection wrote its bf16 rows to qkv ([S][ld], columns
// q | k | v): q rotated -> q_out [S][q_dim] (rope_kv_kernel's arithmetic), k rotated and v quantized into the record of
// (row_seq[s], row_pos[s]) or (the cache at `cache`, pos0 + s); a speculative tree row rotates at its position and stores
// at its slot (row_tree, common.cuh).  Threads of the first loop own q pairs; warps of the
// second own (row, K or V, KV head, block).  Waits for the projection before any global access (PDL).
__global__ void kvq_rope_store_kernel(const uint16_t* __restrict__ qkv, int ld, uint16_t* __restrict__ q_out, int q_dim, int kv_dim,
                                      int head_dim, uint8_t* __restrict__ cache_k, uint8_t* __restrict__ cache_v,
                                      const float* __restrict__ cis, const int32_t* __restrict__ pos_ptr, int S,
                                      const int32_t* __restrict__ row_pos, const int32_t* __restrict__ row_seq, long long seq_stride,
                                      const int32_t* __restrict__ row_tree) {
  pdl_launch_dependents();
  pdl_wait();
  const int pos0 = row_pos ? 0 : *pos_ptr;
  const int64_t nthr = (int64_t)gridDim.x * blockDim.x, gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int qpairs = q_dim / 2;
  for (int64_t i = gtid; i < (int64_t)S * qpairs; i += nthr) {
    const int s = (int)(i / qpairs), n = (int)(i % qpairs) * 2;
    const int pos = row_pos ? row_pos[s] : pos0 + s;
    const float2 fc = *reinterpret_cast<const float2*>(cis + ((size_t)pos * (head_dim / 2) + (n % head_dim) / 2) * 2);
    *reinterpret_cast<uint32_t*>(q_out + (size_t)s * q_dim + n) = rope_pair(*reinterpret_cast<const uint32_t*>(qkv + (size_t)s * ld + n), fc);
  }
  const int n_kv = kv_dim / head_dim, nb = (head_dim + 31) / 32, rowb = kv_row_bytes(kv_dim, n_kv), lane = threadIdx.x & 31;
  const int64_t tasks = (int64_t)S * 2 * n_kv * nb;
  for (int64_t w = gtid >> 5; w < tasks; w += nthr >> 5) {   // warp-uniform
    const int b = (int)(w % nb), h = (int)((w / nb) % n_kv), which = (int)((w / ((int64_t)nb * n_kv)) & 1);
    const int s = (int)(w / ((int64_t)nb * n_kv * 2));
    const int pos = row_pos ? row_pos[s] : pos0 + s;
    const int j = b * 32 + lane, col = h * head_dim + j;
    const bool valid = j < head_dim;
    uint32_t v = valid ? qkv[(size_t)s * ld + q_dim + which * kv_dim + col] : 0u;
    if (which == 0) {   // RoPE pairs (2i, 2i+1) are lanes (2i, 2i+1) of the block
      const uint32_t other = __shfl_xor_sync(0xffffffffu, v, 1);
      if (valid) {
        const uint32_t pair = (lane & 1) ? other | (v << 16) : v | (other << 16);
        const float2 fc = *reinterpret_cast<const float2*>(cis + ((size_t)pos * (head_dim / 2) + j / 2) * 2);
        const uint32_t o = rope_pair(pair, fc);
        v = (lane & 1) ? o >> 16 : o & 0xffffu;
      }
    }
    const int slot = row_tree ? tree_slot(row_tree[s]) : pos;
    uint8_t* rec = (which ? cache_v : cache_k) + (row_seq ? (size_t)row_seq[s] * (size_t)seq_stride : 0) + (size_t)slot * rowb;
    kvq_block(v, valid, rec + h * head_dim + b * 32, rec + kv_dim + h * 4 + b, lane);
  }
}

// n records (rowb bytes apart) -> their decoded bf16 rows [n][kv_l] (lnb_session_read of an MXFP8 cache)
__global__ void kv_dequant_kernel(const uint8_t* __restrict__ rec, int rowb, int kv_l, int head_dim, int64_t n, uint16_t* __restrict__ out) {
  const int cpr = kv_l / 8;   // 8-column chunks never straddle a block (blocks start at multiples of 32 of a head)
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * cpr; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / cpr;
    const int col = (int)(i % cpr) * 8, h = col / head_dim;
    const uint8_t* r = rec + t * rowb;
    *reinterpret_cast<uint4*>(out + t * kv_l + col) =
        kv_decode8(*reinterpret_cast<const uint2*>(r + col), mx_scale(r[kv_l + h * 4 + ((col - h * head_dim) >> 5)]));
  }
}

// lnb_op_kv_quantize_bf16: rows [n][n_kv * head_dim] of bf16 -> codes [n][n_kv * head_dim], scales [n][n_kv][nb] and the
// decoded rows, through kvq_block and kv_dec1.  One warp per (row, KV head, block).
__global__ void kvq_rows_kernel(const uint16_t* __restrict__ rows, int n, int head_dim, int n_kv, uint8_t* __restrict__ codes,
                                uint8_t* __restrict__ scales, uint16_t* __restrict__ deq) {
  const int nb = (head_dim + 31) / 32, kv = n_kv * head_dim, lane = threadIdx.x & 31;
  const int64_t tasks = (int64_t)n * n_kv * nb, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < tasks; w += nw) {
    const int b = (int)(w % nb), h = (int)((w / nb) % n_kv), s = (int)(w / ((int64_t)nb * n_kv));
    const int j = b * 32 + lane;
    const bool valid = j < head_dim;
    const size_t e = (size_t)s * kv + h * head_dim + j;
    const uint32_t sc = kvq_block(valid ? rows[e] : 0u, valid, codes + (size_t)s * kv + h * head_dim + b * 32,
                                  scales + ((size_t)s * n_kv + h) * nb + b, lane);
    __syncwarp();
    if (valid) deq[e] = (uint16_t)kv_dec1(codes[e], mx_scale(sc));
  }
}

}  // namespace lnb
