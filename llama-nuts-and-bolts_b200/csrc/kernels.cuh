// kernels.cuh -- the non-GEMV kernels of the forward path plus generic-shape kernels that
// back the op-level C-ABI.  All of them call pdl_wait() first so that they can sit in a
// programmatic-dependent-launch chain.
#pragma once
#include "common.cuh"
#include "sample_det.h"

namespace lnb {

// ------------------------------------------------------------------------------------------
// Upload-time layout change: row-major W[rows x ld] (a [row0.., col0..] window of it) ->
// panel-major (8-row panels, see gemv.cuh).  dpanel_stride == 1: source row i lands in destination row
// dpanel0 * 8 + i (wq | wk | wv stacked).  dpanel_stride == 2: the w1 | w3 half-panel interleave of the fused
// SwiGLU -- panel p holds the GATE rows of hidden units 4p..4p+3 (w1, dpanel0 == 0) in its rows 0..3 and their UP
// rows (w3, dpanel0 != 0) in rows 4..7, so that gate and up of one unit always meet inside one warp (lane, lane + 4)
// whatever panel range a CTA owns (the persistent engine splits rows at single-panel granularity).
// One thread moves one 16-byte chunk (8 bf16).
LNB_DEVINL int64_t panel_dest_row(int64_t row, int dpanel0, int dpanel_stride) {
  if (dpanel_stride == 2) return (row >> 2) * 8 + (dpanel0 ? 4 : 0) + (row & 3);
  return (int64_t)dpanel0 * 8 + row;
}
__global__ void retile_kernel(const uint16_t* __restrict__ src, int64_t ld, int64_t row0, int64_t col0, int rows,
                              int K, uint16_t* __restrict__ dst, int dpanel0, int dpanel_stride) {
  const int64_t chunks_per_row = K / 8;
  const int64_t total = (int64_t)rows * chunks_per_row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / chunks_per_row, ch = i % chunks_per_row;
    const uint4 v = *reinterpret_cast<const uint4*>(src + (row0 + row) * ld + col0 + ch * 8);
    const int64_t d = panel_dest_row(row, dpanel0, dpanel_stride);
    const int64_t dp = d / 8, rr = d % 8;
    *reinterpret_cast<uint4*>(dst + ((dp * chunks_per_row + ch) * 8 + rr) * 8) = v;
  }
}

// inverse (debug / tests): panel-major -> row-major
__global__ void untile_kernel(const uint16_t* __restrict__ src, int rows, int K, uint16_t* __restrict__ dst,
                              int spanel0, int spanel_stride) {
  const int64_t chunks_per_row = K / 8;
  const int64_t total = (int64_t)rows * chunks_per_row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / chunks_per_row, ch = i % chunks_per_row;
    const int64_t d = panel_dest_row(row, spanel0, spanel_stride);
    const int64_t sp = d / 8, rr = d % 8;
    *reinterpret_cast<uint4*>(dst + row * K + ch * 8) =
        *reinterpret_cast<const uint4*>(src + ((sp * chunks_per_row + ch) * 8 + rr) * 8);
  }
}

// ------------------------------------------------------------------------------------------
// Synthetic checkpoint generator (DESIGN.md "Synthetic weights"): element i of the FULL
// row-major tensor `name` is t((2u-1)*scale + offset), u = top 24 bits of
// splitmix64(seed ^ fnv1a(name), i).  Writes either row-major (panel_major=0) or panel-major.
LNB_DEVINL uint64_t splitmix64_at(uint64_t seed, uint64_t i) { return lnb_splitmix64_at(seed, i); }
LNB_DEVINL uint16_t synth_value(uint64_t seed, uint64_t i, float scale, float offset) {
  const uint64_t z = splitmix64_at(seed, i);
  const float u = __fmul_rn((float)(z >> 40), 1.0f / 16777216.0f);
  const float w = __fadd_rn(__fmul_rn(2.0f, u), -1.0f);
  const float v = __fadd_rn(__fmul_rn(w, scale), offset);
  return f2bf(v);
}
__global__ void synth_fill_kernel(uint64_t seed, float scale, float offset, int64_t ld, int64_t row0, int64_t col0,
                                  int rows, int K, uint16_t* __restrict__ dst, int panel_major, int dpanel0,
                                  int dpanel_stride) {
  const int64_t total = (int64_t)rows * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / K, col = i % K;
    const uint16_t v = synth_value(seed, (uint64_t)((row0 + row) * ld + col0 + col), scale, offset);
    if (panel_major) {
      const int64_t d = panel_dest_row(row, dpanel0, dpanel_stride);
      const int64_t dp = d / 8, rr = d % 8, ch = col / 8, e = col % 8;
      dst[((dp * (K / 8) + ch) * 8 + rr) * 8 + e] = v;
    } else {
      dst[i] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------
// ml.Fwd_Get_Rows (src/ml/operations_impl.go:142-173): x[s,:] = emb[tok[s],:].
// tok_src: tokens of this call, or NULL -> use st->next_token (device-driven decode, S == 1).
__global__ void gather_rows_kernel(const uint16_t* __restrict__ emb, const int32_t* __restrict__ tok_src,
                                   const LnbDevState* st, uint16_t* __restrict__ x, int dim) {
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x;
  const int32_t tok = tok_src ? tok_src[s] : st->next_token;
  const uint4* src = reinterpret_cast<const uint4*>(emb + (size_t)tok * dim);
  uint4* dst = reinterpret_cast<uint4*>(x + (size_t)s * dim);
  for (int i = threadIdx.x; i < dim / 8; i += blockDim.x) dst[i] = src[i];
}

// ------------------------------------------------------------------------------------------
// Attention core of LlamaAttention.Forward (src/model/llamatransformer.go:402-514) for one
// (query row, head) per CTA, reading K/V in place from the cache (attentionRepeatKV :529-559
// becomes kv_head = head / n_rep; the four Transposes :435-449 become index arithmetic).
//   sc_t = t( t(sum_seq_d q_d * k_td) / t(sqrt(hd)) )            MatMul :459, DivToScalar :464
//   (+ mask: entries t > s are -inf -> e = 0, p = 0: skipped; kept entries add 0)   :471
//   e_t = exp_f64(sc_t);  Z = sum_seq_t e_t (f64);  p_t = t(f32(e_t / Z))          Softmax :484-495
//   o_d = t( sum_seq_t p_t * v_td )                                                 MatMul :504
// All sums are in the reference's sequential order in both accumulation modes except Z,
// which LNB_ACC_FAST reduces as a tree in f64.
// grid = (n_heads, S); block = 128; dyn smem = T*(8+4) + hd*4 bytes.
__global__ void __launch_bounds__(128) sdpa_kernel(const uint16_t* __restrict__ q, int ldq,
                                                   const uint16_t* __restrict__ cache_k,
                                                   const uint16_t* __restrict__ cache_v, int kv_dim, int n_rep,
                                                   int hd, uint16_t* __restrict__ out, int ldo,
                                                   const int32_t* __restrict__ pos_ptr, int pos_fixed, int S,
                                                   int causal, int strict, float scale_bf16_as_f32, int out_x8) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t sm[];
  const int H = blockIdx.x, s = blockIdx.y;
  const int pos0 = pos_ptr ? *pos_ptr : pos_fixed;
  const int T = pos0 + S;
  const int Teff = causal ? min(T, pos0 + s + 1) : T;
  double* e = reinterpret_cast<double*>(sm);                  // [T]
  float* pf = reinterpret_cast<float*>(sm + (size_t)T * 8);   // [T]
  float* qs = pf + T;                                         // [hd]
  __shared__ double zsh[4];
  __shared__ double zfinal;
  const int h = H / n_rep;
  const int tid = threadIdx.x;

  for (int d = tid; d < hd; d += blockDim.x) qs[d] = bf2f(q[(size_t)s * ldq + (size_t)H * hd + d]);
  __syncthreads();

  for (int t = tid; t < Teff; t += blockDim.x) {
    const uint16_t* kr = cache_k + (size_t)t * kv_dim + (size_t)h * hd;
    float acc = 0.f;
    for (int d = 0; d < hd; d += 8) {
      const uint4 kv = *reinterpret_cast<const uint4*>(kr + d);
      acc = __fmaf_rn(qs[d + 0], bf_lo(kv.x), acc);
      acc = __fmaf_rn(qs[d + 1], bf_hi(kv.x), acc);
      acc = __fmaf_rn(qs[d + 2], bf_lo(kv.y), acc);
      acc = __fmaf_rn(qs[d + 3], bf_hi(kv.y), acc);
      acc = __fmaf_rn(qs[d + 4], bf_lo(kv.z), acc);
      acc = __fmaf_rn(qs[d + 5], bf_hi(kv.z), acc);
      acc = __fmaf_rn(qs[d + 6], bf_lo(kv.w), acc);
      acc = __fmaf_rn(qs[d + 7], bf_hi(kv.w), acc);
    }
    float sc = trunc_bf(acc);
    sc = trunc_bf(__fdiv_rn(sc, scale_bf16_as_f32));
    e[t] = exp((double)sc);
  }
  __syncthreads();

  if (strict) {
    if (tid == 0) {
      double z = 0.0;
      for (int t = 0; t < Teff; t++) z = __dadd_rn(z, e[t]);
      zfinal = z;
    }
  } else {
    double z = 0.0;
    for (int t = tid; t < Teff; t += blockDim.x) z = __dadd_rn(z, e[t]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z = __dadd_rn(z, __shfl_xor_sync(0xffffffffu, z, o));
    if ((tid & 31) == 0) zsh[tid >> 5] = z;
    __syncthreads();
    if (tid == 0) zfinal = __dadd_rn(__dadd_rn(__dadd_rn(zsh[0], zsh[1]), zsh[2]), zsh[3]);
  }
  __syncthreads();
  const double Z = zfinal;
  for (int t = tid; t < Teff; t += blockDim.x) pf[t] = trunc_bf((float)__ddiv_rn(e[t], Z));
  __syncthreads();

  for (int d = tid; d < hd; d += blockDim.x) {
    const uint16_t* vc = cache_v + (size_t)h * hd + d;
    float acc = 0.f;
    for (int t = 0; t < Teff; t++) acc = __fmaf_rn(pf[t], bf2f(vc[(size_t)t * kv_dim]), acc);
    const int col = H * hd + d;  // Transpose(0,1)+Reshape :508-514
    if (out_x8) {  // tile-major X8 (gemm_tc.cuh x8_index)
      const size_t tile = (size_t)(s >> 7) * (ldo >> 7) + (col >> 7);
      out[(((tile * 16 + ((s >> 3) & 15)) * 16 + ((col >> 3) & 15)) * 8 + (s & 7)) * 8 + (col & 7)] = f2bf(acc);
    }
    else out[(size_t)s * ldo + col] = f2bf(acc);
  }
}

// ------------------------------------------------------------------------------------------
// Decode attention (S == 1), one CTA per KV head serving its n_rep query heads (GQA: K and V are read
// once per KV head instead of once per query head; attentionRepeatKV :529-559 is pure indexing).
// Same arithmetic, truncation points and summation orders as sdpa_kernel.  The K / V rows that were
// complete before this call was enqueued (the prompt) are staged into shared memory with cp.async BEFORE
// griddepcontrol.wait (overlapping the QKV projection's tail); later rows and q are fetched after it.  K rows are padded to hd+8 elements (bank-conflict-free
// 128-bit reads for "one thread = one key").  block = 128 * n_rep threads (thread = (query head, key or d)).
// dyn smem = T_max * ((hd + 8) + hd) * 2  +  n_rep * (hd * 4 + T_max * 12) + 64
LNB_DEVINL void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
LNB_DEVINL void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__global__ void __launch_bounds__(1024) sdpa_decode_kernel(const uint16_t* __restrict__ q, const uint16_t* __restrict__ cache_k,
                                                           const uint16_t* __restrict__ cache_v, int kv_dim, int n_rep, int hd,
                                                           uint16_t* __restrict__ out, const int32_t* __restrict__ pos_ptr,
                                                           int T_max, int strict, float scale_bf16_as_f32,
                                                           const int32_t* __restrict__ pos_arr, long long cache_seq_stride, int ldq,
                                                           const LnbDevState* __restrict__ st, const int32_t* __restrict__ row_seq,
                                                           const int32_t* __restrict__ row_tree) {
  extern __shared__ __align__(16) uint8_t sm[];
  const int kstride = hd + 8;
  uint16_t* sK = reinterpret_cast<uint16_t*>(sm);                       // [T_max][hd + 8]
  uint16_t* sV = sK + (size_t)T_max * kstride;                          // [T_max][hd]
  double* sE = reinterpret_cast<double*>(sV + (size_t)T_max * hd);      // [n_rep][T_max]
  float* sP = reinterpret_cast<float*>(sE + (size_t)n_rep * T_max);     // [n_rep][T_max]
  float* sQ = sP + (size_t)n_rep * T_max;                               // [n_rep][hd]
  double* sZ = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(sQ + (size_t)n_rep * hd) + 15) & ~(uintptr_t)15);  // [n_rep][4] + [n_rep]
  const int h = blockIdx.x;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int hh = tid / 128, tt = tid % 128;
  const int cpr = hd / 8;  // 16-byte chunks per row
  // batched decode: blockIdx.y = row with its own position and q / output row, on the cache of sequence row_seq[blockIdx.y]
  // (speculative verification: several rows of one sequence, the later ones seeing the earlier ones' keys)
  if (pos_arr) {
    const size_t seq = (size_t)row_seq[blockIdx.y];
    pos_ptr = pos_arr + blockIdx.y;
    cache_k += seq * (size_t)cache_seq_stride;
    cache_v += seq * (size_t)cache_seq_stride;
    q += (size_t)blockIdx.y * ldq;
    out += (size_t)blockIdx.y * ldq;
  }

  pdl_launch_dependents();
  // With programmatic dependent launch this code may run while ANY earlier kernel of the stream is still
  // in flight (a kernel may start once its predecessor has started, not finished -- with small grids a
  // whole decode step can be resident at once), so only cache rows that were complete before the host
  // enqueued this call may be touched before the wait: rows [0, safe_rows), fixed by set_state_kernel at
  // the start of the call.  Everything else -- including rows appended by earlier steps of the same
  // device-resident decode run -- is loaded after griddepcontrol.wait.
  const int safe = (pos_arr || !st) ? 0 : max(0, min(st->safe_rows, T_max));
  for (int i = tid; i < safe * cpr; i += nthr) {
    const int t = i / cpr, c = i % cpr;
    cp_async16(sK + (size_t)t * kstride + c * 8, cache_k + (size_t)t * kv_dim + (size_t)h * hd + c * 8);
    cp_async16(sV + (size_t)t * hd + c * 8, cache_v + (size_t)t * kv_dim + (size_t)h * hd + c * 8);
  }
  pdl_wait();
  const int pos = __ldcg(pos_ptr);
  const int T = pos + 1;
  const int lo = min(safe, T);
  const KeyMap km = key_map(row_tree, blockIdx.y, pos);   // tree rows: key t from slot km(t) (row_tree implies pos_arr)
  for (int i = tid; i < (T - lo) * cpr; i += nthr) {
    const int t = lo + i / cpr, c = i % cpr;
    const size_t kt = (size_t)km(t) * kv_dim + (size_t)h * hd + c * 8;
    cp_async16(sK + (size_t)t * kstride + c * 8, cache_k + kt);
    cp_async16(sV + (size_t)t * hd + c * 8, cache_v + kt);
  }
  for (int i = tid; i < n_rep * hd; i += nthr) sQ[i] = bf2f(q[(size_t)(h * n_rep) * hd + i]);
  cp_async_wait_all();
  __syncthreads();

  // scores: sc_t = t( t(sum_seq_d q_d k_td) / t(sqrt(hd)) ); e_t = exp_f64(sc_t)      (:459-464, :484-490)
  const float* qh = sQ + hh * hd;
  for (int t = tt; t < T; t += 128) {
    const uint16_t* kr = sK + (size_t)t * kstride;
    float acc = 0.f;
    for (int d = 0; d < hd; d += 8) {
      const uint4 kv = *reinterpret_cast<const uint4*>(kr + d);
      acc = __fmaf_rn(qh[d + 0], bf_lo(kv.x), acc);
      acc = __fmaf_rn(qh[d + 1], bf_hi(kv.x), acc);
      acc = __fmaf_rn(qh[d + 2], bf_lo(kv.y), acc);
      acc = __fmaf_rn(qh[d + 3], bf_hi(kv.y), acc);
      acc = __fmaf_rn(qh[d + 4], bf_lo(kv.z), acc);
      acc = __fmaf_rn(qh[d + 5], bf_hi(kv.z), acc);
      acc = __fmaf_rn(qh[d + 6], bf_lo(kv.w), acc);
      acc = __fmaf_rn(qh[d + 7], bf_hi(kv.w), acc);
    }
    float sc = trunc_bf(acc);
    sc = trunc_bf(__fdiv_rn(sc, scale_bf16_as_f32));
    sE[(size_t)hh * T_max + t] = exp((double)sc);
  }
  __syncthreads();
  // Z = sum_seq_t e_t (f64): reference order (strict) or a tree (fast)
  double* eh = sE + (size_t)hh * T_max;
  if (strict) {
    if (tt == 0) {
      double z = 0.0;
      for (int t = 0; t < T; t++) z = __dadd_rn(z, eh[t]);
      sZ[n_rep * 4 + hh] = z;
    }
  } else {
    double z = 0.0;
    for (int t = tt; t < T; t += 128) z = __dadd_rn(z, eh[t]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z = __dadd_rn(z, __shfl_xor_sync(0xffffffffu, z, o));
    if ((tt & 31) == 0) sZ[hh * 4 + (tt >> 5)] = z;
  }
  __syncthreads();
  if (!strict && tt == 0)
    sZ[n_rep * 4 + hh] = __dadd_rn(__dadd_rn(__dadd_rn(sZ[hh * 4 + 0], sZ[hh * 4 + 1]), sZ[hh * 4 + 2]), sZ[hh * 4 + 3]);
  __syncthreads();
  const double Z = sZ[n_rep * 4 + hh];
  float* ph = sP + (size_t)hh * T_max;
  for (int t = tt; t < T; t += 128) ph[t] = trunc_bf((float)__ddiv_rn(eh[t], Z));   // t(f32(e/Z))  :493
  __syncthreads();
  // o_d = t( sum_seq_t p_t v_td )                                                      (:504)
  if (tt < hd) {
    const uint16_t* vc = sV + tt;
    float acc = 0.f;
#pragma unroll 4
    for (int t = 0; t < T; t++) acc = __fmaf_rn(ph[t], bf2f(vc[(size_t)t * hd]), acc);
    out[(size_t)(h * n_rep + hh) * hd + tt] = f2bf(acc);
  }
}

// ------------------------------------------------------------------------------------------
// Prompt attention (S > 1, LNB_ACC_FAST prefill path): one CTA per (query head, block of 32 query rows),
// keys streamed through shared memory in tiles of 64, two passes like the reference's data flow demands
// (P must be t(f32(e / Z)) with the FINAL Z, so an online-softmax rescale is not an option, SURVEY H4):
//   pass 1: sc = t(t(sum_seq_d q k)/t(sqrt(hd))), e = exp_f64(sc), Z_row = sum of e   (f64, tile order)
//   pass 2: the same scores again, p = t(f32(e / Z)), o_d += p_t * v_td  with t ascending
// Every score dot runs d = 0..hd-1 sequentially and every (row, d) output accumulates t = 0,1,2,...
// sequentially, i.e. in the reference's order; only the f64 row sum Z is reordered.  Causal mask
// (llamatransformer.go:128-136): keys t > pos0 + s contribute exactly 0 and whole tiles beyond the block
// are skipped.  Output goes straight into the tile-major X8 operand of the Wo GEMM.  hd must be 128.
constexpr int SP_QB = 32, SP_TK = 64, SP_HD = 128, SP_KS = SP_HD + 8;
constexpr int SP_SMEM = SP_QB * SP_HD * 4 + SP_TK * SP_KS * 2 + SP_TK * SP_HD * 2 + SP_QB * SP_TK * 4 + SP_QB * 8;

LNB_DEVINL void sp_scores(const float* __restrict__ Qs, const uint16_t* __restrict__ Ks, int r2, int kq, float (&acc)[2][4]) {
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 4; b++) acc[a][b] = 0.f;
  const float* q0 = Qs + (size_t)(2 * r2) * SP_HD;
  const float* q1 = q0 + SP_HD;
#pragma unroll 2
  for (int d = 0; d < SP_HD; d += 8) {
    const float4 a0 = *reinterpret_cast<const float4*>(q0 + d), a1 = *reinterpret_cast<const float4*>(q0 + d + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(q1 + d), b1 = *reinterpret_cast<const float4*>(q1 + d + 4);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const uint4 kv = *reinterpret_cast<const uint4*>(Ks + (size_t)(kq + 16 * j) * SP_KS + d);
      const float k0 = bf_lo(kv.x), k1 = bf_hi(kv.x), k2 = bf_lo(kv.y), k3 = bf_hi(kv.y);
      const float k4 = bf_lo(kv.z), k5 = bf_hi(kv.z), k6 = bf_lo(kv.w), k7 = bf_hi(kv.w);
      float x = acc[0][j], y = acc[1][j];
      x = __fmaf_rn(a0.x, k0, x); y = __fmaf_rn(b0.x, k0, y);
      x = __fmaf_rn(a0.y, k1, x); y = __fmaf_rn(b0.y, k1, y);
      x = __fmaf_rn(a0.z, k2, x); y = __fmaf_rn(b0.z, k2, y);
      x = __fmaf_rn(a0.w, k3, x); y = __fmaf_rn(b0.w, k3, y);
      x = __fmaf_rn(a1.x, k4, x); y = __fmaf_rn(b1.x, k4, y);
      x = __fmaf_rn(a1.y, k5, x); y = __fmaf_rn(b1.y, k5, y);
      x = __fmaf_rn(a1.z, k6, x); y = __fmaf_rn(b1.z, k6, y);
      x = __fmaf_rn(a1.w, k7, x); y = __fmaf_rn(b1.w, k7, y);
      acc[0][j] = x; acc[1][j] = y;
    }
  }
}

__global__ void __launch_bounds__(256) sdpa_prefill_kernel(const uint16_t* __restrict__ q, int ldq, const uint16_t* __restrict__ cache_k,
                                                           const uint16_t* __restrict__ cache_v, int kv_dim, int n_rep,
                                                           uint16_t* __restrict__ out_x8, int ldo, const int32_t* __restrict__ pos_ptr,
                                                           int S, float scale_bf16_as_f32) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t sm[];
  float* Qs = reinterpret_cast<float*>(sm);                                   // [32][128]
  uint16_t* Ks = reinterpret_cast<uint16_t*>(Qs + SP_QB * SP_HD);             // [64][136]
  uint16_t* Vs = Ks + SP_TK * SP_KS;                                          // [64][128]
  float* Ps = reinterpret_cast<float*>(Vs + SP_TK * SP_HD);                   // [32][64]
  double* Zs = reinterpret_cast<double*>(Ps + SP_QB * SP_TK);                 // [32]
  const int H = blockIdx.x, s0 = blockIdx.y * SP_QB, h = H / n_rep;
  const int tid = threadIdx.x;
  const int pos0 = *pos_ptr;
  const int t_end = min(pos0 + S, pos0 + s0 + SP_QB);   // keys this row block can see
  const int n_tiles = (t_end + SP_TK - 1) / SP_TK;

  for (int i = tid; i < SP_QB * SP_HD; i += 256) {
    const int r = i / SP_HD, d = i % SP_HD;
    Qs[i] = (s0 + r < S) ? bf2f(q[(size_t)(s0 + r) * ldq + (size_t)H * SP_HD + d]) : 0.f;
  }
  const int r2 = tid / 16, kq = tid % 16;   // score block: rows 2*r2, 2*r2+1 ; keys kq + 16*j
  double z0 = 0.0, z1 = 0.0;
  auto load_tile = [&](int tile, bool with_v) {
    const int t0 = tile * SP_TK;
    for (int i = tid; i < SP_TK * (SP_HD / 8); i += 256) {
      const int t = i / (SP_HD / 8), c = i % (SP_HD / 8);
      uint4 kk = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
      if (t0 + t < t_end) {
        kk = *reinterpret_cast<const uint4*>(cache_k + (size_t)(t0 + t) * kv_dim + (size_t)h * SP_HD + c * 8);
        if (with_v) vv = *reinterpret_cast<const uint4*>(cache_v + (size_t)(t0 + t) * kv_dim + (size_t)h * SP_HD + c * 8);
      }
      *reinterpret_cast<uint4*>(Ks + (size_t)t * SP_KS + c * 8) = kk;
      if (with_v) *reinterpret_cast<uint4*>(Vs + (size_t)t * SP_HD + c * 8) = vv;
    }
  };
  // ---------------- pass 1: row sums of exp ----------------------------------------------------
  for (int tile = 0; tile < n_tiles; tile++) {
    __syncthreads();
    load_tile(tile, false);
    __syncthreads();
    float acc[2][4];
    sp_scores(Qs, Ks, r2, kq, acc);
#pragma unroll
    for (int a = 0; a < 2; a++)
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int t = tile * SP_TK + kq + 16 * j, srow = s0 + 2 * r2 + a;
        if (t <= pos0 + srow && t < t_end) {
          float sc = trunc_bf(acc[a][j]);
          sc = trunc_bf(__fdiv_rn(sc, scale_bf16_as_f32));
          const double e = exp((double)sc);
          if (a == 0) z0 = __dadd_rn(z0, e); else z1 = __dadd_rn(z1, e);
        }
      }
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) {   // the 16 threads that share a row pair are 16 consecutive lanes
    z0 = __dadd_rn(z0, __shfl_xor_sync(0xffffffffu, z0, o));
    z1 = __dadd_rn(z1, __shfl_xor_sync(0xffffffffu, z1, o));
  }
  if (kq == 0) { Zs[2 * r2] = z0; Zs[2 * r2 + 1] = z1; }
  // ---------------- pass 2: p = t(f32(e/Z)), o += p v ------------------------------------------
  const int pr = tid / 8, dg = (tid % 8) * 16;   // PV block: row pr, columns dg .. dg+15
  float o[16];
#pragma unroll
  for (int i = 0; i < 16; i++) o[i] = 0.f;
  for (int tile = 0; tile < n_tiles; tile++) {
    __syncthreads();
    load_tile(tile, true);
    __syncthreads();
    float acc[2][4];
    sp_scores(Qs, Ks, r2, kq, acc);
#pragma unroll
    for (int a = 0; a < 2; a++) {
      const double Z = Zs[2 * r2 + a];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int t = tile * SP_TK + kq + 16 * j, srow = s0 + 2 * r2 + a;
        float pv = 0.f;
        if (t <= pos0 + srow && t < t_end) {
          float sc = trunc_bf(acc[a][j]);
          sc = trunc_bf(__fdiv_rn(sc, scale_bf16_as_f32));
          pv = trunc_bf((float)__ddiv_rn(exp((double)sc), Z));
        }
        Ps[(size_t)(2 * r2 + a) * SP_TK + kq + 16 * j] = pv;
      }
    }
    __syncthreads();
    const int tn = min(SP_TK, t_end - tile * SP_TK);
    const float* prow = Ps + (size_t)pr * SP_TK;
    for (int t = 0; t < tn; t++) {
      const float pt = prow[t];
      const uint4 v0 = *reinterpret_cast<const uint4*>(Vs + (size_t)t * SP_HD + dg);
      const uint4 v1 = *reinterpret_cast<const uint4*>(Vs + (size_t)t * SP_HD + dg + 8);
      o[0] = __fmaf_rn(pt, bf_lo(v0.x), o[0]);   o[1] = __fmaf_rn(pt, bf_hi(v0.x), o[1]);
      o[2] = __fmaf_rn(pt, bf_lo(v0.y), o[2]);   o[3] = __fmaf_rn(pt, bf_hi(v0.y), o[3]);
      o[4] = __fmaf_rn(pt, bf_lo(v0.z), o[4]);   o[5] = __fmaf_rn(pt, bf_hi(v0.z), o[5]);
      o[6] = __fmaf_rn(pt, bf_lo(v0.w), o[6]);   o[7] = __fmaf_rn(pt, bf_hi(v0.w), o[7]);
      o[8] = __fmaf_rn(pt, bf_lo(v1.x), o[8]);   o[9] = __fmaf_rn(pt, bf_hi(v1.x), o[9]);
      o[10] = __fmaf_rn(pt, bf_lo(v1.y), o[10]); o[11] = __fmaf_rn(pt, bf_hi(v1.y), o[11]);
      o[12] = __fmaf_rn(pt, bf_lo(v1.z), o[12]); o[13] = __fmaf_rn(pt, bf_hi(v1.z), o[13]);
      o[14] = __fmaf_rn(pt, bf_lo(v1.w), o[14]); o[15] = __fmaf_rn(pt, bf_hi(v1.w), o[15]);
    }
  }
  const int srow = s0 + pr;
  if (srow < S) {
#pragma unroll
    for (int i = 0; i < 16; i += 8) {
      uint4 w;
      w.x = (uint32_t)f2bf(o[i + 0]) | ((uint32_t)f2bf(o[i + 1]) << 16);
      w.y = (uint32_t)f2bf(o[i + 2]) | ((uint32_t)f2bf(o[i + 3]) << 16);
      w.z = (uint32_t)f2bf(o[i + 4]) | ((uint32_t)f2bf(o[i + 5]) << 16);
      w.w = (uint32_t)f2bf(o[i + 6]) | ((uint32_t)f2bf(o[i + 7]) << 16);
      *reinterpret_cast<uint4*>(out_x8 + x8_index(srow, H * SP_HD + dg + i, ldo)) = w;   // 8 consecutive columns = one chunk
    }
  }
}

// ------------------------------------------------------------------------------------------
// Tensor-parallel tail of Wo / w2: h[m,n] = t( res[m,n] + t(sum[m,n]) ) after the fp32
// allreduce (ml.Add, llamatransformer.go:232,248, on the reduced partials).
__global__ void resid_from_f32_kernel(const float* __restrict__ sum, const uint16_t* __restrict__ res,
                                      uint16_t* __restrict__ out, int64_t n) {
  pdl_launch_dependents();
  pdl_wait();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = f2bf(__fadd_rn(bf2f(res[i]), trunc_bf(sum[i])));
}

// ------------------------------------------------------------------------------------------
// Reducer of the peer-memory all-reduce (see LnbP2P in common.cuh): polls the N local slots until the
// words of this epoch have arrived, adds them in rank order and applies the residual:
// out = t( res + t( ((p0 + p1) + p2) + ... ) )   (ml.Add after Wo / w2, llamatransformer.go:232,248).
// The last CTA advances the epoch (local counter only).  Every wait is bounded (p2p_wait_word, common.cuh).
__global__ void __launch_bounds__(256) p2p_reduce_resid_kernel(LnbP2P pp, LnbDevState* st, const uint16_t* __restrict__ res,
                                                               uint16_t* __restrict__ out, int n_elems) {
  pdl_launch_dependents();
  pdl_wait();
  if (*reinterpret_cast<volatile uint32_t*>(&st->ar_error)) return;   // an earlier wait of this session timed out
  const uint32_t epoch = st->ar_epoch;
  const unsigned long long t0 = global_timer_ns();
  const uint2* base = pp.data[pp.rank] + (size_t)(epoch & 1u) * pp.n * pp.slot_elems;
  bool ok = true;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_elems && ok; i += gridDim.x * blockDim.x) {
    float sum = 0.f;
    for (int r = 0; r < pp.n; r++) {
      uint2 w;
      if (!p2p_wait_word(base + (size_t)r * pp.slot_elems + i, epoch, r, pp, st, t0, &w)) { ok = false; break; }
      sum = (r == 0) ? __uint_as_float(w.x) : __fadd_rn(sum, __uint_as_float(w.x));
    }
    if (ok) out[i] = f2bf(__fadd_rn(bf2f(res[i]), trunc_bf(sum)));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int done = atomicAdd(&st->ar_done2, 1u);
    if (done == gridDim.x - 1) {
      st->ar_done2 = 0;
      st->ar_epoch = epoch + 1;
      __threadfence();
    }
  }
}

// Tensor-parallel greedy argmax over peer memory: every rank pushes its 64-bit (value, index) key as two
// LL words to all peers, takes the maximum of the N keys (same on every rank), publishes the token and
// advances the decode state.  One warp.
__global__ void p2p_argmax_kernel(LnbP2P pp, LnbDevState* st, int advance, int32_t* tok_out) {
  pdl_launch_dependents();
  pdl_wait();
  if (*reinterpret_cast<volatile uint32_t*>(&st->ar_error)) return;
  const uint32_t epoch = st->ar_epoch;
  const unsigned long long t0 = global_timer_ns();
  const int lane = threadIdx.x;
  const unsigned long long mykey = st->amax_key;
  const size_t myoff = ((size_t)((epoch & 1u) * pp.n + pp.rank)) * pp.slot_elems;
  if (lane < pp.n) {
    pp.data[lane][myoff] = make_uint2((uint32_t)(mykey & 0xffffffffull), epoch);
    pp.data[lane][myoff + 1] = make_uint2((uint32_t)(mykey >> 32), epoch);
  }
  unsigned long long key = LNB_ARGMAX_EMPTY;
  bool ok = true;
  if (lane < pp.n) {
    const uint2* src = pp.data[pp.rank] + ((size_t)((epoch & 1u) * pp.n + lane)) * pp.slot_elems;
    uint2 lo = make_uint2(0, 0), hi = make_uint2(0, 0);
    ok = p2p_wait_word(src, epoch, lane, pp, st, t0, &lo) && p2p_wait_word(src + 1, epoch, lane, pp, st, t0, &hi);
    key = ((unsigned long long)hi.x << 32) | lo.x;
  }
  if (__any_sync(0xffffffffu, !ok)) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
    key = other > key ? other : key;
  }
  if (lane == 0) {
    const int32_t tok = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
    st->next_token = tok;
    st->amax_key = LNB_ARGMAX_EMPTY;
    st->done_ctr = 0;
    st->ar_epoch = epoch + 1;
    if (advance) {
      if (tok_out) tok_out[st->step] = tok;
      st->step += 1;
      st->pos += 1;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Generic-shape kernels behind the op-level C-ABI (any S, K, N): one thread per output,
// reference order.  Used when a shape does not meet the panel GEMV's constraints
// (e.g. the reference's own 2x3 . 4x3^T golden case).
__global__ void linear_naive_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ w,
                                    uint16_t* __restrict__ out, int S, int K, int N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)S * N) return;
  const int s = (int)(i / N), n = (int)(i % N);
  float acc = 0.f;
  for (int k = 0; k < K; k++) acc = __fmaf_rn(bf2f(x[(size_t)s * K + k]), bf2f(w[(size_t)n * K + k]), acc);
  out[i] = f2bf(acc);
}

// ml.MatMul BF16 (operations_matmul.go:24-60): out[g,m,n] = t(sum_seq_k a[g,m,k]*b[g,k,n])
__global__ void matmul_naive_kernel(const uint16_t* __restrict__ a, const uint16_t* __restrict__ b,
                                    uint16_t* __restrict__ out, int B, int M, int K, int N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * M * N) return;
  const int n = (int)(i % N);
  const int64_t gm = i / N;
  const int g = (int)(gm / M);
  const uint16_t* ar = a + gm * K;
  const uint16_t* bg = b + (size_t)g * K * N;
  float acc = 0.f;
  for (int k = 0; k < K; k++) acc = __fmaf_rn(bf2f(ar[k]), bf2f(bg[(size_t)k * N + n]), acc);
  out[i] = f2bf(acc);
}

// RMSNorm.Forward (llamatransformer.go:633-660), one CTA (256 threads) per row.
// strict: sequential sum; fast: the same 256-way interleave + butterfly as gemv.cuh's prologue.
__global__ void __launch_bounds__(256) rmsnorm_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ w,
                                                      uint16_t* __restrict__ out, int D, float eps, int strict,
                                                      const float* __restrict__ rscale) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float wsum[8];
  __shared__ float rs;
  const uint16_t* xr = x + (size_t)blockIdx.x * D;
  const int tid = threadIdx.x;
  if (rscale) {  // 1/rms already computed (rms_scale_kernel / rms_scale_scan_kernel)
    if (tid == 0) rs = rscale[blockIdx.x];
  } else if (strict) {
    if (tid == 0) {
      float sum = 0.f;
      for (int k = 0; k < D; k++) {
        const float v = bf2f(xr[k]);
        sum = __fmaf_rn(v, v, sum);
      }
      const float me = __fadd_rn(__fdiv_rn(sum, (float)D), eps);
      rs = (float)(1.0 / sqrt((double)me));
    }
  } else {
    float sum = 0.f;
    for (int k = tid; k < D; k += 256) {
      const float v = bf2f(xr[k]);
      sum = __fmaf_rn(v, v, sum);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
    if ((tid & 31) == 0) wsum[tid >> 5] = sum;
    __syncthreads();
    if (tid == 0) {
      float tot = 0.f;
      for (int i = 0; i < 8; i++) tot = __fadd_rn(tot, wsum[i]);
      const float me = __fadd_rn(__fdiv_rn(tot, (float)D), eps);
      rs = (float)(1.0 / sqrt((double)me));
    }
  }
  __syncthreads();
  const float r = rs;
  for (int k = tid; k < D; k += 256) {
    const float n1 = trunc_bf(__fmul_rn(bf2f(xr[k]), r));
    out[(size_t)blockIdx.x * D + k] = f2bf(__fmul_rn(n1, bf2f(w[k])));
  }
}

// LNB_ACC_STRICT RMSNorm scale, once per row instead of once per GEMV CTA:
//   r[m] = f32( 1 / sqrt( f64( (sum_seq_k x[m,k]^2) / D + eps ) ) )     (llamatransformer.go:641-656)
// The sum is the reference's strictly sequential f32 chain (4 cycles per element on one thread);
// the squares (exact in f32) are staged in shared memory by the whole CTA first and the chain
// reads them with double-buffered 128-bit loads so that only the FADD latency is exposed.
// grid = rows, block = 128, dyn smem = D * 4.
__global__ void __launch_bounds__(128) rms_scale_kernel(const uint16_t* __restrict__ x, int ldx, float* __restrict__ r,
                                                        int D, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) float sq[];
  const uint16_t* xr = x + (size_t)blockIdx.x * ldx;
  for (int k = threadIdx.x * 2; k < D; k += 256) {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(xr + k);
    const float a = bf_lo(w), b = bf_hi(w);
    sq[k] = __fmul_rn(a, a);
    sq[k + 1] = __fmul_rn(b, b);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
    const float4* q4 = reinterpret_cast<const float4*>(sq);
    const int n4 = D / 4;
    constexpr int B = 8;
    int i = 0;
    if (n4 >= 2 * B) {
      float4 a[B], b[B];
#pragma unroll
      for (int u = 0; u < B; u++) a[u] = q4[u];
      for (; i + 2 * B <= n4; i += 2 * B) {
#pragma unroll
        for (int u = 0; u < B; u++) b[u] = q4[i + B + u];
#pragma unroll
        for (int u = 0; u < B; u++) {
          sum = __fadd_rn(sum, a[u].x); sum = __fadd_rn(sum, a[u].y);
          sum = __fadd_rn(sum, a[u].z); sum = __fadd_rn(sum, a[u].w);
        }
        if (i + 3 * B <= n4) {
#pragma unroll
          for (int u = 0; u < B; u++) a[u] = q4[i + 2 * B + u];
        }
#pragma unroll
        for (int u = 0; u < B; u++) {
          sum = __fadd_rn(sum, b[u].x); sum = __fadd_rn(sum, b[u].y);
          sum = __fadd_rn(sum, b[u].z); sum = __fadd_rn(sum, b[u].w);
        }
      }
    }
    for (int k = i * 4; k < D; k++) sum = __fadd_rn(sum, sq[k]);
    const float me = __fadd_rn(__fdiv_rn(sum, (float)D), eps);
    r[blockIdx.x] = (float)(1.0 / sqrt((double)me));
  }
}

// applyRotaryEmbeddings (llamatransformer.go:753-790) standalone: x[S,H,hd]
__global__ void rope_kernel(const uint16_t* __restrict__ x, const float* __restrict__ cis, uint16_t* __restrict__ out,
                            int S, int H, int hd, int start_pos) {
  const int half = hd / 2;
  const int64_t total = (int64_t)S * H * half;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ii = (int)(i % half);
    const int64_t sh = i / half;
    const int s = (int)(sh / H);
    const uint32_t w = *reinterpret_cast<const uint32_t*>(x + sh * hd + 2 * ii);
    const double a = (double)bf_lo(w), b = (double)bf_hi(w);
    const float2 fc = *reinterpret_cast<const float2*>(cis + ((size_t)(start_pos + s) * half + ii) * 2);
    const double c = (double)fc.x, d = (double)fc.y;
    const float re = (float)(a * c - b * d);
    const float im = (float)(a * d + b * c);
    *reinterpret_cast<uint32_t*>(out + sh * hd + 2 * ii) = (uint32_t)f2bf(re) | ((uint32_t)f2bf(im) << 16);
  }
}

__global__ void silu_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ tab,
                            uint16_t* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = tab[x[i]];
}
__global__ void add_kernel(const uint16_t* __restrict__ a, const uint16_t* __restrict__ b, uint16_t* __restrict__ out,
                           int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = f2bf(__fadd_rn(bf2f(a[i]), bf2f(b[i])));
}
__global__ void mul_kernel(const uint16_t* __restrict__ a, const uint16_t* __restrict__ b, uint16_t* __restrict__ out,
                           int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = f2bf(__fmul_rn(bf2f(a[i]), bf2f(b[i])));
}

// ml.Softmax (operations_impl.go:478-511): one CTA per row; the f64 sum is sequential
// (reference order) -- this op-level kernel is only used by the ml.Softmax shim.
__global__ void softmax_f32_kernel(const float* __restrict__ x, float* __restrict__ out, int cols) {
  __shared__ double zs;
  const float* xr = x + (size_t)blockIdx.x * cols;
  if (threadIdx.x == 0) {
    double z = 0.0;
    for (int c = 0; c < cols; c++) z = __dadd_rn(z, exp((double)xr[c]));
    zs = z;
  }
  __syncthreads();
  const double z = zs;
  for (int c = threadIdx.x; c < cols; c += blockDim.x)
    out[(size_t)blockIdx.x * cols + c] = (float)__ddiv_rn(exp((double)xr[c]), z);
}

// ml.Argmax (operations_impl.go:513-548): first maximum wins, NaN and values <= -MaxFloat32
// are never selected (-1 if nothing is).
__global__ void __launch_bounds__(256) argmax_f32_kernel(const float* __restrict__ x, int cols, int32_t* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();  // also used inside the forward chain (batched decode)
  __shared__ unsigned long long best[8];
  const float* xr = x + (size_t)blockIdx.x * cols;
  unsigned long long key = LNB_ARGMAX_EMPTY;
  for (int c = threadIdx.x; c < cols; c += 256) {
    const float v = xr[c];
    if (v > -3.402823466e+38f) {
      const unsigned long long k2 = argmax_key(v, (uint32_t)c);
      key = k2 > key ? k2 : key;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
    key = other > key ? other : key;
  }
  if ((threadIdx.x & 31) == 0) best[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; i++) key = best[i] > key ? best[i] : key;
    out[blockIdx.x] = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
  }
}

}  // namespace lnb
