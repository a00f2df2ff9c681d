// sdpa_stream.cuh -- attention whose key history streams from HBM in tiles, for every row the shared-memory kernels
// (sdpa_kernel, sdpa_decode_kernel) cannot hold: long SequenceLength sessions, batched decode beyond the decode kernel's
// fit, and lnb_op_attention_bf16 beyond sdpa_kernel's T limit.
//
// One description covers every caller: query row r (global index r of the call) has its own cache base
// (cache + row_seq[r] * row_cache_stride: batched, ragged and speculative calls, where rows of one sequence follow each
// other; cache without a row map) and its own position p_r (pos_arr[r], or base + pos_step * r: S = 1
// decode, a prompt or chunked prefill under the [S,T] mask, or pos_step = 0 for the op's unmasked form) and sees keys
// 0..p_r (a speculative tree row reads key t from slot KeyMap(t) of its row_tree word, common.cuh).  The arithmetic is
// sdpa_kernel's (llamatransformer.go:459-514):
//   sc_t = t( t(sum_seq_d q_d k_td) / t(sqrt(hd)) );  e_t = exp_f64(sc_t);  p_t = t(f32(e_t / Z));  o_d = t(sum_t p_t v_td)
// Because sc_t is a bf16 value, e_t is recomputed from the 2-byte score wherever it is needed instead of being kept
// as 8 bytes.  Three launches per group of rows, all reading and writing a per-session scratch:
//   ss_scores_kernel  grid (kv head, row, chunk of SS_CH keys): K tiles through shared memory, every score dot runs
//                     d = 0..hd-1 sequentially, the bf16 score goes to sc[row][head][t]; FAST also writes the chunk's
//                     partial Z (f64: per thread in t order, then a fixed xor tree, then the 4 warps in order).
//   STRICT: ss_zsum_kernel  grid (query head, row): Z = sum_t e_t in t order by one thread while the other warps
//                     compute the next tile of e; then p_t overwrites sc_t in place.
//           ss_out_kernel   grid (kv head x d-range, row): one fp32 chain per (query head, d) over t = 0..p_r.
//   FAST:   ss_out_kernel   grid (kv head, row, chunk): Z = the chunk partials added in chunk order (every CTA
//                     redundantly), p from the score, one fp32 chain per (query head, d) over the chunk's keys -> opart.
//           ss_combine_kernel grid (query head, row): o_d = t(sum of the chunk partials in chunk order).
// So STRICT is bit-identical to sdpa_kernel's strict form; FAST has the order above (DESIGN §3).  No float atomics.
// PDL: every kernel waits (griddepcontrol.wait) before its first global access, so nothing is read or written while an
// earlier kernel of the stream may still run.
// MXFP8 caches (KVF = KVF_MXFP8, kvcache.cuh): ss_scores_kernel and ss_out_kernel copy each tile's codes (8-byte pieces)
// and its keys' 4-byte scale slots with cp.async, decode them into the bf16 tile the bf16 form copies, and then run the
// bf16 form's arithmetic unchanged.  cache_k / cache_v then point at the records, kv_dim is the record's byte size and
// row_cache_stride counts bytes.
#pragma once
#include "kvcache.cuh"

namespace lnb {

constexpr int SS_CH = 1024;   // keys per chunk (FAST: one CTA per chunk; both modes: one score CTA per chunk)
constexpr int SS_KT = 128;    // keys per K tile of ss_scores_kernel (one key per thread)
constexpr int SS_VT = 256;    // keys per V / p tile of ss_out_kernel (two stages)
constexpr int SS_ZT = 1024;   // e values per buffer of ss_zsum_kernel (two buffers)

struct StreamAttn {
  const uint16_t* q;            // row r, query head H: q + r * ldq + H * hd
  int ldq;
  const uint16_t* cache_k;
  const uint16_t* cache_v;
  int kv_dim;
  long long row_cache_stride;   // elements between the caches of consecutive sequences
  const int32_t* row_seq;       // rows of several sequences: row r reads the cache of sequence row_seq[r]; NULL: cache_k
  const int32_t* row_tree;      // speculative tree rows: row r's slot and ancestor mask (common.cuh KeyMap); NULL: key t = slot t
  int n_rep, hd, n_heads;       // n_heads: query heads of this rank
  const int32_t* pos_arr;       // per-row positions, or NULL:
  const int32_t* pos_ptr;       //   p_r = (pos_ptr ? *pos_ptr : pos_fixed) + pos_step * r
  int pos_fixed, pos_step;
  int row0;                     // first row of this launch group (scratch row = r - row0)
  int t_stride;                 // keys per scratch row (a multiple of SS_VT, >= every T)
  int n_chunks;                 // t_stride / SS_CH rounded up
  uint16_t* sc;                 // [rows][n_heads][t_stride] bf16 scores (STRICT: then p)
  double* zpart;                // FAST: [rows][n_heads][n_chunks]
  float* opart;                 // FAST: [rows][n_heads][n_chunks][hd]
  uint16_t* out;                // row r, column c: out[r * ldo + c], or the X8 operand of the Wo GEMM (out_x8)
  int ldo, out_x8;
  float scale;                  // t(sqrt(hd)) as f32
  int strict;
};

LNB_DEVINL int ss_keys(const StreamAttn& P, int r) {   // keys row r sees (call only after pdl_wait)
  const int p = P.pos_arr ? __ldcg(P.pos_arr + r) : (P.pos_ptr ? __ldcg(P.pos_ptr) : P.pos_fixed) + P.pos_step * r;
  return p + 1;
}
LNB_DEVINL KeyMap ss_key_map(const StreamAttn& P, int r, int T) { return key_map(P.row_tree, r, T - 1); }   // (after pdl_wait)
LNB_DEVINL size_t ss_cache_base(const StreamAttn& P, int r) {   // (call only after pdl_wait)
  return P.row_seq ? (size_t)__ldcg(P.row_seq + r) * (size_t)P.row_cache_stride : 0;
}
LNB_DEVINL uint16_t* ss_score_row(const StreamAttn& P, int rl, int H) {
  return P.sc + ((size_t)rl * P.n_heads + H) * (size_t)P.t_stride;
}
LNB_DEVINL void ss_store(const StreamAttn& P, int r, int col, float v) {
  if (P.out_x8) P.out[x8_index(r, col, P.ldo)] = f2bf(v);
  else P.out[(size_t)r * P.ldo + col] = f2bf(v);
}
LNB_DEVINL void ss_cp16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
LNB_DEVINL void ss_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
LNB_DEVINL void ss_cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// dyn smem = SS_KT * (hd + 8) * 2 + n_rep * hd * 4 (MXFP8: + the tile's codes and scale slots, SS_KT * (hd + 4))
inline size_t ss_scores_smem(int hd, int n_rep, int kvf) {
  return (size_t)SS_KT * (hd + 8) * 2 + (size_t)n_rep * hd * 4 + (kvf == KVF_MXFP8 ? (size_t)SS_KT * (hd + 4) : 0);
}
LNB_DEVINL void ss_cp8(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
LNB_DEVINL void ss_cp4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
// MXFP8: issue the copies of keys [k0, k0 + n) of head h (key t in the record at slot km(t) of rec, rowb bytes apart; codes
// of the head's columns [c0, c0 + w)) into codes [n][w] and slots [n]
LNB_DEVINL void ss_issue_fp8(const uint8_t* rec, int rowb, int kv_l, int h, int hd, int c0, int w, int k0, int n, const KeyMap& km,
                             uint8_t* codes, uint32_t* slots, int tid, int nthr) {
  const int cpr = w / 8;
  for (int i = tid; i < n * cpr; i += nthr) {
    const int t = i / cpr, cc = i % cpr;
    ss_cp8(codes + (size_t)t * w + cc * 8, rec + (size_t)km(k0 + t) * rowb + h * hd + c0 + cc * 8);
  }
  for (int t = tid; t < n; t += nthr) ss_cp4(slots + t, rec + (size_t)km(k0 + t) * rowb + kv_l + h * 4);
}
// MXFP8: decode the copied codes [n][w] (columns [c0, c0 + w) of the head) into the bf16 tile [n][ld]
LNB_DEVINL void ss_decode_fp8(const uint8_t* codes, const uint32_t* slots, int c0, int w, int n, uint16_t* out, int ld, int tid, int nthr) {
  const int cpr = w / 8;
  for (int i = tid; i < n * cpr; i += nthr) {
    const int t = i / cpr, cc = i % cpr;
    const uint32_t e8m0 = (slots[t] >> (8 * ((c0 + cc * 8) >> 5))) & 0xffu;
    *reinterpret_cast<uint4*>(out + (size_t)t * ld + cc * 8) =
        kv_decode8(*reinterpret_cast<const uint2*>(codes + (size_t)t * w + cc * 8), mx_scale(e8m0));
  }
}

template <int KVF>
__global__ void __launch_bounds__(SS_KT) ss_scores_kernel(const StreamAttn P) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t sm[];
  __shared__ double zw[8][SS_KT / 32];
  const int h = blockIdx.x, rl = blockIdx.y, c = blockIdx.z, r = P.row0 + rl;
  const int tid = threadIdx.x;
  const int T = ss_keys(P, r);
  const int t0 = c * SS_CH;
  if (t0 >= T) return;
  const int t1 = min(T, t0 + SS_CH);
  const KeyMap km = ss_key_map(P, r, T);
  const int hd = P.hd, n_rep = P.n_rep, ks = hd + 8, cpr = hd / 8;
  uint16_t* sK = reinterpret_cast<uint16_t*>(sm);                     // [SS_KT][hd + 8]
  float* sQ = reinterpret_cast<float*>(sK + (size_t)SS_KT * ks);      // [n_rep][hd]
  uint32_t* sSl = reinterpret_cast<uint32_t*>(sQ + (size_t)n_rep * hd);  // MXFP8: [SS_KT] scale slots, then [SS_KT][hd] codes
  uint8_t* sC = reinterpret_cast<uint8_t*>(sSl + SS_KT);
  const uint16_t* kb = P.cache_k + ss_cache_base(P, r) + (size_t)h * hd;
  const uint8_t* kr8 = reinterpret_cast<const uint8_t*>(P.cache_k) + ss_cache_base(P, r);
  for (int i = tid; i < n_rep * hd; i += SS_KT) sQ[i] = bf2f(P.q[(size_t)r * P.ldq + (size_t)h * n_rep * hd + i]);
  double z[8];
#pragma unroll
  for (int j = 0; j < 8; j++) z[j] = 0.0;
  for (int k0 = t0; k0 < t1; k0 += SS_KT) {
    const int n = min(SS_KT, t1 - k0);
    __syncthreads();
    if constexpr (KVF == KVF_MXFP8) {
      ss_issue_fp8(kr8, P.kv_dim, P.n_heads / n_rep * hd, h, hd, 0, hd, k0, n, km, sC, sSl, tid, SS_KT);
    } else {
      for (int i = tid; i < n * cpr; i += SS_KT) {
        const int t = i / cpr, cc = i % cpr;
        ss_cp16(sK + (size_t)t * ks + cc * 8, kb + (size_t)km(k0 + t) * P.kv_dim + cc * 8);
      }
    }
    ss_cp_commit();
    ss_cp_wait<0>();
    __syncthreads();
    if constexpr (KVF == KVF_MXFP8) {
      ss_decode_fp8(sC, sSl, 0, hd, n, sK, ks, tid, SS_KT);
      __syncthreads();
    }
    if (tid < n) {
      const uint16_t* kr = sK + (size_t)tid * ks;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; j++) acc[j] = 0.f;
      for (int d = 0; d < hd; d += 8) {
        const uint4 kv = *reinterpret_cast<const uint4*>(kr + d);
        const float k0f = bf_lo(kv.x), k1 = bf_hi(kv.x), k2 = bf_lo(kv.y), k3 = bf_hi(kv.y);
        const float k4 = bf_lo(kv.z), k5 = bf_hi(kv.z), k6 = bf_lo(kv.w), k7 = bf_hi(kv.w);
#pragma unroll
        for (int j = 0; j < 8; j++) {
          if (j < n_rep) {
            const float* qh = sQ + j * hd + d;
            float a = acc[j];
            a = __fmaf_rn(qh[0], k0f, a); a = __fmaf_rn(qh[1], k1, a);
            a = __fmaf_rn(qh[2], k2, a);  a = __fmaf_rn(qh[3], k3, a);
            a = __fmaf_rn(qh[4], k4, a);  a = __fmaf_rn(qh[5], k5, a);
            a = __fmaf_rn(qh[6], k6, a);  a = __fmaf_rn(qh[7], k7, a);
            acc[j] = a;
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 8; j++) {
        if (j < n_rep) {
          float sc = trunc_bf(acc[j]);
          sc = trunc_bf(__fdiv_rn(sc, P.scale));
          ss_score_row(P, rl, h * n_rep + j)[k0 + tid] = f2bf(sc);
          if (!P.strict) z[j] = __dadd_rn(z[j], exp((double)sc));
        }
      }
    }
  }
  if (P.strict) return;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    if (j < n_rep) {
      double v = z[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
      if ((tid & 31) == 0) zw[j][tid >> 5] = v;
    }
  }
  __syncthreads();
  if (tid < n_rep)
    P.zpart[((size_t)rl * P.n_heads + h * n_rep + tid) * P.n_chunks + c] =
        __dadd_rn(__dadd_rn(__dadd_rn(zw[tid][0], zw[tid][1]), zw[tid][2]), zw[tid][3]);
}

// STRICT: Z in the reference's order, then p in place of the scores.  block = 128: thread 0 adds buffer k while
// warps 1..3 fill buffer k + 1 with e.
__global__ void __launch_bounds__(128) ss_zsum_kernel(const StreamAttn P) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sE[2][SS_ZT];
  __shared__ double zfinal;
  const int H = blockIdx.x, rl = blockIdx.y, r = P.row0 + rl;
  const int tid = threadIdx.x;
  const int T = ss_keys(P, r);
  uint16_t* row = ss_score_row(P, rl, H);
  const int nt = (T + SS_ZT - 1) / SS_ZT;
  for (int k = -1; k < nt; k++) {   // k = -1 only fills buffer 0
    const int base = k * SS_ZT;
    if (tid == 0 && k >= 0) {
      const double* e = sE[k & 1];
      const int n = min(SS_ZT, T - base);
      double z = k ? zfinal : 0.0;
#pragma unroll 8
      for (int i = 0; i < n; i++) z = __dadd_rn(z, e[i]);
      zfinal = z;
    } else if (tid >= 32 && k + 1 < nt) {
      double* e = sE[(k + 1) & 1];
      const int n = min(SS_ZT, T - base - SS_ZT);
      for (int i = tid - 32; i < n; i += 96) e[i] = exp((double)bf2f(row[base + SS_ZT + i]));
    }
    __syncthreads();
  }
  const double Z = zfinal;
  for (int t = tid; t < T; t += 128) row[t] = f2bf(trunc_bf((float)__ddiv_rn(exp((double)bf2f(row[t])), Z)));
}

// dyn smem = 2 stages x (SS_VT x dw V columns + n_rep x SS_VT bf16 scores) + n_rep x SS_VT f32 p
// (MXFP8: + 2 stages of the tile's codes and scale slots, SS_VT x (dw + 4) each)
inline size_t ss_out_smem(int hd, int n_rep, int dsplit, int kvf) {
  const int dw = hd / dsplit;
  return (size_t)2 * ((size_t)SS_VT * dw * 2 + (size_t)n_rep * SS_VT * 2) + (size_t)n_rep * SS_VT * 4 +
         (kvf == KVF_MXFP8 ? (size_t)2 * SS_VT * (dw + 4) : 0);
}

// block = n_rep * (hd / dsplit): thread = (query head hh of the group, column d of the CTA's d-range)
template <int KVF>
__global__ void __launch_bounds__(1024) ss_out_kernel(const StreamAttn P, int dsplit) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t sm[];
  __shared__ double sZ[8];
  const int h = blockIdx.x / dsplit, g = blockIdx.x % dsplit, rl = blockIdx.y, c = blockIdx.z, r = P.row0 + rl;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int n_rep = P.n_rep, dw = P.hd / dsplit, cpr = dw / 8;
  const int T = ss_keys(P, r);
  int t0 = 0, t1 = T;
  if (!P.strict) {
    t0 = c * SS_CH;
    if (t0 >= T) return;
    t1 = min(T, t0 + SS_CH);
  }
  const KeyMap km = ss_key_map(P, r, T);
  uint16_t* sV = reinterpret_cast<uint16_t*>(sm);                       // [2][SS_VT][dw]
  uint16_t* sS = sV + (size_t)2 * SS_VT * dw;                           // [2][n_rep][SS_VT] raw bf16 (score or p)
  float* sP = reinterpret_cast<float*>(sS + (size_t)2 * n_rep * SS_VT); // [n_rep][SS_VT]
  uint32_t* sSl = reinterpret_cast<uint32_t*>(sP + (size_t)n_rep * SS_VT);   // MXFP8: [2][SS_VT] scale slots, [2][SS_VT][dw] codes
  uint8_t* sC = reinterpret_cast<uint8_t*>(sSl + 2 * SS_VT);
  const int hh = tid / dw, dd = tid % dw;
  if (!P.strict && tid < n_rep) {   // Z: the chunk partials in chunk order
    const double* zp = P.zpart + ((size_t)rl * P.n_heads + h * n_rep + tid) * P.n_chunks;
    const int nch = (T + SS_CH - 1) / SS_CH;
    double z = 0.0;
    for (int k = 0; k < nch; k++) z = __dadd_rn(z, zp[k]);
    sZ[tid] = z;
  }
  const uint16_t* vb = P.cache_v + ss_cache_base(P, r) + (size_t)h * P.hd + (size_t)g * dw;
  const uint8_t* vr8 = reinterpret_cast<const uint8_t*>(P.cache_v) + ss_cache_base(P, r);
  auto issue = [&](int k0, int stage) {
    const int n = min(SS_VT, t1 - k0);
    if constexpr (KVF == KVF_MXFP8) {
      ss_issue_fp8(vr8, P.kv_dim, P.n_heads / n_rep * P.hd, h, P.hd, g * dw, dw, k0, n, km, sC + (size_t)stage * SS_VT * dw,
                   sSl + stage * SS_VT, tid, nthr);
    } else {
      uint16_t* v = sV + (size_t)stage * SS_VT * dw;
      for (int i = tid; i < n * cpr; i += nthr) {
        const int t = i / cpr, cc = i % cpr;
        ss_cp16(v + (size_t)t * dw + cc * 8, vb + (size_t)km(k0 + t) * P.kv_dim + cc * 8);
      }
    }
    uint16_t* s = sS + (size_t)stage * n_rep * SS_VT;
    const int n8 = (n + 7) / 8;   // whole 16-byte pieces (t_stride is a multiple of SS_VT: never past the row)
    for (int i = tid; i < n_rep * n8; i += nthr) {
      const int j = i / n8, cc = i % n8;
      ss_cp16(s + (size_t)j * SS_VT + cc * 8, ss_score_row(P, rl, h * n_rep + j) + k0 + cc * 8);
    }
    ss_cp_commit();
  };
  float acc = 0.f;
  issue(t0, 0);
  int stage = 0;
  for (int k0 = t0; k0 < t1; k0 += SS_VT, stage ^= 1) {
    const int n = min(SS_VT, t1 - k0);
    if (k0 + SS_VT < t1) {
      issue(k0 + SS_VT, stage ^ 1);
      ss_cp_wait<1>();
    } else {
      ss_cp_wait<0>();
    }
    __syncthreads();
    if constexpr (KVF == KVF_MXFP8)
      ss_decode_fp8(sC + (size_t)stage * SS_VT * dw, sSl + stage * SS_VT, g * dw, dw, n, sV + (size_t)stage * SS_VT * dw, dw, tid, nthr);
    const uint16_t* s = sS + (size_t)stage * n_rep * SS_VT;
    for (int i = tid; i < n_rep * n; i += nthr) {
      const int j = i / n, t = i % n;
      const float b = bf2f(s[(size_t)j * SS_VT + t]);
      sP[(size_t)j * SS_VT + t] = P.strict ? b : trunc_bf((float)__ddiv_rn(exp((double)b), sZ[j]));   // t(f32(e/Z)) :493
    }
    __syncthreads();
    if (hh < n_rep) {
      const float* ph = sP + (size_t)hh * SS_VT;
      const uint16_t* vc = sV + (size_t)stage * SS_VT * dw + dd;
#pragma unroll 8
      for (int t = 0; t < n; t++) acc = __fmaf_rn(ph[t], bf2f(vc[(size_t)t * dw]), acc);
    }
    __syncthreads();   // stage and sP are refilled next
  }
  if (hh >= n_rep) return;
  const int H = h * n_rep + hh, d = g * dw + dd;
  if (P.strict) ss_store(P, r, H * P.hd + d, acc);
  else P.opart[(((size_t)rl * P.n_heads + H) * P.n_chunks + c) * P.hd + d] = acc;
}

// FAST: o_d = t(sum of the chunk partials in chunk order).  grid (query head, row), block = hd.
__global__ void ss_combine_kernel(const StreamAttn P) {
  pdl_launch_dependents();
  pdl_wait();
  const int H = blockIdx.x, rl = blockIdx.y, r = P.row0 + rl, d = threadIdx.x;
  const int nch = (ss_keys(P, r) + SS_CH - 1) / SS_CH;
  const float* op = P.opart + ((size_t)rl * P.n_heads + H) * P.n_chunks * P.hd + d;
  float acc = 0.f;
  for (int k = 0; k < nch; k++) acc = __fadd_rn(acc, op[(size_t)k * P.hd]);
  ss_store(P, r, H * P.hd + d, acc);
}

}  // namespace lnb
