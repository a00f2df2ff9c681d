// engine.cuh -- the persistent decode engine: ONE kernel launch runs n_steps complete S=1 forward passes
// (LlamaTransformer.Forward, src/model/llamatransformer.go:145-180, driven like generateTokensInternal,
// src/inference/inference.go:194-253) on a grid of one CTA per SM.
//
// Why: a decode step is 160+ short dependent kernels.  As separate launches every one of them pays its own
// launch gap, its own barrier init, its own pipeline ramp (the first weight tile arrives ~1.5 us after the
// kernel starts) and -- with rows / 32 CTAs -- its own wave quantisation (28672 rows of w1|w3 = 896 CTAs on 296
// slots = 3.03 waves: the dominant kernel sat at 0.78 of the HBM roofline for that reason alone).  At 8 GPUs the
// per-kernel work shrinks 8x and the fixed costs are all that is left (round 1: 1.35 ms per token against a
// 0.29 ms roofline).  Here:
//   * the step is a PHASE LIST in device memory (EnginePhase[]: projection, attention, all-reduce, argmax exchange);
//     every CTA walks the same list, phases are separated by a grid barrier (one atomic + one spin per CTA);
//   * every projection's rows are split STATICALLY and evenly over the CTAs at 8-row panel granularity
//     (3584 panels of w1|w3 over 132 CTAs = 27 or 28 each: balance 0.97);
//   * warp 0 of every CTA is a bulk-copy producer that walks the phase list AHEAD of the consumers: weights do not
//     depend on activations, so while the consumers wait at a grid barrier (or for a peer GPU) the ring already
//     fills with the next projection's first tiles -- no ramp;
//   * the arithmetic is the arithmetic of gemv.cuh / kernels.cuh, expression for expression (same truncation points,
//     same summation orders in both accumulation modes): the engine path and the kernel-chain path produce identical
//     bits (tests/test_gpu_engine.py), and LNB_ACC_STRICT stays bit-identical to the oracle.
//
// Thread roles (288 threads): warp 0 = producer (every lane issues one panel's cp.async.bulk per stage of a 4 x 32 KB
// ring), 256 consumers.
//   LNB_ACC_FAST   (KS = 8): row tile = 8 panels (64 rows); consumer (r = c % 32, j = c / 32) owns rows r and r + 32 of the
//                            tile (two independent accumulation chains per thread) in k-stream j.
//   LNB_ACC_STRICT (KS = 1): row tile = up to 16 panels; consumer c < 128 = row c of the tile, one sequential chain per row,
//                            the four chain warps sit on four different schedulers (a CTA that owns <= 4 panels of a
//                            latency-bound projection runs ONE chain warp with its scheduler to itself).
// Shared memory: 1 KB header (mbarriers, scalars, the phase's GemvParams) + 128 KB weight ring + 84 KB work area
// (the activation vector as f32 / the attention phase's K, V, scores).
//
// Everything that can wait on another CTA or another GPU is bounded: grid barrier, stage barriers and peer waits give up
// after (a multiple of) timeout_ns, write the reason to a host-mapped word and trap -- a late or dead rank becomes an
// error on its peers (LNB_ETIMEOUT / LNB_ECUDA with the reason in lnb_last_error), never a hung GPU.
#pragma once
#include "gemv.cuh"
#include "kernels.cuh"
#include "seqsum.cuh"
#include "wpack.cuh"

namespace lnb {

enum { EP_GEMV = 0, EP_SDPA = 1, EP_REDUCE = 2, EP_ARGMAX = 3 };
enum {
  EF_X_TOKEN = 1,    // x   = embedding row of the step's input token (ml.Fwd_Get_Rows, operations_impl.go:142-173)
  EF_RES_TOKEN = 2,  // res = the same row (the residual stream of layer 0 is the embedding)
  EF_GRID_SYNC = 4   // grid barrier after this phase (the LM head: its argmax key must be complete before anyone reads it)
};

struct EnginePhase {
  int type, pro, epi, flags;
  int N, K, kt, ldx;
  const uint16_t* W;
  const uint8_t* Wp;        // STRICT: the packed copy of W (wpack.cuh) and its unit bytes [N/8][k-tiles], NULL: stream W
  const uint8_t* Wu;
  const uint16_t* x;        // GEMV: activations [K] / REDUCE: residual [dim]
  const uint16_t* norm_w;
  const uint16_t* res;
  uint16_t* out_bf16;       // GEMV output / REDUCE output
  float* out_f32;
  int ldo, n_offset;
  uint16_t* cache_k;        // this layer's caches (offset to the active sequence): QKV epilogue, SDPA
  uint16_t* cache_v;
  const uint16_t* q;        // SDPA in / out (plain buffers; unused when the tagged vectors are set)
  uint16_t* o;
  int q_dim, kv_dim;        // local widths (per tensor-parallel rank)
  // Activations between phases of one step travel as self-validating 4-byte words {tag:16 | bf16:16}: the consumer polls
  // the words of the vector it needs until they carry the producer phase's tag -- no grid barrier, and the wait is the load.
  // tag(step, phase) = tag_base + step * n_phases + phase (the host keeps it below 2^16 and the buffers' old tags dead).
  const uint32_t* x_t;      // tagged input vector (GEMV prologue / SDPA: q | k | v of this step), NULL: plain `x` / token
  const uint32_t* res_t;    // tagged residual (EPI_RESID / REDUCE), NULL: plain `res` / token
  uint32_t* out_t;          // tagged output vector, NULL: plain outputs
  int x_delta, res_delta;   // how many phases earlier (same step) the tagged input / residual was produced
};

struct EngineParams {
  const EnginePhase* phases;
  int n_phases, n_steps;
  LnbDevState* st;
  const uint16_t* emb;
  int dim, head_dim, n_rep, seq_len;
  const float* cis;
  const uint16_t* silu_tab;
  float eps, attn_scale;
  int strict;
  int32_t* tok_out;
  unsigned int* bar_ctr;    // grid barrier counter, zeroed by the host before the launch
  LnbP2P p2p;
  int tp;
  unsigned long long timeout_ns;
  volatile uint32_t* err_host;   // host-mapped word: why the engine trapped (see eng_fail)
  unsigned int pf_window;        // bytes of a projection's stream each CTA prefetches into L2 beyond its ring when it reaches the phase (0: none)
  unsigned int tag_base;         // tag of (step 0, phase 0)
  unsigned long long* prof;      // NULL, or [gridDim.x][ENG_NPROF] cycle sums of consumer thread 0: 0 grid barrier, 1 prologue,
                                 // 2 main loop (stage waits included), 3 combine + epilogue, 4 attention, 5 peer reduce / argmax
  int advance;              // 1: decode-loop bookkeeping (tok_out[step], st->pos / st->step advance)
};

constexpr int ENG_NCONS = 256;
constexpr int ENG_THREADS = ENG_NCONS + 64;                // + producer warp (warp 0) + L2-prefetch warp (warp 9)
constexpr int ENG_RING = 128 * 1024;
constexpr int ENG_WORK = 84 * 1024;
constexpr int ENG_XMAX = 56 * 1024;                       // f32 activation vector: K <= 14336
constexpr int ENG_PART_OFF = ENG_XMAX;                    // [8][64] f32 stream partials (FAST), 2 KB
constexpr int ENG_SCAN_OFF = ENG_XMAX + 2048;             // seg-scan scratch (STRICT RMSNorm), 4 KB
constexpr int ENG_NPROF = 12;                              // per-CTA cycle counters (LNB_ENGINE_PROF): see EngineParams.prof
constexpr int ENG_SMEM = 1024 + ENG_RING + ENG_WORK;
template <int KS> struct EngCfg {
  static constexpr int kNST = 4;
  static constexpr int kStage = ENG_RING / kNST;          // 32 KB
  static constexpr int kPT = (KS == 1) ? 16 : 8;          // panels per row tile
  // STRICT: consumer warps 0..3 are the chain warps (hardware warps 1..4 = one per scheduler); warps 4..7 only help with
  // prologues / attention / reductions and park at the phase's closing barrier meanwhile (bar.sync costs no issue slots)
  static constexpr int kChainWarps = (KS == 1) ? 4 : 8;
};

// host + device: panels [lo, hi) of a matrix with P panels owned by CTA b of G
__host__ __device__ inline void eng_split(int P, int b, int G, int* lo, int* hi) {
  *lo = (int)(((long long)P * b) / G);
  *hi = (int)(((long long)P * (b + 1)) / G);
}
// k-tile of a row tile with np panels: the phase's kt (sized for full tiles), doubled while the stage has room -- a row
// tile of 1 panel at kt = 256 would move 4 KB per stage and crawl at the ring's latency (4 stages x 4 KB per ~1.2 us).
// FAST only: the STRICT chain tiles are compile-time unrolled for kt <= 512.
__host__ __device__ inline int eng_tile_kt(int ks, int np, int K, int kt, int stage_bytes) {
  if (ks == 1 || true) return kt;   // (k-tile scaling: kept for the record, disabled)
  while (kt * 2 <= K && kt * 2 <= 2048 && np * (kt * 2) * 16 <= stage_bytes && K % (kt * 2) == 0) kt *= 2;
  return kt;
}
// shared-memory need of the attention phase for T_max rows
__host__ __device__ inline size_t eng_sdpa_smem(int T_max, int hd, int n_rep) {
  return (size_t)T_max * ((hd + 8) + hd) * 2 + (size_t)n_rep * ((size_t)T_max * 12 + (size_t)hd * 4) + (size_t)n_rep * 5 * 8 + 64;
}

struct EngCtl {            // in the header, after the barriers
  int pos;
  int tok;
  volatile unsigned long long ld_bytes;   // weight bytes the producer has issued so far (the prefetch warp stays ahead of it)
};

// Fatal, loud, never a hang: the reason goes to a host-mapped word (readable after the context died), then trap.
// codes: 0xC0000000 | barrier target  = a CTA never reached a grid barrier;  0xD0000000 | stage  = a weight tile never
// arrived / was never released;  0x80000000 | epoch << 4 | rank  = a tensor-parallel peer never delivered (common.cuh).
LNB_DEVINL void eng_fail(volatile uint32_t* err_host, uint32_t code) {
  if (err_host) {
    *err_host = code;
    __threadfence_system();
  }
  __trap();
}

LNB_DEVINL uint32_t ld_acquire_u32(const unsigned int* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
LNB_DEVINL uint4 ldcg_u4(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
LNB_DEVINL uint32_t ldcg_u32(const void* p) { return __ldcg(reinterpret_cast<const unsigned int*>(p)); }
LNB_DEVINL uint16_t ldcg_u16(const void* p) { return __ldcg(reinterpret_cast<const unsigned short*>(p)); }

// bounded mbarrier wait (a stage that never completes is a bug or a dead copy engine: trap instead of hanging the GPU)
LNB_DEVINL void eng_mbar_wait(uint64_t* bar, uint32_t parity, volatile uint32_t* err_host, unsigned long long timeout_ns, bool backoff,
                              uint32_t what) {
  uint32_t spins = 0;
  unsigned long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (backoff) __nanosleep(LNB_BACKOFF_NS);
    if ((++spins & 4095u) == 0u && timeout_ns) {
      const unsigned long long now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4 * timeout_ns) eng_fail(err_host, 0xD0000000u | (what & 0xffffffu));
    }
  }
}

// Grid barrier among the consumers of all CTAs (the producer warps never take part).  Called by all ENG_NCONS
// consumer threads; `target` = barriers so far * gridDim.x.
LNB_DEVINL void eng_grid_barrier(const EngineParams& P, unsigned int target, int c) {
  named_bar_sync(1, ENG_NCONS);                      // every consumer's stores happen-before thread 0's release
  if (c == 0) {
#ifdef ENG_OLD_BARRIER
    __threadfence();
    atomicAdd(P.bar_ctr, 1u);
#else
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(P.bar_ctr) : "memory");
#endif
    unsigned long long t0 = 0;
    uint32_t spins = 0;
    while (ld_acquire_u32(P.bar_ctr) < target) {
      if ((++spins & 1023u) == 0u && P.timeout_ns) {
        const unsigned long long now = global_timer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > 2 * P.timeout_ns) eng_fail(P.err_host, 0xC0000000u | (target & 0xffffffu));
      }
    }
#ifdef ENG_OLD_BARRIER
    __threadfence();
#endif
  }
  named_bar_sync(1, ENG_NCONS);
}
// peer wait inside the engine: the bounded wait of common.cuh, fatal on timeout
LNB_DEVINL uint2 eng_wait_word(const EngineParams& P, const uint2* src, uint32_t epoch, int r, unsigned long long t0) {
  uint2 w;
  if (!p2p_wait_word(src, epoch, r, P.p2p, P.st, t0, &w)) eng_fail(P.err_host, 0x80000000u | ((epoch & 0xffffffu) << 4) | (uint32_t)(r & 15));
  return w;
}

// ---- LNB_ACC_STRICT RMSNorm sum of squares: the one-pass binade scan of seqsum.cuh (rms_scale_seg_kernel) for the
// consumers of an engine CTA.  s_x = the row as f32 in shared memory (D = NT * CH elements); threads t >= NT only
// take part in the barriers.  Returns the reference's sequential fp32 sum (valid on every thread via *s_out).
template <int CH>
LNB_DEVINL void eng_seq_sumsq(const float* s_x, int t, int NT, uint8_t* scratch, float* s_out, unsigned long long* prof = nullptr) {
  long long tp0 = (prof && t == 0) ? clock64() : 0;   // profile slots 7 (squares, prediction, maps, warp scan), 9 (walk)
  uint32_t* s_run_i0 = reinterpret_cast<uint32_t*>(scratch);            // [256]
  uint32_t* s_run_i1 = s_run_i0 + 256;                                   // [256]
  uint16_t* s_run_end = reinterpret_cast<uint16_t*>(s_run_i1 + 256);     // [256]
  uint8_t* s_code = reinterpret_cast<uint8_t*>(s_run_end + 256);         // [256]
  float* s_wsum = reinterpret_cast<float*>(s_code + 256);                // [8]
  const int lane = t & 31, wid = t >> 5, nw = NT >> 5;
  const bool on = t < NT;
  float sq[CH];
  float inc = 0.f;
  if (on) {
    // 128-bit loads: a thread's CH consecutive floats, read one by one, would be a CH-way bank conflict (stride CH words)
    if (CH % 4 == 0) {
#pragma unroll
      for (int k = 0; k < CH; k += 4) {
        const float4 v = *reinterpret_cast<const float4*>(s_x + t * CH + k);
        sq[k] = __fmul_rn(v.x, v.x); sq[k + 1] = __fmul_rn(v.y, v.y);
        sq[k + 2] = __fmul_rn(v.z, v.z); sq[k + 3] = __fmul_rn(v.w, v.w);
      }
    } else {
#pragma unroll
      for (int k = 0; k < CH; k++) {
        const float v = s_x[t * CH + k];
        sq[k] = __fmul_rn(v, v);
      }
    }
    float cs = 0.f;
#pragma unroll
    for (int k = 0; k < CH; k++) cs = __fadd_rn(cs, sq[k]);
    inc = cs;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const float v = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc = __fadd_rn(inc, v);
    }
    if (lane == 31) s_wsum[wid] = inc;
    s_run_end[t] = 0;
  }
  named_bar_sync(1, ENG_NCONS);
  if (on) {
    // approximate prefix sums (any rounding will do: they only PREDICT the binade of every chunk)
    float wpre = 0.f;
    {
      float wv = (lane < nw) ? s_wsum[lane] : 0.f;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, wv, d);
        if (lane >= d) wv = __fadd_rn(wv, u);
      }
      const float p = __shfl_sync(0xffffffffu, wv, (wid + 31) & 31);
      if (wid > 0) wpre = p;
    }
    float before = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) before = 0.f;
    before = __fadd_rn(before, wpre);
    const float after = __fadd_rn(inc, wpre);
    const int code = (t == 0) ? 0 : seq_predict(before, after);
    s_code[t] = (uint8_t)code;
    SeqSeg v;
    v.m.i0 = v.m.i1 = 0u;
    if (code) {
#pragma unroll
      for (int k = 0; k < CH; k++) v.m = seq_compose(v.m, seq_term(__float_as_uint(sq[k]), code));
    }
    // runs of equally predicted chunks, folded into one parity map per run -- WITHIN the warp only: a run that crosses a
    // warp boundary is published as two runs (the walk takes one more jump; the cross-warp scan and two barriers are gone)
    const int pc = __shfl_up_sync(0xffffffffu, code, 1), nc = __shfl_down_sync(0xffffffffu, code, 1);
    v.flag = (code == 0 || pc != code || lane == 0) ? 1u : 0u;   // uncertain chunks are runs of their own (never jumped)
    v.head = (uint32_t)t;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      SeqSeg o;
      o.flag = __shfl_up_sync(0xffffffffu, v.flag, d);
      o.head = __shfl_up_sync(0xffffffffu, v.head, d);
      o.m.i0 = __shfl_up_sync(0xffffffffu, v.m.i0, d);
      o.m.i1 = __shfl_up_sync(0xffffffffu, v.m.i1, d);
      if (lane >= d) v = seq_seg_op(o, v);
    }
    if (code && (nc != code || lane == 31)) {        // last chunk of a run: publish the run at its head
      s_run_end[v.head] = (uint16_t)(t + 1);
      s_run_i0[v.head] = v.m.i0;
      s_run_i1[v.head] = v.m.i1;
    }
  }
  named_bar_sync(1, ENG_NCONS);
  if (prof && t == 0) { const long long n_ = clock64(); prof[7] += (unsigned long long)(n_ - tp0); tp0 = n_; }
  if (t == 0) {                                      // the walk: jump over runs, real FADDs everywhere else
    uint32_t sb = 0u;
    int cidx = 0;
    while (cidx < NT) {
      const int e = (int)s_run_end[cidx];
      const int E = (int)s_code[cidx];
      SeqInc run;
      run.i0 = s_run_i0[cidx]; run.i1 = s_run_i1[cidx];
      uint32_t nb;
      if (e > cidx && seq_try_jump(sb, E, run, &nb)) { sb = nb; cidx = e; continue; }
      float s = __uint_as_float(sb);
      float xs[CH];
#pragma unroll
      for (int k = 0; k < CH; k++) xs[k] = s_x[cidx * CH + k];       // (vectorised by the compiler: the row is 16-byte aligned)
#pragma unroll
      for (int k = 0; k < CH; k++) s = __fadd_rn(s, __fmul_rn(xs[k], xs[k]));
      sb = __float_as_uint(s);
      cidx++;
    }
    *s_out = __uint_as_float(sb);
    if (prof) { const long long n_ = clock64(); prof[9] += (unsigned long long)(n_ - tp0); prof[10] += 1ull; }
  }
  named_bar_sync(1, ENG_NCONS);
}
// (CH, NT) for a row of D elements with at most 256 threads; false: no engine for this model width
__host__ __device__ inline bool eng_scan_shape(int D, int* ch, int* nt) {
  const int cand[4] = {16, 8, 4, 2};
  for (int i = 0; i < 4; i++) {
    const int c = cand[i];
    if (D % c == 0 && (D / c) % 32 == 0 && D / c <= ENG_NCONS && D / c >= 32) { *ch = c; *nt = D / c; return true; }
  }
  return false;
}

// One k-tile of NG groups of 4 chunks (NG * 32 elements) of ONE row's sequential accumulation chain: register
// double-buffered like gemv.cuh's MB == 1 branch -- the LDS of group g+1 are in flight while the 32 dependent FMAs of
// group g issue -- and fully unrolled (a run-time group loop left ptxas with two rotating temporaries and a chain that
// ran at 12 cycles per element instead of 5).
template <int NG>
LNB_DEVINL float eng_chain_tile(const uint8_t* __restrict__ tile, const float* __restrict__ xt, float acc) {
  uint4 wa[4], wb[4];
  float4 xa0[4], xa1[4], xb0[4], xb1[4];
#define ENG_LOAD(gi, W_, X0_, X1_)                                            \
  _Pragma("unroll") for (int q_ = 0; q_ < 4; q_++) {                          \
    const int ch_ = (gi) * 4 + q_;                                            \
    W_[q_] = *reinterpret_cast<const uint4*>(tile + ch_ * 128);               \
    X0_[q_] = *reinterpret_cast<const float4*>(xt + ch_ * 8);                 \
    X1_[q_] = *reinterpret_cast<const float4*>(xt + ch_ * 8 + 4);             \
  }
#define ENG_FMA(W_, X0_, X1_)                                                 \
  _Pragma("unroll") for (int q_ = 0; q_ < 4; q_++) {                          \
    float a_ = acc;                                                           \
    a_ = __fmaf_rn(X0_[q_].x, bf_lo(W_[q_].x), a_);                           \
    a_ = __fmaf_rn(X0_[q_].y, bf_hi(W_[q_].x), a_);                           \
    a_ = __fmaf_rn(X0_[q_].z, bf_lo(W_[q_].y), a_);                           \
    a_ = __fmaf_rn(X0_[q_].w, bf_hi(W_[q_].y), a_);                           \
    a_ = __fmaf_rn(X1_[q_].x, bf_lo(W_[q_].z), a_);                           \
    a_ = __fmaf_rn(X1_[q_].y, bf_hi(W_[q_].z), a_);                           \
    a_ = __fmaf_rn(X1_[q_].z, bf_lo(W_[q_].w), a_);                           \
    a_ = __fmaf_rn(X1_[q_].w, bf_hi(W_[q_].w), a_);                           \
    acc = a_;                                                                 \
  }
  ENG_LOAD(0, wa, xa0, xa1)
#pragma unroll
  for (int gi = 0; gi < NG; gi += 2) {
    if (gi + 1 < NG) { ENG_LOAD(gi + 1, wb, xb0, xb1) }
    ENG_FMA(wa, xa0, xa1)
    if (gi + 2 < NG) { ENG_LOAD(gi + 2, wa, xa0, xa1) }
    if (gi + 1 < NG) { ENG_FMA(wb, xb0, xb1) }
  }
#undef ENG_LOAD
#undef ENG_FMA
  return acc;
}
// The same chain over a packed unit (wpack.cuh): NG groups of 384 bytes, each decoded to the bf16 words eng_chain_tile
// reads and fed to the same FMAs in the same order.  The decode does not depend on the accumulator, so it is software-
// pipelined: the pair words of group g + 1 are decoded between the dependent FMAs of group g (decoded just before its own
// FMAs, a chunk cost its decode latency on top of its FMA chain: ~14 cycles per weight instead of the issue rate), and the
// packed words of group g + 2 are loaded meanwhile.  NG = 0: a run-time number of groups (unit lengths other than 64..512).
LNB_DEVINL uint32_t eng_wp_pair(const uint4 (&w)[3], int q, int p, uint32_t bb) {
  const uint4& s = (q < 2) ? w[0] : w[1];                    // sign|mantissa bytes: chunks 0, 1 then 2, 3
  const uint32_t sm = (q & 1) ? ((p < 2) ? s.z : s.w) : ((p < 2) ? s.x : s.y);
  const uint32_t cw = (q == 0) ? w[2].x : (q == 1) ? w[2].y : (q == 2) ? w[2].z : w[2].w;
  switch (p) {
    case 0: return wp_pair<0>(sm, cw, bb);
    case 1: return wp_pair<1>(sm, cw, bb);
    case 2: return wp_pair<2>(sm, cw, bb);
    default: return wp_pair<3>(sm, cw, bb);
  }
}
template <int NG>
LNB_DEVINL float eng_chain_tile_wp(const uint8_t* __restrict__ unit, const float* __restrict__ xt, float acc, uint32_t bb, int ng = NG) {
  auto ld = [&](int g, uint4 (&w)[3]) {
    w[0] = *reinterpret_cast<const uint4*>(unit + g * WP_GROUP_BYTES);
    w[1] = *reinterpret_cast<const uint4*>(unit + g * WP_GROUP_BYTES + 128);
    w[2] = *reinterpret_cast<const uint4*>(unit + g * WP_GROUP_BYTES + 256);
  };
  auto fma_pair = [&](const float* x, uint32_t w) {
    acc = __fmaf_rn(x[0], bf_lo(w), acc);
    acc = __fmaf_rn(x[1], bf_hi(w), acc);
  };
  if (NG == 0) {
    for (int g = 0; g < ng; g++) {
      uint4 w[3];
      ld(g, w);
#pragma unroll
      for (int q = 0; q < 4; q++)
#pragma unroll
        for (int p = 0; p < 4; p++) fma_pair(xt + g * 32 + q * 8 + p * 2, eng_wp_pair(w, q, p, bb));
    }
    return acc;
  }
  uint4 pw[2][3];                 // packed words: group g + 1 in pw[(g + 1) & 1], group g + 2 loading into pw[g & 1]
  uint32_t cur[16], nxt[16];      // pair words of groups g and g + 1
  ld(0, pw[0]);
  if (NG > 1) ld(1, pw[1]);
#pragma unroll
  for (int i = 0; i < 16; i++) cur[i] = eng_wp_pair(pw[0], i >> 2, i & 3, bb);
#pragma unroll
  for (int g = 0; g < NG; g++) {
    if (g + 2 < NG) ld(g + 2, pw[g & 1]);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const float4 x0 = *reinterpret_cast<const float4*>(xt + g * 32 + q * 8);
      const float4 x1 = *reinterpret_cast<const float4*>(xt + g * 32 + q * 8 + 4);
      const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
      for (int p = 0; p < 4; p++) {
        if (g + 1 < NG) nxt[q * 4 + p] = eng_wp_pair(pw[(g + 1) & 1], q, p, bb);
        fma_pair(xs + p * 2, cur[q * 4 + p]);
      }
    }
#pragma unroll
    for (int i = 0; i < 16; i++) cur[i] = nxt[i];
  }
  return acc;
}

// four consecutive words of a tagged vector, polled until all of them carry `tag_hi`
// (relaxed at gpu scope, not volatile: volatile loads are kept in order by the hardware, one L2 round trip each -- a
// thread's 4..14 polling loads of a prologue must be in flight together)
LNB_DEVINL uint4 ld_volatile_u4(const uint32_t* p) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
LNB_DEVINL bool tags_ok(const uint4& v, uint32_t tag_hi) {
  return (((v.x ^ tag_hi) | (v.y ^ tag_hi) | (v.z ^ tag_hi) | (v.w ^ tag_hi)) & 0xffff0000u) == 0u;
}
LNB_DEVINL uint4 wait_tagged4(const uint32_t* p, uint32_t tag_hi, volatile uint32_t* err_host, unsigned long long timeout_ns) {
  uint4 v = ld_volatile_u4(p);
  uint32_t spins = 0;
  unsigned long long t0 = 0;
  while (!tags_ok(v, tag_hi)) {
    if ((++spins & 1023u) == 0u && timeout_ns) {
      const unsigned long long now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 2 * timeout_ns) eng_fail(err_host, 0xE0000000u | (tag_hi >> 16));   // 0xE...: a tagged activation never arrived
    }
    v = ld_volatile_u4(p);
  }
  return v;
}
LNB_DEVINL float tagged_f32(uint32_t w) { return __uint_as_float(w << 16); }

LNB_DEVINL void l2_prefetch_bulk(const void* gsrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}

// The engine's scan as a kernel of its own (op-level C-ABI, algo 4): one row per CTA, 256 threads -- lets the adversarial-row
// tests of the standalone scan kernels (zeros, subnormals, binade crossings, inf) run against this variant too.
template <int CH>
__global__ void __launch_bounds__(ENG_NCONS) eng_rms_scale_kernel(const uint16_t* __restrict__ x, int ldx, float* __restrict__ r, int D, float eps) {
  extern __shared__ __align__(16) uint8_t sm[];
  float* s_x = reinterpret_cast<float*>(sm);
  uint8_t* scr = sm + (size_t)D * 4;
  __shared__ float s_sum;
  const int t = threadIdx.x;
  for (int k = t; k < D; k += ENG_NCONS) s_x[k] = bf2f(x[(size_t)blockIdx.x * ldx + k]);
  named_bar_sync(1, ENG_NCONS);
  eng_seq_sumsq<CH>(s_x, t, D / CH, scr, &s_sum);
  if (t == 0) {
    const float me = __fadd_rn(__fdiv_rn(s_sum, (float)D), eps);
    r[blockIdx.x] = (float)(1.0 / sqrt((double)me));
  }
}

// ------------------------------------------------------------------------------------------------------------
template <int KS>
__global__ void __launch_bounds__(ENG_THREADS, 1) decode_engine_kernel(const EngineParams P) {
  using Cfg = EngCfg<KS>;
  constexpr int NST = Cfg::kNST, STAGE = Cfg::kStage, PT = Cfg::kPT;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);              // [NST]
  uint64_t* empty_bar = full_bar + NST;                                // [NST]
  uint8_t* s_unit = smem + 64;                                         // [NST][PT] unit bytes of a packed phase's stages
  static_assert(64 + NST * PT <= 256, "unit bytes must fit below s_scalar");
  float* s_scalar = reinterpret_cast<float*>(smem + 256);              // rms scale etc.
  EngCtl* ctl = reinterpret_cast<EngCtl*>(smem + 320);
  GemvParams* gp = reinterpret_cast<GemvParams*>(smem + 512);          // the running phase as the epilogues see it
  uint8_t* s_ring = smem + 1024;
  uint8_t* s_work = s_ring + ENG_RING;
  float* s_x = reinterpret_cast<float*>(s_work);
  float* s_part = reinterpret_cast<float*>(s_work + ENG_PART_OFF);
  static_assert(sizeof(GemvParams) <= 512, "GemvParams must fit the header");

  const int tid = threadIdx.x;
  const int G = gridDim.x, bid = blockIdx.x;
  if (tid == 0) {
    for (int s = 0; s < NST; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], Cfg::kChainWarps * 32);
    }
    mbar_fence_init();
    ctl->ld_bytes = 0ull;
  }
  __syncthreads();

  if (tid < 32) {
    // =========================== producer: walks the phase list ahead of the consumers ===========================
    // lanes 0..np-1 issue one panel's copy of a stage each (ptxas serialises them through the uniform datapath: ~50 cycles
    // per copy, which is why copies are kept >= 2 KB); lane 0 owns the barrier bookkeeping.
    const uint64_t pol = l2_policy_evict_first();
    uint32_t seq = 0;
    unsigned long long issued = 0;
    for (int step = 0; step < P.n_steps; step++) {
      for (int ph = 0; ph < P.n_phases; ph++) {
        const EnginePhase* E = P.phases + ph;
        if (E->type != EP_GEMV) continue;
        const int K = E->K, kt = E->kt;
        const int n_tiles = (K + kt - 1) / kt;
        int p0, p1;
        eng_split(E->N / 8, bid, G, &p0, &p1);
        const uint8_t* wbase = reinterpret_cast<const uint8_t*>(E->W);
        const uint8_t* pbase = (KS == 1) ? E->Wp : nullptr;   // packed phase: each panel's unit byte picks its source
        for (int rt = p0; rt < p1; rt += PT) {
          const int np = min(PT, p1 - rt);
          const uint8_t* src_row = wbase + (size_t)(rt + tid) * (size_t)K * 16u;
          const uint8_t* psrc_row = pbase ? pbase + (size_t)(rt + tid) * (size_t)K * 12u : nullptr;
          const int kt = eng_tile_kt(KS, np, K, E->kt, STAGE);
          const int n_tiles = (K + kt - 1) / kt;
          const uint8_t* urow = pbase ? E->Wu + (size_t)(rt + tid) * (size_t)n_tiles : nullptr;
          uint32_t u_next = (pbase && tid < np) ? (uint32_t)__ldg(urow) : (uint32_t)WP_RAW;
          for (int t = 0; t < n_tiles; t++, seq++) {
            const int s = seq % NST;
            const uint32_t par = (seq / NST) & 1u;
            const int k0 = t * kt;
            const uint32_t len = (uint32_t)min(kt, K - k0);
            // the unit byte of the next k-tile is loaded one stage ahead: its latency hides behind this stage's wait and issue
            const uint32_t u = u_next;
            if (pbase && tid < np && t + 1 < n_tiles) u_next = (uint32_t)__ldg(urow + t + 1);
            const bool packed = u != (uint32_t)WP_RAW;
            const uint32_t my_bytes = tid < np ? len * (packed ? 12u : 16u) : 0u;
            const uint32_t stage_bytes = pbase ? __reduce_add_sync(0xffffffffu, my_bytes) : len * 16u * (uint32_t)np;
            // every issuing lane observes the stage's release itself (an acquire by lane 0 plus __syncwarp orders the
            // other lanes' copies too, but compute-sanitizer's racecheck does not follow that edge for async-proxy writes)
            eng_mbar_wait(&empty_bar[s], par ^ 1u, P.err_host, P.timeout_ns, false, seq);
            if (pbase && tid < np) s_unit[s * PT + tid] = (uint8_t)u;   // published by lane 0's arrive below
            __syncwarp();
            if (tid == 0) mbar_expect_tx(&full_bar[s], stage_bytes);
            __syncwarp();
            if (tid < np)
              bulk_g2s(s_ring + (size_t)s * STAGE + (size_t)tid * ((size_t)kt * 16),
                       packed ? psrc_row + (size_t)k0 * 12u : src_row + (size_t)k0 * 16u, my_bytes, &full_bar[s], pol);
            issued += (unsigned long long)stage_bytes;
            if (tid == 0) ctl->ld_bytes = issued;
          }
        }
      }
    }
    return;
  }
  if (tid >= 32 + ENG_NCONS) {
    // =========================== L2 prefetcher: the same walk, pf_window bytes ahead of the producer ==============
    // The ring holds 128 KB per SM = 19 MB per chip = 3 us of HBM time, but a phase boundary (inputs of the next projection
    // still being produced, prologue, attention) stalls the consumers longer than that.  This warp asks L2 for the stream
    // beyond the ring, so that HBM keeps working through the stall and the ring then refills at L2 speed.
    if (P.pf_window == 0) return;
    const int lane = tid & 31;
    unsigned long long pf = 0;
    const unsigned long long lead = (unsigned long long)NST * STAGE;   // the ring itself: not worth prefetching
    for (int step = 0; step < P.n_steps; step++) {
      for (int ph = 0; ph < P.n_phases; ph++) {
        const EnginePhase* E = P.phases + ph;
        if (E->type != EP_GEMV) continue;
        const int K = E->K, kt = E->kt;
        const int n_tiles = (K + kt - 1) / kt;
        int p0, p1;
        eng_split(E->N / 8, bid, G, &p0, &p1);
        // (a packed phase: the packed copy, whatever the units' bytes say -- a hint, not a copy)
        const bool pk = KS == 1 && E->Wp;
        const uint8_t* wbase = pk ? E->Wp : reinterpret_cast<const uint8_t*>(E->W);
        const uint32_t epc = pk ? 12u : 16u;   // bytes per column of a panel
        for (int rt = p0; rt < p1; rt += PT) {
          const int np = min(PT, p1 - rt);
          const int kt = eng_tile_kt(KS, np, K, E->kt, STAGE);
          const int n_tiles = (K + kt - 1) / kt;
          for (int t = 0; t < n_tiles; t++) {
            const uint32_t bpp = (uint32_t)min(kt, K - t * kt) * epc;
            const unsigned long long tile_bytes = (unsigned long long)bpp * (unsigned long long)np;
            unsigned long long ld = ctl->ld_bytes;
            uint32_t spins = 0;
            while (pf > ld + lead + (unsigned long long)P.pf_window) {   // far enough ahead: wait for the producer
              __nanosleep(200);
              ld = ctl->ld_bytes;
              if (++spins > (1u << 26)) return;
            }
            if (pf >= ld + lead && lane < np)
              l2_prefetch_bulk(wbase + ((size_t)(rt + lane) * (size_t)K + (size_t)t * kt) * epc, bpp);
            pf += tile_bytes;
          }
        }
      }
    }
    return;
  }

  // ======================================= consumers =============================================================
  const int c = tid - 32;
  const int lane = tid & 31;
  const int cw = c >> 5;
  const int r = (KS == 1) ? c : (c & 31);     // row within the row tile
  const int j = (KS == 1) ? 0 : (c >> 5);     // k-stream
  uint32_t seq = 0;                           // stages consumed so far (same count as the producer's)
  unsigned int n_bar = 0;                     // grid barriers passed
  uint32_t epoch = (P.tp > 1) ? P.st->ar_epoch : 0u;
  int pos = P.st->pos;
  int tok = P.st->next_token;
  // the greedy-argmax key is double-buffered by step parity: with ONE grid barrier per step the key of step s can only be
  // cleared once every CTA has passed the barrier of step s + 1 (everyone read it right after barrier s)
  unsigned long long* const keys[2] = {&P.st->amax_key, &P.st->amax_key_b};
  if (bid == 0 && c == 0) {
    *keys[0] = LNB_ARGMAX_EMPTY;
    *keys[1] = LNB_ARGMAX_EMPTY;
    __threadfence();                          // before any of this CTA's outputs, which every LM-head atomicMax depends on
  }
  long long t_mark = (P.prof && c == 0) ? clock64() : 0;       // LNB_ENGINE_PROF: where consumer thread 0 spends its cycles

  for (int step = 0; step < P.n_steps; step++) {
    if (c == 0) { ctl->pos = pos; ctl->tok = tok; }
    for (int ph = 0; ph < P.n_phases; ph++) {
      const EnginePhase* E = P.phases + ph;
      const int type = E->type;
      const uint32_t tag_now = P.tag_base + (uint32_t)step * (uint32_t)P.n_phases + (uint32_t)ph;
      if (type == EP_GEMV) {
        const int K = E->K, kt = E->kt;
        const int n_tiles = (K + kt - 1) / kt;
        int p0, p1;
        eng_split(E->N / 8, bid, G, &p0, &p1);
        const int flags = E->flags;
        const uint16_t* xg = (flags & EF_X_TOKEN) ? P.emb + (size_t)tok * P.dim : E->x;
        const uint32_t* xtg = (flags & EF_X_TOKEN) ? nullptr : E->x_t;
        const uint32_t x_tag_hi = (tag_now - (uint32_t)E->x_delta) << 16;
        if (p1 > p0) {
          // ---- prologue: activations -> f32 in shared memory (gemv.cuh prologue, MB = 1) -----------------------
          // all global loads of a thread are issued before the first shared-memory store (the compiler cannot prove
          // that the generic pointers do not alias shared memory and would serialise them, one L2 round trip each)
          float* s_nw = s_x + K;                              // RMSNorm weights as f32 (K = dim here: 2 * K * 4 <= ENG_XMAX)
          {
            const int n_ch = K / 8;
            const bool with_w = (E->pro == PRO_RMSNORM);
            for (int base = 0; base < n_ch; base += ENG_NCONS * 4) {
              uint4 xv[4], xv2[4], wv[4];
#pragma unroll
              for (int u = 0; u < 4; u++) {
                const int ch = base + u * ENG_NCONS + c;
                if (ch < n_ch) {
                  if (xtg) {   // tagged words: 8 elements = 2 x 16 bytes; validated below
                    xv[u] = ld_volatile_u4(xtg + (size_t)ch * 8);
                    xv2[u] = ld_volatile_u4(xtg + (size_t)ch * 8 + 4);
                  } else {
                    xv[u] = ldcg_u4(xg + (size_t)ch * 8);
                  }
                  if (with_w) wv[u] = __ldg(reinterpret_cast<const uint4*>(E->norm_w + (size_t)ch * 8));
                }
              }
          // ---- the phase as gemv_epilogue sees it ------------------------------------------------------------
                  if (c == 0 && base == 0) {   // (while this thread's input loads are in flight)
                GemvParams g{};
                g.W = E->W; g.N = E->N; g.K = K; g.M = 1;
                g.x = xg; g.ldx = E->ldx; g.norm_w = E->norm_w; g.eps = P.eps;
                g.out_bf16 = E->out_bf16; g.out_f32 = E->out_f32; g.ldo = E->ldo;
                g.res = (flags & EF_RES_TOKEN) ? P.emb + (size_t)tok * P.dim : E->res;
                g.q_dim = E->q_dim; g.kv_dim = E->kv_dim; g.head_dim = P.head_dim;
                g.cache_k = E->cache_k; g.cache_v = E->cache_v; g.pos_arr = nullptr; g.cache_seq_stride = 0;
                g.cis = P.cis; g.silu_tab = P.silu_tab;
                g.n_offset = E->n_offset; g.st = P.st; g.amax_key_ptr = keys[step & 1]; g.argmax_row = 0; g.publish = 0; g.advance = 0; g.tok_out = nullptr;
                g.pos_ptr = &ctl->pos; g.m_off = 0;
                g.p2p = P.p2p;
                g.ar_epoch_override = epoch;
                g.out_t = E->out_t; g.tag_hi = tag_now << 16;
                g.res_t = (flags & EF_RES_TOKEN) ? nullptr : E->res_t; g.res_tag_hi = (tag_now - (uint32_t)E->res_delta) << 16;
                *gp = g;
              }
#pragma unroll
              for (int u = 0; u < 4; u++) {
                const int ch = base + u * ENG_NCONS + c;
                if (ch < n_ch) {
                  float4* d = reinterpret_cast<float4*>(s_x + (size_t)ch * 8);
                  if (xtg) {
                    if (!tags_ok(xv[u], x_tag_hi)) xv[u] = wait_tagged4(xtg + (size_t)ch * 8, x_tag_hi, P.err_host, P.timeout_ns);
                    if (!tags_ok(xv2[u], x_tag_hi)) xv2[u] = wait_tagged4(xtg + (size_t)ch * 8 + 4, x_tag_hi, P.err_host, P.timeout_ns);
                    d[0] = make_float4(tagged_f32(xv[u].x), tagged_f32(xv[u].y), tagged_f32(xv[u].z), tagged_f32(xv[u].w));
                    d[1] = make_float4(tagged_f32(xv2[u].x), tagged_f32(xv2[u].y), tagged_f32(xv2[u].z), tagged_f32(xv2[u].w));
                  } else {
                    d[0] = make_float4(bf_lo(xv[u].x), bf_hi(xv[u].x), bf_lo(xv[u].y), bf_hi(xv[u].y));
                    d[1] = make_float4(bf_lo(xv[u].z), bf_hi(xv[u].z), bf_lo(xv[u].w), bf_hi(xv[u].w));
                  }
                  if (with_w) {
                    float4* dw = reinterpret_cast<float4*>(s_nw + (size_t)ch * 8);
                    dw[0] = make_float4(bf_lo(wv[u].x), bf_hi(wv[u].x), bf_lo(wv[u].y), bf_hi(wv[u].y));
                    dw[1] = make_float4(bf_lo(wv[u].z), bf_hi(wv[u].z), bf_lo(wv[u].w), bf_hi(wv[u].w));
                  }
                }
              }
            }
          }
          named_bar_sync(1, ENG_NCONS);
          if (P.prof && c == 0) { const long long t_now = clock64(); P.prof[bid * ENG_NPROF + 6] += (unsigned long long)(t_now - t_mark); t_mark = t_now; }
          if (E->pro == PRO_RMSNORM) {
            if (P.strict) {
              int ch = 0, nt = 0;
              eng_scan_shape(K, &ch, &nt);
              uint8_t* scr = s_work + ENG_SCAN_OFF;
              float* s_sum = s_scalar + 4;
              unsigned long long* pr = P.prof ? P.prof + (size_t)bid * ENG_NPROF : nullptr;
              switch (ch) {
                case 16: eng_seq_sumsq<16>(s_x, c, nt, scr, s_sum, pr); break;
                case 8: eng_seq_sumsq<8>(s_x, c, nt, scr, s_sum, pr); break;
                case 4: eng_seq_sumsq<4>(s_x, c, nt, scr, s_sum, pr); break;
                default: eng_seq_sumsq<2>(s_x, c, nt, scr, s_sum, pr); break;
              }
              if (c == 0) {
                const float me = __fadd_rn(__fdiv_rn(*s_sum, (float)K), P.eps);
                s_scalar[0] = (float)(1.0 / sqrt((double)me));
              }
            } else {
              // FAST: 256 interleaved partial sums, butterfly within each warp, then sequentially over the 8 warps
              float sum = 0.f;
              for (int k = c; k < K; k += ENG_NCONS) sum = __fmaf_rn(s_x[k], s_x[k], sum);
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
              if (lane == 0) s_part[cw] = sum;
              named_bar_sync(1, ENG_NCONS);
              if (c == 0) {
                float tot = 0.f;
                for (int w = 0; w < ENG_NCONS / 32; w++) tot = __fadd_rn(tot, s_part[w]);
                const float me = __fadd_rn(__fdiv_rn(tot, (float)K), P.eps);
                s_scalar[0] = (float)(1.0 / sqrt((double)me));
              }
            }
            named_bar_sync(1, ENG_NCONS);
            const float rs = s_scalar[0];
            for (int k = c; k < K; k += ENG_NCONS) {
              const float n1 = trunc_bf(__fmul_rn(s_x[k], rs));
              s_x[k] = trunc_bf(__fmul_rn(n1, s_nw[k]));
            }
            named_bar_sync(1, ENG_NCONS);
          }
          if (P.prof && c == 0) { const long long t_now = clock64(); P.prof[bid * ENG_NPROF + 1] += (unsigned long long)(t_now - t_mark); t_mark = t_now; }
          // ---- row tiles --------------------------------------------------------------------------------------
          if (KS > 1 || cw < Cfg::kChainWarps) {
            for (int rt = p0; rt < p1; rt += PT) {
              const int np = min(PT, p1 - rt);
              const int kt = eng_tile_kt(KS, np, K, E->kt, STAGE);
              const int n_tiles = (K + kt - 1) / kt;
              // FAST: this thread's rows are r and r + 32 of the 64-row tile; STRICT: row c of the 128-row tile
              const int pp0 = r >> 3, rr = r & 7;
              const int pp1 = pp0 + 4;
              const bool on0 = pp0 < np;
              const bool on1 = (KS > 1) && (pp1 < np);
              float acc0 = 0.f, acc1 = 0.f;
              const bool warp_on = (KS == 1) ? ((cw * 4) < np) : true;   // a chain warp without rows only keeps the ring moving
              for (int t = 0; t < n_tiles; t++, seq++) {
                const int s = seq % NST;
                const uint32_t par = (seq / NST) & 1u;
                eng_mbar_wait(&full_bar[s], par, P.err_host, P.timeout_ns, !warp_on, seq);
                const int k0 = t * kt;
                const int nchunks = min(kt, K - k0) / 8;
                // (rows without a panel in this tile read the stage's panel 0 -- data this thread has synchronised with -- and
                //  are never stored: `valid` is false for them)
                const uint8_t* tile0 = s_ring + (size_t)s * STAGE + (on0 ? (size_t)pp0 * ((size_t)kt * 16) : (size_t)0) + rr * 16;
                const float* xt = s_x + k0;
                // packed phase: this panel's unit byte, published with the stage (a lane with a raw panel runs the bf16 chain)
                const uint32_t ub = (KS == 1 && E->Wp && on0) ? (uint32_t)s_unit[s * PT + pp0] : (uint32_t)WP_RAW;
                if (KS == 1 && ub != (uint32_t)WP_RAW) {
                  const uint32_t bb = (ub - 15u) << 7;
                  if (nchunks == 64) acc0 = eng_chain_tile_wp<16>(tile0, xt, acc0, bb);
                  else if (nchunks == 32) acc0 = eng_chain_tile_wp<8>(tile0, xt, acc0, bb);
                  else if (nchunks == 16) acc0 = eng_chain_tile_wp<4>(tile0, xt, acc0, bb);
                  else if (nchunks == 8) acc0 = eng_chain_tile_wp<2>(tile0, xt, acc0, bb);
                  else acc0 = eng_chain_tile_wp<0>(tile0, xt, acc0, bb, nchunks / 4);
                } else if (KS == 1) {
                  if (on0) {
                    if (nchunks == 64) acc0 = eng_chain_tile<16>(tile0, xt, acc0);
                    else if (nchunks == 32) acc0 = eng_chain_tile<8>(tile0, xt, acc0);
                    else if (nchunks == 16) acc0 = eng_chain_tile<4>(tile0, xt, acc0);
                    else if (nchunks == 8) acc0 = eng_chain_tile<2>(tile0, xt, acc0);
                    else {
                      for (int ch = 0; ch < nchunks; ch++) {
                        const uint4 wv = *reinterpret_cast<const uint4*>(tile0 + ch * 128);
                        const float4 xa = *reinterpret_cast<const float4*>(xt + ch * 8);
                        const float4 xb = *reinterpret_cast<const float4*>(xt + ch * 8 + 4);
                        float a = acc0;
                        a = __fmaf_rn(xa.x, bf_lo(wv.x), a); a = __fmaf_rn(xa.y, bf_hi(wv.x), a);
                        a = __fmaf_rn(xa.z, bf_lo(wv.y), a); a = __fmaf_rn(xa.w, bf_hi(wv.y), a);
                        a = __fmaf_rn(xb.x, bf_lo(wv.z), a); a = __fmaf_rn(xb.y, bf_hi(wv.z), a);
                        a = __fmaf_rn(xb.z, bf_lo(wv.w), a); a = __fmaf_rn(xb.w, bf_hi(wv.w), a);
                        acc0 = a;
                      }
                    }
                  }
                } else {
                  // FAST: stream j owns the chunks ch = j, j + 8, ...
                  // Row tiles with <= 4 panels (wo, w2, the tail tile of the others) have no second row at all: one chain per
                  // thread.  Otherwise two independent chains; a row without a panel reads the stage's panel 0 (data this thread
                  // has synchronised with -- never memory a bulk copy may be writing) and is not stored (`valid` is false).
                  // The next chunk's operands are loaded before the current chunk's FMAs issue.
                  if (np <= 4) {
                    int ch = j;
                    float4 xa, xb;
                    uint4 w0;
                    if (ch < nchunks) {
                      xa = *reinterpret_cast<const float4*>(xt + ch * 8);
                      xb = *reinterpret_cast<const float4*>(xt + ch * 8 + 4);
                      w0 = *reinterpret_cast<const uint4*>(tile0 + ch * 128);
                    }
#pragma unroll 2
                    for (; ch < nchunks; ch += KS) {
                      const float4 ca = xa, cb = xb;
                      const uint4 c0 = w0;
                      const int nx = ch + KS;
                      if (nx < nchunks) {
                        xa = *reinterpret_cast<const float4*>(xt + nx * 8);
                        xb = *reinterpret_cast<const float4*>(xt + nx * 8 + 4);
                        w0 = *reinterpret_cast<const uint4*>(tile0 + nx * 128);
                      }
                      float a = acc0;
                      a = __fmaf_rn(ca.x, bf_lo(c0.x), a); a = __fmaf_rn(ca.y, bf_hi(c0.x), a);
                      a = __fmaf_rn(ca.z, bf_lo(c0.y), a); a = __fmaf_rn(ca.w, bf_hi(c0.y), a);
                      a = __fmaf_rn(cb.x, bf_lo(c0.z), a); a = __fmaf_rn(cb.y, bf_hi(c0.z), a);
                      a = __fmaf_rn(cb.z, bf_lo(c0.w), a); a = __fmaf_rn(cb.w, bf_hi(c0.w), a);
                      acc0 = a;
                    }
                  } else {
                    const uint8_t* tile1 = s_ring + (size_t)s * STAGE + (on1 ? (size_t)pp1 * ((size_t)kt * 16) : (size_t)0) + rr * 16;
                    int ch = j;
                    float4 xa, xb;
                    uint4 w0, w1;
                    if (ch < nchunks) {
                      xa = *reinterpret_cast<const float4*>(xt + ch * 8);
                      xb = *reinterpret_cast<const float4*>(xt + ch * 8 + 4);
                      w0 = *reinterpret_cast<const uint4*>(tile0 + ch * 128);
                      w1 = *reinterpret_cast<const uint4*>(tile1 + ch * 128);
                    }
#pragma unroll 2
                    for (; ch < nchunks; ch += KS) {
                      const float4 ca = xa, cb = xb;
                      const uint4 c0 = w0, c1 = w1;
                      const int nx = ch + KS;
                      if (nx < nchunks) {
                        xa = *reinterpret_cast<const float4*>(xt + nx * 8);
                        xb = *reinterpret_cast<const float4*>(xt + nx * 8 + 4);
                        w0 = *reinterpret_cast<const uint4*>(tile0 + nx * 128);
                        w1 = *reinterpret_cast<const uint4*>(tile1 + nx * 128);
                      }
                      float a = acc0, b = acc1;
                      a = __fmaf_rn(ca.x, bf_lo(c0.x), a); b = __fmaf_rn(ca.x, bf_lo(c1.x), b);
                      a = __fmaf_rn(ca.y, bf_hi(c0.x), a); b = __fmaf_rn(ca.y, bf_hi(c1.x), b);
                      a = __fmaf_rn(ca.z, bf_lo(c0.y), a); b = __fmaf_rn(ca.z, bf_lo(c1.y), b);
                      a = __fmaf_rn(ca.w, bf_hi(c0.y), a); b = __fmaf_rn(ca.w, bf_hi(c1.y), b);
                      a = __fmaf_rn(cb.x, bf_lo(c0.z), a); b = __fmaf_rn(cb.x, bf_lo(c1.z), b);
                      a = __fmaf_rn(cb.y, bf_hi(c0.z), a); b = __fmaf_rn(cb.y, bf_hi(c1.z), b);
                      a = __fmaf_rn(cb.z, bf_lo(c0.w), a); b = __fmaf_rn(cb.z, bf_lo(c1.w), b);
                      a = __fmaf_rn(cb.w, bf_hi(c0.w), a); b = __fmaf_rn(cb.w, bf_hi(c1.w), b);
                      acc0 = a; acc1 = b;
                    }
                  }
                }
                // every lane releases the stage it read.  (One elected lane after a warp barrier is formally enough -- release
                // is cumulative over what the barrier ordered before it -- but compute-sanitizer's racecheck does not follow
                // that edge and reports the next bulk copy into the stage as a WAR hazard against the other lanes' reads.)
                mbar_arrive(&empty_bar[s]);
              }
              if (P.prof && c == 0) { const long long t_now = clock64(); P.prof[bid * ENG_NPROF + 2] += (unsigned long long)(t_now - t_mark); t_mark = t_now; }
              // ---- combine the KS streams in stream order, then the fused epilogue -------------------------------
              if (KS > 1) {
                s_part[j * 64 + r] = acc0;
                s_part[j * 64 + 32 + r] = acc1;
                named_bar_sync(1, ENG_NCONS);
                if (c < 64) {
                  float v = s_part[c];
#pragma unroll
                  for (int jj = 1; jj < KS; jj++) v = __fadd_rn(v, s_part[jj * 64 + c]);
                  const int er = c;                              // row of the 64-row tile; lane == er % 32
                  const int n = (rt + (er >> 3)) * 8 + (er & 7);
                  const bool valid = (er >> 3) < np;
                  switch (E->epi) {
                    case EPI_BF16: gemv_epilogue<EPI_BF16>(*gp, v, n, 0, valid, rt + (er >> 3), er, lane); break;
                    case EPI_RESID: gemv_epilogue<EPI_RESID>(*gp, v, n, 0, valid, rt + (er >> 3), er, lane); break;
                    case EPI_LOGITS: gemv_epilogue<EPI_LOGITS>(*gp, v, n, 0, valid, rt + (er >> 3), er, lane); break;
                    case EPI_QKV_ROPE: gemv_epilogue<EPI_QKV_ROPE>(*gp, v, n, 0, valid, rt + (er >> 3), er, lane); break;
                    case EPI_SWIGLU: gemv_epilogue<EPI_SWIGLU>(*gp, v, n, 0, valid, rt + (er >> 3), er, lane); break;
                    case EPI_P2P: gemv_epilogue<EPI_P2P>(*gp, v, n, 0, valid, rt + (er >> 3), er, lane); break;
                    default: gemv_epilogue<EPI_F32RAW>(*gp, v, n, 0, valid, rt + (er >> 3), er, lane); break;
                  }
                }
                named_bar_sync(1, ENG_NCONS);                    // s_part is reused by the next row tile
              } else {
                const int n = (rt + pp0) * 8 + rr;               // global row of W
                switch (E->epi) {
                  case EPI_BF16: gemv_epilogue<EPI_BF16>(*gp, acc0, n, 0, on0, rt + pp0, r, lane); break;
                  case EPI_RESID: gemv_epilogue<EPI_RESID>(*gp, acc0, n, 0, on0, rt + pp0, r, lane); break;
                  case EPI_LOGITS: gemv_epilogue<EPI_LOGITS>(*gp, acc0, n, 0, on0, rt + pp0, r, lane); break;
                  case EPI_QKV_ROPE: gemv_epilogue<EPI_QKV_ROPE>(*gp, acc0, n, 0, on0, rt + pp0, r, lane); break;
                  case EPI_SWIGLU: gemv_epilogue<EPI_SWIGLU>(*gp, acc0, n, 0, on0, rt + pp0, r, lane); break;
                  case EPI_P2P: gemv_epilogue<EPI_P2P>(*gp, acc0, n, 0, on0, rt + pp0, r, lane); break;
                  default: gemv_epilogue<EPI_F32RAW>(*gp, acc0, n, 0, on0, rt + pp0, r, lane); break;
                }
              }
              if (P.prof && c == 0) { const long long t_now = clock64(); P.prof[bid * ENG_NPROF + 3] += (unsigned long long)(t_now - t_mark); t_mark = t_now; }
            }
          }
        }
      } else if (type == EP_SDPA) {
        // ---- decode attention, one CTA per QUERY head (the four heads of a GQA group stage the same K / V rows from L2):
        // sdpa_decode_kernel's arithmetic (kernels.cuh) -- the same 128 threads per head for the f64 row sum, so the bits
        // are the kernel chain's in both modes.  The other CTAs go straight on to the next phase's inputs.
        const int hd = P.head_dim, n_rep = P.n_rep;
        const int n_qh = E->q_dim / hd;
        if (bid < n_qh) {
          const int H = bid, h = H / n_rep;
          const int T = pos + 1, T_max = P.seq_len;
          const int kstride = hd + 8, cpr = hd / 8;
          uint16_t* sK = reinterpret_cast<uint16_t*>(s_work);
          uint16_t* sV = sK + (size_t)T_max * kstride;
          double* sE = reinterpret_cast<double*>(sV + (size_t)T_max * hd);
          float* sP = reinterpret_cast<float*>(sE + (size_t)T_max);
          // the query is stored as float4, so it starts on a 16-byte boundary: sE and sP take 12 * T_max bytes, which left sQ
          // misaligned whenever T_max % 4 != 0 (eng_sdpa_smem's slack covers the padding)
          float* sQ = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(sP + (size_t)T_max) + 15) & ~(uintptr_t)15);
          double* sZ = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(sQ + (size_t)hd) + 15) & ~(uintptr_t)15);
          // rows of earlier positions come from the cache (complete since the previous step's grid barrier); this step's
          // k / v row and the query head come from the tagged q | k | v vector the projection phase is writing right now
          for (int i = c; i < (T - 1) * cpr; i += ENG_NCONS) {
            const int t = i / cpr, cc = i % cpr;
            *reinterpret_cast<uint4*>(sK + (size_t)t * kstride + cc * 8) = ldcg_u4(E->cache_k + (size_t)t * E->kv_dim + (size_t)h * hd + cc * 8);
            *reinterpret_cast<uint4*>(sV + (size_t)t * hd + cc * 8) = ldcg_u4(E->cache_v + (size_t)t * E->kv_dim + (size_t)h * hd + cc * 8);
          }
          {
            const uint32_t qtag = (tag_now - (uint32_t)E->x_delta) << 16;
            const int n4 = hd / 4;
            for (int i = c; i < 3 * n4; i += ENG_NCONS) {
              if (i < n4) {
                const uint4 w = wait_tagged4(E->x_t + (size_t)H * hd + (size_t)i * 4, qtag, P.err_host, P.timeout_ns);
                *reinterpret_cast<float4*>(sQ + (size_t)i * 4) = make_float4(tagged_f32(w.x), tagged_f32(w.y), tagged_f32(w.z), tagged_f32(w.w));
              } else {
                const bool is_v = i >= 2 * n4;
                const int e4 = i - (is_v ? 2 * n4 : n4);
                const uint4 w = wait_tagged4(E->x_t + (size_t)E->q_dim + (is_v ? (size_t)E->kv_dim : 0) + (size_t)h * hd + (size_t)e4 * 4, qtag,
                                             P.err_host, P.timeout_ns);
                uint16_t* dst = is_v ? sV + (size_t)(T - 1) * hd + e4 * 4 : sK + (size_t)(T - 1) * kstride + e4 * 4;
                *reinterpret_cast<uint2*>(dst) = make_uint2((w.x & 0xffffu) | (w.y << 16), (w.z & 0xffffu) | (w.w << 16));
              }
            }
          }
          named_bar_sync(1, ENG_NCONS);
          for (int t = c; t < T; t += ENG_NCONS) {
            const uint16_t* kr = sK + (size_t)t * kstride;
            float a = 0.f;
            for (int d = 0; d < hd; d += 8) {
              const uint4 kv = *reinterpret_cast<const uint4*>(kr + d);
              a = __fmaf_rn(sQ[d + 0], bf_lo(kv.x), a);
              a = __fmaf_rn(sQ[d + 1], bf_hi(kv.x), a);
              a = __fmaf_rn(sQ[d + 2], bf_lo(kv.y), a);
              a = __fmaf_rn(sQ[d + 3], bf_hi(kv.y), a);
              a = __fmaf_rn(sQ[d + 4], bf_lo(kv.z), a);
              a = __fmaf_rn(sQ[d + 5], bf_hi(kv.z), a);
              a = __fmaf_rn(sQ[d + 6], bf_lo(kv.w), a);
              a = __fmaf_rn(sQ[d + 7], bf_hi(kv.w), a);
            }
            float sc = trunc_bf(a);
            sc = trunc_bf(__fdiv_rn(sc, P.attn_scale));
            sE[t] = exp((double)sc);
          }
          named_bar_sync(1, ENG_NCONS);
          if (P.strict) {
            if (c == 0) {
              double z = 0.0;
              for (int t = 0; t < T; t++) z = __dadd_rn(z, sE[t]);
              sZ[4] = z;
            }
          } else if (c < 128) {
            double z = 0.0;
            for (int t = c; t < T; t += 128) z = __dadd_rn(z, sE[t]);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) z = __dadd_rn(z, __shfl_xor_sync(0xffffffffu, z, o));
            if ((c & 31) == 0) sZ[c >> 5] = z;
          }
          named_bar_sync(1, ENG_NCONS);
          if (!P.strict && c == 0) sZ[4] = __dadd_rn(__dadd_rn(__dadd_rn(sZ[0], sZ[1]), sZ[2]), sZ[3]);
          named_bar_sync(1, ENG_NCONS);
          {
            const double Z = sZ[4];
            for (int t = c; t < T; t += ENG_NCONS) sP[t] = trunc_bf((float)__ddiv_rn(sE[t], Z));
          }
          named_bar_sync(1, ENG_NCONS);
          if (c < hd) {
            const uint16_t* vc = sV + c;
            float a = 0.f;
#pragma unroll 4
            for (int t = 0; t < T; t++) a = __fmaf_rn(sP[t], bf2f(vc[(size_t)t * hd]), a);
            E->out_t[(size_t)H * hd + c] = (tag_now << 16) | f2bf(a);
          }
        }
      } else if (type == EP_REDUCE) {
        // ---- peer all-reduce of the partials the previous phase pushed: out = t(res + t(p0 + p1 + ...)), rank order ----
        const int per = (P.dim + G - 1) / G;
        const int i = bid * per + c;
        if (c < per && i < P.dim) {
          const unsigned long long t0 = global_timer_ns();
          const uint2* base = P.p2p.data[P.p2p.rank] + (size_t)(epoch & 1u) * P.p2p.n * P.p2p.slot_elems;
          float sum = 0.f;
          for (int rk = 0; rk < P.p2p.n; rk++) {
            const uint2 w = eng_wait_word(P, base + (size_t)rk * P.p2p.slot_elems + i, epoch, rk, t0);
            sum = (rk == 0) ? __uint_as_float(w.x) : __fadd_rn(sum, __uint_as_float(w.x));
          }
          float rsd;
          if (E->flags & EF_RES_TOKEN) rsd = bf2f(ldcg_u16(P.emb + (size_t)tok * P.dim + i));
          else rsd = tagged_f32(wait_tagged_word(E->res_t + i, (tag_now - (uint32_t)E->res_delta) << 16));
          E->out_t[i] = (tag_now << 16) | f2bf(__fadd_rn(rsd, trunc_bf(sum)));
        }
        epoch++;
      } else if (type == EP_ARGMAX) {
        // ---- tensor-parallel greedy argmax: CTA 0 pushes this rank's key to every peer; every CTA takes the max ----
        // (runs after the LM head's grid barrier: st->amax_key is final)
        const unsigned long long t0 = global_timer_ns();
        const size_t myoff = ((size_t)((epoch & 1u) * P.p2p.n + P.p2p.rank)) * P.p2p.slot_elems;
        if (bid == 0 && c < P.p2p.n) {
          const unsigned long long mykey = __ldcg(keys[step & 1]);
          P.p2p.data[c][myoff] = make_uint2((uint32_t)(mykey & 0xffffffffull), epoch);
          P.p2p.data[c][myoff + 1] = make_uint2((uint32_t)(mykey >> 32), epoch);
        }
        if (c < 32) {
          unsigned long long key = LNB_ARGMAX_EMPTY;
          if (c < P.p2p.n) {
            const uint2* src = P.p2p.data[P.p2p.rank] + ((size_t)((epoch & 1u) * P.p2p.n + c)) * P.p2p.slot_elems;
            const uint2 lo = eng_wait_word(P, src, epoch, c, t0), hi = eng_wait_word(P, src + 1, epoch, c, t0);
            key = ((unsigned long long)hi.x << 32) | lo.x;
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
            key = other > key ? other : key;
          }
          if (c == 0) ctl->tok = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
        }
        epoch++;
        named_bar_sync(1, ENG_NCONS);
        tok = ctl->tok;
        continue;                                  // purely local result: no grid barrier
      }
      // ---- end of phase ---------------------------------------------------------------------------------------------
      if (P.prof && c == 0) {
        const long long t_now = clock64();
        if (type == EP_SDPA) P.prof[bid * ENG_NPROF + 4] += (unsigned long long)(t_now - t_mark);
        else if (type == EP_REDUCE) P.prof[bid * ENG_NPROF + 5] += (unsigned long long)(t_now - t_mark);
        t_mark = t_now;
      }
      if (!(E->flags & EF_GRID_SYNC)) {
        named_bar_sync(1, ENG_NCONS);              // the CTA's own scratch (gp, s_x, s_part) changes hands
        continue;
      }
      // the LM head: its argmax key is an atomic maximum over all CTAs -> one real grid barrier per step.  It also orders
      // this step's plain stores (KV cache rows) before the next step's plain loads.
      n_bar++;
      eng_grid_barrier(P, n_bar * (unsigned int)G, c);
      if (P.prof && c == 0) { const long long t_now = clock64(); P.prof[bid * ENG_NPROF + 0] += (unsigned long long)(t_now - t_mark); t_mark = t_now; }
      if (type == EP_GEMV && E->epi == EPI_LOGITS && P.tp == 1) {
        const unsigned long long key = __ldcg(keys[step & 1]);
        tok = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
      }
      if (bid == 0 && c == 0) {                    // everyone is past the previous step's reads of the other key
        atomicExch(keys[(step + 1) & 1], LNB_ARGMAX_EMPTY);
        __threadfence();
      }
    }
    // ---- end of step: greedy token known to every CTA ------------------------------------------------------------
    if (bid == 0 && c == 0 && P.advance && P.tok_out) P.tok_out[P.st->step + step] = tok;
    pos += 1;
  }
  if (bid == 0 && c == 0) {
    // n_bar >= 1 barriers have passed since any CTA read the state at the top
    P.st->next_token = tok;      // (amax_key is reset by set_state_kernel / at the start of the next launch: other CTAs may
    P.st->done_ctr = 0;          //  still be reading it here)
    if (P.tp > 1) P.st->ar_epoch = epoch;
    if (P.advance) {
      P.st->step += P.n_steps;
      P.st->pos += P.n_steps;
    }
  }
}

}  // namespace lnb
