// gemv.cuh -- the projection kernel of the decode path (M = 1..8 rows of activations
// against a bf16 weight matrix that is streamed from HBM exactly once).
//
// Replaces ml.LinearTransformation (src/ml/operations_impl.go:427-447 ->
// operations_lineartransform.go:37-70,145-207) for Wq/Wk/Wv, Wo, w1/w3, w2 and the LM
// head, with the neighbouring elementwise ops of LlamaAttention / LlamaFeedForward /
// RMSNorm fused into its prologue and epilogue (each fused op keeps the reference's
// truncation point; see the EPI_* / PRO_* notes).
//
// HBM layout of a weight matrix W[N,K] ("panel-major", built once at upload):
//   panel p = rows 8p..8p+7;  chunk c = k 8c..8c+7;
//   address(p, c, r, e) = ((p * K/8 + c) * 8 + r) * 8 + e        (bf16 elements)
// i.e. the matrix is stored as 8-row x 16-byte "core matrices" (128 B each), k-chunks of a panel
// back to back.  A (panel, k-range) block is ONE contiguous byte range -> a single bulk-async copy
// (TMA engine, cp.async.bulk + mbarrier complete_tx) per panel per stage; in shared memory the 8 rows
// of a chunk are 128 contiguous bytes -> conflict-free 128-bit LDS for "one thread = one output row"
// (each quarter-warp reads one core matrix), and any number of consecutive panels forms a wgmma
// K-major / no-swizzle operand with a uniform 8-row-group stride (gemm_tc.cuh reads the SAME bytes).
//
// Thread roles: warp 0 = producer (one lane issues bulk copies into an NST-stage ring);
// the other TN*KS threads are consumers.  Consumer (r, j): output row r of the CTA's TN
// rows, k-stream j of KS.  Stream j owns the 8-element chunks g with g % KS == j and
// accumulates them sequentially (fp32 FMA; bf16*bf16 products are exact in fp32, so FMA ==
// mul-then-add).  KS == 1 (LNB_ACC_STRICT) is exactly the reference's k = 0,1,2,... order.
// KS > 1 (LNB_ACC_FAST): out = ((p0 + p1) + p2) + ... + p_{KS-1}, combined in stream order.
//
// MXFP8 weights (FMT == WF_MXFP8, mxfp8.cuh): the same producer streams each panel's E4M3 codes (64 B per chunk) and its
// E8M0 scales; a stage carries twice the k-range of the bf16 config it mirrors, so as many bytes are in flight.  Consumers
// decode every weight to the exact fp32 value of the bf16 number it stands for and run the same FMAs in the same order.
// MXFP4 weights (FMT == WF_MXFP4, mxfp4.cuh) likewise, with 32 B of codes per chunk and the largest k-tile whose stage is
// no larger than its bf16 twin's (gemv_kt), so an MXFP4 matrix gets the row block of the bf16 matrix it stands for.
#pragma once
#include "common.cuh"
#include "mxfp8.cuh"
#include "mxfp4.cuh"

namespace lnb {

enum { PRO_PLAIN = 0, PRO_RMSNORM = 1 };
enum {
  EPI_BF16 = 0,      // out_bf16[m,n] = t(acc)                                  (ToBFloat16, :205)
  EPI_F32RAW = 1,    // out_f32[m,n] = acc     (tensor-parallel partial, reduced over ranks before truncation)
  EPI_RESID = 2,     // out_bf16[m,n] = t(res[m,n] + t(acc))                    (ml.Add, llamatransformer.go:232,248)
  EPI_LOGITS = 3,    // out_f32[m,n] = f32(t(acc)); greedy argmax of row n_rows-1 (llamatransformer.go:170-175; inference.go:207-216)
  EPI_QKV_ROPE = 4,  // q -> rope -> q_out ; k -> rope -> cacheK[pos+m] ; v -> cacheV[pos+m]   (llamatransformer.go:374-403)
  EPI_SWIGLU = 5,    // panels alternate w1/w3: out[m,i] = t( silu_tab[t(g)] * t(u) )          (llamatransformer.go:601-614)
  EPI_P2P = 6        // tensor-parallel partial pushed into every peer's all-reduce slot over NVLink (fused collective)
};

struct GemvParams {
  const uint16_t* W;       // panel-major weights (MXFP8: the codes; their scales are the kernel's second argument)
  int N, K;                // N = rows of W (multiple of 8), K multiple of 8
  int M;                   // activation rows in this launch (<= MB)
  // prologue
  const uint16_t* x;       // [M, ldx] bf16 activations (PRO_PLAIN) / residual stream (PRO_RMSNORM)
  int ldx;
  const uint16_t* norm_w;  // [K] bf16 (PRO_RMSNORM)
  float eps;
  int strict_norm;         // 1: sequential sum of squares (reference order)
  const float* rscale;     // [M] precomputed f32(1/sqrt(mean+eps)) per row (rms_scale_kernel); NULL: computed in-CTA
  // epilogue
  uint16_t* out_bf16;      // EPI_BF16 / EPI_RESID / EPI_SWIGLU(out [M, N/2]) / EPI_QKV_ROPE(q_out [M, q_dim])
  float* out_f32;          // EPI_F32RAW / EPI_LOGITS (may be NULL for LOGITS)
  int ldo;                 // row pitch of the output in elements
  const uint16_t* res;     // EPI_RESID residual [M, ldo]
  // EPI_QKV_ROPE
  int q_dim, kv_dim, head_dim;
  uint16_t* cache_k;       // [seq_len, kv_dim]  (batched decode: sequence b at + b * cache_seq_stride)
  uint16_t* cache_v;
  const int32_t* pos_arr;  // batched decode (one row per independent sequence): position of row m; NULL -> *pos_ptr + m
  long long cache_seq_stride;  // elements between the caches of consecutive sequences (batched decode)
  const int32_t* row_seq;  // rows of several sequences: row m's sequence (cache at + row_seq[m] * cache_seq_stride); NULL: cache_k
  const int32_t* row_tree; // with pos_arr, speculative tree rows: K and V of row m go to slot tree_slot(row_tree[m]); NULL: pos
  const float* cis;        // [rows][head_dim/2][2]
  // EPI_SWIGLU
  const uint16_t* silu_tab;
  // EPI_LOGITS
  int n_offset;            // global index of row 0 (vocab shard offset)
  LnbDevState* st;         // device state: pos, argmax key, next token (NULL: no argmax in this launch)
  int argmax_row;          // activation row of this launch whose greedy argmax is wanted (-1: none)
  int publish;             // 1: the last CTA decodes the key into st->next_token (tp_size == 1)
  int advance;             // 1: last CTA also advances st->pos and appends the token to tok_out (device-driven decode)
  int32_t* tok_out;        // device [n_steps] (advance mode)
  const int32_t* pos_ptr;  // == &st->pos (kept separate so op-level calls can pass a plain int buffer)
  int m_off;               // index of activation row 0 of this launch inside the forward call (row blocking)
  LnbP2P p2p;              // EPI_P2P: peer regions (st must be set: epoch / done counters live in the device state)
  uint32_t ar_epoch_override;  // EPI_P2P inside the persistent engine: the epoch is tracked per CTA, not in st (0: use st)
  // persistent engine only: activations travel between phases as self-validating words {tag:16 | bf16:16} (engine.cuh)
  unsigned long long* amax_key_ptr;  // EPI_LOGITS: the argmax key to maximise (NULL: &st->amax_key)
  unsigned long long* amax_keys_row; // batch engine: one key per activation row (every row is the last row of its own sequence)
  int cm;                  // batch engine: bf16 activations are CHUNK-MAJOR [K/8][8 rows][8]: element (row m, col n) at cm_idx(m, n)
  uint32_t* out_t;         // tagged output vector (NULL: plain bf16 output)
  uint32_t tag_hi;         // this phase's tag << 16
  const uint32_t* res_t;   // tagged residual vector (NULL: plain `res`)
  uint32_t res_tag_hi;     // tag << 16 of the phase that produced the residual
};

// the k-tile of format F for a bf16 k-tile kt: MXFP8 twice kt; MXFP4 the largest multiple of 64 whose codes, pad and
// scales (kt4 * 4 + 32 + kt4 / 4 bytes per panel) fit in the bf16 panel's kt * 16 bytes
constexpr int gemv_kt(int kt, int F) { return F == WF_MXFP4 ? ((64 * kt - 128) / 17) & ~63 : kt << F; }

template <int TN, int KS, int MB, int KT, int NST, int FMT = WF_BF16>
struct GemvCfg {
  static constexpr int kTN = TN, kKS = KS, kMB = MB, kKT = KT, kNST = NST, kFmt = FMT;
  static constexpr int kP = TN / 8;                    // 8-row panels per CTA
  static constexpr int kNCons = TN * KS;               // consumer threads
  static constexpr int kThreads = kNCons + 32;         // + producer warp
  // MXFP8: a panel's codes take KT * 8 bytes plus 64 bytes of padding, so the two panels a half-warp reads sit in opposite
  // halves of the banks (conflict-free 8-byte loads); the panels' scales (KT / 4 bytes each) follow
  // MXFP4: KT * 4 bytes plus 32, so the four panels a warp reads (4 bytes a lane) start in four different 8-bank groups
  static constexpr int kPanelBytes = FMT == WF_MXFP8 ? KT * 8 + 64 : FMT == WF_MXFP4 ? KT * 4 + 32 : KT * 16;
  static constexpr int kScaleOff = kP * kPanelBytes;
  static constexpr int kStageBytes = FMT != WF_BF16 ? kScaleOff + kP * (KT / 4) : TN * KT * 2;
  static constexpr int kChunksPerTile = KT / 8;
  static_assert(TN % 32 == 0 && TN <= 128, "TN");
  static_assert(kNCons % 32 == 0, "consumer warps");
  static_assert(kChunksPerTile % KS == 0, "k-tile must hold a whole number of chunk rounds");
  static_assert(FMT == WF_BF16 || KT % 64 == 0, "MX k-tiles hold whole, 16-byte-aligned scale ranges");
  static size_t smem_bytes(int K) {
    size_t b = 1024;                                   // barriers + scalars (first 1 KB)
    b += (size_t)NST * kStageBytes;
    b += (size_t)MB * K * 4;                           // activations as f32
    b += (size_t)KS * MB * TN * 4;                     // partial sums for the stream combine
    return b;
  }
};

// chunk-major activation layout of the batch engine: 8 sequences' values of one 8-element k-chunk are 128 contiguous bytes, so
// the k-range of a k-tile is ONE contiguous block for all rows (engine_batch.cuh)
LNB_HDINL size_t cm_idx(int m, int n) { return ((((size_t)(n >> 3)) * 8 + (size_t)m) << 3) + (size_t)(n & 7); }

// one word of a tagged activation vector, as soon as its producer has stored it (bounded: a word that never comes is a
// bug or a dead SM -> trap, never a hang)
LNB_DEVINL uint32_t wait_tagged_word(const uint32_t* p, uint32_t tag_hi) {
  uint32_t w, spins = 0;
  for (;;) {
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(w) : "l"(p));
    if ((w & 0xffff0000u) == tag_hi) return w;
    if (++spins > (1u << 28)) __trap();
  }
}

// ------------------------------------------------------------------------------------------
// Epilogue of one output element: v = the untruncated fp32 dot product of activation row em with
// weight row n.  Must be called by all 32 lanes of a warp (it shuffles); lane == tile row % 32.
template <int EPI>
LNB_DEVINL void gemv_epilogue(const GemvParams& p, float v, int n, int em, bool valid, int panel, int er, int lane) {
  if (EPI == EPI_BF16) {
    if (valid) p.out_bf16[(size_t)em * p.ldo + n] = f2bf(v);
  } else if (EPI == EPI_F32RAW) {
    if (valid) p.out_f32[(size_t)em * p.ldo + n] = v;
  } else if (EPI == EPI_P2P) {
    if (valid) {
      const uint32_t epoch = p.ar_epoch_override ? p.ar_epoch_override : p.st->ar_epoch;   // epochs start at 1
      const size_t off = ((size_t)((epoch & 1u) * p.p2p.n + p.p2p.rank)) * p.p2p.slot_elems + (size_t)(p.m_off + em) * p.ldo + n;
      const uint2 w = make_uint2(__float_as_uint(v), epoch);
#pragma unroll
      for (int r = 0; r < 8; r++)
        if (r < p.p2p.n) p.p2p.data[r][off] = w;   // 32 lanes -> 256 contiguous bytes per peer, one 8-byte word each
    }
  } else if (EPI == EPI_RESID) {
    if (valid) {
      float a = trunc_bf(v);
      const size_t oi = p.cm ? cm_idx(p.m_off + em, n) : (size_t)em * p.ldo + n;
      float rsd = p.res_t ? __uint_as_float(wait_tagged_word(p.res_t + n, p.res_tag_hi) << 16) : bf2f(p.res[oi]);
      const uint16_t o = f2bf(__fadd_rn(rsd, a));
      if (p.out_t) p.out_t[n] = p.tag_hi | o;
      else p.out_bf16[oi] = o;
    }
  } else if (EPI == EPI_LOGITS) {
    float lv = trunc_bf(v);
    if (valid && p.out_f32) p.out_f32[(size_t)em * p.ldo + n] = lv;
    unsigned long long key = LNB_ARGMAX_EMPTY;
    if (valid && (em == p.argmax_row || p.amax_keys_row) && lv > -3.402823466e+38f) key = argmax_key(lv, (uint32_t)(n + p.n_offset));
    if (p.amax_keys_row) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
        key = other > key ? other : key;
      }
      if (lane == 0 && key != LNB_ARGMAX_EMPTY) atomicMax(&p.amax_keys_row[p.m_off + em], key);
    } else if (p.st) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
        key = other > key ? other : key;
      }
      if (lane == 0 && key != LNB_ARGMAX_EMPTY) atomicMax(p.amax_key_ptr ? p.amax_key_ptr : &p.st->amax_key, key);
    }
  } else if (EPI == EPI_QKV_ROPE) {
    // rows [0,q_dim) = q, [q_dim, q_dim+kv_dim) = k, rest = v.  RoPE pairs (2i,2i+1) are
    // adjacent rows == adjacent lanes.  Go evaluates complex64*complex64 through float64
    // (operations_impl.go:414-417; SURVEY F16-A1), products are exact in f64.
    const float mine = trunc_bf(v);                                     // t(linear)  (:306-344)
    const float other = __shfl_xor_sync(0xffffffffu, mine, 1);
    if (valid) {
      const int row = p.m_off + em;
      int pos, slot;   // RoPE at the position, the cache row at the slot
      if (p.pos_arr) {
        pos = p.pos_arr[row];
        slot = p.row_tree ? tree_slot(p.row_tree[row]) : pos;
      } else {
        pos = slot = *p.pos_ptr + row;
      }
      const size_t cb = p.row_seq ? (size_t)p.row_seq[row] * (size_t)p.cache_seq_stride : 0;
      uint16_t* ck = p.cache_k + cb;
      uint16_t* cv = p.cache_v + cb;
      if (n < p.q_dim + p.kv_dim) {
        const int nn = (n < p.q_dim) ? n : n - p.q_dim;
        const int i = (nn % p.head_dim) >> 1;
        const float2 fc = *reinterpret_cast<const float2*>(p.cis + ((size_t)pos * (p.head_dim / 2) + i) * 2);
        const double cc = (double)fc.x, dd = (double)fc.y;
        float o;
        if ((n & 1) == 0) {
          const double a = (double)mine, b = (double)other;
          o = (float)(a * cc - b * dd);
        } else {
          const double a = (double)other, b = (double)mine;
          o = (float)(a * dd + b * cc);
        }
        if (p.out_t) p.out_t[n] = p.tag_hi | f2bf(o);                   // engine: q, and this step's k row for the attention phase
        if (n < p.q_dim) { if (!p.out_t) p.out_bf16[p.cm ? cm_idx(p.m_off + em, n) : (size_t)em * p.ldo + n] = f2bf(o); }
        else ck[(size_t)slot * p.kv_dim + nn] = f2bf(o);                 // SetSlice :402
      } else {
        if (p.out_t) p.out_t[n] = p.tag_hi | f2bf(mine);
        cv[(size_t)slot * p.kv_dim + (n - p.q_dim - p.kv_dim)] = f2bf(mine);        // :403
      }
    }
  } else if (EPI == EPI_SWIGLU) {
    // every panel of the stacked w1|w3 matrix holds the gate rows of hidden units 4*panel .. 4*panel+3 in its rows
    // 0..3 and their up rows in rows 4..7 (retile_kernel, dpanel_stride == 2); `panel` = the panel of this row; the
    // partner of tile row er (er % 8 < 4) is er + 4 == lane + 4 of the same warp
    const float mine = trunc_bf(v);
    const float up = __shfl_down_sync(0xffffffffu, mine, 4);
    if (valid && (er & 4) == 0) {
      const uint16_t sg = p.silu_tab[f2bf(mine)];                       // t(TABLE_SILU[bits]) activations.go:38
      const float mm = __fmul_rn(bf2f(sg), up);                         // MultiplyElementwise :614
      const int col = panel * 4 + (er & 3);
      if (p.out_t) p.out_t[col] = p.tag_hi | f2bf(mm);
      else p.out_bf16[p.cm ? cm_idx(p.m_off + em, col) : (size_t)em * p.ldo + col] = f2bf(mm);
    }
  }
}

// LM head, tp_size == 1: the last CTA to finish decodes the argmax key into the greedy token and
// (device-driven decode) advances the per-session state.  Called by ONE thread per CTA after that
// CTA's atomicMax contributions are fenced.
LNB_DEVINL void logits_publish(const GemvParams& p) {
  const unsigned int done = atomicAdd(&p.st->done_ctr, 1u);
  if (done == gridDim.x - 1) {
    __threadfence();
    const unsigned long long key = atomicExch(&p.st->amax_key, LNB_ARGMAX_EMPTY);
    const int32_t tok = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
    p.st->next_token = tok;
    p.st->done_ctr = 0;
    if (p.advance) {
      if (p.tok_out) p.tok_out[p.st->step] = tok;
      p.st->step += 1;
      p.st->pos += 1;
    }
    __threadfence();
  }
}

// ------------------------------------------------------------------------------------------
template <class Cfg, int PRO, int EPI>
__global__ void __launch_bounds__(Cfg::kThreads) gemv_kernel(const GemvParams p, const uint8_t* Ws) {   // Ws: MX scales
  constexpr int TN = Cfg::kTN, KS = Cfg::kKS, MB = Cfg::kMB, KT = Cfg::kKT, NST = Cfg::kNST;
  constexpr int P = Cfg::kP, NCONS = Cfg::kNCons, STAGE = Cfg::kStageBytes;
  constexpr int CPT = Cfg::kChunksPerTile;
  static_assert(CPT % KS == 0, "chunks per tile");

  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);            // [NST]
  uint64_t* empty_bar = full_bar + NST;                              // [NST]
  float* s_scalar = reinterpret_cast<float*>(smem + 512);            // [MB] rms scale, + scratch
  uint8_t* s_stage = smem + 1024;
  float* s_x = reinterpret_cast<float*>(s_stage + (size_t)NST * STAGE);  // [MB][K]
  float* s_part = s_x + (size_t)MB * p.K;                                // [KS][MB][TN]

  const int tid = threadIdx.x;
  const int K = p.K;
  const int n_tiles = (K + KT - 1) / KT;
  const int panel0 = blockIdx.x * P;
  const int n_panels_total = p.N / 8;
  const int my_panels = min(P, n_panels_total - panel0);

  if (tid == 0) {
    for (int s = 0; s < NST; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], NCONS / 32);
    }
    mbar_fence_init();
  }
  __syncthreads();
  // let the next kernel in the stream start its own weight prefetch as early as possible
  pdl_launch_dependents();

  if (tid < 32) {
    // ===================== producer: weights never depend on the previous kernel ==========
    if (tid == 0) {
      const uint64_t pol = l2_policy_evict_first();
      const uint8_t* wbase = reinterpret_cast<const uint8_t*>(p.W);
      for (int t = 0; t < n_tiles; t++) {
        const int s = t % NST;
        const uint32_t ph = (uint32_t)(t / NST) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u);
        const int k0 = t * KT;
        const int kt = min(KT, K - k0);
        if constexpr (Cfg::kFmt != WF_BF16) {
          constexpr uint32_t cb = Cfg::kFmt == WF_MXFP8 ? 8u : 4u;               // code bytes per column of a panel
          const uint32_t code_bytes = (uint32_t)kt * cb;                          // kt/8 chunks * 64 B (MXFP4: 32 B)
          const uint32_t scale_bytes = (uint32_t)(((kt + 31) / 32 + 1) & ~1) * 8u;  // whole 16-byte pairs of blocks
          const int nbp = mx_nbp(K);
          mbar_expect_tx(&full_bar[s], (code_bytes + scale_bytes) * (uint32_t)my_panels);
          for (int pp = 0; pp < my_panels; pp++) {
            const size_t panel = (size_t)(panel0 + pp);
            bulk_g2s(s_stage + (size_t)s * STAGE + (size_t)pp * Cfg::kPanelBytes, wbase + (panel * (size_t)K + (size_t)k0) * cb,
                     code_bytes, &full_bar[s], pol);
            bulk_g2s(s_stage + (size_t)s * STAGE + Cfg::kScaleOff + (size_t)pp * (KT / 4), Ws + (panel * nbp + k0 / 32) * 8u,
                     scale_bytes, &full_bar[s], pol);
          }
        } else {
          const uint32_t bytes_per_panel = (uint32_t)kt * 16u;  // kt/8 chunks * 128 B
          mbar_expect_tx(&full_bar[s], bytes_per_panel * (uint32_t)my_panels);
          for (int pp = 0; pp < my_panels; pp++) {
            const uint8_t* src = wbase + ((size_t)(panel0 + pp) * (size_t)K + (size_t)k0) * 16u;
            bulk_g2s(s_stage + (size_t)s * STAGE + (size_t)pp * (KT * 16), src, bytes_per_panel, &full_bar[s], pol);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers ========================================================
  const int c = tid - 32;
  const int r = c % TN;        // row within the CTA tile
  const int j = c / TN;        // k-stream
  const int pp = r / 8, rr = r % 8;
  const int cw = c / 32;       // consumer warp index
  const int lane = tid & 31;

  pdl_wait();  // activations come from the previous kernel

  // ---- prologue: activations -> f32 in shared memory -----------------------------------
  if (PRO == PRO_PLAIN) {
    for (int m = 0; m < MB; m++)
      for (int k = c * 2; k < K; k += NCONS * 2) {
        float2 v = make_float2(0.f, 0.f);
        if (m < p.M) {
          uint32_t w = *reinterpret_cast<const uint32_t*>(p.x + (size_t)m * p.ldx + k);
          v.x = bf_lo(w);
          v.y = bf_hi(w);
        }
        *reinterpret_cast<float2*>(s_x + (size_t)m * K + k) = v;
      }
  } else {
    // RMSNorm.Forward (llamatransformer.go:633-660): Pow(x,2) -> f32, sequential f32 Mean,
    // +eps, f32(1/sqrt(f64)), t(x*r), t(.*w)
    for (int m = 0; m < MB; m++)
      for (int k = c * 2; k < K; k += NCONS * 2) {
        float2 v = make_float2(0.f, 0.f);
        if (m < p.M) {
          uint32_t w = *reinterpret_cast<const uint32_t*>(p.x + (size_t)m * p.ldx + k);
          v.x = bf_lo(w);
          v.y = bf_hi(w);
        }
        *reinterpret_cast<float2*>(s_x + (size_t)m * K + k) = v;
      }
    named_bar_sync(1, NCONS);
    if (p.rscale) {
      if (c < MB) s_scalar[c] = (c < p.M) ? p.rscale[c] : 0.f;
    } else if (p.strict_norm) {
      // reference order: one sequential chain per row; rows are spread over threads
      if (c < MB) {
        float sum = 0.f;
        const float* xr = s_x + (size_t)c * K;
        for (int k = 0; k < K; k++) sum = __fmaf_rn(xr[k], xr[k], sum);  // x*x exact (16-bit mantissa)
        float me = __fadd_rn(__fdiv_rn(sum, (float)K), p.eps);
        s_scalar[c] = (float)(1.0 / sqrt((double)me));
      }
    } else {
      // FAST: NCONS interleaved partial sums (element i -> partial i % NCONS), butterfly within
      // each warp, then sequentially over warps.
      for (int m = 0; m < MB; m++) {
        float sum = 0.f;
        const float* xr = s_x + (size_t)m * K;
        for (int k = c; k < K; k += NCONS) sum = __fmaf_rn(xr[k], xr[k], sum);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
        if (lane == 0) s_part[m * (NCONS / 32) + cw] = sum;
      }
      named_bar_sync(1, NCONS);
      if (c < MB) {
        float sum = 0.f;
        for (int w = 0; w < NCONS / 32; w++) sum = __fadd_rn(sum, s_part[c * (NCONS / 32) + w]);
        float me = __fadd_rn(__fdiv_rn(sum, (float)K), p.eps);
        s_scalar[c] = (float)(1.0 / sqrt((double)me));
      }
    }
    named_bar_sync(1, NCONS);
    for (int m = 0; m < MB; m++) {
      const float rs = s_scalar[m];
      for (int k = c; k < K; k += NCONS) {
        float n1 = trunc_bf(__fmul_rn(s_x[(size_t)m * K + k], rs));
        s_x[(size_t)m * K + k] = trunc_bf(__fmul_rn(n1, bf2f(p.norm_w[k])));
      }
    }
  }
  named_bar_sync(1, NCONS);

  // ---- main loop ------------------------------------------------------------------------
  float acc[MB];
#pragma unroll
  for (int m = 0; m < MB; m++) acc[m] = 0.f;

  constexpr int NI = CPT / KS;  // chunks of one thread per full k-tile
  for (int t = 0; t < n_tiles; t++) {
    const int s = t % NST;
    const uint32_t ph = (uint32_t)(t / NST) & 1u;
    mbar_wait(&full_bar[s], ph);
    const int k0 = t * KT;
    const int nchunks = min(KT, K - k0) / 8;
    if constexpr (Cfg::kFmt == WF_MXFP8) {
      const uint8_t* ctile = s_stage + (size_t)s * STAGE + (size_t)pp * Cfg::kPanelBytes + rr * 8;
      const uint8_t* stile = s_stage + (size_t)s * STAGE + Cfg::kScaleOff + (size_t)pp * (KT / 4) + rr;
      constexpr int UNROLL = MB > 2 ? 1 : 4;   // eight rows' accumulators and operands fill the registers already
#pragma unroll UNROLL
      for (int ch = j; ch < nchunks; ch += KS) {
        float w[8];
        mx_decode8(*reinterpret_cast<const uint2*>(ctile + ch * 64), mx_scale(stile[(ch >> 2) * 8]), w);
        const float* xk = s_x + k0 + ch * 8;
#pragma unroll
        for (int m = 0; m < MB; m++) {
          const float4 xa = *reinterpret_cast<const float4*>(xk + (size_t)m * K);
          const float4 xb = *reinterpret_cast<const float4*>(xk + (size_t)m * K + 4);
          float a = acc[m];
          a = __fmaf_rn(xa.x, w[0], a);
          a = __fmaf_rn(xa.y, w[1], a);
          a = __fmaf_rn(xa.z, w[2], a);
          a = __fmaf_rn(xa.w, w[3], a);
          a = __fmaf_rn(xb.x, w[4], a);
          a = __fmaf_rn(xb.y, w[5], a);
          a = __fmaf_rn(xb.z, w[6], a);
          a = __fmaf_rn(xb.w, w[7], a);
          acc[m] = a;
        }
      }
    } else if constexpr (Cfg::kFmt == WF_MXFP4) {
      const uint8_t* ctile = s_stage + (size_t)s * STAGE + (size_t)pp * Cfg::kPanelBytes + rr * 4;
      const uint8_t* stile = s_stage + (size_t)s * STAGE + Cfg::kScaleOff + (size_t)pp * (KT / 4) + rr;
      constexpr int UNROLL = MB > 2 ? 1 : 4;
#pragma unroll UNROLL
      for (int ch = j; ch < nchunks; ch += KS) {
        uint32_t P[4];   // P[g] = {column g, column g + 4}
        mx4_decode8(*reinterpret_cast<const uint32_t*>(ctile + ch * 32), mx4_scale2(stile[(ch >> 2) * 8]), P);
        const float* xk = s_x + k0 + ch * 8;
#pragma unroll
        for (int m = 0; m < MB; m++) {
          const float4 xa = *reinterpret_cast<const float4*>(xk + (size_t)m * K);
          const float4 xb = *reinterpret_cast<const float4*>(xk + (size_t)m * K + 4);
          float a = acc[m];
          a = __fmaf_rn(xa.x, bf_lo(P[0]), a);
          a = __fmaf_rn(xa.y, bf_lo(P[1]), a);
          a = __fmaf_rn(xa.z, bf_lo(P[2]), a);
          a = __fmaf_rn(xa.w, bf_lo(P[3]), a);
          a = __fmaf_rn(xb.x, bf_hi(P[0]), a);
          a = __fmaf_rn(xb.y, bf_hi(P[1]), a);
          a = __fmaf_rn(xb.z, bf_hi(P[2]), a);
          a = __fmaf_rn(xb.w, bf_hi(P[3]), a);
          acc[m] = a;
        }
      }
    } else {
    const uint8_t* tile = s_stage + (size_t)s * STAGE + (size_t)pp * (KT * 16) + rr * 16;
    if (MB == 1 && NI % 4 == 0 && nchunks == CPT) {
      // Full tile, one activation row: groups of 4 chunks with register double buffering, so the
      // shared-memory loads of group g+1 are in flight while the 32 dependent FMAs of group g
      // issue (the chain is the critical path in LNB_ACC_STRICT: 4 cycles per k).
      constexpr int G = 4, NG = NI / G;
      uint4 wa[G], wb[G];
      float4 xa0[G], xa1[G], xb0[G], xb1[G];
      const float* xt = s_x + k0;
#define LNB_LOAD_GROUP(gi, W_, X0_, X1_)                                      \
  _Pragma("unroll") for (int q_ = 0; q_ < G; q_++) {                          \
    const int ch_ = j + KS * ((gi) * G + q_);                                 \
    W_[q_] = *reinterpret_cast<const uint4*>(tile + ch_ * 128);               \
    X0_[q_] = *reinterpret_cast<const float4*>(xt + ch_ * 8);                 \
    X1_[q_] = *reinterpret_cast<const float4*>(xt + ch_ * 8 + 4);             \
  }
#define LNB_FMA_GROUP(W_, X0_, X1_)                                           \
  _Pragma("unroll") for (int q_ = 0; q_ < G; q_++) {                          \
    float a_ = acc[0];                                                        \
    a_ = __fmaf_rn(X0_[q_].x, bf_lo(W_[q_].x), a_);                           \
    a_ = __fmaf_rn(X0_[q_].y, bf_hi(W_[q_].x), a_);                           \
    a_ = __fmaf_rn(X0_[q_].z, bf_lo(W_[q_].y), a_);                           \
    a_ = __fmaf_rn(X0_[q_].w, bf_hi(W_[q_].y), a_);                           \
    a_ = __fmaf_rn(X1_[q_].x, bf_lo(W_[q_].z), a_);                           \
    a_ = __fmaf_rn(X1_[q_].y, bf_hi(W_[q_].z), a_);                           \
    a_ = __fmaf_rn(X1_[q_].z, bf_lo(W_[q_].w), a_);                           \
    a_ = __fmaf_rn(X1_[q_].w, bf_hi(W_[q_].w), a_);                           \
    acc[0] = a_;                                                              \
  }
      LNB_LOAD_GROUP(0, wa, xa0, xa1)
#pragma unroll
      for (int gi = 0; gi < NG; gi += 2) {
        if (gi + 1 < NG) { LNB_LOAD_GROUP(gi + 1, wb, xb0, xb1) }
        LNB_FMA_GROUP(wa, xa0, xa1)
        if (gi + 2 < NG) { LNB_LOAD_GROUP(gi + 2, wa, xa0, xa1) }
        if (gi + 1 < NG) { LNB_FMA_GROUP(wb, xb0, xb1) }
      }
#undef LNB_LOAD_GROUP
#undef LNB_FMA_GROUP
    } else {
#pragma unroll 4
      for (int ch = j; ch < nchunks; ch += KS) {
        const uint4 wv = *reinterpret_cast<const uint4*>(tile + ch * 128);
        const float w0 = bf_lo(wv.x), w1 = bf_hi(wv.x), w2 = bf_lo(wv.y), w3 = bf_hi(wv.y);
        const float w4 = bf_lo(wv.z), w5 = bf_hi(wv.z), w6 = bf_lo(wv.w), w7 = bf_hi(wv.w);
        const float* xk = s_x + k0 + ch * 8;
#pragma unroll
        for (int m = 0; m < MB; m++) {
          const float4 xa = *reinterpret_cast<const float4*>(xk + (size_t)m * K);
          const float4 xb = *reinterpret_cast<const float4*>(xk + (size_t)m * K + 4);
          float a = acc[m];
          a = __fmaf_rn(xa.x, w0, a);
          a = __fmaf_rn(xa.y, w1, a);
          a = __fmaf_rn(xa.z, w2, a);
          a = __fmaf_rn(xa.w, w3, a);
          a = __fmaf_rn(xb.x, w4, a);
          a = __fmaf_rn(xb.y, w5, a);
          a = __fmaf_rn(xb.z, w6, a);
          a = __fmaf_rn(xb.w, w7, a);
          acc[m] = a;
        }
      }
    }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }

  // ---- combine the KS streams in stream order --------------------------------------------
  if (KS > 1) {
#pragma unroll
    for (int m = 0; m < MB; m++) s_part[((size_t)j * MB + m) * TN + r] = acc[m];
    named_bar_sync(1, NCONS);
  }
  // after the combine, thread e < TN*MB owns output (row e % TN, activation row e / TN)
  constexpr int NOUT = TN * MB;
  static_assert(NOUT % 32 == 0, "epilogue shuffles need whole warps");
  for (int e = c; e < NOUT; e += NCONS) {
    const int er = e % TN, em = e / TN;
    float v;
    if (KS > 1) {
      v = s_part[(size_t)em * TN + er];
      for (int jj = 1; jj < KS; jj++) v = __fadd_rn(v, s_part[((size_t)jj * MB + em) * TN + er]);
    } else {
      v = 0.f;
#pragma unroll
      for (int m = 0; m < MB; m++)
        if (m == em) v = acc[m];
    }
    const int n = (panel0 + er / 8) * 8 + (er % 8);  // global row of W
    const bool valid = (em < p.M) && (er / 8 < my_panels);
    gemv_epilogue<EPI>(p, v, n, em, valid, panel0 + er / 8, er, lane);
  }

  if (EPI == EPI_LOGITS) {
    if (p.st && p.publish) {
      __threadfence();
      named_bar_sync(1, NCONS);
      if (c == 0) logits_publish(p);
    }
  }
}


}  // namespace lnb
