// engine_batch.cuh -- the persistent decode engine for n <= 8 concurrent sequences (BASELINE config 5): ONE kernel launch
// advances all sequences by one token, every weight matrix streamed from HBM once for all of them.
//
// Why a second kernel: with 8 activation rows the activations of a projection no longer fit shared memory as f32
// (8 x 14336 x 4 B for w2; the kernel chain fell back to 2-row blocks and streamed w2 FOUR times per step), and the
// arithmetic per weight byte is 8x the single-sequence engine's: the step is bound by FFMA issue and the weight stream
// together, not by dependency latency.  Design:
//   * same skeleton as engine.cuh: a phase list, a static balanced panel split (eng_split), warp 0 = run-ahead bulk-copy
//     producer into a 4 x 32 KB ring, 256 consumers;
//   * activations between phases are plain bf16 in a CHUNK-MAJOR layout [K/8][8 rows][8] (cm_idx): the k-range of a k-tile
//     is one contiguous, coalesced block for all rows.  Every consumer thread fetches 16 bytes of the NEXT k-tile's
//     activations (ld.global.cg, one tile ahead, hidden behind the current tile's FMAs), converts its 8 values to f32 --
//     applying RMSNorm on the way: t(t(x * r[m]) * w[k]) -- into a double-buffered shared tile, and all rows of all warps
//     then read them as warp-wide broadcasts;
//   * phases are separated by a grid barrier (the activations are plain words here, and at 8 rows per step the ~2 us
//     barrier is a few per cent of a phase);
//   * the RMSNorm scale r[m] is a phase of its own (one CTA per sequence; STRICT: the binade scan of engine.cuh);
//   * FAST: two weight rows per thread x 8 sequences = 16 independent chains; STRICT: one weight row x 4 sequences per
//     thread (the two warps that share 32 rows split the sequences), each chain in the reference's k = 0, 1, 2, ... order --
//     with four independent chains per lane and two warps per scheduler the reference order stops being latency-bound.
// Per sequence the arithmetic is that of its own S=1 Forward (src/model/llamatransformer.go:145-180), expression for
// expression: STRICT results are bit-identical to independent oracle contexts (tests/test_gpu_model.py, tools/tp_check.py).
//
// LNB_ACC_FAST, tensor-core form (batch_engine_kernel<0>, LNB_BATCH_TC=1; the FMA-pipe form batch_engine_kernel<8> is the FAST
// default, it measured faster on an H100): the FAST projections run on the tensor cores as warpgroup MMAs (wgmma.cuh):
//   D[64 x 32] (registers, fp32)  +=  X[64 x 16k] (registers, bf16; row m = sequence m, rows >= 8 are zero)  .  W[32 x 16k]^T
// with the weight tile of a ring stage as the B operand -- it IS a K-major, no-swizzle operand already (8-row x 16-byte core
// matrices = the panels, as in gemm_tc.cuh); a tile of np panels takes ceil(np / 4) such 32-row slices, so a CTA with 3
// panels spends 4 panels' worth of tensor-core time.  Warp roles: 0 = weight producer (as before); 9 = activation blocks
// global -> shared (bulk copies of 128 k x 8 rows = 2 KB, after the phase's grid barrier); 4..7 = the MMA warpgroup (it loads
// the activation fragments from the shared block, issues the MMAs and hands the 8 accumulator rows over through shared
// memory); 1, 2, 3 and 8 = the per-row epilogue (bt_epilogue).
// RMSNorm moves into the SCALE phase, which stores the normalised row t(t(x * r) * w) next to r.  The accumulation order
// is the tensor core's: FAST only (documented reorder); STRICT stays on the FMA pipes in the reference's order.
#pragma once
#include "engine.cuh"
#include "gemm_tc.cuh"

namespace lnb {

enum { BP_GEMV = 0, BP_SDPA = 1, BP_REDUCE = 2, BP_SCALE = 3, BP_TOKENS = 4 };

struct BatchPhase {
  int type, pro, epi, flags;
  int N, K, kt, pad;
  const uint16_t* W;
  const uint16_t* x;        // GEMV / SCALE / SDPA(q) input, chunk-major bf16 [K/8][8][8]
  const uint16_t* norm_w;   // PRO_RMSNORM: weights applied while the activation tile is converted
  const uint16_t* res;      // chunk-major residual (EPI_RESID / REDUCE)
  uint16_t* out;            // chunk-major bf16 output (SCALE with EF_X_TOKEN: where the gathered embedding rows go)
  uint16_t* xn;             // SCALE, tensor-core form: the normalised row t(t(x * r[m]) * norm_w[k]), chunk-major (else NULL)
  float* out_f32;           // EPI_LOGITS: [8][ldo] f32 (row-major) or NULL
  int ldo, n_offset;
  uint16_t* cache_k;        // this layer's caches, sequence 0 (row m's sequence at + that sequence * cache_seq_stride)
  uint16_t* cache_v;
  int q_dim, kv_dim;
};

// the sequence whose cache row m reads and appends to: row_seq[m] (a batched step: one row per sequence; speculative
// verification: consecutive positions of one sequence)
LNB_DEVINL size_t be_cache_base(const int32_t* row_seq, int m, long long cache_seq_stride) {
  return (size_t)row_seq[m] * (size_t)cache_seq_stride;
}

struct BatchParams {
  const BatchPhase* phases;
  int n_phases, n;          // n = sequences in this step (<= 8)
  LnbDevState* st;
  const uint16_t* emb;
  int dim, head_dim, n_rep, seq_len;
  const float* cis;
  const uint16_t* silu_tab;
  float eps, attn_scale;
  int strict;
  const int32_t* tokens;    // [n] input token of every sequence
  const int32_t* pos_arr;   // [n] position it is fed at
  const int32_t* row_seq;   // [n] sequence of every row (its KV cache)
  const int32_t* row_tree;  // [n] speculative tree rows: slot and ancestor mask of every row (common.cuh KeyMap); else NULL
  long long cache_seq_stride;
  float* rscale;            // [8] RMSNorm scales of the running norm
  unsigned long long* keys; // [8] greedy-argmax keys (cleared by the host before the launch)
  int32_t* next_arr;        // [n] greedy tokens
  unsigned int* bar_ctr;
  LnbP2P p2p;
  int tp;
  unsigned long long timeout_ns;
  volatile uint32_t* err_host;
  unsigned long long* prof;  // NULL, or [gridDim.x][ENG_NPROF] cycle sums of consumer thread 0 (LNB_ENGINE_PROF): 0 grid barrier,
                             // 1 projection setup, 2 activation tile (convert + hand-over), 3 weight-stage wait, 4 FMAs,
                             // 5 epilogue, 6 SCALE, 7 attention, 8 other phases, 9 tiles
};

constexpr int BE_NW_OFF = 0;                 // f32 norm weights [K <= 4096]            16 KB   (SCALE: the row as f32)
constexpr int BE_XT_OFF = 16 * 1024;         // 2 x activation tile f32 [kt/8][8][8]    2 x 16 KB
constexpr int BE_PART_OFF = 48 * 1024;       // FAST stream partials [8 streams][8 rows][64]   16 KB
constexpr int BE_SCAN_OFF = 64 * 1024;       // binade-scan scratch 4 KB
constexpr int BE_R_OFF = 68 * 1024;          // r[8]
// tensor-core form: activation blocks of 128 k (2 KB) in a ring inside the work area; a block of mbarriers behind the work
// area; the accumulators of a row tile reach the epilogue warps through a double-buffered hand-over area
constexpr int BT_NXS = 8;                    // activation blocks in shared memory
constexpr int BT_KT_MAX = 512;
constexpr int BT_XB = 128 * 16;              // one block: 128 k x 8 rows x 2 B
constexpr int BT_X_OFF = 16 * 1024;          // 8 x 2 KB in the work area
constexpr int BT_D_OFF = 48 * 1024;          // accumulator hand-over [2][8][129] f32
constexpr int BT_SMEM = ENG_SMEM + 512;      // + the mbarriers of this form
constexpr int BT_NEPI = 128;                 // epilogue threads (consumer warps 0, 1, 2 and 7)
static_assert(BT_SMEM <= 227 * 1024, "shared memory per CTA");

// ---- one k-tile of the activations: this thread's 16-byte pieces of the chunk-major block [k0, k0 + kt) ------------------
// piece i (i < kt): chunk i >> 3 of the tile, row i & 7  ->  consecutive threads read consecutive 16 bytes
LNB_DEVINL void be_fetch(const uint16_t* __restrict__ x, int k0, int kt, int c, uint4 (&v)[2]) {
#pragma unroll
  for (int u = 0; u < 2; u++) {
    const int i = c + u * ENG_NCONS;
    if (i < kt) v[u] = ldcg_u4(x + (size_t)k0 * 8 + (size_t)i * 8);
  }
}
// convert to f32 (RMSNorm on the way when nw != NULL: t(t(x * r[m]) * w[k]), llamatransformer.go:633-660) into the shared tile
LNB_DEVINL void be_convert(const uint4 (&v)[2], int k0, int kt, int c, int n, const float* __restrict__ s_r, const float* __restrict__ s_nw,
                           float* __restrict__ dst) {
#pragma unroll
  for (int u = 0; u < 2; u++) {
    const int i = c + u * ENG_NCONS;
    if (i < kt) {
      const int m = i & 7, ch = i >> 3;
      float f[8] = {bf_lo(v[u].x), bf_hi(v[u].x), bf_lo(v[u].y), bf_hi(v[u].y), bf_lo(v[u].z), bf_hi(v[u].z), bf_lo(v[u].w), bf_hi(v[u].w)};
      if (m >= n) {
#pragma unroll
        for (int e = 0; e < 8; e++) f[e] = 0.f;
      } else if (s_nw) {
        const float rs = s_r[m];
        const float* w = s_nw + k0 + ch * 8;
#pragma unroll
        for (int e = 0; e < 8; e++) f[e] = trunc_bf(__fmul_rn(trunc_bf(__fmul_rn(f[e], rs)), w[e]));
      }
      float4* d = reinterpret_cast<float4*>(dst + (size_t)i * 8);
      d[0] = make_float4(f[0], f[1], f[2], f[3]);
      d[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
  }
}


// ---- tensor-core form: the fused epilogues for one (panel, sequence) = 8 consecutive weight rows of one sequence ----------
// Same arithmetic as gemv_epilogue (gemv.cuh), expression for expression, on 8 rows at once: in the chunk-major layout those
// are 16 contiguous bytes, so every input is ONE vector load issued before anything is stored (under a saturated weight
// stream a dependent global round trip costs microseconds), and the RoPE / SwiGLU partners are in the same thread.
// Called by all 32 lanes; lane = 8 * (panel % 4) + m.
LNB_DEVINL void bt_epilogue(const GemvParams& p, int epi, const float (&v)[8], int panel, int m, bool valid, int lane) {
  const int n0 = panel * 8;
  if (epi == EPI_RESID) {
    if (valid) {
      const size_t oi = cm_idx(m, n0);
      const uint4 r = ldcg_u4(p.res + oi);
      const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
      uint32_t o[4];
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const float lo = __fadd_rn(bf_lo(rw[e]), trunc_bf(v[2 * e]));          // ml.Add(x, t(linear))  llamatransformer.go:232,248
        const float hi = __fadd_rn(bf_hi(rw[e]), trunc_bf(v[2 * e + 1]));
        o[e] = (__float_as_uint(lo) >> 16) | (__float_as_uint(hi) & 0xffff0000u);
      }
      *reinterpret_cast<uint4*>(p.out_bf16 + oi) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  } else if (epi == EPI_P2P) {
    if (valid) {
      const uint32_t epoch = p.ar_epoch_override;
      const size_t off = ((size_t)((epoch & 1u) * p.p2p.n + p.p2p.rank)) * p.p2p.slot_elems + (size_t)m * p.ldo + n0;
#pragma unroll
      for (int r = 0; r < 8; r++) {
        if (r < p.p2p.n) {
          uint4* dst = reinterpret_cast<uint4*>(p.p2p.data[r] + off);          // 8 {value, epoch} words = 64 contiguous bytes per peer
#pragma unroll
          for (int e = 0; e < 4; e++) dst[e] = make_uint4(__float_as_uint(v[2 * e]), epoch, __float_as_uint(v[2 * e + 1]), epoch);
        }
      }
    }
  } else if (epi == EPI_LOGITS) {
    unsigned long long key = LNB_ARGMAX_EMPTY;
    float lv[8];
#pragma unroll
    for (int e = 0; e < 8; e++) {
      lv[e] = trunc_bf(v[e]);
      if (valid && lv[e] > -3.402823466e+38f) {
        const unsigned long long k2 = argmax_key(lv[e], (uint32_t)(n0 + e + p.n_offset));
        key = k2 > key ? k2 : key;
      }
    }
    if (valid && p.out_f32) {
      float4* dst = reinterpret_cast<float4*>(p.out_f32 + (size_t)m * p.ldo + n0);
      dst[0] = make_float4(lv[0], lv[1], lv[2], lv[3]);
      dst[1] = make_float4(lv[4], lv[5], lv[6], lv[7]);
    }
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {                 // the four panels of this warp that belong to sequence m
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
      key = other > key ? other : key;
    }
    if (lane < 8 && key != LNB_ARGMAX_EMPTY) atomicMax(&p.amax_keys_row[m], key);
  } else if (epi == EPI_QKV_ROPE) {
    if (valid) {
      const int pos = p.pos_arr[m], slot = p.row_tree ? tree_slot(p.row_tree[m]) : pos;   // RoPE at pos, stored at slot
      uint16_t* ck = p.cache_k + be_cache_base(p.row_seq, m, p.cache_seq_stride);
      uint16_t* cv = p.cache_v + be_cache_base(p.row_seq, m, p.cache_seq_stride);
      uint32_t o[4];
      if (n0 < p.q_dim + p.kv_dim) {
        const int nn0 = (n0 < p.q_dim) ? n0 : n0 - p.q_dim;
        const int i0 = (nn0 % p.head_dim) >> 1;
        const float4* fc = reinterpret_cast<const float4*>(p.cis + ((size_t)pos * (p.head_dim / 2) + i0) * 2);
        const float4 c01 = fc[0], c23 = fc[1];
        const float cs[8] = {c01.x, c01.y, c01.z, c01.w, c23.x, c23.y, c23.z, c23.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
          // complex64 * complex64 through float64 (operations_impl.go:414-417; SURVEY F16-A1), products exact in f64
          const double a = (double)trunc_bf(v[2 * i]), b = (double)trunc_bf(v[2 * i + 1]);
          const double cc = (double)cs[2 * i], dd = (double)cs[2 * i + 1];
          const float re = (float)(a * cc - b * dd), im = (float)(a * dd + b * cc);
          o[i] = (__float_as_uint(re) >> 16) | (__float_as_uint(im) & 0xffff0000u);
        }
        uint16_t* dst = (n0 < p.q_dim) ? p.out_bf16 + cm_idx(m, n0) : ck + (size_t)slot * p.kv_dim + nn0;         // SetSlice :402
        *reinterpret_cast<uint4*>(dst) = make_uint4(o[0], o[1], o[2], o[3]);
      } else {
#pragma unroll
        for (int i = 0; i < 4; i++) o[i] = (__float_as_uint(v[2 * i]) >> 16) | (__float_as_uint(v[2 * i + 1]) & 0xffff0000u);
        *reinterpret_cast<uint4*>(cv + (size_t)slot * p.kv_dim + (n0 - p.q_dim - p.kv_dim)) = make_uint4(o[0], o[1], o[2], o[3]);  // :403
      }
    }
  } else if (epi == EPI_SWIGLU) {
    // rows 0..3 of the panel = gate rows of hidden units 4*panel .. +3, rows 4..7 their up rows (retile_kernel)
    if (valid) {
      uint16_t sg[4];
#pragma unroll
      for (int e = 0; e < 4; e++) sg[e] = p.silu_tab[f2bf(v[e])];                 // t(TABLE_SILU[bits]) activations.go:38
      uint16_t o[4];
#pragma unroll
      for (int e = 0; e < 4; e++) o[e] = f2bf(__fmul_rn(bf2f(sg[e]), trunc_bf(v[e + 4])));   // MultiplyElementwise :614
      *reinterpret_cast<uint2*>(p.out_bf16 + cm_idx(m, panel * 4)) =
          make_uint2((uint32_t)o[0] | ((uint32_t)o[1] << 16), (uint32_t)o[2] | ((uint32_t)o[3] << 16));
    }
  }
}

template <int KS>
__global__ void __launch_bounds__(ENG_THREADS, 1) batch_engine_kernel(const BatchParams P) {
  using Cfg = EngCfg<KS>;
  constexpr bool TC = (KS == 0);
  constexpr int NST = Cfg::kNST, STAGE = Cfg::kStage, PT = TC ? 16 : Cfg::kPT;
  constexpr int MB = 8;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + NST;
  uint64_t* fullxs_bar = reinterpret_cast<uint64_t*>(smem + ENG_SMEM);   // (tensor-core form) activation blocks, shared
  uint64_t* emptyxs_bar = fullxs_bar + BT_NXS;
  uint64_t* accfull_bar = emptyxs_bar + BT_NXS;    // the two accumulator hand-over buffers
  uint64_t* accempty_bar = accfull_bar + 2;
  float* s_scalar = reinterpret_cast<float*>(smem + 256);
  GemvParams* gp = reinterpret_cast<GemvParams*>(smem + 512);
  uint8_t* s_ring = smem + 1024;
  uint8_t* s_work = s_ring + ENG_RING;
  float* s_nw = reinterpret_cast<float*>(s_work + BE_NW_OFF);
  float* s_xt = reinterpret_cast<float*>(s_work + BE_XT_OFF);
  float* s_part = reinterpret_cast<float*>(s_work + BE_PART_OFF);
  float* s_r = reinterpret_cast<float*>(s_work + BE_R_OFF);

  const int tid = threadIdx.x;
  const int G = gridDim.x, bid = blockIdx.x;
  const int n = P.n;
  if (tid == 0) {
    for (int s = 0; s < NST; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], TC ? 1 : ENG_NCONS);     // every consumer thread reads every stage / the MMAs' commit
    }
    if (TC) {
      for (int s = 0; s < BT_NXS; s++) { mbar_init(&fullxs_bar[s], 1); mbar_init(&emptyxs_bar[s], 1); }
      for (int b = 0; b < 2; b++) { mbar_init(&accfull_bar[b], 1); mbar_init(&accempty_bar[b], BT_NEPI); }
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (tid < 32) {
    // =========================== producer: the weights of every projection, ahead of the consumers ================
    const uint64_t pol = l2_policy_evict_first();
    uint32_t seq = 0;
    for (int ph = 0; ph < P.n_phases; ph++) {
      const BatchPhase* E = P.phases + ph;
      if (E->type != BP_GEMV) continue;
      const int K = E->K, kt = E->kt;
      const int n_tiles = (K + kt - 1) / kt;
      int p0, p1;
      eng_split(E->N / 8, bid, G, &p0, &p1);
      const uint8_t* wbase = reinterpret_cast<const uint8_t*>(E->W);
      for (int rt = p0; rt < p1; rt += PT) {
        const int np = min(PT, p1 - rt);
        const uint8_t* src_row = wbase + (size_t)(rt + tid) * (size_t)K * 16u;
        for (int t = 0; t < n_tiles; t++, seq++) {
          const int s = seq % NST;
          const uint32_t par = (seq / NST) & 1u;
          const int k0 = t * kt;
          const uint32_t bytes_per_panel = (uint32_t)min(kt, K - k0) * 16u;
          eng_mbar_wait(&empty_bar[s], par ^ 1u, P.err_host, P.timeout_ns, false, seq);
          if (tid == 0) mbar_expect_tx(&full_bar[s], bytes_per_panel * (uint32_t)np);
          __syncwarp();
          if (tid < np)
            bulk_g2s(s_ring + (size_t)s * STAGE + (size_t)tid * ((size_t)kt * 16), src_row + (size_t)k0 * 16u, bytes_per_panel, &full_bar[s], pol);
        }
      }
    }
    return;
  }
  if (tid >= 32 + ENG_NCONS) {
    // ====================== tensor-core form: the activation blocks of every projection, global -> shared ===========
    // (one thread; a projection's input is complete once the grid barrier that closed the previous phase has been passed
    // by everybody: phases 0 .. ph-1 each end with one barrier)
    if (!TC || tid != 32 + ENG_NCONS) return;
    const uint64_t polx = l2_policy_evict_last();
    uint8_t* xring = s_work + BT_X_OFF;
    uint32_t seqx = 0;
    for (int ph = 0; ph < P.n_phases; ph++) {
      const BatchPhase* E = P.phases + ph;
      if (E->type != BP_GEMV) continue;
      int p0, p1;
      eng_split(E->N / 8, bid, G, &p0, &p1);
      if (p1 <= p0) continue;
      {
        const unsigned int target = (unsigned int)ph * (unsigned int)G;
        unsigned long long t0 = 0;
        uint32_t spins = 0;
        while (ld_acquire_u32(P.bar_ctr) < target) {
          if ((++spins & 1023u) == 0u && P.timeout_ns) {
            const unsigned long long now = global_timer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 4 * P.timeout_ns) eng_fail(P.err_host, 0xC1000000u | (target & 0xffffffu));
          }
        }
        fence_proxy_async();                       // the other CTAs' plain stores, then this thread's bulk-copy reads
      }
      const int K = E->K;
      const int n_blk = (K + 127) / 128;
      const uint8_t* xb = reinterpret_cast<const uint8_t*>(E->x);
      for (int rt = p0; rt < p1; rt += PT) {
        for (int b = 0; b < n_blk; b++, seqx++) {
          const int s = seqx % BT_NXS;
          const uint32_t par = (seqx / BT_NXS) & 1u;
          const uint32_t bytes = (uint32_t)min(128, K - b * 128) * 16u;
          eng_mbar_wait(&emptyxs_bar[s], par ^ 1u, P.err_host, P.timeout_ns, false, seqx);
          mbar_expect_tx(&fullxs_bar[s], bytes);
          bulk_g2s(xring + (size_t)s * BT_XB, xb + (size_t)b * BT_XB, bytes, &fullxs_bar[s], polx);
        }
      }
    }
    return;
  }

  // ======================================= consumers =============================================================
  const int c = tid - 32;
  const int lane = tid & 31;
  const int cw = c >> 5;
  const int cw_u = __shfl_sync(0xffffffffu, cw, 0);     // (the same value, known to the compiler as warp-uniform)
  // FAST: thread = (rows r and r + 32 of the 64-row tile, k-stream j), all 8 sequences.
  // STRICT: thread = (row r of the 128-row tile, sequences mh*4 .. mh*4+3): two warps share 32 rows, each takes half of the
  // sequences -- four independent reference-order chains per lane, two warps per scheduler.
  const int r = (KS == 1) ? (c & 127) : (c & 31);
  const int j = (KS == 1) ? 0 : (c >> 5);
  const int mh = (KS == 1) ? (c >> 7) : 0;
  uint32_t seq = 0;
  uint32_t seqx = 0, acc_cnt = 0;           // (tensor-core form) activation stages and accumulators used so far
  unsigned int mma_acc = 0, mma_w = 0, mma_x = 0, mma_issue = 0;   // LNB_ENGINE_PROF, MMA issuer: cycles waiting for a free
                                            // accumulator / a weight stage / an activation block, and issuing
  unsigned int n_bar = 0;
  uint32_t epoch = (P.tp > 1) ? P.st->ar_epoch : 0u;
  EngineParams BP{};                        // (eng_grid_barrier / eng_wait_word take the single-sequence parameter block)
  BP.bar_ctr = P.bar_ctr; BP.timeout_ns = P.timeout_ns; BP.err_host = P.err_host; BP.p2p = P.p2p; BP.st = P.st;
  const bool prof_on = P.prof != nullptr && c == 0;
  unsigned long long* pr = prof_on ? P.prof + (size_t)bid * ENG_NPROF : nullptr;
  long long t_mark = prof_on ? clock64() : 0;
  // (cycle sums stay in registers until the kernel ends: a global read-modify-write per mark would itself wait microseconds
  // behind the weight stream and land in the next section)
  unsigned int pacc[ENG_NPROF];
#pragma unroll
  for (int k = 0; k < ENG_NPROF; k++) pacc[k] = 0u;
#define BE_PROF(slot) do { if (prof_on) { const long long n_ = clock64(); pacc[slot] += (unsigned int)(n_ - t_mark); t_mark = n_; } } while (0)

  for (int ph = 0; ph < P.n_phases; ph++) {
    const BatchPhase* E = P.phases + ph;
    const int type = E->type;
    if (type == BP_SCALE) {
      // ---- RMSNorm scale of row m = bid (one CTA per sequence); EF_X_TOKEN: the row is the embedding of the sequence's
      // input token and is also stored as the residual stream of layer 0 (ml.Fwd_Get_Rows, operations_impl.go:142-173) ----
      if (bid < n) {
        const int m = bid, K = E->K;
        float* s_x = s_nw;   // the row as f32 (the GEMV phases' norm-weight area is free during this phase)
        const bool from_tok = (E->flags & EF_X_TOKEN) != 0;
        const uint16_t* row = from_tok ? P.emb + (size_t)P.tokens[m] * P.dim : nullptr;
        for (int chk = c; chk < K / 8; chk += ENG_NCONS) {
          const uint4 v = from_tok ? ldcg_u4(row + (size_t)chk * 8) : ldcg_u4(E->x + ((size_t)chk * 8 + m) * 8);
          if (from_tok) *reinterpret_cast<uint4*>(E->out + ((size_t)chk * 8 + m) * 8) = v;
          float4* d = reinterpret_cast<float4*>(s_x + (size_t)chk * 8);
          d[0] = make_float4(bf_lo(v.x), bf_hi(v.x), bf_lo(v.y), bf_hi(v.y));
          d[1] = make_float4(bf_lo(v.z), bf_hi(v.z), bf_lo(v.w), bf_hi(v.w));
        }
        named_bar_sync(1, ENG_NCONS);
        if (P.strict) {
          int ch = 0, nt = 0;
          eng_scan_shape(K, &ch, &nt);
          uint8_t* scr = s_work + BE_SCAN_OFF;
          float* s_sum = s_scalar + 4;
          switch (ch) {
            case 16: eng_seq_sumsq<16>(s_x, c, nt, scr, s_sum); break;
            case 8: eng_seq_sumsq<8>(s_x, c, nt, scr, s_sum); break;
            case 4: eng_seq_sumsq<4>(s_x, c, nt, scr, s_sum); break;
            default: eng_seq_sumsq<2>(s_x, c, nt, scr, s_sum); break;
          }
          if (c == 0) {
            const float me = __fadd_rn(__fdiv_rn(*s_sum, (float)K), P.eps);
            P.rscale[m] = s_scalar[8] = (float)(1.0 / sqrt((double)me));
          }
        } else {
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
            P.rscale[m] = s_scalar[8] = (float)(1.0 / sqrt((double)me));
          }
        }
        if (E->xn) {
          // the normalised row for the tensor-core projections: t(t(x * r) * w[k]) (llamatransformer.go:633-660), chunk-major
          named_bar_sync(1, ENG_NCONS);
          const float rs = s_scalar[8];
          for (int chk = c; chk < K / 8; chk += ENG_NCONS) {
            const uint4 w = __ldg(reinterpret_cast<const uint4*>(E->norm_w + (size_t)chk * 8));
            const float wf[8] = {bf_lo(w.x), bf_hi(w.x), bf_lo(w.y), bf_hi(w.y), bf_lo(w.z), bf_hi(w.z), bf_lo(w.w), bf_hi(w.w)};
            const float* xs = s_x + (size_t)chk * 8;
            uint32_t o[4];
#pragma unroll
            for (int e = 0; e < 4; e++) {
              const float lo = trunc_bf(__fmul_rn(trunc_bf(__fmul_rn(xs[2 * e], rs)), wf[2 * e]));
              const float hi = trunc_bf(__fmul_rn(trunc_bf(__fmul_rn(xs[2 * e + 1], rs)), wf[2 * e + 1]));
              o[e] = (__float_as_uint(lo) >> 16) | (__float_as_uint(hi) & 0xffff0000u);
            }
            *reinterpret_cast<uint4*>(E->xn + ((size_t)chk * 8 + m) * 8) = make_uint4(o[0], o[1], o[2], o[3]);
          }
        }
      }
    } else if (type == BP_GEMV && TC) {
      // ---- tensor-core projection: D[seq, weight row] += X[seq, 16k] . W[weight row, 16k] per k16 step ------------------
      const int K = E->K, kt = E->kt;
      const int n_tiles = (K + kt - 1) / kt;
      int p0, p1;
      eng_split(E->N / 8, bid, G, &p0, &p1);
      if (p1 > p0) {
        if (cw_u < 3 || cw_u == 7) {
          // -- epilogue warps (hardware warps 1, 2, 3, 8): thread ec = (panel of the tile, sequence)
          if (c == 0) {
            GemvParams g{};
            g.W = E->W; g.N = E->N; g.K = K; g.M = n; g.eps = P.eps;
            g.out_bf16 = E->out; g.out_f32 = E->out_f32; g.ldo = E->ldo; g.res = E->res; g.cm = 1;
            g.q_dim = E->q_dim; g.kv_dim = E->kv_dim; g.head_dim = P.head_dim;
            g.cache_k = E->cache_k; g.cache_v = E->cache_v; g.pos_arr = P.pos_arr; g.cache_seq_stride = P.cache_seq_stride;
            g.row_seq = P.row_seq; g.row_tree = P.row_tree;
            g.cis = P.cis; g.silu_tab = P.silu_tab;
            g.n_offset = E->n_offset; g.st = nullptr; g.argmax_row = -1; g.amax_keys_row = P.keys;
            g.pos_ptr = P.pos_arr; g.m_off = 0;
            g.p2p = P.p2p; g.ar_epoch_override = epoch;
            if (E->epi == EPI_P2P) g.st = P.st;
            *gp = g;
          }
          const float* s_d = reinterpret_cast<const float*>(s_work + BT_D_OFF);
          const int ec = (cw_u == 7) ? c - 128 : c;
          const int pp = ec >> 3, m = ec & 7;
          const int epi = E->epi;
          named_bar_sync(2, BT_NEPI);
          const GemvParams& g = *gp;
          BE_PROF(1);
          for (int rt = p0; rt < p1; rt += PT) {
            const int np = min(PT, p1 - rt);
            const int buf = acc_cnt & 1;
            eng_mbar_wait(&accfull_bar[buf], (acc_cnt >> 1) & 1u, P.err_host, P.timeout_ns, false, acc_cnt);
            acc_cnt++;
            BE_PROF(3);
            const float* sd = s_d + (size_t)buf * (8 * 129);
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; e++) v[e] = sd[m * 129 + pp * 8 + e];
            mbar_arrive(&accempty_bar[buf]);              // the MMA warpgroup may hand the tile after next over in this buffer
            bt_epilogue(g, epi, v, rt + pp, m, pp < np && m < n, lane);
            BE_PROF(5);
          }
          fence_proxy_async();      // these stores are read by the next projection's bulk copies (after the grid barrier)
        } else {
          // -- the MMA warpgroup (hardware warps 4..7).  Warp 4 holds accumulator rows 0..7 = the sequences (fragment row
          //    l / 4 of lane l); it alone loads activations (the other warps' rows of A are zero) and hands the results over
          const int wl = cw_u - 3;                       // warp of the warpgroup
          const int g8 = lane >> 2, cq = 2 * (lane & 3);
          const bool pm = P.prof != nullptr && wl == 0 && lane == 0;
          long long tm = pm ? clock64() : 0;
#define BT_MARK(var) do { if (pm) { const long long n_ = clock64(); var += (unsigned int)(n_ - tm); tm = n_; } } while (0)
          const uint8_t* xring = s_work + BT_X_OFF;
          float* s_d = reinterpret_cast<float*>(s_work + BT_D_OFF);
          for (int rt = p0; rt < p1; rt += PT) {
            const int np = min(PT, p1 - rt);
            const int nsl = (np + 3) >> 2;               // 32-row slices of the tile
            float d[4][16];
#pragma unroll
            for (int q = 0; q < 4; q++)
#pragma unroll
              for (int i = 0; i < 16; i++) d[q][i] = 0.f;
            uint32_t accum = 0u;
            for (int t = 0; t < n_tiles; t++) {
              const int ktt = min(kt, K - t * kt);
              const int sw = seq % NST;
              eng_mbar_wait(&full_bar[sw], (seq / NST) & 1u, P.err_host, P.timeout_ns, false, seq);
              BT_MARK(mma_w);
              seq++;
              const uint32_t w_base = smem_u32(s_ring + (size_t)sw * STAGE);
              for (int kb0 = 0; kb0 < ktt; kb0 += 128) {
                const int ss = seqx % BT_NXS;
                if (wl == 0) eng_mbar_wait(&fullxs_bar[ss], (seqx / BT_NXS) & 1u, P.err_host, P.timeout_ns, false, seqx);
                BT_MARK(mma_x);
                seqx++;
                // A fragments of the (up to) 8 k16 steps of this block: chunk-major [16 chunks][8 rows][8] = core matrices
                const int nk16 = min(128, ktt - kb0) / 16;
                uint32_t a[8][4];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                  a[j][0] = a[j][1] = a[j][2] = a[j][3] = 0u;
                  if (wl == 0 && j < nk16) {
                    const uint8_t* xs = xring + (size_t)ss * BT_XB + g8 * 16 + cq * 2;
                    a[j][0] = *reinterpret_cast<const uint32_t*>(xs + (2 * j) * 128);
                    a[j][2] = *reinterpret_cast<const uint32_t*>(xs + (2 * j + 1) * 128);
                  }
                }
                __syncwarp();
                if (wl == 0 && lane == 0) mbar_arrive(&emptyxs_bar[ss]);   // the block is in registers: it may be overwritten
                // B: next k-chunk 128 B, next panel kt * 16 B, next k16 step 256 B (= 16 in the descriptor's address field);
                // slice q = panels 4q .. 4q+3
                const uint64_t b0 = gmma_desc(w_base + (uint32_t)kb0 * 16u, 128, (uint32_t)kt * 16u);
                const uint64_t slice = (uint64_t)(((uint32_t)kt * 64u) >> 4);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 8; j++) {
                  if (j < nk16) {
#pragma unroll
                    for (int q = 0; q < 4; q++)
                      if (q < nsl) wgmma_rs_n32(d[q], a[j], b0 + (uint64_t)q * slice + (uint64_t)(16 * j), accum);
                    accum = 1u;
                  }
                }
                wgmma_commit();
                BT_MARK(mma_issue);
              }
              wgmma_wait<0>();                             // this stage's MMAs have read the weights
              if (wl == 0 && lane == 0) mbar_arrive(&empty_bar[sw]);
            }
#pragma unroll
            for (int q = 0; q < 4; q++) wgmma_fence_regs(d[q]);
            if (wl == 0) {
              const int buf = acc_cnt & 1;
              eng_mbar_wait(&accempty_bar[buf], ((acc_cnt >> 1) & 1u) ^ 1u, P.err_host, P.timeout_ns, false, acc_cnt);
              BT_MARK(mma_acc);
              float* sd = s_d + (size_t)buf * (8 * 129) + g8 * 129 + cq;
#pragma unroll
              for (int q = 0; q < 4; q++)
                if (q < nsl) {
#pragma unroll
                  for (int cb = 0; cb < 4; cb++) { sd[q * 32 + cb * 8] = d[q][4 * cb]; sd[q * 32 + cb * 8 + 1] = d[q][4 * cb + 1]; }
                }
              __syncwarp();
              if (lane == 0) mbar_arrive(&accfull_bar[buf]);
            }
            acc_cnt++;
          }
#undef BT_MARK
        }
      }
    } else if (!TC && type == BP_GEMV) {
      const int K = E->K, kt = E->kt;
      const int n_tiles = (K + kt - 1) / kt;
      int p0, p1;
      eng_split(E->N / 8, bid, G, &p0, &p1);
      if (p1 > p0) {
        const bool with_norm = (E->pro == PRO_RMSNORM);
        uint4 xv[2];
        be_fetch(E->x, 0, min(kt, K), c, xv);              // the first tile's activations are in flight during the setup
        if (c == 0) {
          GemvParams g{};
          g.W = E->W; g.N = E->N; g.K = K; g.M = n; g.eps = P.eps;
          g.out_bf16 = E->out; g.out_f32 = E->out_f32; g.ldo = E->ldo; g.res = E->res; g.cm = 1;
          g.q_dim = E->q_dim; g.kv_dim = E->kv_dim; g.head_dim = P.head_dim;
          g.cache_k = E->cache_k; g.cache_v = E->cache_v; g.pos_arr = P.pos_arr; g.cache_seq_stride = P.cache_seq_stride;
          g.row_seq = P.row_seq; g.row_tree = P.row_tree;
          g.cis = P.cis; g.silu_tab = P.silu_tab;
          g.n_offset = E->n_offset; g.st = nullptr; g.argmax_row = -1; g.amax_keys_row = P.keys;
          g.pos_ptr = P.pos_arr; g.m_off = 0;
          g.p2p = P.p2p; g.ar_epoch_override = epoch;
          if (E->epi == EPI_P2P) g.st = P.st;
          *gp = g;
        }
        if (with_norm) {
          for (int k = c * 8; k < K; k += ENG_NCONS * 8) {
            const uint4 w = __ldg(reinterpret_cast<const uint4*>(E->norm_w + k));
            float4* d = reinterpret_cast<float4*>(s_nw + k);
            d[0] = make_float4(bf_lo(w.x), bf_hi(w.x), bf_lo(w.y), bf_hi(w.y));
            d[1] = make_float4(bf_lo(w.z), bf_hi(w.z), bf_lo(w.w), bf_hi(w.w));
          }
          if (c < MB) s_r[c] = (c < n) ? __ldcg(P.rscale + c) : 0.f;
        }
        named_bar_sync(1, ENG_NCONS);
        BE_PROF(1);
        for (int rt = p0; rt < p1; rt += PT) {
          const int np = min(PT, p1 - rt);
          const int pp0 = r >> 3, rr = r & 7, pp1 = pp0 + 4;
          const bool on0 = pp0 < np;
          const bool on1 = (KS > 1) && (pp1 < np);
          const bool chain = true;
          float acc0[MB], acc1[MB];
#pragma unroll
          for (int m = 0; m < MB; m++) { acc0[m] = 0.f; acc1[m] = 0.f; }
          if (rt > p0) be_fetch(E->x, 0, min(kt, K), c, xv);         // (a new row tile starts over at k = 0)
          for (int t = 0; t < n_tiles; t++) {
            const int k0 = t * kt;
            const int ktt = min(kt, K - k0);
            float* xt = s_xt + (size_t)(t & 1) * (size_t)(kt * 8);
            // this tile's activations: registers -> f32 tile; the next tile's: HBM/L2 -> registers (hidden behind the FMAs)
            be_convert(xv, k0, ktt, c, n, s_r, with_norm ? s_nw : nullptr, xt);
            if (t + 1 < n_tiles) be_fetch(E->x, k0 + kt, min(kt, K - k0 - kt), c, xv);
            named_bar_sync(1, ENG_NCONS);
            BE_PROF(2);
            if (chain) {
              const int s = seq % NST;
              const uint32_t par = (seq / NST) & 1u;
              eng_mbar_wait(&full_bar[s], par, P.err_host, P.timeout_ns, false, seq);
              seq++;
              BE_PROF(3);
              if (prof_on) pacc[9] += 1u;
              const int nchunks = ktt / 8;
              const uint8_t* tile0 = s_ring + (size_t)s * STAGE + (on0 ? (size_t)pp0 * ((size_t)kt * 16) : (size_t)0) + rr * 16;
              const uint8_t* tile1 = s_ring + (size_t)s * STAGE + (on1 ? (size_t)pp1 * ((size_t)kt * 16) : (size_t)0) + rr * 16;
              if (KS == 1) {
                if (on0) {
#pragma unroll 2
                  for (int ch = 0; ch < nchunks; ch++) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(tile0 + ch * 128);
                    const float w0 = bf_lo(wv.x), w1 = bf_hi(wv.x), w2 = bf_lo(wv.y), w3 = bf_hi(wv.y);
                    const float w4 = bf_lo(wv.z), w5 = bf_hi(wv.z), w6 = bf_lo(wv.w), w7 = bf_hi(wv.w);
                    const float* xc = xt + (size_t)ch * 64 + mh * 32;
#pragma unroll
                    for (int m = 0; m < 4; m++) {
                      const float4 xa = *reinterpret_cast<const float4*>(xc + m * 8);
                      const float4 xb = *reinterpret_cast<const float4*>(xc + m * 8 + 4);
                      float a = acc0[m];
                      a = __fmaf_rn(xa.x, w0, a); a = __fmaf_rn(xa.y, w1, a); a = __fmaf_rn(xa.z, w2, a); a = __fmaf_rn(xa.w, w3, a);
                      a = __fmaf_rn(xb.x, w4, a); a = __fmaf_rn(xb.y, w5, a); a = __fmaf_rn(xb.z, w6, a); a = __fmaf_rn(xb.w, w7, a);
                      acc0[m] = a;
                    }
                  }
                }
              } else {
                for (int ch = j; ch < nchunks; ch += KS) {
                  const uint4 wa = *reinterpret_cast<const uint4*>(tile0 + ch * 128);
                  const uint4 wb = *reinterpret_cast<const uint4*>(tile1 + ch * 128);
                  const float a0 = bf_lo(wa.x), a1 = bf_hi(wa.x), a2 = bf_lo(wa.y), a3 = bf_hi(wa.y);
                  const float a4 = bf_lo(wa.z), a5 = bf_hi(wa.z), a6 = bf_lo(wa.w), a7 = bf_hi(wa.w);
                  const float b0 = bf_lo(wb.x), b1 = bf_hi(wb.x), b2 = bf_lo(wb.y), b3 = bf_hi(wb.y);
                  const float b4 = bf_lo(wb.z), b5 = bf_hi(wb.z), b6 = bf_lo(wb.w), b7 = bf_hi(wb.w);
                  const float* xc = xt + (size_t)ch * 64;
#pragma unroll
                  for (int m = 0; m < MB; m++) {
                    const float4 xa = *reinterpret_cast<const float4*>(xc + m * 8);
                    const float4 xb = *reinterpret_cast<const float4*>(xc + m * 8 + 4);
                    float a = acc0[m], b = acc1[m];
                    a = __fmaf_rn(xa.x, a0, a); b = __fmaf_rn(xa.x, b0, b);
                    a = __fmaf_rn(xa.y, a1, a); b = __fmaf_rn(xa.y, b1, b);
                    a = __fmaf_rn(xa.z, a2, a); b = __fmaf_rn(xa.z, b2, b);
                    a = __fmaf_rn(xa.w, a3, a); b = __fmaf_rn(xa.w, b3, b);
                    a = __fmaf_rn(xb.x, a4, a); b = __fmaf_rn(xb.x, b4, b);
                    a = __fmaf_rn(xb.y, a5, a); b = __fmaf_rn(xb.y, b5, b);
                    a = __fmaf_rn(xb.z, a6, a); b = __fmaf_rn(xb.z, b6, b);
                    a = __fmaf_rn(xb.w, a7, a); b = __fmaf_rn(xb.w, b7, b);
                    acc0[m] = a; acc1[m] = b;
                  }
                }
              }
              mbar_arrive(&empty_bar[s]);
              BE_PROF(4);
            }
          }
          // ---- combine the KS streams in stream order, then the fused epilogue, row by row -------------------------------
          if (KS > 1) {
#pragma unroll
            for (int m = 0; m < MB; m++) {
              s_part[((size_t)j * MB + m) * 64 + r] = acc0[m];
              s_part[((size_t)j * MB + m) * 64 + 32 + r] = acc1[m];
            }
            named_bar_sync(1, ENG_NCONS);
            if (c < 64) {
              const int er = c;
              const int nrow = (rt + (er >> 3)) * 8 + (er & 7);
              const bool valid = (er >> 3) < np;
              for (int m = 0; m < n; m++) {
                float v = s_part[(size_t)m * 64 + er];
#pragma unroll
                for (int jj = 1; jj < KS; jj++) v = __fadd_rn(v, s_part[((size_t)jj * MB + m) * 64 + er]);
                switch (E->epi) {
                  case EPI_RESID: gemv_epilogue<EPI_RESID>(*gp, v, nrow, m, valid, rt + (er >> 3), er, lane); break;
                  case EPI_LOGITS: gemv_epilogue<EPI_LOGITS>(*gp, v, nrow, m, valid, rt + (er >> 3), er, lane); break;
                  case EPI_QKV_ROPE: gemv_epilogue<EPI_QKV_ROPE>(*gp, v, nrow, m, valid, rt + (er >> 3), er, lane); break;
                  case EPI_SWIGLU: gemv_epilogue<EPI_SWIGLU>(*gp, v, nrow, m, valid, rt + (er >> 3), er, lane); break;
                  case EPI_P2P: gemv_epilogue<EPI_P2P>(*gp, v, nrow, m, valid, rt + (er >> 3), er, lane); break;
                  default: gemv_epilogue<EPI_BF16>(*gp, v, nrow, m, valid, rt + (er >> 3), er, lane); break;
                }
              }
            }
            named_bar_sync(1, ENG_NCONS);
          } else {
            const int nrow = (rt + pp0) * 8 + rr;
            for (int mm = 0; mm < 4; mm++) {
              const int m = mh * 4 + mm;
              if (m >= n) break;                      // (warp-uniform: mh and n are)
              float v = 0.f;
#pragma unroll
              for (int q = 0; q < 4; q++)
                if (q == mm) v = acc0[q];
              switch (E->epi) {
                case EPI_RESID: gemv_epilogue<EPI_RESID>(*gp, v, nrow, m, on0, rt + pp0, r, lane); break;
                case EPI_LOGITS: gemv_epilogue<EPI_LOGITS>(*gp, v, nrow, m, on0, rt + pp0, r, lane); break;
                case EPI_QKV_ROPE: gemv_epilogue<EPI_QKV_ROPE>(*gp, v, nrow, m, on0, rt + pp0, r, lane); break;
                case EPI_SWIGLU: gemv_epilogue<EPI_SWIGLU>(*gp, v, nrow, m, on0, rt + pp0, r, lane); break;
                case EPI_P2P: gemv_epilogue<EPI_P2P>(*gp, v, nrow, m, on0, rt + pp0, r, lane); break;
                default: gemv_epilogue<EPI_BF16>(*gp, v, nrow, m, on0, rt + pp0, r, lane); break;
              }
            }
          }
          if (KS == 1) named_bar_sync(1, ENG_NCONS);   // the activation tile buffers change hands at the row-tile boundary
          BE_PROF(5);
        }
      }
    } else if (type == BP_SDPA) {
      // ---- decode attention per (query head, sequence): sdpa_decode_kernel's arithmetic; every sequence has its own cache,
      // position and history length ----
      const int hd = P.head_dim, n_rep = P.n_rep;
      const int n_qh = E->q_dim / hd;
      const int T_max = P.seq_len;
      const int kstride = hd + 8, cpr = hd / 8;
      uint16_t* sK = reinterpret_cast<uint16_t*>(s_work);
      uint16_t* sV = sK + (size_t)T_max * kstride;
      double* sE = reinterpret_cast<double*>(sV + (size_t)T_max * hd);
      float* sP = reinterpret_cast<float*>(sE + (size_t)T_max);
      float* sQ = sP + (size_t)T_max;
      double* sZ = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(sQ + (size_t)hd) + 15) & ~(uintptr_t)15);
      for (int item = bid; item < n_qh * n; item += G) {
        const int H = item % n_qh, m = item / n_qh, h = H / n_rep;
        const int T = P.pos_arr[m] + 1;   // keys 0 .. pos: earlier rows of the same sequence appended theirs in the QKV phase
        const KeyMap km = key_map(P.row_tree, m, T - 1);   // tree rows: key t from slot km(t)
        const uint16_t* ck = E->cache_k + be_cache_base(P.row_seq, m, P.cache_seq_stride);
        const uint16_t* cv = E->cache_v + be_cache_base(P.row_seq, m, P.cache_seq_stride);
        for (int i = c; i < T * cpr; i += ENG_NCONS) {
          const int t = i / cpr, cc = i % cpr;
          const size_t kt = (size_t)km(t) * E->kv_dim + (size_t)h * hd + cc * 8;
          *reinterpret_cast<uint4*>(sK + (size_t)t * kstride + cc * 8) = ldcg_u4(ck + kt);
          *reinterpret_cast<uint4*>(sV + (size_t)t * hd + cc * 8) = ldcg_u4(cv + kt);
        }
        for (int d = c; d < hd; d += ENG_NCONS) sQ[d] = bf2f(ldcg_u16(E->x + cm_idx(m, H * hd + d)));
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
          E->out[cm_idx(m, H * hd + c)] = f2bf(a);
        }
        named_bar_sync(1, ENG_NCONS);              // the staging area is reused by the CTA's next (head, sequence)
      }
    } else if (type == BP_REDUCE) {
      // ---- peer all-reduce of the n x dim partials the previous phase pushed: out = t(res + t(p0 + p1 + ...)), rank order ----
      const int total = n * P.dim;
      const int per = (total + G - 1) / G;
      const unsigned long long t0 = global_timer_ns();
      const uint2* base = P.p2p.data[P.p2p.rank] + (size_t)(epoch & 1u) * P.p2p.n * P.p2p.slot_elems;
      for (int i = bid * per + c; i < min(total, (bid + 1) * per); i += ENG_NCONS) {
        const int m = i / P.dim, col = i % P.dim;
        float sum = 0.f;
        for (int rk = 0; rk < P.p2p.n; rk++) {
          const uint2 w = eng_wait_word(BP, base + (size_t)rk * P.p2p.slot_elems + i, epoch, rk, t0);
          sum = (rk == 0) ? __uint_as_float(w.x) : __fadd_rn(sum, __uint_as_float(w.x));
        }
        const size_t oi = cm_idx(m, col);
        E->out[oi] = f2bf(__fadd_rn(bf2f(ldcg_u16(E->res + oi)), trunc_bf(sum)));
      }
      epoch++;
    } else if (type == BP_TOKENS) {
      // ---- greedy tokens: the LM head's per-row keys are complete (grid barrier before this phase) ----
      if (P.tp > 1) {
        const unsigned long long t0 = global_timer_ns();
        const size_t myoff = ((size_t)((epoch & 1u) * P.p2p.n + P.p2p.rank)) * P.p2p.slot_elems;
        if (bid == 0 && c < P.p2p.n) {
          for (int m = 0; m < n; m++) {
            const unsigned long long mykey = __ldcg(&P.keys[m]);
            P.p2p.data[c][myoff + 2 * m] = make_uint2((uint32_t)(mykey & 0xffffffffull), epoch);
            P.p2p.data[c][myoff + 2 * m + 1] = make_uint2((uint32_t)(mykey >> 32), epoch);
          }
        }
        if (bid == 0 && c < 32) {
          for (int m = 0; m < n; m++) {
            unsigned long long key = LNB_ARGMAX_EMPTY;
            if (c < P.p2p.n) {
              const uint2* src = P.p2p.data[P.p2p.rank] + ((size_t)((epoch & 1u) * P.p2p.n + c)) * P.p2p.slot_elems + 2 * m;
              const uint2 lo = eng_wait_word(BP, src, epoch, c, t0), hi = eng_wait_word(BP, src + 1, epoch, c, t0);
              key = ((unsigned long long)hi.x << 32) | lo.x;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
              key = other > key ? other : key;
            }
            if (c == 0) P.next_arr[m] = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
          }
        }
        epoch++;
      } else if (bid == 0 && c < n) {
        const unsigned long long key = __ldcg(&P.keys[c]);
        P.next_arr[c] = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
      }
      continue;                                    // last phase: no barrier
    }
    // ---- end of phase: everybody's outputs become visible to everybody ------------------------------------------------
    if (type == BP_SCALE) BE_PROF(6);
    else if (type == BP_SDPA) BE_PROF(7);
    else if (type != BP_GEMV) BE_PROF(8);
    n_bar++;
    eng_grid_barrier(BP, n_bar * (unsigned int)G, c);
    BE_PROF(0);
  }
#undef BE_PROF
  if (prof_on) {
#pragma unroll
    for (int k = 0; k < ENG_NPROF; k++) pr[k] += (unsigned long long)pacc[k];
  }
  if (TC && P.prof && cw == 3 && lane == 0) {         // (slots 2, 4, 10, 11 are free in the tensor-core form)
    unsigned long long* q = P.prof + (size_t)bid * ENG_NPROF;
    q[2] += mma_acc; q[4] += mma_w; q[10] += mma_x; q[11] += mma_issue;
  }
  if (bid == 0 && c == 0 && P.tp > 1) P.st->ar_epoch = epoch;
}

}  // namespace lnb
