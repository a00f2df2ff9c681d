// gemm_tc.cuh -- the prompt-processing projection: C[M,N] = X[M,K] . W[N,K]^T on the Hopper tensor cores (wgmma, bf16 in,
// fp32 accumulate in registers), operands staged into shared memory by the TMA engine's bulk-async copies.  Replaces
// ml.LinearTransformation (src/ml/operations_impl.go:427-447 -> operations_lineartransform.go:145-207) when S is large
// (prefill); the decode path (S = 1..8) uses gemv.cuh.
//
// Numerics: products are exact, accumulation is fp32 in the tensor core's own order, the result is
// truncated to bf16 exactly like the reference's ToBFloat16 (:205).  The accumulation ORDER is the
// hardware's, so this path belongs to LNB_ACC_FAST; LNB_ACC_STRICT keeps the sequential GEMV.
//
// Operand layouts (both K-major, no swizzle: 8-row x 16-byte core matrices, wgmma.cuh):
//   W  : the same panel-major HBM layout the GEMV streams (8-row panels = core matrices, gemv.cuh): the 16
//        panels of a 128-row tile are copied panel by panel (KT*16 B each) and form ONE N=128 B operand:
//        LBO = 128 B (next k-chunk), SBO = KT*16 B (next panel).
//   X  : "X8" activations written by the preceding kernel, tile-major: [M/128][K/128] tiles of
//        [16 row-groups][16 k-chunks][8 rows][8 elems] = 32 KB contiguous -> ONE bulk copy per stage;
//        LBO = 128 B (next k-chunk), SBO = 2048 B (next 8 rows).
// One CTA computes a 128 x 128 tile.  Warps 0..7 = two consumer warpgroups, warpgroup g owns rows 64g .. 64g+63 of the
// tile (64 fp32 accumulators per thread) and runs the epilogue from its registers; warp 8 = bulk-copy producer (a stage is
// 17 copies: lanes 0..15 copy one weight panel each, lane 16 the activation tile, so the copies are issued in parallel).
#pragma once
#include "wgmma.cuh"

namespace lnb {

enum { TC_EPI_BF16 = 0, TC_EPI_RESID = 1, TC_EPI_F32TRUNC = 2, TC_EPI_F32RAW = 3, TC_EPI_SWIGLU = 4 };

struct GemmTcParams {
  const uint16_t* X8;   // activations, X8 layout, M padded to a multiple of 128 (padding rows are zero)
  const uint16_t* W;    // weights, 16-row panel-major
  int M, N, K;          // M = valid rows; N % 128 == 0; K % 64 == 0
  uint16_t* out_bf16;   // [M, ldo] row-major (TC_EPI_BF16 / TC_EPI_RESID)
  float* out_f32;       // [M, ldo] (TC_EPI_F32TRUNC: f32(t(acc)); TC_EPI_F32RAW: acc)
  const uint16_t* res;  // [M, ldo] residual (TC_EPI_RESID)
  int ldo;
  // TC_EPI_SWIGLU (W = the stacked w1|w3 matrix, half-panel interleave: columns 8p..8p+3 = gate of hidden units 4p..4p+3,
  // 8p+4..8p+7 = their up values): out_bf16 = the X8 operand of the w2 GEMM, ldo = its K (ffn), m = t(t(TABLE_SILU[t(g)]) * t(u))
  // (llamatransformer.go:601-614); padding rows of the last M tile are written too (they come out as 0)
  const uint16_t* silu_tab;
};

constexpr int TC_BM = 128, TC_BN = 128, TC_KT = 128, TC_NS = 3;
constexpr int TC_A_STAGE = TC_BM * TC_KT * 2;  // 32 KB
constexpr int TC_B_STAGE = TC_BN * TC_KT * 2;  // 32 KB
constexpr int TC_SMEM = 1024 + TC_NS * (TC_A_STAGE + TC_B_STAGE);
constexpr int TC_CONSUMERS = 256;
constexpr int TC_THREADS = TC_CONSUMERS + 32;
static_assert(TC_SMEM <= 227 * 1024, "shared memory per CTA");

// ---- layout helpers for the tensor-core path (X8 = tile-major activations, see the header comment)
// X8 address of element (row, col) of a [*, K] activation matrix
LNB_HDINL size_t x8_index(int row, int col, int K) {
  const size_t tile = (size_t)(row >> 7) * (K >> 7) + (col >> 7);                 // [M/128][K/128]
  const int g = (row >> 3) & 15, ch = (col >> 3) & 15;                            // [16 groups][16 chunks]
  return (((tile * 16 + g) * 16 + ch) * 8 + (row & 7)) * 8 + (col & 7);
}

template <int EPI>
__global__ void __launch_bounds__(TC_THREADS, 1) gemm_tc_kernel(const GemmTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);  // [NS] stage loaded
  uint64_t* empty_bar = full_bar + TC_NS;                  // [NS] stage read by every consumer's MMAs
  uint8_t* sA = smem + 1024;
  uint8_t* sB = sA + TC_NS * TC_A_STAGE;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // blockIdx.x walks the M tiles: consecutive CTAs share one weight tile (read from HBM once, then L2 hits)
  const int m0 = blockIdx.x * TC_BM;   // first activation row
  const int n0 = blockIdx.y * TC_BN;   // first weight row of this tile
  const int n_kt = p.K / TC_KT;

  if (tid == 0) {
    for (int s = 0; s < TC_NS; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], TC_CONSUMERS); }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp == TC_CONSUMERS / 32) {
    // ===================== producer: lane j < 16 copies weight panel j, lane 16 the activation tile ==================
    pdl_wait();  // the activations come from the previous kernel (weights alone could go earlier)
    const uint64_t pol_w = l2_policy_evict_first();
    const uint64_t pol_x = l2_policy_evict_last();   // every N-tile re-reads the same activations
    const uint8_t* xb = reinterpret_cast<const uint8_t*>(p.X8);
    const uint8_t* wb = reinterpret_cast<const uint8_t*>(p.W);
    for (int t = 0; t < n_kt; t++) {
      const int s = t % TC_NS;
      mbar_wait(&empty_bar[s], (((uint32_t)(t / TC_NS)) & 1u) ^ 1u);
      if (lane == 0) mbar_expect_tx(&full_bar[s], TC_A_STAGE + TC_B_STAGE);
      __syncwarp();
      const size_t k0 = (size_t)t * TC_KT;
      if (lane < 16)   // B: 16 panels of 8 rows, each (8 rows x KT) = KT*16 contiguous bytes
        bulk_g2s(sB + (size_t)s * TC_B_STAGE + (size_t)lane * (TC_KT * 16), wb + ((size_t)(n0 / 8 + lane) * p.K + k0) * 16, TC_KT * 16,
                 &full_bar[s], pol_w);
      else if (lane == 16)   // A: one contiguous 128 x 128 tile of the tile-major X8 layout
        bulk_g2s(sA + (size_t)s * TC_A_STAGE, xb + ((size_t)(m0 / TC_BM) * (p.K / TC_KT) + t) * TC_A_STAGE, TC_A_STAGE,
                 &full_bar[s], pol_x);
    }
    return;
  }

  // ===================== consumers: warpgroup wg computes rows 64 wg .. 64 wg + 63 of the tile ===========================
  const int wg = warp >> 2;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) acc[i] = 0.f;
  for (int t = 0; t < n_kt; t++) {
    const int s = t % TC_NS;
    mbar_wait(&full_bar[s], ((uint32_t)(t / TC_NS)) & 1u);
    // A: this warpgroup's 8 row groups start 8 x 2048 B into the stage; next k16 step = +256 B = +16 in the address field
    uint64_t a_desc = gmma_desc(smem_u32(sA + (size_t)s * TC_A_STAGE + (size_t)wg * 8 * (TC_KT * 16)), 128, TC_KT * 16);
    uint64_t b_desc = gmma_desc(smem_u32(sB + (size_t)s * TC_B_STAGE), 128, TC_KT * 16);
    wgmma_fence();
#pragma unroll
    for (int k16 = 0; k16 < TC_KT / 16; k16++) {
      wgmma_ss_n128(acc, a_desc, b_desc, (t > 0 || k16 > 0) ? 1u : 0u);   // 64 x 128 x 16 per instruction
      a_desc += 16; b_desc += 16;
    }
    wgmma_commit();
    // the previous stage's MMAs are complete once at most this stage's group is in flight: hand that stage back
    wgmma_wait<1>();
    if (t > 0) mbar_arrive(&empty_bar[(t - 1) % TC_NS]);
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);

  // ===================== epilogue: registers -> global ========================================================
  const int row0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows row0 (acc[4c], acc[4c+1]) and row0 + 8 (acc[4c+2..3])
  const int cq = 2 * (lane & 3);                                    // columns 8c + cq, 8c + cq + 1
  if (EPI == TC_EPI_RESID) pdl_wait();    // residual operand is written by an earlier kernel
#pragma unroll
  for (int c = 0; c < TC_BN / 8; c++) {
    if (EPI == TC_EPI_SWIGLU) {
      // columns 8c..8c+3 are gates, 8c+4..8c+7 the up values of the same hidden units: the lane two to the right holds them
      float up[4];
#pragma unroll
      for (int e = 0; e < 4; e++) up[e] = __shfl_xor_sync(0xffffffffu, acc[4 * c + e], 2);
      if (cq < 4) {
#pragma unroll
        for (int hr = 0; hr < 2; hr++) {
          const float g0 = acc[4 * c + 2 * hr], g1 = acc[4 * c + 2 * hr + 1];
          const uint16_t s0 = p.silu_tab[__float_as_uint(g0) >> 16], s1 = p.silu_tab[__float_as_uint(g1) >> 16];   // t(TABLE_SILU[t(gate)])
          const float lo = __fmul_rn(bf2f(s0), trunc_bf(up[2 * hr]));
          const float hi = __fmul_rn(bf2f(s1), trunc_bf(up[2 * hr + 1]));
          *reinterpret_cast<uint32_t*>(p.out_bf16 + x8_index(row0 + 8 * hr, (n0 >> 1) + 4 * c + cq, p.ldo)) =
              (__float_as_uint(lo) >> 16) | (__float_as_uint(hi) & 0xffff0000u);
        }
      }
    } else {
#pragma unroll
      for (int hr = 0; hr < 2; hr++) {
        const int row = row0 + 8 * hr;
        if (row >= p.M) continue;
        const size_t o = (size_t)row * p.ldo + n0 + 8 * c + cq;
        float a = acc[4 * c + 2 * hr], b = acc[4 * c + 2 * hr + 1];
        if (EPI == TC_EPI_BF16 || EPI == TC_EPI_RESID) {
          if (EPI == TC_EPI_RESID) {
            const uint32_t rw = *reinterpret_cast<const uint32_t*>(p.res + o);
            a = __fadd_rn(bf_lo(rw), trunc_bf(a));   // ml.Add(x, t(linear))  llamatransformer.go:232,248
            b = __fadd_rn(bf_hi(rw), trunc_bf(b));
          }
          *reinterpret_cast<uint32_t*>(p.out_bf16 + o) = (uint32_t)f2bf(a) | ((uint32_t)f2bf(b) << 16);
        } else {
          if (EPI == TC_EPI_F32TRUNC) { a = trunc_bf(a); b = trunc_bf(b); }
          *reinterpret_cast<float2*>(p.out_f32 + o) = make_float2(a, b);
        }
      }
    }
  }
}

// ---- -----------------------------------------------------
// row-major [M, K] bf16 -> X8 ([Mpad/8][K/8][8][8]); rows >= M are written as zeros
__global__ void pack_x8_kernel(const uint16_t* __restrict__ src, int ld, int M, int Mpad, int K, uint16_t* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t chunks = K / 8, total = (int64_t)Mpad * chunks;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / chunks, ch = i % chunks;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row < M) v = *reinterpret_cast<const uint4*>(src + row * ld + ch * 8);
    *reinterpret_cast<uint4*>(dst + x8_index((int)row, (int)ch * 8, K)) = v;
  }
}

// X8 -> row-major [M, K] (tests / op-level API)
__global__ void unpack_x8_kernel(const uint16_t* __restrict__ src, int M, int K, uint16_t* __restrict__ dst, int ld) {
  const int64_t chunks = K / 8, total = (int64_t)M * chunks;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / chunks, ch = i % chunks;
    *reinterpret_cast<uint4*>(dst + row * ld + ch * 8) = *reinterpret_cast<const uint4*>(src + x8_index((int)row, (int)ch * 8, K));
  }
}

// RMSNorm.Forward (llamatransformer.go:633-660) for the prefill path: one CTA (256 threads) per row,
// LNB_ACC_FAST reduction order (256 interleaved partial sums, butterfly, then over warps -- the same
// order as gemv.cuh's prologue), output written straight into the X8 layout the tensor-core GEMM reads.
// Rows in [M, Mpad) are zero-filled (grid = Mpad).
__global__ void __launch_bounds__(256) rmsnorm_x8_kernel(const uint16_t* __restrict__ x, int ldx, const uint16_t* __restrict__ w,
                                                         uint16_t* __restrict__ out_x8, int M, int D, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float wsum[8];
  __shared__ float rs;
  const int row = blockIdx.x, tid = threadIdx.x;
  if (row >= M) {
    for (int k = tid; k < D; k += 256) out_x8[x8_index(row, k, D)] = 0;
    return;
  }
  const uint16_t* xr = x + (size_t)row * ldx;
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
  __syncthreads();
  const float r = rs;
  for (int k = tid; k < D; k += 256) {
    const float n1 = trunc_bf(__fmul_rn(bf2f(xr[k]), r));
    out_x8[x8_index(row, k, D)] = f2bf(__fmul_rn(n1, bf2f(w[k])));
  }
}

// RoPE of one pair: w holds columns (2i, 2i+1) as bf16 (low half first), fc = cis[pos][i]; the rotated pair, same packing
// (the MXFP8 cache writer, kvcache.cuh, rotates its K rows with it too)
LNB_DEVINL uint32_t rope_pair(uint32_t w, float2 fc) {
  const double a = (double)bf_lo(w), b = (double)bf_hi(w), c = (double)fc.x, d = (double)fc.y;
  return (uint32_t)f2bf((float)(a * c - b * d)) | ((uint32_t)f2bf((float)(a * d + b * c)) << 16);
}

// After the fused wq|wk|wv GEMM of the prefill path: RoPE on q and k (f64 intermediates, see
// gemv.cuh EPI_QKV_ROPE), q -> q_out [S, q_dim], k -> cacheK[pos0+s], v -> cacheV[pos0+s]
// (llamatransformer.go:374-403).  One thread per (row, pair of columns).  Ragged calls (rows of several sequences):
// row s sits at row_pos[s] of the cache of sequence row_seq[s] (+ row_seq[s] * seq_stride); both NULL otherwise.
__global__ void rope_kv_kernel(const uint16_t* __restrict__ qkv, int ld, uint16_t* __restrict__ q_out, int q_dim, int kv_dim,
                               int head_dim, uint16_t* __restrict__ cache_k, uint16_t* __restrict__ cache_v,
                               const float* __restrict__ cis, const int32_t* __restrict__ pos_ptr, int S,
                               const int32_t* __restrict__ row_pos, const int32_t* __restrict__ row_seq, long long seq_stride) {
  pdl_launch_dependents();
  pdl_wait();
  const int pairs = (q_dim + 2 * kv_dim) / 2;
  const int64_t total = (int64_t)S * pairs;
  const int pos0 = row_pos ? 0 : *pos_ptr;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int s = (int)(i / pairs), n = (int)(i % pairs) * 2;
    const uint32_t w = *reinterpret_cast<const uint32_t*>(qkv + (size_t)s * ld + n);
    const int pos = row_pos ? row_pos[s] : pos0 + s;
    const size_t cb = row_seq ? (size_t)row_seq[s] * (size_t)seq_stride : 0;
    if (n < q_dim + kv_dim) {
      const int nn = (n < q_dim) ? n : n - q_dim;
      const int ii = (nn % head_dim) >> 1;
      const float2 fc = *reinterpret_cast<const float2*>(cis + ((size_t)pos * (head_dim / 2) + ii) * 2);
      const uint32_t o = rope_pair(w, fc);
      if (n < q_dim) *reinterpret_cast<uint32_t*>(q_out + (size_t)s * q_dim + n) = o;
      else *reinterpret_cast<uint32_t*>(cache_k + cb + (size_t)pos * kv_dim + nn) = o;
    } else {
      *reinterpret_cast<uint32_t*>(cache_v + cb + (size_t)pos * kv_dim + (n - q_dim - kv_dim)) = w;
    }
  }
}

// After the fused w1|w3 GEMM (columns follow the half-panel interleave of the stacked matrix:
// 4 gate columns, then the 4 up columns of the same hidden units): m = t( t(TABLE_SILU[g]) * u )
// (llamatransformer.go:601-614), written in X8 layout for the w2 GEMM.  Rows in [M, Mpad) -> 0.
__global__ void swiglu_x8_kernel(const uint16_t* __restrict__ gu, int ld, const uint16_t* __restrict__ silu_tab,
                                 uint16_t* __restrict__ out_x8, int M, int Mpad, int ffn) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = (int64_t)Mpad * ffn;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int row = (int)(i / ffn), c = (int)(i % ffn);
    uint16_t o = 0;
    if (row < M) {
      const size_t base = (size_t)row * ld + (size_t)(c >> 2) * 8 + (c & 3);
      const uint16_t sg = silu_tab[gu[base]];
      o = f2bf(__fmul_rn(bf2f(sg), bf2f(gu[base + 4])));
    }
    out_x8[x8_index(row, c, ffn)] = o;
  }
}

}  // namespace lnb
