// sdpa_tc.cuh -- the attention core of a prompt call on the Hopper tensor cores (LNB_ACC_FAST prefill, head_dim 128).
// Replaces, for S >= 32 rows, the scaled-dot-product block of LlamaAttention.Forward (src/model/llamatransformer.go:402-514):
//   sc_st = t( t(sum_d q_sd * k_td) / t(sqrt(hd)) )                MatMul :459, DivToScalar :464
//   masked entries (t > pos0 + s) contribute nothing               :471
//   e_st = exp_f64(sc_st);  Z_s = sum_t e_st (f64);  p_st = t(f32(e_st / Z_s))     Softmax :484-495  (here e_st * (1 / Z_s))
//   o_sd = t( sum_t p_st * v_td )                                  MatMul :504
// Truncation points, the f64 exponentials and the f64 division are the reference's; the two inner sums (over d for the
// scores, over t for the output) run in the tensor core's order and Z is added per thread and then across the four threads
// of a row -- a documented reorder, which is why this kernel belongs to LNB_ACC_FAST (STRICT keeps sdpa_kernel).
//
// One CTA = (query head H, 128 query rows), 256 threads = two warpgroups; warpgroup g owns query rows 64g .. 64g+63 and
// keeps its scores and its output rows in registers (wgmma.cuh fragment layout).  Per 64-key tile:
//   S[64 x 64] = Q . K^T      8 x wgmma m64n64k16, A = Q tile, B = K tile, both K-major core-matrix tiles in shared memory
//                             ([row groups][16 chunks][8 rows][8 elems], the X8 tile of gemm_tc.cuh)
//   pass 1: every thread adds exp_f64 of its entries (row sums Z)
//   pass 2: S again (recomputing 8 MMAs is cheaper than keeping every tile), p = t(f32(e / Z)) packed straight into the bf16
//           A fragments of O[64 x 128] += P . V (4 x wgmma m64n128k16, A from registers), B = V^T staged by the threads
//           (V rows are key-major in the cache; the transposing copy is 32 two-byte stores per thread and tile)
// K tiles are double-buffered and arrive with cp.async one tile ahead (zero-filled past the last key).
// exp_f64 of a score is a TABLE LOOKUP: the score is a bf16 value, so exp_tab[bits] = exp((double)bf16(bits)), filled once per
// device by the same device exp() the other attention kernels call (exp_tab_kernel), has exactly the bits an inline call
// would produce; the live part of the table (|score| of a few units: a few thousand entries) stays in L1.
#pragma once
#include "gemm_tc.cuh"

namespace lnb {

constexpr int ST_BK = 64;                            // keys per tile
constexpr int ST_QTILE = 128 * 128 * 2;              // 32 KB: [128 rows][128 d], A operand of S (SBO 2048)
constexpr int ST_KTILE = ST_BK * 128 * 2;            // 16 KB: [64 keys][128 d], B operand of S (N = 64, K = 128): SBO 2048
constexpr int ST_VTILE = 128 * ST_BK * 2;            // 16 KB: [128 d][64 keys], B operand of O (N = 128, K = 64): SBO 1024
constexpr int ST_SMEM = ST_QTILE + 2 * ST_KTILE + ST_VTILE;

// exp_tab[b] = exp((double)bf16(b)) for all 65536 bit patterns
__global__ void exp_tab_kernel(double* __restrict__ tab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 65536) tab[i] = exp((double)bf2f((uint16_t)i));
}

// element (r, c) of a K-major operand tile with 128 columns: core matrix (r / 8, c / 8) = 128 contiguous bytes
LNB_DEVINL uint32_t st_off(int r, int c) { return (uint32_t)((((r >> 3) * 16 + (c >> 3)) * 8 + (r & 7)) * 16 + (c & 7) * 2); }
// element (r, c) of a K-major operand tile with 64 columns
LNB_DEVINL uint32_t sx_off64(int r, int c) { return (uint32_t)((((r >> 3) * 8 + (c >> 3)) * 8 + (r & 7)) * 16 + (c & 7) * 2); }
LNB_DEVINL void cp_async16_zfill(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t n = valid ? 16u : 0u;          // src-size 0: the 16 bytes are written as zeros, nothing is read
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(n) : "memory");
}
LNB_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
LNB_DEVINL void cp_async_wait0() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// exp_f64 of the scores of one row: two consecutive keys t, t + 1 (a masked entry reads exp(-inf) = 0, which adds nothing to Z
// and gives p = 0); both table loads are issued before either is used
LNB_DEVINL void st_exp2(float a0, float a1, int t, int qpos, int t_end, float scale, const double* __restrict__ tab, double& e0,
                        double& e1) {
  float s0 = trunc_bf(__fdiv_rn(trunc_bf(a0), scale)), s1 = trunc_bf(__fdiv_rn(trunc_bf(a1), scale));
  const uint32_t i0 = (t <= qpos && t < t_end) ? (__float_as_uint(s0) >> 16) : 0xff80u;        // 0xff80 = bf16 -inf
  const uint32_t i1 = (t + 1 <= qpos && t + 1 < t_end) ? (__float_as_uint(s1) >> 16) : 0xff80u;
  e0 = __ldg(tab + i0);
  e1 = __ldg(tab + i1);
}

__global__ void __launch_bounds__(256, 1) sdpa_tc_kernel(const uint16_t* __restrict__ q, int ldq, const uint16_t* __restrict__ cache_k,
                                                         const uint16_t* __restrict__ cache_v, int kv_dim, int n_rep,
                                                         uint16_t* __restrict__ out_x8, int ldo, const int32_t* __restrict__ pos_ptr,
                                                         int S, float scale_bf16_as_f32, const double* __restrict__ exp_tab) {
  pdl_launch_dependents();
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + ST_QTILE;                                  // [2] K tiles
  uint8_t* sV = sK + 2 * ST_KTILE;                              // V^T: row = d, column = key

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int H = blockIdx.x, h = H / n_rep;
  const int qt = (int)gridDim.y - 1 - (int)blockIdx.y;          // the long (late) query tiles start first
  const int s0 = qt * 128;
  pdl_wait();
  const int pos0 = *pos_ptr;
  const int t_end = min(pos0 + S, pos0 + s0 + 128);             // keys this row block can see
  const int n_tiles = (t_end + ST_BK - 1) / ST_BK;
  // this thread's rows of the tile (fragment layout: row r_lo for accumulators 4c, 4c+1; r_lo + 8 for 4c+2, 4c+3) and columns
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const int qpos_lo = pos0 + s0 + r_lo, qpos_hi = qpos_lo + 8;  // keys t <= qpos are visible to a row

  // Q tile: 2048 pieces of 16 bytes (row r, chunk c8)
  for (int i = tid; i < 2048; i += 256) {
    const int r = i >> 4, c8 = i & 15;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (s0 + r < S) v = *reinterpret_cast<const uint4*>(q + (size_t)(s0 + r) * ldq + (size_t)H * 128 + c8 * 8);
    *reinterpret_cast<uint4*>(sQ + st_off(r, c8 * 8)) = v;
  }
  // K tile j -> buffer j & 1, asynchronously (4 pieces of 16 bytes per thread)
  auto prefetch_k = [&](int tile) {
    const int t0 = tile * ST_BK;
    uint8_t* dst = sK + (size_t)(tile & 1) * ST_KTILE;
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int i = tid + u * 256, r = i >> 4, c8 = i & 15;
      const bool ok = t0 + r < t_end;
      const uint16_t* src = cache_k + (size_t)(ok ? t0 + r : 0) * kv_dim + (size_t)h * 128 + c8 * 8;
      cp_async16_zfill(dst + st_off(r, c8 * 8), src, ok);
    }
    cp_async_commit();
  };
  // S = Q . K_tile^T for this warpgroup's 64 rows (M 64, N 64, K 128: 8 MMAs), complete on return
  auto scores = [&](int tile, float (&sacc)[32]) {
    uint64_t a_desc = gmma_desc(smem_u32(sQ) + (uint32_t)wg * 8u * 2048u, 128, 2048);
    uint64_t b_desc = gmma_desc(smem_u32(sK + (size_t)(tile & 1) * ST_KTILE), 128, 2048);
    wgmma_fence();
#pragma unroll
    for (int k16 = 0; k16 < 8; k16++) {
      wgmma_ss_n64(sacc, a_desc, b_desc, k16 > 0 ? 1u : 0u);
      a_desc += 16; b_desc += 16;
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sacc);
  };

  // ---------------- pass 1: row sums of exp ------------------------------------------------------------------------
  double z_lo = 0.0, z_hi = 0.0;
  float sacc[32];
#pragma unroll
  for (int i = 0; i < 32; i++) sacc[i] = 0.f;
  prefetch_k(0);
  for (int tile = 0; tile < n_tiles; tile++) {
    cp_async_wait0();                                           // this thread's pieces of K_tile have landed
    fence_proxy_async_smem();
    __syncthreads();                                            // ... everybody's; and the other buffer's MMAs are complete
    if (tile + 1 < n_tiles) prefetch_k(tile + 1);
    scores(tile, sacc);
    const int t0 = tile * ST_BK + cq;
#pragma unroll
    for (int c = 0; c < 8; c++) {
      double e0, e1, e2, e3;
      st_exp2(sacc[4 * c], sacc[4 * c + 1], t0 + 8 * c, qpos_lo, t_end, scale_bf16_as_f32, exp_tab, e0, e1);
      st_exp2(sacc[4 * c + 2], sacc[4 * c + 3], t0 + 8 * c, qpos_hi, t_end, scale_bf16_as_f32, exp_tab, e2, e3);
      z_lo = __dadd_rn(__dadd_rn(z_lo, e0), e1);
      z_hi = __dadd_rn(__dadd_rn(z_hi, e2), e3);
    }
  }
  // the four threads of a row: (z0 + z1) + (z2 + z3), the same bits in all four
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    z_lo = __dadd_rn(z_lo, __shfl_xor_sync(0xffffffffu, z_lo, o));
    z_hi = __dadd_rn(z_hi, __shfl_xor_sync(0xffffffffu, z_hi, o));
  }
  // p = t(f32(e * (1/Z))): the reference divides (e / Z); multiplying by the f64 reciprocal differs from the quotient by at most
  // one f64 ulp, which survives the rounding to f32 AND the truncation to bf16 with probability ~2^-45 per element -- and an
  // f64 division per score is ~30 FP64 instructions against one (this kernel is LNB_ACC_FAST only)
  const double rz_lo = __ddiv_rn(1.0, z_lo), rz_hi = __ddiv_rn(1.0, z_hi);

  // ---------------- pass 2: p = t(f32(e / Z)), O += P . V -----------------------------------------------------------
  float oacc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) oacc[i] = 0.f;
  __syncthreads();                                              // every pass-1 MMA is complete: both K buffers are free
  prefetch_k(0);
  for (int tile = 0; tile < n_tiles; tile++) {
    // V rows of this tile: 4 pieces of 16 bytes per thread (consecutive lanes = consecutive keys)
    uint4 vreg[4];
    {
      const int t0v = tile * ST_BK;
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int i = tid + u * 256, tl = i & 63, c8 = i >> 6;
        vreg[u] = make_uint4(0u, 0u, 0u, 0u);
        if (t0v + tl < t_end) vreg[u] = *reinterpret_cast<const uint4*>(cache_v + (size_t)(t0v + tl) * kv_dim + (size_t)h * 128 + c8 * 8);
      }
    }
    cp_async_wait0();
    __syncthreads();                                            // the previous tile's O MMAs are complete: V^T is free
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int i = tid + u * 256, tl = i & 63, c8 = i >> 6;
      const uint32_t w[4] = {vreg[u].x, vreg[u].y, vreg[u].z, vreg[u].w};
#pragma unroll
      for (int e = 0; e < 8; e++)
        *reinterpret_cast<uint16_t*>(sV + sx_off64(c8 * 8 + e, tl)) = (uint16_t)((e & 1) ? (w[e >> 1] >> 16) : (w[e >> 1] & 0xffffu));
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (tile + 1 < n_tiles) prefetch_k(tile + 1);
    scores(tile, sacc);
    // P as the A fragments of 4 k16 steps: step j covers keys 16j .. 16j+15 = score blocks 2j and 2j+1; fragment registers
    // 0, 1, 2, 3 = (row r_lo, block 2j), (r_lo + 8, 2j), (r_lo, 2j+1), (r_lo + 8, 2j+1)
    uint32_t pa[4][4];
    const int t0 = tile * ST_BK + cq;
#pragma unroll
    for (int c = 0; c < 8; c++) {
      double e0, e1, e2, e3;
      st_exp2(sacc[4 * c], sacc[4 * c + 1], t0 + 8 * c, qpos_lo, t_end, scale_bf16_as_f32, exp_tab, e0, e1);
      st_exp2(sacc[4 * c + 2], sacc[4 * c + 3], t0 + 8 * c, qpos_hi, t_end, scale_bf16_as_f32, exp_tab, e2, e3);
      const float p0 = (float)__dmul_rn(e0, rz_lo), p1 = (float)__dmul_rn(e1, rz_lo);
      const float p2 = (float)__dmul_rn(e2, rz_hi), p3 = (float)__dmul_rn(e3, rz_hi);
      pa[c >> 1][(c & 1) * 2 + 0] = (__float_as_uint(p0) >> 16) | (__float_as_uint(p1) & 0xffff0000u);
      pa[c >> 1][(c & 1) * 2 + 1] = (__float_as_uint(p2) >> 16) | (__float_as_uint(p3) & 0xffff0000u);
    }
    uint64_t b_desc = gmma_desc(smem_u32(sV), 128, 1024);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; j++) {                               // O += P . V   (M 64, N 128, K 64: 4 MMAs)
      wgmma_rs_n128(oacc, pa[j], b_desc, 1u);
      b_desc += 16;
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(oacc);
  }

  // ---------------- O -> t(.) -> the X8 operand of the Wo GEMM ------------------------------------------------------
#pragma unroll
  for (int hr = 0; hr < 2; hr++) {
    const int srow = s0 + r_lo + 8 * hr;
    if (srow < S) {
#pragma unroll
      for (int c = 0; c < 16; c++)
        *reinterpret_cast<uint32_t*>(out_x8 + x8_index(srow, H * 128 + 8 * c + cq, ldo)) =
            (__float_as_uint(oacc[4 * c + 2 * hr]) >> 16) | (__float_as_uint(oacc[4 * c + 2 * hr + 1]) & 0xffff0000u);
    }
  }
}

}  // namespace lnb
