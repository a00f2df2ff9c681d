// Round-2 experiment (prepared without a GPU): STRICT accumulation at M = 8 (batched decode).  Each lane owns one
// weight row and EIGHT independent accumulation chains (one per batch row), so the warp is issue-bound, not
// latency-bound.  How many such warps does an SM need before the FFMA pipe saturates, and what does one k cost?
// Expectation: ~11 instructions per k per warp (8 FFMA + 1 cvt + 2 LDS.128 of x + 1/8 LDS.128 of w); with W warps per
// scheduler the SM should approach 128 FFMA / clk.  Today's CfgS8 runs ONE warp per SM.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o chain_mb8 tools/micro/chain_mb8.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(__byte_perm(w, 0u, 0x1044)); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

constexpr int KT = 256;   // k per resident weight tile (reused for every tile: timing needs the bytes, not their values)

// smem: per warp a bf16 tile [KT/8 chunks][32 rows][8] (one LDS.128 per lane per chunk, conflict-free),
//       shared x as [k][8 batch rows] f32 (two LDS.128 broadcasts per k)
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) mb8(float* out, long long* cyc, int K) {
  extern __shared__ __align__(16) uint8_t sm[];
  uint4* wt = reinterpret_cast<uint4*>(sm);                                   // WARPS * (KT/8) * 32 uint4
  float4* xs = reinterpret_cast<float4*>(sm + (size_t)WARPS * (KT / 8) * 32 * 16);   // KT * 2 float4 (reused per tile)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < WARPS * (KT / 8) * 32; i += WARPS * 32) wt[i] = make_uint4(0x3f803f00u + i, 0x3e803f80u, 0x3f003e80u, 0x3f803f80u);
  for (int i = tid; i < KT * 2; i += WARPS * 32) xs[i] = make_float4(1.0f + i * 1e-4f, 0.5f, 0.25f, 2.0f);
  __syncthreads();
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const uint4* my = wt + (size_t)warp * (KT / 8) * 32;
  const long long t0 = clock64();
  for (int k0 = 0; k0 < K; k0 += KT) {
#pragma unroll 2
    for (int c = 0; c < KT / 8; c++) {
      const uint4 w = my[c * 32 + lane];
      const float wv[8] = {bf_lo(w.x), bf_hi(w.x), bf_lo(w.y), bf_hi(w.y), bf_lo(w.z), bf_hi(w.z), bf_lo(w.w), bf_hi(w.w)};
#pragma unroll
      for (int e = 0; e < 8; e++) {
        const float4 x0 = xs[(c * 8 + e) * 2], x1 = xs[(c * 8 + e) * 2 + 1];
        a[0] = __fmaf_rn(x0.x, wv[e], a[0]); a[1] = __fmaf_rn(x0.y, wv[e], a[1]);
        a[2] = __fmaf_rn(x0.z, wv[e], a[2]); a[3] = __fmaf_rn(x0.w, wv[e], a[3]);
        a[4] = __fmaf_rn(x1.x, wv[e], a[4]); a[5] = __fmaf_rn(x1.y, wv[e], a[5]);
        a[6] = __fmaf_rn(x1.z, wv[e], a[6]); a[7] = __fmaf_rn(x1.w, wv[e], a[7]);
      }
    }
  }
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int m = 0; m < 8; m++) s += a[m];
  out[(blockIdx.x * WARPS + warp) * 32 + lane] = s;
  if (tid == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int WARPS>
static void run(int K) {
  const int NB = 132;
  float* o;
  long long* c;
  cudaMalloc(&o, (size_t)NB * WARPS * 32 * 4);
  cudaMalloc(&c, NB * 8);
  const size_t smem = (size_t)WARPS * (KT / 8) * 32 * 16 + (size_t)KT * 2 * 16;
  cudaFuncSetAttribute(mb8<WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  for (int rep = 0; rep < 2; rep++) mb8<WARPS><<<NB, WARPS * 32, smem>>>(o, c, K);
  if (cudaDeviceSynchronize() != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError())); return; }
  long long t;
  cudaMemcpy(&t, c, 8, cudaMemcpyDeviceToHost);
  const double cyc_per_k = (double)t / K;
  printf("warps/SM %2d: %.2f cycles per k per warp  ->  %.1f FFMA/clk/SM (peak 128), %d rows x 8 chains per SM\n", WARPS, cyc_per_k,
         WARPS * 32 * 8 / cyc_per_k, WARPS * 32);
  cudaFree(o);
  cudaFree(c);
}

int main() {
  const int K = 4096;
  run<1>(K); run<2>(K); run<4>(K); run<8>(K); run<16>(K);
  return 0;
}
