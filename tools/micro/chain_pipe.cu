// Round-2 experiment (prepared without a GPU): the STRICT accumulation chain fed with f32 weights that a HELPER warp
// converts from bf16 on another scheduler, so that the chain warp issues 1.5 instead of 2.4 instructions per k
// (a lone warp issues ~1 instruction per 2 cycles; the dependent FFMA needs ~4.5 cycles).
//   warp 0 (helper): bf16 core-matrix tile in smem -> f32 sub-tiles [k/4][row][4] in a ring (full/empty mbarriers)
//   warp 1 (chain) : acc = fma(x[k], wf[k][row], acc), k strictly increasing -- the reference's order
// Kernel `direct` is today's inner loop (conversion inside the chain warp) on the same data; both must print the same
// checksum.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 --fmad=false -o chain_pipe tools/micro/chain_pipe.cu
// Run under a timeout (mbarrier protocol untested on hardware): timeout 20 ./chain_pipe
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(__byte_perm(w, 0u, 0x1044)); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ bool mbar_test(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) { while (!mbar_test(b, parity)) {} }

constexpr int KT = 512;     // bf16 tile (k) resident in smem, reused for every tile of the row (timing only needs the bytes)
constexpr int SK = 128;     // k per f32 sub-tile
constexpr int Q = 4;        // ring depth
constexpr int ROWS = 32;

// bf16 tile layout = the library's panel-major stage: [panel 0..3][chunk c][row in panel 0..7][8 bf16]
__device__ __forceinline__ const uint4* tile_ptr(const uint8_t* tile, int row, int chunk) {
  return reinterpret_cast<const uint4*>(tile + ((size_t)((row >> 3) * (KT / 8) + chunk) * 8 + (row & 7)) * 16);
}

__global__ void __launch_bounds__(64) pipe(float* out, long long* cyc, int K) {
  extern __shared__ __align__(16) uint8_t sm[];
  uint8_t* tile = sm;                                                    // ROWS * KT * 2
  float* xs = reinterpret_cast<float*>(sm + ROWS * KT * 2);              // K floats
  float4* ring = reinterpret_cast<float4*>(xs + K);                      // Q * (SK/4) * ROWS float4
  __shared__ uint64_t full[Q], empty[Q];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < ROWS * KT / 2; i += 64) reinterpret_cast<uint32_t*>(tile)[i] = 0x3f003e80u + (uint32_t)(i * 2654435761u >> 26) * 0x00010001u;
  for (int i = tid; i < K; i += 64) xs[i] = 1.0f + (float)(i % 97) * 0.0078125f;
  if (tid == 0)
    for (int q = 0; q < Q; q++) { mbar_init(&full[q], 1); mbar_init(&empty[q], 1); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  const int n_sub = K / SK;
  const long long t0 = clock64();
  if (warp == 0) {
    // ---- helper: convert sub-tile s into ring slot s % Q ----
    for (int s = 0; s < n_sub; s++) {
      const int q = s % Q;
      if (s >= Q) mbar_wait(&empty[q], ((s / Q) - 1) & 1);
      float4* dst = ring + (size_t)q * (SK / 4) * ROWS;
      const int c0 = (s * SK % KT) / 8;
#pragma unroll 4
      for (int c = 0; c < SK / 8; c++) {
        const uint4 w = *tile_ptr(tile, lane, c0 + c);
        dst[(size_t)(2 * c) * ROWS + lane] = make_float4(bf_lo(w.x), bf_hi(w.x), bf_lo(w.y), bf_hi(w.y));
        dst[(size_t)(2 * c + 1) * ROWS + lane] = make_float4(bf_lo(w.z), bf_hi(w.z), bf_lo(w.w), bf_hi(w.w));
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[q]);   // mbarrier.arrive has release semantics for the warp's prior writes after __syncwarp
    }
  } else {
    // ---- chain ----
    float a = 0.f;
    for (int s = 0; s < n_sub; s++) {
      const int q = s % Q;
      mbar_wait(&full[q], (s / Q) & 1);
      const float4* src = ring + (size_t)q * (SK / 4) * ROWS;
      const float4* xp = reinterpret_cast<const float4*>(xs + (size_t)s * SK);
#pragma unroll 8
      for (int g = 0; g < SK / 4; g++) {
        const float4 w = src[(size_t)g * ROWS + lane];
        const float4 x = xp[g];
        a = __fmaf_rn(x.x, w.x, a);
        a = __fmaf_rn(x.y, w.y, a);
        a = __fmaf_rn(x.z, w.z, a);
        a = __fmaf_rn(x.w, w.w, a);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[q]);
    }
    out[blockIdx.x * ROWS + lane] = a;
    if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
  }
}

// today's loop: the chain warp converts its own operands
__global__ void __launch_bounds__(32) direct(float* out, long long* cyc, int K) {
  extern __shared__ __align__(16) uint8_t sm[];
  uint8_t* tile = sm;
  float* xs = reinterpret_cast<float*>(sm + ROWS * KT * 2);
  const int lane = threadIdx.x;
  for (int i = lane; i < ROWS * KT / 2; i += 32) reinterpret_cast<uint32_t*>(tile)[i] = 0x3f003e80u + (uint32_t)(i * 2654435761u >> 26) * 0x00010001u;
  for (int i = lane; i < K; i += 32) xs[i] = 1.0f + (float)(i % 97) * 0.0078125f;
  __syncthreads();
  const long long t0 = clock64();
  float a = 0.f;
  for (int k0 = 0; k0 < K; k0 += KT) {
#pragma unroll 8
    for (int c = 0; c < KT / 8; c++) {
      const uint4 w = *tile_ptr(tile, lane, c);
      const float4 x0 = *reinterpret_cast<const float4*>(xs + k0 + c * 8), x1 = *reinterpret_cast<const float4*>(xs + k0 + c * 8 + 4);
      a = __fmaf_rn(x0.x, bf_lo(w.x), a); a = __fmaf_rn(x0.y, bf_hi(w.x), a);
      a = __fmaf_rn(x0.z, bf_lo(w.y), a); a = __fmaf_rn(x0.w, bf_hi(w.y), a);
      a = __fmaf_rn(x1.x, bf_lo(w.z), a); a = __fmaf_rn(x1.y, bf_hi(w.z), a);
      a = __fmaf_rn(x1.z, bf_lo(w.w), a); a = __fmaf_rn(x1.w, bf_hi(w.w), a);
    }
  }
  out[blockIdx.x * ROWS + lane] = a;
  if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
}

int main() {
  const int K = 14336, NB = 132;
  float *o1, *o2;
  long long *c1, *c2;
  cudaMalloc(&o1, NB * ROWS * 4); cudaMalloc(&o2, NB * ROWS * 4); cudaMalloc(&c1, NB * 8); cudaMalloc(&c2, NB * 8);
  const size_t sm_direct = ROWS * KT * 2 + (size_t)K * 4, sm_pipe = sm_direct + (size_t)Q * SK * ROWS * 4;
  cudaFuncSetAttribute(pipe, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_pipe);
  cudaFuncSetAttribute(direct, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_direct);
  for (int rep = 0; rep < 2; rep++) {
    direct<<<NB, 32, sm_direct>>>(o1, c1, K);
    pipe<<<NB, 64, sm_pipe>>>(o2, c2, K);
  }
  if (cudaDeviceSynchronize() != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
  float h1[ROWS], h2[ROWS];
  long long t1, t2;
  cudaMemcpy(h1, o1, sizeof(h1), cudaMemcpyDeviceToHost); cudaMemcpy(h2, o2, sizeof(h2), cudaMemcpyDeviceToHost);
  cudaMemcpy(&t1, c1, 8, cudaMemcpyDeviceToHost); cudaMemcpy(&t2, c2, 8, cudaMemcpyDeviceToHost);
  int same = 1;
  for (int i = 0; i < ROWS; i++) same &= (h1[i] == h2[i]);
  printf("K=%d  direct %.2f cycles/k   helper-fed %.2f cycles/k   results %s (row0 %.6f)\n", K, (double)t1 / K, (double)t2 / K,
         same ? "IDENTICAL" : "DIFFER", h1[0]);
  return same ? 0 : 1;
}
