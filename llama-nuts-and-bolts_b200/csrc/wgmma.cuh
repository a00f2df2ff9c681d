// wgmma.cuh -- the Hopper tensor-core primitives the prompt-processing kernels and the FAST batch engine use (sm_90a):
// warpgroup MMAs (wgmma.mma_async, bf16 in, fp32 accumulate in registers) on operands in shared memory, plus the
// shared-memory matrix descriptor.  Every operand here is "K-major, no swizzle": 8-row x 16-byte core matrices of 128
// contiguous bytes; LBO = the byte distance of the next core matrix along K, SBO = that of the next 8 rows.
// Accumulator fragment of warp w (0..3) of the warpgroup, lane l, n8 block c: d[4c + e] = D[16w + l/4 + 8(e/2)][8c + 2(l%4) + e%2].
#pragma once
#include "common.cuh"

namespace lnb {

// shared-memory matrix descriptor, no swizzle (start address, LBO and SBO in 16-byte units; layout type 0)
LNB_DEVINL uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fffu);            // start address  [0,14)
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;  // leading byte offset [16,30)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32;  // stride byte offset  [32,46)
  return d;
}
LNB_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
LNB_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
LNB_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// after a wait: the accumulator registers are final (keeps the compiler from touching them earlier)
template <int R>
LNB_DEVINL void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// generic-proxy writes (st.shared / cp.async by threads) before async-proxy reads (wgmma operands)
LNB_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// generic-proxy global stores before bulk copies of the same bytes
LNB_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

// accumulator operands 8k .. 8k+7 of a wrapper below
#define LNB_D8(k) "+f"(d[8 * (k)]), "+f"(d[8 * (k) + 1]), "+f"(d[8 * (k) + 2]), "+f"(d[8 * (k) + 3]), "+f"(d[8 * (k) + 4]), \
    "+f"(d[8 * (k) + 5]), "+f"(d[8 * (k) + 6]), "+f"(d[8 * (k) + 7])
// D[64 x 64] (+)= A[64 x 16] . B[64 x 16]^T, both operands K-major in shared memory
LNB_DEVINL void wgmma_ss_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
               : LNB_D8(0), LNB_D8(1), LNB_D8(2), LNB_D8(3) : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, both operands K-major in shared memory
LNB_DEVINL void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
               : LNB_D8(0), LNB_D8(1), LNB_D8(2), LNB_D8(3), LNB_D8(4), LNB_D8(5), LNB_D8(6), LNB_D8(7) : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// D[64 x 32] (+)= A[64 x 16] . B[32 x 16]^T, A in registers (the m16n8k16 A fragment per warp), B K-major in shared memory
LNB_DEVINL void wgmma_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
               : LNB_D8(0), LNB_D8(1) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}

// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, A in registers (the m16n8k16 A fragment per warp), B K-major in shared memory
LNB_DEVINL void wgmma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
               : LNB_D8(0), LNB_D8(1), LNB_D8(2), LNB_D8(3), LNB_D8(4), LNB_D8(5), LNB_D8(6), LNB_D8(7) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
}

#undef LNB_D8

}  // namespace lnb
