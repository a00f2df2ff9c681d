// common.cuh -- shared device helpers for liblnb.so (sm_90a only).
//
// bf16 <-> f32 follow the reference exactly: widening is a 16-bit shift, narrowing
// is TRUNCATION (src/dtype/bfloat16.go:19-21,59-61), never round-to-nearest.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define LNB_DEVINL __device__ __forceinline__
#define LNB_HDINL __host__ __device__ __forceinline__   // layout helpers the host also uses (lnb_session_read de-tiles with them)

LNB_DEVINL float bf2f(uint16_t b) { return __uint_as_float(((uint32_t)b) << 16); }
LNB_DEVINL uint16_t f2bf(float f) { return (uint16_t)(__float_as_uint(f) >> 16); }  // truncation
// a 32-bit word holding two consecutive bf16 (little endian: element 0 in the low half)
// PRMT (ALU pipe) instead of a shift: ptxas would turn `w << 16` into IMAD.U32 on the FMA pipe,
// where it competes with the dependent-FFMA accumulation chains of the GEMV.
LNB_DEVINL float bf_lo(uint32_t w) { return __uint_as_float(__byte_perm(w, 0u, 0x1044)); }
LNB_DEVINL float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
LNB_DEVINL float trunc_bf(float f) { return __uint_as_float(__float_as_uint(f) & 0xffff0000u); }  // bf2f(f2bf(f))

LNB_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier (shared::cta) ------------------------------------------------------------
LNB_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
LNB_DEVINL void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
LNB_DEVINL void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
LNB_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
LNB_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
LNB_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// polite variant for warps that are NOT on the critical path: back off between polls so that the
// spinning warp does not steal issue slots from the accumulation-chain warp on the same scheduler
#ifndef LNB_BACKOFF_NS
#define LNB_BACKOFF_NS 64
#endif
LNB_DEVINL void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) __nanosleep(LNB_BACKOFF_NS);
}

// ---- bulk async copy global -> shared (TMA engine, 1-D; SASS: UBLKCP) -------------------
LNB_DEVINL uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
LNB_DEVINL uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// size multiple of 16, src/dst 16-byte aligned; completes `bytes` on the mbarrier
LNB_DEVINL void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// ---- programmatic dependent launch -----------------------------------------------------
LNB_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
LNB_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- rows of a speculative tree (lnb_forward_speculative_tree, DESIGN.md §9c) ----------
// A tree call's row map carries one word per row: the cache slot the row's K and V go to (low 24 bits) and its ancestor
// mask (high 8 bits: the segment-local rows of its path root .. itself; ancestors precede their descendants, so the set
// bits in ascending order ARE the path).  A row at position pos of a segment starting at base = pos + 1 - popc(mask)
// sees logical keys 0 .. pos: key t < base is slot t, key base + d is slot base + (the d-th set bit of the mask).  Every
// summation runs over logical keys, so a tree row computes what the chain row over its path computes.  Rows of every
// other call carry no words (row_tree NULL): slot = position, and KeyMap's identity costs no load.
constexpr int TREE_SLOT_BITS = 24;
LNB_HDINL int tree_slot(int32_t w) { return w & ((1 << TREE_SLOT_BITS) - 1); }
struct KeyMap {
  int base = 0x7fffffff;
  uint32_t mask = 0;
  LNB_DEVINL int operator()(int t) const {
    if (t < base) return t;
    uint32_t m = mask;
    for (int d = t - base; d > 0; d--) m &= m - 1;   // drop the lower set bits: the path's first d rows
    return base + __ffs(m) - 1;
  }
};
// the key map of row r at position pos (call only after the row map may be read: pdl_wait)
LNB_DEVINL KeyMap key_map(const int32_t* row_tree, int r, int pos) {
  KeyMap k;
  if (row_tree) {
    k.mask = (uint32_t)__ldcg(row_tree + r) >> TREE_SLOT_BITS;
    k.base = pos + 1 - __popc(k.mask);
  }
  return k;
}

// ---- named barrier among a subset of the CTA -------------------------------------------
LNB_DEVINL void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---- greedy-argmax key: larger f32 first, then LOWER index (ml.Argmax keeps the first
// maximum: strict '<' scan, src/ml/operations_impl.go:529-541).  NaN never wins. --------
LNB_DEVINL unsigned long long argmax_key(float v, uint32_t idx) {
  uint32_t u = __float_as_uint(v);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // order-preserving map of finite floats / infs
  return ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - idx);
}
// key of "nothing selected": below the key of every value > -MaxFloat32
#define LNB_ARGMAX_EMPTY 0ull

// per-step device state shared by the kernels of one session (lets a captured CUDA graph
// be replayed for every position)
struct LnbDevState {
  int32_t pos;                   // start position of the current forward call
  int32_t n_rows;                // S of the current forward call
  unsigned long long amax_key;   // running argmax key of the last row
  uint32_t done_ctr;             // CTAs of the LM-head kernel that finished
  int32_t next_token;            // greedy token of the last row
  int32_t step;                  // decode-run step counter
  int32_t safe_rows;             // KV rows [0, safe_rows) were complete before this call was enqueued (host-synchronised)
  uint32_t ar_epoch;             // sequence number of the next peer all-reduce (same on every rank)
  uint32_t ar_error;             // sticky: 0 = ok, else 0x80000000 | (epoch & 0xffffff) << 4 | late rank  (a peer never delivered
                                 // within LnbP2P.timeout_ns: every later peer kernel of the session exits at once)
  uint32_t ar_done2;             // CTAs of the reducing kernel that have finished
  uint32_t pad2;
  unsigned long long amax_key_b; // persistent engine: the argmax key of odd steps (engine.cuh)
};

// One-shot all-reduce over NVLink peer memory (tensor-parallel decode), "LL" style: every value travels
// as an 8-byte word {fp32 bits, epoch}; an 8-byte store is delivered atomically, so the receiver needs no
// fence, flag or barrier -- it polls the word until its epoch field matches.  Every rank owns a region
//   [2 parities][N ranks][slot_elems] x 8 bytes
// that all peers map (CUDA IPC).  Producer (GEMV epilogue): each thread stores its fp32 partial into slot
// `rank` of EVERY peer's region (st.global.v2 over NVLink).  Reducer: polls the N local slots and adds them
// IN RANK ORDER (every rank gets the same bits), then applies the residual add.
// parity = epoch & 1 double-buffers the region (a rank can be at most one all-reduce ahead of a peer).
struct LnbP2P {
  uint2* data[8];      // peer r's region base (device pointers valid on this GPU)
  int rank, n, slot_elems;
  unsigned long long timeout_ns;   // budget of one wait for a peer's words (%globaltimer); 0 = wait forever
};

LNB_DEVINL unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
LNB_DEVINL uint2 ld_volatile_u2(const uint2* p) {
  uint2 v;
  asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
// Bounded wait for one LL word of `epoch` from rank r.  A late or dead peer must not hang the GPU (and with it
// the whole box): after timeout_ns the first waiter records (epoch, rank) in st->ar_error, every other waiter
// sees the flag within 1024 polls, and all of them return false.  The host turns the flag into LNB_ETIMEOUT.
LNB_DEVINL bool p2p_wait_word(const uint2* src, uint32_t epoch, int r, const LnbP2P& pp, LnbDevState* st,
                              unsigned long long t_start, uint2* out) {
  uint2 w = ld_volatile_u2(src);
  uint32_t spins = 0;
  while (w.y != epoch) {
    if ((++spins & 1023u) == 0u) {
      if (*reinterpret_cast<volatile uint32_t*>(&st->ar_error)) return false;
      if (pp.timeout_ns && global_timer_ns() - t_start > pp.timeout_ns) {
        atomicCAS(&st->ar_error, 0u, 0x80000000u | ((epoch & 0xffffffu) << 4) | (uint32_t)(r & 15));
        return false;
      }
    }
    w = ld_volatile_u2(src);
  }
  *out = w;
  return true;
}
