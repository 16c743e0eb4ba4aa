// Execution primitives of the device program.
//
// The scheduling program (hived_core.h) is written once against these primitives:
//   * CUDA build (the product, sm_90a): one CTA; warp 0 is the "leader warp" that executes the
//     sequential control flow warp-uniformly (all 32 lanes run the same scalar code; stores are
//     done by lane 0 and ordered with __syncwarp), the other warps sleep in the hardware barrier
//     until the leader posts a data-parallel operation (cluster-view pass) in shared memory.
//   * HIVED_EMU build (tests/ only, never shipped or loaded by the package): a 1-thread, 1-lane
//     instantiation of the same source on the host so the kernel LOGIC can be unit-tested in a
//     container without a GPU.  It is not a fallback: the product library contains no host path.
#pragma once
#include <cstdint>

#ifdef HIVED_EMU
#define HIVED_DEV inline
#define HIVED_DEV_NOINLINE
#define HIVED_WARPSZ 1
namespace hived {
struct ExecShim {};
inline int hv_lane() { return 0; }
inline int hv_tid() { return 0; }
inline int hv_nth() { return 1; }
inline int hv_warp() { return 0; }
inline int hv_nwarps() { return 1; }
inline bool hv_is_runahead() { return false; }
inline bool hv_in_lead_group() { return true; }
inline void hv_regs_lead_group() {}
inline void hv_regs_other_group() {}
inline void hv_nanosleep() {}
inline void hv_touch(const void*) {}
inline void hv_cta_sync() {}
inline void hv_publish_smem(int* p, int v) { *(volatile int*)p = v; }
inline int hv_peek_smem(int* p) { return *(volatile int*)p; }
inline void hv_warp_sync() {}
inline void hv_phase() {}
inline unsigned hv_ballot(bool p) { return p ? 1u : 0u; }
inline unsigned hv_match(int) { return 1u; }
inline unsigned hv_lanemask_lt() { return 0u; }
inline int hv_popc(unsigned m) { return __builtin_popcount(m); }
inline int hv_ffs(unsigned m) { return __builtin_ffs((int)m); }
inline int hv_hibit(unsigned m) { return m ? 31 - __builtin_clz(m) : -1; }  // index of the highest set bit
inline int hv_fns(unsigned m, int k) {  // position of the (k+1)-th set bit, -1 if there is none
  for (int b = 0; b < 32; b++) if ((m >> b) & 1u) { if (k == 0) return b; k--; }
  return -1;
}
inline int hv_shfl(int v, int) { return v; }
inline int hv_shfl_up(int v, int) { return v; }
inline int hv_shfl_xor(int v, int) { return v; }
inline int hv_atomic_min(int* a, int v) { int o = *a; if (v < o) *a = v; return o; }
inline int hv_atomic_add(int* a, int v) { int o = *a; *a = o + v; return o; }
inline void hv_red_max(int* a, int v) { if (v > *a) *a = v; }
inline long long hv_clock() { return 0; }
#ifdef HIVED_EMU_MT
// several 1-lane CTAs on host threads (tests/emu/hived_emu_mt.cpp: the CPU comparator of bench.py): the ordered
// shared sections between CTAs use the same progress protocol, with host atomics
extern thread_local int hv_tls_cta;
inline int hv_ld_volatile(const int* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void hv_st_volatile(int* p, int v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
inline void hv_fence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline void hv_atomic_add64(long long* a, long long v) { __atomic_fetch_add(a, v, __ATOMIC_RELAXED); }
inline void hv_atomic_or64(long long* a, long long v) { __atomic_fetch_or(a, v, __ATOMIC_RELAXED); }
inline int hv_cta() { return hv_tls_cta; }
#else
inline int hv_ld_volatile(const int* p) { return *p; }
inline void hv_st_volatile(int* p, int v) { *p = v; }
inline void hv_fence() {}
inline void hv_atomic_add64(long long* a, long long v) { *a += v; }
inline void hv_atomic_or64(long long* a, long long v) { *a |= v; }
inline int hv_cta() { return 0; }
#endif
inline void hv_prefetch(const void*) {}
// asynchronous 16-byte global -> shared copies (host emulation: plain copy, nothing to wait for)
inline void hv_cp_async16(void* smem, const void* gmem) { __builtin_memcpy(smem, gmem, 16); }
inline void hv_cp_async_wait() {}
inline int hv_reduce_max(int v) { return v; }
inline int hv_reduce_min(int v) { return v; }
inline int hv_reduce_add(int v) { return v; }
}  // namespace hived
#define HV_ST(ptr, val) (*(ptr) = (val))
#elif defined(HIVED_SIMT_EMU)
// tests/emu/simt_rt.h: the same program with the real geometry (32 lanes, several warps, several CTAs), every CUDA
// thread a fiber on one host thread — functional checking of the warp-level code without a GPU (test only)
#define HIVED_DEV inline
#define HIVED_DEV_NOINLINE
#define HIVED_WARPSZ 32
namespace hived {
inline int hv_lane() { return simt::lane(); }
inline int hv_tid() { return simt::tid(); }
// the last warp of a CTA with three or more warps is the run-ahead (prefetch) warp: it takes no part in the CTA-wide
// passes, whose barrier spans the other warps only
inline bool hv_has_runahead() { return simt::nth() >= 96; }
inline int hv_nth() { return simt::nth() - (hv_has_runahead() ? 32 : 0); }
inline int hv_warp() { return simt::warp(); }
inline int hv_nwarps() { return hv_nth() / 32; }
inline bool hv_is_runahead() { return hv_has_runahead() && simt::warp() == hv_nwarps(); }
// the roles of the CUDA build's register split (below); the reallocation itself has no host counterpart
inline bool hv_in_lead_group() { return simt::warp() < 4 && !hv_is_runahead(); }
inline void hv_regs_lead_group() {}
inline void hv_regs_other_group() {}
inline void hv_nanosleep() { simt::yield_to_scheduler(); }
inline void hv_touch(const void* p) { (void)*(const volatile char*)p; }
inline void hv_cta_sync() { simt::cta_barrier_n(hv_nth()); }
inline void hv_publish_smem(int* p, int v) { *(volatile int*)p = v; }
inline int hv_peek_smem(int* p) { simt::yield_to_scheduler(); return *(volatile int*)p; }
inline void hv_warp_sync() { simt::warp_collective(0, [](const int*, int*) {}); }
// phase boundary: every lane has finished the reads of the phase before any lane starts the writes of the next one
inline void hv_phase() { hv_warp_sync(); }
inline unsigned hv_ballot(bool p) {
  return (unsigned)simt::warp_collective(p ? 1 : 0, [](const int* v, int* r) {
    unsigned m = 0;
    for (int i = 0; i < 32; i++) if (v[i]) m |= 1u << i;
    for (int i = 0; i < 32; i++) r[i] = (int)m;
  });
}
inline unsigned hv_match(int x) {
  return (unsigned)simt::warp_collective(x, [](const int* v, int* r) {
    for (int i = 0; i < 32; i++) { unsigned m = 0; for (int j = 0; j < 32; j++) if (v[j] == v[i]) m |= 1u << j; r[i] = (int)m; }
  });
}
inline unsigned hv_lanemask_lt() { return (1u << simt::lane()) - 1u; }
inline int hv_popc(unsigned m) { return __builtin_popcount(m); }
inline int hv_ffs(unsigned m) { return __builtin_ffs((int)m); }
inline int hv_hibit(unsigned m) { return m ? 31 - __builtin_clz(m) : -1; }
inline int hv_fns(unsigned m, int k) {
  for (int b = 0; b < 32; b++) if ((m >> b) & 1u) { if (k == 0) return b; k--; }
  return -1;
}
inline int hv_shfl(int x, int src) {
  // every lane names its own source: deposit the values, then read the named one
  simt::warp_collective(x, [](const int* v, int* r) { for (int i = 0; i < 32; i++) r[i] = v[i]; });
  int got = simt::rt().cur->w->res[src & 31];
  simt::warp_collective(0, [](const int*, int*) {});  // nobody overwrites res[] before every lane has read
  return got;
}
inline int hv_shfl_up(int x, int d) {
  return simt::warp_collective(x, [d](const int* v, int* r) { for (int i = 0; i < 32; i++) r[i] = i >= d ? v[i - d] : v[i]; });
}
inline int hv_shfl_xor(int x, int m) {
  return simt::warp_collective(x, [m](const int* v, int* r) { for (int i = 0; i < 32; i++) r[i] = v[i ^ m]; });
}
inline int hv_atomic_min(int* a, int v) { int o = *a; if (v < o) *a = v; return o; }
inline int hv_atomic_add(int* a, int v) { int o = *a; *a = o + v; return o; }
inline void hv_red_max(int* a, int v) { if (v > *a) *a = v; }
inline long long hv_clock() { return 0; }
inline int hv_ld_volatile(const int* p) { simt::yield_to_scheduler(); return *(const volatile int*)p; }
inline void hv_st_volatile(int* p, int v) { *(volatile int*)p = v; }
inline void hv_fence() {}
inline void hv_atomic_add64(long long* a, long long v) { *a += v; }
inline void hv_atomic_or64(long long* a, long long v) { *a |= v; }
inline int hv_cta() { return simt::cta(); }
inline void hv_prefetch(const void*) {}
inline void hv_cp_async16(void* smem, const void* gmem) { __builtin_memcpy(smem, gmem, 16); }
inline void hv_cp_async_wait() {}
inline int hv_reduce_max(int x) {
  return simt::warp_collective(x, [](const int* v, int* r) { int m = v[0]; for (int i = 1; i < 32; i++) if (v[i] > m) m = v[i]; for (int i = 0; i < 32; i++) r[i] = m; });
}
inline int hv_reduce_min(int x) {
  return simt::warp_collective(x, [](const int* v, int* r) { int m = v[0]; for (int i = 1; i < 32; i++) if (v[i] < m) m = v[i]; for (int i = 0; i < 32; i++) r[i] = m; });
}
inline int hv_reduce_add(int x) {
  return simt::warp_collective(x, [](const int* v, int* r) { int m = 0; for (int i = 0; i < 32; i++) m += v[i]; for (int i = 0; i < 32; i++) r[i] = m; });
}
}  // namespace hived
#define HV_ST(ptr, val)                      \
  do {                                       \
    if (hived::hv_lane() == 0) *(ptr) = (val); \
    hived::hv_warp_sync();                   \
  } while (0)
#else
#define HIVED_DEV __device__ __forceinline__
#define HIVED_DEV_NOINLINE __device__ __noinline__
#define HIVED_WARPSZ 32
namespace hived {
__device__ __forceinline__ int hv_lane() { return threadIdx.x & 31; }
__device__ __forceinline__ int hv_tid() { return threadIdx.x; }
// The last warp of the CTA is the run-ahead (prefetch) warp (hived_core.h: runAhead): it takes no part in the
// CTA-wide passes, whose barrier (a named barrier) spans the other warps only.
__device__ __forceinline__ int hv_nth() { return blockDim.x - 32; }
__device__ __forceinline__ int hv_warp() { return threadIdx.x >> 5; }
__device__ __forceinline__ int hv_nwarps() { return (blockDim.x >> 5) - 1; }
__device__ __forceinline__ bool hv_is_runahead() { return (threadIdx.x >> 5) == (blockDim.x >> 5) - 1; }
// Register split between the warpgroups of the 512-thread CTA (setmaxnreg, sm_90a).  __launch_bounds__(512, 1) caps
// every thread at 128 registers, yet only the leader warp runs the long sequential code.  Warpgroup 0 (the leader and
// workers 1-3) grows to HV_REGS_LEAD, warpgroups 1-3 (the other workers and the run-ahead warp) shrink to
// HV_REGS_OTHER: 128 x 240 + 384 x 88 = 64 512 of the SM's 65 536.  The instruction is warpgroup-collective (all four
// warps execute the same one).  ptxas compiles code that both groups reach under the smaller limit, so each group's
// roles stay in a branch of their own until they are done (Core::run / Core::serve).
constexpr int HV_REGS_LEAD = 240, HV_REGS_OTHER = 88;
__device__ __forceinline__ bool hv_in_lead_group() { return threadIdx.x < 128; }
__device__ __forceinline__ void hv_regs_lead_group() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(HV_REGS_LEAD)); }
__device__ __forceinline__ void hv_regs_other_group() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(HV_REGS_OTHER)); }
__device__ __forceinline__ void hv_nanosleep() { __nanosleep(200); }
// pull a line towards L1 without a register target
__device__ __forceinline__ void hv_touch(const void* p) {
  // an ordinary cached load whose result nobody waits for: unlike prefetch.global.L1 (a hint), it is certain to
  // allocate the line in L1
  unsigned t;
  asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(t) : "l"(p));
}
// named barrier 1 over the leader + worker warps (the run-ahead warp never joins).  The leader and the workers reach it
// from different instructions, so it is the UNALIGNED form (PTX: bar.sync == barrier.sync.aligned asks every
// participant to execute the same barrier instruction; compute-sanitizer synccheck enforces that).
#ifdef HIVED_AB_ALIGNED_BAR  // (A/B builds only)
__device__ __forceinline__ void hv_cta_sync() { asm volatile("bar.sync 1, %0;" ::"r"(blockDim.x - 32) : "memory"); }
#else
__device__ __forceinline__ void hv_cta_sync() { asm volatile("barrier.sync 1, %0;" ::"r"(blockDim.x - 32) : "memory"); }
#endif
// a progress word in SHARED memory polled by another warp of the CTA (the run-ahead warp follows the leader): atomic
// on both sides, so that the intended concurrent access is not a data race (compute-sanitizer racecheck)
#ifdef HIVED_AB_VOLATILE_PUBLISH  // (A/B builds only)
__device__ __forceinline__ void hv_publish_smem(int* p, int v) { *(volatile int*)p = v; }
#else
__device__ __forceinline__ void hv_publish_smem(int* p, int v) { atomicExch(p, v); }
#endif
__device__ __forceinline__ int hv_peek_smem(int* p) { return atomicAdd(p, 0); }
__device__ __forceinline__ void hv_warp_sync() { __syncwarp(); }
// phase boundary of the leader warp's uniform code (all lanes read, then one or all lanes write the same locations).
// The warp is converged there (uniform control flow, no divergent call in between), so the hardware executes the
// reads of all lanes before the writes; the functional emulator (tests/emu/simt_rt.h), which runs lanes one after
// the other, makes the boundary explicit.  -DHIVED_STRICT_PHASES turns it into a real __syncwarp().
#ifdef HIVED_STRICT_PHASES
__device__ __forceinline__ void hv_phase() { __syncwarp(); }
#else
__device__ __forceinline__ void hv_phase() {}
#endif
__device__ __forceinline__ unsigned hv_ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
__device__ __forceinline__ unsigned hv_match(int v) { return __match_any_sync(0xffffffffu, v); }
__device__ __forceinline__ unsigned hv_lanemask_lt() { return (1u << (threadIdx.x & 31)) - 1u; }
__device__ __forceinline__ int hv_popc(unsigned m) { return __popc(m); }
__device__ __forceinline__ int hv_ffs(unsigned m) { return __ffs((int)m); }
__device__ __forceinline__ int hv_hibit(unsigned m) { return 31 - __clz((int)m); }  // index of the highest set bit, -1 if none
__device__ __forceinline__ int hv_fns(unsigned m, int k) { return (int)__fns(m, 0, k + 1); }  // (k+1)-th set bit, -1 if none
__device__ __forceinline__ int hv_shfl(int v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ int hv_shfl_up(int v, int delta) { return __shfl_up_sync(0xffffffffu, v, delta); }
__device__ __forceinline__ int hv_shfl_xor(int v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
__device__ __forceinline__ int hv_atomic_min(int* a, int v) { return atomicMin(a, v); }
__device__ __forceinline__ int hv_atomic_add(int* a, int v) { return atomicAdd(a, v); }
// fire-and-forget maximum (RED.MAX: no return value, nothing waits for the old value)
__device__ __forceinline__ void hv_red_max(int* a, int v) { atomicMax(a, v); }
__device__ __forceinline__ long long hv_clock() { return clock64(); }
__device__ __forceinline__ int hv_ld_volatile(const int* p) { return *(const volatile int*)p; }
__device__ __forceinline__ void hv_st_volatile(int* p, int v) { *(volatile int*)p = v; }
__device__ __forceinline__ void hv_fence() { __threadfence(); }
__device__ __forceinline__ void hv_atomic_add64(long long* a, long long v) { atomicAdd((unsigned long long*)a, (unsigned long long)v); }
__device__ __forceinline__ void hv_atomic_or64(long long* a, long long v) { atomicOr((unsigned long long*)a, (unsigned long long)v); }
__device__ __forceinline__ int hv_cta() { return blockIdx.x; }
// asynchronous 16-byte global -> shared copy (LDGSTS): no register target, completes in the background
__device__ __forceinline__ void hv_cp_async16(void* smem, const void* gmem) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void hv_cp_async_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// warp-wide integer reductions: one REDUX instruction (sm_80+) instead of a five-step shuffle butterfly
__device__ __forceinline__ int hv_reduce_max(int v) { return __reduce_max_sync(0xffffffffu, v); }
__device__ __forceinline__ int hv_reduce_min(int v) { return __reduce_min_sync(0xffffffffu, v); }
__device__ __forceinline__ int hv_reduce_add(int v) { return __reduce_add_sync(0xffffffffu, v); }
__device__ __forceinline__ void hv_prefetch(const void* p) { asm volatile("prefetch.L1 [%0];" ::"l"(p)); }
}  // namespace hived
// leader-warp store: one lane writes, the warp is re-converged and the store ordered before later loads
#define HV_ST(ptr, val)                      \
  do {                                       \
    if (hived::hv_lane() == 0) *(ptr) = (val); \
    __syncwarp();                            \
  } while (0)
#endif
