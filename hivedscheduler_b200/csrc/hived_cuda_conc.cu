// libhived_cuda.so, third translation unit: the device program of hived_core.h built for concurrent contexts
// (HIVED_OPT_CONCURRENT, include/hived.h).  Concurrent slot s of a device keeps its context's Dev in constant slot s
// (g_hived_devs[s]) from creation to destruction; every launch for it carries s as its dynamic shared-memory byte count
// (hv_slot_base, hived_core.h), so one kernel serves every slot.  The joint build (hived_cuda_many.cu) indexes its slots
// by blockIdx.y, which a launch of one context's CTAs cannot choose; the slot base is kept out of it so that the joint
// kernels stay as they were.
#define HIVED_CONC_BUILD 1
#include "hived_many.h"
#include "hived_core.h"

namespace hived {
namespace conc {

constexpr int NT = 512;  // as hived_cuda.cu: 16 warps, the whole register file of one SM

// one batch of the context: CTA x of its C CTAs (grid (C, 1)), arguments as for hived_events_kernel
__global__ void __launch_bounds__(NT, 1) hived_events_conc_kernel(const __grid_constant__ ManySlot q) {
  // (runCta's body, written out as in hived_events_many_kernel, for the same reason)
  Sm& sm = g_hived_sm;
  const int cta = blockIdx.x;
  if (threadIdx.x == 0) {
    sm.cmd = CMD_IDLE;
    sm.panic = 0;
    sm.lead_k = -1;
    sm.pool_off = ctaWords(q.words, cta).poolOff;
  }
  __syncthreads();
  Core core(g_hived_devs[hv_slot_base()], &sm, q.pool, ctaWords(q.words, cta).poolEnd, q.C);
  const int32_t* ownOff = q.own ? q.own + q.n : nullptr;
  const int nOwn = q.own ? ownOff[cta + 1] - ownOff[cta] : q.n;
  core.calm = ctaWords(q.words, cta).calm != 0;
  core.run(q.events, q.n, q.results, q.sugg, nullptr, nullptr, q.nPinnedOrder, q.nBad, q.own ? q.own + ownOff[cta] : nullptr, nOwn);
  __syncthreads();
  if (threadIdx.x == 0) {
    ctaWords(q.words, cta).poolOff = sm.pool_off;
    ctaWords(q.words, cta).calm = sm.panic;
    ctaWords(q.words, cta).mg = sm.stop_k;
  }
}

// one CTA: the repair pass of hived_repair_kernel after a VC-parallel batch
__global__ void __launch_bounds__(NT, 1) hived_repair_conc_kernel() {
  Core core(g_hived_devs[hv_slot_base()], &g_hived_sm, nullptr, 0, 1);
  core.repairSharedAncestors();
}

// the context's resident per-call kernel: hived_serve_kernel of hived_cuda.cu, one CTA
__global__ void __launch_bounds__(NT, 1)
hived_serve_conc_kernel(volatile int32_t* slot, int seq0, int idleSpins, hived_result_t* stageRes, uint32_t* dSugg,
                        int32_t* dAux, int nPinnedOrder, int nBad, int32_t* pool) {
  serveCta(g_hived_devs[hv_slot_base()], slot, seq0, idleSpins, stageRes, dSugg, dAux, nPinnedOrder, nBad, pool);
}

}  // namespace conc

cudaError_t concLoadDev(const Dev& dev, int s, cudaStream_t st) {
  // the kernels want L1, not shared memory, as hived_cuda.cu's
  cudaFuncSetAttribute(conc::hived_serve_conc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
  cudaFuncSetAttribute(conc::hived_events_conc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
  cudaFuncSetAttribute(conc::hived_repair_conc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
  return cudaMemcpyToSymbolAsync(conc::g_hived_devs, &dev, sizeof(Dev), (size_t)s * sizeof(Dev), cudaMemcpyHostToDevice, st);
}

cudaError_t concServeLaunch(int s, volatile int32_t* slot, int seq0, int idleSpins, hived_result_t* stageRes, uint32_t* dSugg,
                            int32_t* dAux, int nPinnedOrder, int nBad, int32_t* pool, cudaStream_t st) {
  void* args[] = {&slot, &seq0, &idleSpins, &stageRes, &dSugg, &dAux, &nPinnedOrder, &nBad, &pool};
  return cudaLaunchKernel((const void*)conc::hived_serve_conc_kernel, dim3(1), dim3(conc::NT), args, (size_t)s, st);
}

cudaError_t concBatchLaunch(int s, const ManySlot& q, cudaStream_t st) {
  void* args[] = {(void*)&q};
  cudaError_t e = q.C > 1
      ? cudaLaunchCooperativeKernel((const void*)conc::hived_events_conc_kernel, dim3(q.C), dim3(conc::NT), args, (size_t)s, st)
      : cudaLaunchKernel((const void*)conc::hived_events_conc_kernel, dim3(1), dim3(conc::NT), args, (size_t)s, st);
  if (e != cudaSuccess || q.C <= 1) return e;
  return cudaLaunchKernel((const void*)conc::hived_repair_conc_kernel, dim3(1), dim3(conc::NT), nullptr, (size_t)s, st);
}

}  // namespace hived
