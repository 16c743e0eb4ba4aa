// Joint launches (include/hived_multictx.h) and concurrent contexts (HIVED_OPT_CONCURRENT): the interface between
// hived_cuda.cu (host side: streams, the per-context staging and bookkeeping) and the other two builds of the device
// program: hived_cuda_many.cu, which reads context y's Dev from constant slot y, and hived_cuda_conc.cu, which reads
// concurrent slot s's Dev from its constant slot s (the launch's dynamic shared-memory byte count names s).
#pragma once
#include <cuda_runtime.h>

#include "../../include/hived_multictx.h"
#include "hived_dev.h"

namespace hived {

// what CTA (x, y) of a joint launch needs of context y besides its Dev: the arguments of hived_events_kernel
struct ManySlot {
  const hived_event_t* events;
  hived_result_t* results;
  const uint32_t* sugg;     // nullptr: no suggested-node pool
  int32_t* pool;
  CtaWords* words;          // the launch words of every CTA, as for hived_events_kernel
  const int32_t* own;       // VC-parallel run: owner-sorted event list, then the C + 1 list offsets; else nullptr
  int n, C, nPinnedOrder, nBad;
};
struct ManyArgs {
  ManySlot slot[HIVED_MANY_MAX];
};

// contexts' CTAs that fit on the device at once (occupancy of the joint kernel x SM count); 0 if it cannot be queried
int manyCoResident(int device);
// one launch over devs[0..k) (slot y = context y): copies every Dev into its constant slot, then runs the joint events
// kernel on a (max C, k) grid — cooperatively when some context runs VC-parallel, whose CTAs wait for each other — and
// the joint repair kernel for those contexts.  Everything is queued on `st`; the caller synchronises.
cudaError_t manyLaunch(const Dev* const* devs, const ManyArgs& a, int k, cudaStream_t st);

// concurrent contexts (HIVED_OPT_CONCURRENT, hived_cuda_conc.cu): concurrent slot s (0 <= s < HIVED_CONCURRENT_MAX) is
// constant slot s of that build.  concLoadDev queues the copy of the context's Dev into it on `st`; the caller synchronises before
// the first launch.  concServeLaunch queues the slot's resident per-call kernel (Core::serve, arguments as for
// hived_serve_kernel) on `st`.
cudaError_t concLoadDev(const Dev& dev, int s, cudaStream_t st);
cudaError_t concServeLaunch(int s, volatile int32_t* slot, int seq0, int idleSpins, hived_result_t* stageRes, uint32_t* dSugg,
                            int32_t* dAux, int nPinnedOrder, int nBad, int32_t* pool, cudaStream_t st);
// concBatchLaunch queues one batch of the context in concurrent slot s (q, whose C CTAs run it) on `st`: the events
// kernel on C CTAs, cooperatively when C > 1, then the repair kernel when C > 1.  The caller synchronises.
cudaError_t concBatchLaunch(int s, const ManySlot& q, cudaStream_t st);

}  // namespace hived
