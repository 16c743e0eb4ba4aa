// Joint launches (include/hived_multictx.h): the interface between hived_cuda.cu (host side, one stream, the per-context
// staging and bookkeeping) and hived_cuda_many.cu (the second build of the device program, which reads context y's Dev
// from constant slot y).
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
  long long* scalars;       // 4 words per CTA, as for hived_events_kernel
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

}  // namespace hived
