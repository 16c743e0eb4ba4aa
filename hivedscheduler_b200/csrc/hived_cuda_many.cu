// libhived_cuda.so, second translation unit: the device program of hived_core.h built once more for joint launches
// (include/hived_multictx.h).  The only difference from hived_cuda.cu's build is where a CTA finds the scheduler state:
// context y's Dev sits in constant slot y (g_hived_devs[blockIdx.y]) instead of the single g_hived_dev, so the kernels
// of hived_cuda.cu — and the turn-taking of single-context calls around g_hived_dev — stay exactly as they are.
#define HIVED_MANY_BUILD 1
#include "hived_many.h"
#include "hived_core.h"

namespace hived {
namespace many {

constexpr int NT = 512;  // as hived_cuda.cu: 16 warps, the whole register file of one SM

// CTA (x, y) is CTA x of context y; a context with fewer CTAs than the grid's width leaves the rest idle
__global__ void __launch_bounds__(NT, 1) hived_events_many_kernel(const __grid_constant__ ManyArgs a) {
  const ManySlot& q = a.slot[blockIdx.y];
  const int cta = blockIdx.x;
  if (cta >= q.C) return;
  Sm& sm = g_hived_sm;
  if (threadIdx.x == 0) {
    sm.cmd = CMD_IDLE;
    sm.panic = 0;
    sm.lead_k = -1;
    sm.pool_off = q.scalars[cta * 4 + 0];
  }
  __syncthreads();
  Core core(g_hived_devs[blockIdx.y], &sm, q.pool, q.scalars[cta * 4 + 1], q.C);
  const int32_t* ownOff = q.own ? q.own + q.n : nullptr;
  const int nOwn = q.own ? ownOff[cta + 1] - ownOff[cta] : q.n;
  core.run(q.events, q.n, q.results, q.sugg, nullptr, nullptr, q.nPinnedOrder, q.nBad, q.own ? q.own + ownOff[cta] : nullptr, nOwn);
  __syncthreads();
  if (threadIdx.x == 0) {
    q.scalars[cta * 4 + 0] = sm.pool_off;
    q.scalars[cta * 4 + 2] = sm.panic;
    q.scalars[cta * 4 + 3] = sm.stop_k;
  }
}

// grid (1, k): the repair pass of hived_repair_kernel for the contexts that ran VC-parallel
__global__ void __launch_bounds__(NT, 1) hived_repair_many_kernel(const __grid_constant__ ManyArgs a) {
  if (a.slot[blockIdx.y].C <= 1) return;
  Core core(g_hived_devs[blockIdx.y], &g_hived_sm, nullptr, 0, 1);
  core.repairSharedAncestors();
}

}  // namespace many

int manyCoResident(int device) {
  static int cached[64] = {0};
  const int dv = device >= 0 && device < 64 ? device : 0;
  if (cached[dv]) return cached[dv];
  int perSm = 0, sms = 0;
  cudaFuncSetAttribute(many::hived_events_many_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
  cudaFuncSetAttribute(many::hived_repair_many_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, many::hived_events_many_kernel, many::NT, 0) != cudaSuccess ||
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess)
    return 0;
  cached[dv] = perSm * sms;
  return cached[dv];
}

cudaError_t manyLaunch(const Dev* const* devs, const ManyArgs& a, int k, cudaStream_t st) {
  int cmax = 1;
  bool parallel = false;
  for (int y = 0; y < k; y++) {
    cudaError_t e = cudaMemcpyToSymbolAsync(many::g_hived_devs, devs[y], sizeof(Dev), (size_t)y * sizeof(Dev), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    if (a.slot[y].C > cmax) cmax = a.slot[y].C;
    if (a.slot[y].C > 1) parallel = true;
  }
  void* args[] = {(void*)&a};
  cudaError_t e = parallel
      ? cudaLaunchCooperativeKernel((const void*)many::hived_events_many_kernel, dim3(cmax, k), dim3(many::NT), args, 0, st)
      : cudaLaunchKernel((const void*)many::hived_events_many_kernel, dim3(cmax, k), dim3(many::NT), args, 0, st);
  if (e != cudaSuccess) return e;
  if (parallel) e = cudaLaunchKernel((const void*)many::hived_repair_many_kernel, dim3(1, k), dim3(many::NT), args, 0, st);
  return e;
}

}  // namespace hived
