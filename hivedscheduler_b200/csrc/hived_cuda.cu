// libhived_cuda.so — the product: CUDA backend (sm_90a) of include/hived.h.
//
// One kernel, `hived_events_kernel`, runs the scheduling program of hived_core.h over an ordered
// batch of events with ALL scheduler state resident in HBM (hived_dev.h).  It is launched with one
// CTA per group of virtual clusters (one CTA when the batch must run strictly sequentially): in every CTA
// warp 0 walks its share of the batch (the reference's contract is sequential, pkg/internal/types.go:64-71;
// VCs only meet in ordered shared sections), the remaining warps are woken through the hardware barrier for
// the data-parallel cluster-view pass of every scheduling decision.  There is no host implementation
// of the algorithm in this library: if no CUDA device is usable hived_create fails with
// HIVED_ERR_NO_DEVICE.
#include <cuda_runtime.h>

#include <mutex>

#define HIVED_BK_LAUNCH_MANY 1  // the joint launch below
#include "hived_engine.hpp"
#include "hived_many.h"

namespace hived {

constexpr int NT = 512;  // threads per CTA (16 warps); the kernel needs the full register file of one SM

// scalars: 4 words per CTA — [0] pool offset (in: start of the CTA's slice, out: first unused word),
// [1] end of the slice, [2] out: initialisation panic code
__global__ void __launch_bounds__(NT, 1)
hived_events_kernel(const hived_event_t* __restrict__ events, int n, hived_result_t* results,
                    const uint32_t* suggPool, const int32_t* aux, const int32_t* initLists, int nPinnedOrder, int nBad,
                    int32_t* pool, long long* scalars, const int32_t* own, const int32_t* ownOff) {
  Sm& sm = g_hived_sm;
  const int cta = blockIdx.x;
  if (threadIdx.x == 0) {
    sm.cmd = CMD_IDLE;
    sm.panic = 0;
    sm.lead_k = -1;
    sm.pool_off = scalars[cta * 4 + 0];
  }
  __syncthreads();
  Core core(g_hived_dev, &sm, pool, scalars[cta * 4 + 1], gridDim.x);
  int nOwn = own ? ownOff[cta + 1] - ownOff[cta] : n;
  // multi-GPU partition: [start, limit) of this CTA's list and the mode, packed by launchProgram (0: an ordinary run)
  const long long mg = scalars[cta * 4 + 3];
  if (mg) { core.setMultiGpu((int)((mg >> 62) & 3), (int)(mg & 0x7fffffff)); nOwn = (int)((mg >> 31) & 0x7fffffff); }
  core.run(events, n, results, suggPool, aux, initLists, nPinnedOrder, nBad, own ? own + ownOff[cta] : nullptr, nOwn);
  __syncthreads();
  if (threadIdx.x == 0) {
    scalars[cta * 4 + 0] = sm.pool_off;
    scalars[cta * 4 + 2] = sm.panic;
    scalars[cta * 4 + 3] = sm.stop_k;
  }
}

__global__ void __launch_bounds__(NT, 1) hived_repair_kernel() {
  Sm& sm = g_hived_sm;
  Core core(g_hived_dev, &sm, nullptr, 0, 1);
  core.repairSharedAncestors();
}

// The per-call path, resident: one CTA that stays on an SM while calls keep coming (Core::serve).
__global__ void __launch_bounds__(NT, 1)
hived_serve_kernel(volatile int32_t* slot, int seq0, int idleSpins, hived_result_t* stageRes,
                   uint32_t* dSugg, int32_t* dAux, int nPinnedOrder, int nBad, int32_t* pool) {
  Sm& sm = g_hived_sm;
  if (threadIdx.x == 0) {
    sm.cmd = CMD_IDLE;
    sm.panic = 0;
    sm.lead_k = 0x7fffffff;
    sm.pool_off = 0;
  }
  __syncthreads();
  Core core(g_hived_dev, &sm, pool, 0, 1);
  core.serve(slot, seq0, idleSpins, stageRes, dSugg, dAux, nPinnedOrder, nBad);
}

static bool cudaOk(cudaError_t e, std::string& err, const char* what) {
  if (e == cudaSuccess) return true;
  err = std::string(what) + ": " + cudaGetErrorString(e);
  return false;
}

void* bk_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  return p;
}
void bk_free(void* p) { cudaFree(p); }
// The copy hooks have no return value (the engine is backend-neutral): the first failure of the calling thread is kept
// and reported by the next launchProgram / bk_run_small as a platform error (bk_init, i.e. hived_create, starts clean).
static thread_local cudaError_t g_copyErr = cudaSuccess;
static inline void noteCopy(cudaError_t e) { if (e != cudaSuccess && g_copyErr == cudaSuccess) g_copyErr = e; }
static int takeCopyError(std::string& err) {
  if (g_copyErr == cudaSuccess) return 0;
  err = std::string("a device copy failed: ") + cudaGetErrorString(g_copyErr);
  g_copyErr = cudaSuccess;
  cudaGetLastError();
  return HIVED_ERR_PLATFORM;
}
void bk_h2d(void* dst, const void* src, size_t bytes) { if (bytes) noteCopy(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); }
void bk_d2h(void* dst, const void* src, size_t bytes) { if (bytes) noteCopy(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost)); }
void bk_d2d(void* dst, const void* src, size_t bytes) { if (bytes) noteCopy(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToDevice)); }
void bk_zero(void* dst, size_t bytes) { if (bytes) noteCopy(cudaMemset(dst, 0, bytes)); }

void bk_flush_l2() {  // one buffer per device (the current one)
  static void* bufs[64] = {nullptr};
  int dv = 0;
  if (cudaGetDevice(&dv) != cudaSuccess || dv < 0 || dv >= 64) return;
  const size_t bytes = 256u << 20;  // several times the 50 MB L2 of an H100
  if (!bufs[dv] && cudaMalloc(&bufs[dv], bytes) != cudaSuccess) { bufs[dv] = nullptr; return; }
  static int v = 0;
  cudaMemset(bufs[dv], ++v & 0xff, bytes);
  cudaDeviceSynchronize();
}

void bk_use_device(int device) {
  int cur = -1;
  if (cudaGetDevice(&cur) == cudaSuccess && cur != device) cudaSetDevice(device);
}

int bk_init(int& device, std::string& err) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    err = std::string("no usable CUDA device (") + (e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e)) +
          "); libhived_cuda has no CPU fallback";
    return HIVED_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= count) device = 0;
  if (!cudaOk(cudaSetDevice(device), err, "cudaSetDevice")) return HIVED_ERR_NO_DEVICE;
  g_copyErr = cudaSuccess;
  // (the device program does not recurse — explicit stacks in hived_core.h — so its stack frame is known to the
  // compiler and cudaLimitStackSize stays at the driver's default; HIVED_STACK_BYTES overrides it for experiments)
  if (const char* sb = getenv("HIVED_STACK_BYTES")) {
    const long v = atol(sb);
    if (v > 0 && !cudaOk(cudaDeviceSetLimit(cudaLimitStackSize, (size_t)v), err, "cudaDeviceSetLimit")) return HIVED_ERR_NO_DEVICE;
  }
  return 0;
}

struct CudaTimers {
  cudaEvent_t start = nullptr, stop = nullptr;
  cudaStream_t stream = nullptr;
  // resident per-call kernel (bk_run_small): a non-blocking stream of its own, one request slot in mapped host memory
  cudaStream_t serveStream = nullptr;
  volatile int32_t* slotHost = nullptr;  // cudaHostAlloc(mapped)
  int32_t* slotDev = nullptr;
  hived_result_t* stageRes = nullptr;
  uint32_t* dSugg = nullptr;
  int32_t* dAux = nullptr;
  int32_t* servePool = nullptr;
  long long servePoolCap = 0;
  int seq = 0;
  bool alive = false;    // a serve kernel was launched and has not been seen to exit
  bool disabled = false; // HIVED_NO_RESIDENT=1, or setting it up failed: one launch per call
  long long served = 0, launches = 0;
};

// ---- whose Dev is in the constant bank (g_hived_dev, hived_core.h) of each device ---------------------------------
// One context per device at a time.  Every section that launches a kernel or talks to a resident one holds g_devMu
// (contexts of one process take turns on the GPU; a context by itself is single-threaded per the ABI), makes sure its
// own Dev is the one loaded, and leaves nothing of its own running except the resident per-call kernel — which the
// next owner stops (bk_quiesce) before it overwrites the constant bank.
static std::recursive_mutex g_devMu;
static Engine* g_devOwner[64] = {nullptr};

void bk_quiesce(Engine& e);
static int ensureDevLoaded(Engine& e) {  // g_devMu held, the context's device current
  const int dv = e.deviceOrdinal >= 0 && e.deviceOrdinal < 64 ? e.deviceOrdinal : 0;
  if (g_devOwner[dv] == &e) return 0;
  if (g_devOwner[dv]) bk_quiesce(*g_devOwner[dv]);
  g_devOwner[dv] = nullptr;
  cudaError_t ce = cudaMemcpyToSymbol(g_hived_dev, &e.dev, sizeof(Dev));  // synchronous: nothing of ours is running
  if (ce != cudaSuccess) { e.err = std::string("cudaMemcpyToSymbol(g_hived_dev): ") + cudaGetErrorString(ce); return HIVED_ERR_PLATFORM; }
  g_devOwner[dv] = &e;
  return 0;
}
void bk_forget(Engine& e) {  // the context is going away
  std::lock_guard<std::recursive_mutex> lk(g_devMu);
  for (auto& o : g_devOwner) if (o == &e) o = nullptr;
}

// Stop the resident kernel (if any) and wait until it has left: before anything else launches on or writes to the
// scheduler state.  Called with the context's device current.
void bk_quiesce(Engine& e) {
  std::lock_guard<std::recursive_mutex> lk(g_devMu);
  CudaTimers* t = (CudaTimers*)e.stream;
  if (!t || !t->alive) return;
  volatile int32_t* s = t->slotHost;
  if (!s[SERVE_DONE_OFF + 4]) {
    s[1] = 0;  // n = 0: STOP
    __sync_synchronize();
    s[0] = ++t->seq;
  }
  cudaStreamSynchronize(t->serveStream);
  t->alive = false;
}

static_assert(NT / 32 <= MAX_WARPS, "the shared counters are sized for MAX_WARPS warps per CTA");

int launchProgram(Engine& e, int n, bool withInit) {
  std::lock_guard<std::recursive_mutex> lk(g_devMu);
  if (!e.stream) {
    // the kernel wants L1, not shared memory: ask for the smallest carveout that holds its ~18 KB of static smem
    cudaFuncSetAttribute(hived_events_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
    CudaTimers* t = new CudaTimers();
    if (!cudaOk(cudaStreamCreate(&t->stream), e.err, "cudaStreamCreate")) return HIVED_ERR_NO_DEVICE;
    cudaEventCreate(&t->start);
    cudaEventCreate(&t->stop);
    e.stream = t;
  }
  CudaTimers* t = (CudaTimers*)e.stream;
  bk_quiesce(e);
  if (int rc = takeCopyError(e.err)) return rc;  // a staging copy of this batch (or of create()) failed
  if (int rc = ensureDevLoaded(e)) return rc;
  const int mgMode = withInit ? 0 : e.mgMode;
  if (mgMode == 3) {  // end of a multi-GPU partition run: the repair pass alone
    hived_repair_kernel<<<1, NT, 0, t->stream>>>();
    cudaError_t err = cudaStreamSynchronize(t->stream);
    if (err != cudaSuccess) { e.err = std::string("hived_repair_kernel failed: ") + cudaGetErrorString(err); return HIVED_ERR_PLATFORM; }
    e.kernelLaunches++;
    return 0;
  }
  const int C = withInit ? 1 : e.launchCta;
  long long scal[MAX_CTAS * 4] = {0};
  for (int c = 0; c < C; c++) {
    scal[c * 4 + 0] = withInit ? 0 : (mgMode ? e.mgPoolCur[c] : e.poolBase[c]);
    scal[c * 4 + 1] = withInit ? 0 : e.poolBase[c + 1];
    if (mgMode) scal[c * 4 + 3] = ((long long)mgMode << 62) | ((long long)e.mgLimit[c] << 31) | (long long)e.mgCursor[c];
  }
  cudaMemcpyAsync(e.dScalars.p, scal, sizeof scal, cudaMemcpyHostToDevice, t->stream);
  cudaEventRecord(t->start, t->stream);
  const int32_t* own = (C > 1 || mgMode) ? (const int32_t*)e.dOwn.p : nullptr;
  if (C > 1 && !mgMode) {
    // The CTAs of a VC-parallel batch wait for each other (ordered shared sections): launch them cooperatively, so
    // that the runtime guarantees that all of them are resident at the same time.
    const hived_event_t* aEvents = (const hived_event_t*)e.dEvents.p;
    int aN = n;
    hived_result_t* aResults = (hived_result_t*)e.dResults.p;
    const uint32_t* aSugg = e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr;
    const int32_t* aAux = e.hasAux ? (const int32_t*)e.dAux.p : nullptr;
    const int32_t* aInit = nullptr;
    int aPinned = e.nPinnedOrder, aBad = e.nBad;
    int32_t* aPool = (int32_t*)e.dPool.p;
    long long* aScal = (long long*)e.dScalars.p;
    const int32_t* aOwn = own;
    const int32_t* aOwnOff = own + n;
    void* args[] = {&aEvents, &aN, &aResults, &aSugg, &aAux, &aInit, &aPinned, &aBad, &aPool, &aScal, &aOwn, &aOwnOff};
    cudaError_t le = cudaLaunchCooperativeKernel((const void*)hived_events_kernel, dim3(C), dim3(NT), args, 0, t->stream);
    if (le != cudaSuccess) {
      e.err = std::string("cooperative launch of hived_events_kernel failed: ") + cudaGetErrorString(le);
      return HIVED_ERR_PLATFORM;
    }
  } else {
    hived_events_kernel<<<C, NT, 0, t->stream>>>(
        (const hived_event_t*)e.dEvents.p, n, (hived_result_t*)e.dResults.p,
        e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, e.hasAux ? (const int32_t*)e.dAux.p : nullptr,
        withInit ? (const int32_t*)e.dInit.p : nullptr, e.nPinnedOrder, e.nBad, (int32_t*)e.dPool.p, (long long*)e.dScalars.p, own,
        own ? own + n : nullptr);
  }
  if (C > 1 && !mgMode) hived_repair_kernel<<<1, NT, 0, t->stream>>>();
  cudaEventRecord(t->stop, t->stream);
  cudaMemcpyAsync(scal, e.dScalars.p, sizeof scal, cudaMemcpyDeviceToHost, t->stream);
  cudaError_t err = cudaStreamSynchronize(t->stream);
  if (err != cudaSuccess || (err = cudaGetLastError()) != cudaSuccess) {
    e.err = std::string("hived_events_kernel failed: ") + cudaGetErrorString(err);
    return HIVED_ERR_PLATFORM;
  }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, t->start, t->stop);
  e.lastKernelMs = ms;
  e.kernelMsTotal += ms;
  e.kernelLaunches += (C > 1 && !mgMode) ? 2 : 1;
  e.poolEnd.assign(C, 0);
  for (int c = 0; c < C; c++) e.poolEnd[c] = scal[c * 4 + 0];
  if (mgMode) { e.mgStopOut.assign(C, 0); for (int c = 0; c < C; c++) e.mgStopOut[c] = (int32_t)scal[c * 4 + 3]; }
  e.poolOff = scal[0];
  if (withInit && scal[2]) { e.err = "initialisation panicked on the device"; return (int)scal[2]; }
  return 0;
}

// ---- joint launches (include/hived_multictx.h, hived_cuda_many.cu) ------------------------------------------------
// The staged batches of several contexts of one device run in one launch, each context on CTAs of its own, on the first
// context's stream.  g_hived_dev and its owner are not touched; but every resident per-call kernel of the device is
// stopped first — the participants' (they would write the same state) and the owner's (it holds an SM the joint launch
// may need to have all its CTAs resident).  Contexts whose CTAs do not fit on the device together go to further
// launches (rounds), greedily in list order.
int bk_launch_many(Engine* const* es, int k) {
  std::lock_guard<std::recursive_mutex> lk(g_devMu);
  Engine& e0 = *es[0];
  const int dv = e0.deviceOrdinal >= 0 && e0.deviceOrdinal < 64 ? e0.deviceOrdinal : 0;
  for (int y = 0; y < k; y++) bk_quiesce(*es[y]);
  if (g_devOwner[dv]) bk_quiesce(*g_devOwner[dv]);
  auto fail = [&](const std::string& why) {
    for (int y = 0; y < k; y++) es[y]->err = why;
    return HIVED_ERR_PLATFORM;
  };
  std::string err;
  if (takeCopyError(err)) return fail(err);  // a staging copy of one of the batches failed
  const int fit = manyCoResident(e0.deviceOrdinal);
  if (fit <= 0) return fail("joint launch: cannot query the co-resident CTA limit");
  CudaTimers* t = (CudaTimers*)e0.stream;
  std::vector<long long> scal((size_t)k * MAX_CTAS * 4, 0);
  ManyArgs a;
  const Dev* devs[HIVED_MANY_MAX];
  for (int y = 0; y < k; y++) {
    Engine& e = *es[y];
    const int C = e.launchCta;
    long long* s = &scal[(size_t)y * MAX_CTAS * 4];
    for (int c = 0; c < C; c++) { s[c * 4 + 0] = e.poolBase[c]; s[c * 4 + 1] = e.poolBase[c + 1]; }
    cudaMemcpyAsync(e.dScalars.p, s, MAX_CTAS * 4 * sizeof(long long), cudaMemcpyHostToDevice, t->stream);
    a.slot[y] = ManySlot{(const hived_event_t*)e.dEvents.p, (hived_result_t*)e.dResults.p,
                         e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, (int32_t*)e.dPool.p, (long long*)e.dScalars.p,
                         C > 1 ? (const int32_t*)e.dOwn.p : nullptr, e.stagedN, C, e.nPinnedOrder, e.nBad};
    devs[y] = &e.dev;
  }
  cudaEventRecord(t->start, t->stream);
  for (int y0 = 0; y0 < k;) {  // one round: the longest prefix of the rest whose (widest C) x (count) fits
    int y1 = y0 + 1, cmax = a.slot[y0].C;
    while (y1 < k) {
      const int c = a.slot[y1].C > cmax ? a.slot[y1].C : cmax;
      if ((long long)c * (y1 - y0 + 1) > fit) break;
      cmax = c;
      y1++;
    }
    ManyArgs r;
    for (int y = y0; y < y1; y++) r.slot[y - y0] = a.slot[y];
    cudaError_t le = manyLaunch(devs + y0, r, y1 - y0, t->stream);
    if (le != cudaSuccess) { cudaStreamSynchronize(t->stream); cudaGetLastError(); return fail(std::string("joint launch failed: ") + cudaGetErrorString(le)); }
    y0 = y1;
  }
  cudaEventRecord(t->stop, t->stream);
  for (int y = 0; y < k; y++)
    cudaMemcpyAsync(&scal[(size_t)y * MAX_CTAS * 4], es[y]->dScalars.p, MAX_CTAS * 4 * sizeof(long long), cudaMemcpyDeviceToHost, t->stream);
  cudaError_t ce = cudaStreamSynchronize(t->stream);
  if (ce != cudaSuccess || (ce = cudaGetLastError()) != cudaSuccess) return fail(std::string("hived_events_many_kernel failed: ") + cudaGetErrorString(ce));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, t->start, t->stop);
  for (int y = 0; y < k; y++) {
    Engine& e = *es[y];
    const int C = e.launchCta;
    const long long* s = &scal[(size_t)y * MAX_CTAS * 4];
    e.lastKernelMs = ms;
    e.kernelMsTotal += ms;
    e.kernelLaunches += C > 1 ? 2 : 1;
    e.poolEnd.assign(C, 0);
    for (int c = 0; c < C; c++) e.poolEnd[c] = s[c * 4 + 0];
    e.poolOff = s[0];
  }
  return 0;
}

// ---- per-call path ------------------------------------------------------------------------------------------
// hived_schedule / hived_add_allocated_pod / hived_delete_* and tiny batches: one pinned staging buffer laid out as
// [events | scalars | suggested bitmaps | aux | results | pool window]; H2D, kernel and D2H are queued on the stream
// and the host waits once.  (The general path issues ~6 blocking copies per call.)
struct SmallStage {  // never freed: a few KB of pinned memory per calling thread, and no CUDA call at thread exit
  char* host = nullptr;
  size_t bytes = 0;
};
static constexpr int64_t SMALL_POOL_WINDOW = 16384;  // words copied back with the results; more on demand

// ---- resident per-call path -------------------------------------------------------------------------------------
// One request slot in mapped, pinned host memory.  The host writes the payload, then the header's sequence number
// (x86 stores are observed in order); the resident leader warp polls the header over PCIe, runs the events, writes
// results and pool words back into the slot, fences system-wide and stores `done`.  No launch, no cudaMemcpy, no
// stream synchronisation per call.  The kernel leaves after ~2 ms without a request and is relaunched on demand.
static bool serveSetup(Engine& e, CudaTimers* t) {
  if (t->disabled) return false;
  if (t->slotHost) return true;
  const char* off = getenv("HIVED_NO_RESIDENT");
  if (off && *off && *off != '0') { t->disabled = true; return false; }
  void* h = nullptr;
  if (cudaStreamCreateWithFlags(&t->serveStream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaHostAlloc(&h, (size_t)SERVE_SLOT_WORDS * 4, cudaHostAllocMapped) != cudaSuccess) { t->disabled = true; return false; }
  memset(h, 0, (size_t)SERVE_SLOT_WORDS * 4);
  t->slotHost = (volatile int32_t*)h;
  void* d = nullptr;
  if (cudaHostGetDevicePointer(&d, h, 0) != cudaSuccess) { t->disabled = true; return false; }
  t->slotDev = (int32_t*)d;
  t->servePoolCap = 3ll * e.dev.S.LS + 2 * 4096 + 64 > SERVE_POOL_WINDOW ? 3ll * e.dev.S.LS + 2 * 4096 + 64 : SERVE_POOL_WINDOW;
  t->servePoolCap *= SERVE_MAX_EVENTS;
  if (cudaMalloc((void**)&t->stageRes, sizeof(hived_result_t) * SERVE_MAX_EVENTS) != cudaSuccess ||
      cudaMalloc((void**)&t->dSugg, (size_t)SERVE_SUGG_MAX * 4) != cudaSuccess || cudaMalloc((void**)&t->dAux, (size_t)SERVE_AUX_MAX * 4) != cudaSuccess ||
      cudaMalloc((void**)&t->servePool, (size_t)t->servePoolCap * 4) != cudaSuccess) { t->disabled = true; return false; }
  cudaFuncSetAttribute(hived_serve_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
  return true;
}

static int serveCall(Engine& e, CudaTimers* t, const hived_event_t* events, int n, const uint32_t* suggPool, int64_t suggWords,
                     const int32_t* aux, int64_t auxWords, hived_result_t* res, int32_t* pool, int64_t poolCap) {
  const bool hasSugg = suggPool != nullptr && suggWords > 0, hasAux = aux != nullptr && auxWords > 0;
  if (n > SERVE_MAX_EVENTS || (hasSugg && suggWords > SERVE_SUGG_MAX) || (hasAux && auxWords > SERVE_AUX_MAX)) return -2;
  if (!serveSetup(e, t)) return -2;
  const long long cap = poolCap < t->servePoolCap ? poolCap : t->servePoolCap;
  e.notePriorities(events, n);
  e.launchCta = 1;
  e.hasSugg = hasSugg; e.hasAux = hasAux;
  e.poolCapWords = poolCap; e.stagedN = n; e.stagedEvents = events; e.canonicalDone = false;
  volatile int32_t* s = t->slotHost;
  int32_t* pay = (int32_t*)(s + SERVE_EV_OFF);
  memcpy(pay, events, (size_t)n * sizeof(hived_event_t));
  int32_t* hs = pay + SERVE_MAX_EVENTS * (int)(sizeof(hived_event_t) / 4);
  if (hasSugg) memcpy(hs, suggPool, (size_t)suggWords * 4);
  if (hasAux) memcpy(hs + (hasSugg ? suggWords : 0), aux, (size_t)auxWords * 4);
  s[1] = n; s[2] = hasSugg ? (int32_t)suggWords : 0; s[3] = hasAux ? (int32_t)auxWords : 0; s[4] = (int32_t)cap;
  const int seq = ++t->seq;
  __sync_synchronize();
  s[0] = seq;
  auto launch = [&]() {
    s[SERVE_DONE_OFF + 4] = 0;
    __sync_synchronize();
    // 1500 polls over PCIe: the kernel leaves after 1.5-2 ms without a request on an H100
    // (profiles/micro/resident_idle_timeout.py)
    hived_serve_kernel<<<1, NT, 0, t->serveStream>>>(t->slotDev, seq - 1, 1500, t->stageRes, t->dSugg, t->dAux, e.nPinnedOrder,
                                                      e.nBad, t->servePool);
    t->alive = true;
    t->launches++;
    e.kernelLaunches++;
  };
  if (!t->alive) launch();
  // wait for `done`; a kernel that left just before the request arrived is replaced
  long long spins = 0;
  while (s[SERVE_DONE_OFF] != seq) {
    if (s[SERVE_DONE_OFF + 4] && s[SERVE_DONE_OFF] != seq) {
      cudaError_t err = cudaStreamSynchronize(t->serveStream);
      if (err != cudaSuccess) { e.err = std::string("hived_serve_kernel failed: ") + cudaGetErrorString(err); t->alive = false; return HIVED_ERR_PLATFORM; }
      if (s[SERVE_DONE_OFF] == seq) break;
      launch();
    }
    if ((++spins & 0xfffff) == 0) {  // every ~million polls: is the kernel still healthy?
      cudaError_t err = cudaStreamQuery(t->serveStream);
      if (err != cudaSuccess && err != cudaErrorNotReady) {
        e.err = std::string("hived_serve_kernel failed: ") + cudaGetErrorString(err);
        t->alive = false;
        return HIVED_ERR_PLATFORM;
      }
    }
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
  __sync_synchronize();
  t->served++;
  const long long used = (long long)(uint32_t)s[SERVE_DONE_OFF + 1] | ((long long)s[SERVE_DONE_OFF + 2] << 32);
  e.poolOff = used;
  e.poolEnd.assign(1, used);
  e.lastKernelMs = 0.f;
  if (used > cap) return HIVED_ERR_CAPACITY;
  memcpy(res, (const void*)(s + SERVE_RES_OFF), (size_t)n * sizeof(hived_result_t));
  const long long got = used < SERVE_POOL_WINDOW ? used : SERVE_POOL_WINDOW;
  if (got > 0) memcpy(pool, (const void*)(s + SERVE_RES_OFF + SERVE_MAX_EVENTS * (int)(sizeof(hived_result_t) / 4)), (size_t)got * 4);
  if (used > SERVE_POOL_WINDOW)
    cudaMemcpy(pool + SERVE_POOL_WINDOW, t->servePool + SERVE_POOL_WINDOW, (size_t)(used - SERVE_POOL_WINDOW) * 4, cudaMemcpyDeviceToHost);
  return 0;
}

int bk_run_small(Engine& e, const hived_event_t* events, int n, const uint32_t* suggPool, int64_t suggWords, const int32_t* aux,
                 int64_t auxWords, hived_result_t* res, int32_t* pool, int64_t poolCap) {
  if (!e.stream) return -1;  // the first launch (initialisation) creates the stream
  std::lock_guard<std::recursive_mutex> lk(g_devMu);
  CudaTimers* t = (CudaTimers*)e.stream;
  if (int rc = ensureDevLoaded(e)) return rc;
  {
    int rc = serveCall(e, t, events, n, suggPool, suggWords, aux, auxWords, res, pool, poolCap);
    if (rc != -2) return rc;  // -2: the resident path does not take this call
  }
  static thread_local SmallStage stage;  // per host thread; the shim serialises calls per context anyway
  const bool hasSugg = suggPool != nullptr && suggWords > 0, hasAux = aux != nullptr && auxWords > 0;
  const int64_t window = poolCap < SMALL_POOL_WINDOW ? poolCap : SMALL_POOL_WINDOW;
  const size_t oEv = 0, oScal = oEv + (size_t)n * sizeof(hived_event_t), oSugg = oScal + 4 * sizeof(long long),
               oAux = oSugg + (hasSugg ? (size_t)suggWords * 4 : 0), oRes = (oAux + (hasAux ? (size_t)auxWords * 4 : 0) + 15) & ~(size_t)15,
               oPool = oRes + (size_t)n * sizeof(hived_result_t), total = oPool + (size_t)(window > 0 ? window : 1) * 4;
  if (total > stage.bytes) {
    if (stage.host) cudaFreeHost(stage.host);
    stage.host = nullptr;
    stage.bytes = 0;
    if (cudaMallocHost((void**)&stage.host, total * 2) != cudaSuccess) return -1;
    stage.bytes = total * 2;
  }
  e.notePriorities(events, n);
  e.launchCta = 1;
  e.ownOff.assign(2, 0); e.ownOff[1] = n;
  e.poolBase.assign(2, 0); e.poolBase[1] = poolCap;
  e.dEvents.ensure((size_t)n * sizeof(hived_event_t));
  e.dResults.ensure((size_t)n * sizeof(hived_result_t));
  e.dPool.ensure((size_t)(poolCap > 0 ? poolCap : 1) * 4);
  if (hasSugg) e.dSugg.ensure((size_t)suggWords * 4);
  if (hasAux) e.dAux.ensure((size_t)auxWords * 4);
  if (e.buffersFailed()) { e.err = "out of device memory while staging the call"; return HIVED_ERR_CAPACITY; }
  e.hasSugg = hasSugg; e.hasAux = hasAux;
  e.poolCapWords = poolCap; e.stagedN = n; e.stagedEvents = events; e.canonicalDone = false;
  char* h = stage.host;
  memcpy(h + oEv, events, (size_t)n * sizeof(hived_event_t));
  long long* scal = (long long*)(h + oScal);
  scal[0] = 0; scal[1] = poolCap; scal[2] = 0; scal[3] = 0;
  if (hasSugg) memcpy(h + oSugg, suggPool, (size_t)suggWords * 4);
  if (hasAux) memcpy(h + oAux, aux, (size_t)auxWords * 4);
  cudaStream_t st = t->stream;
  cudaMemcpyAsync(e.dEvents.p, h + oEv, (size_t)n * sizeof(hived_event_t), cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(e.dScalars.p, scal, 4 * sizeof(long long), cudaMemcpyHostToDevice, st);
  if (hasSugg) cudaMemcpyAsync(e.dSugg.p, h + oSugg, (size_t)suggWords * 4, cudaMemcpyHostToDevice, st);
  if (hasAux) cudaMemcpyAsync(e.dAux.p, h + oAux, (size_t)auxWords * 4, cudaMemcpyHostToDevice, st);
  cudaEventRecord(t->start, st);
  hived_events_kernel<<<1, NT, 0, st>>>((const hived_event_t*)e.dEvents.p, n, (hived_result_t*)e.dResults.p,
                                        hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, hasAux ? (const int32_t*)e.dAux.p : nullptr,
                                        nullptr, e.nPinnedOrder, e.nBad, (int32_t*)e.dPool.p, (long long*)e.dScalars.p, nullptr, nullptr);
  cudaEventRecord(t->stop, st);
  cudaMemcpyAsync(scal, e.dScalars.p, 4 * sizeof(long long), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(h + oRes, e.dResults.p, (size_t)n * sizeof(hived_result_t), cudaMemcpyDeviceToHost, st);
  if (window > 0) cudaMemcpyAsync(h + oPool, e.dPool.p, (size_t)window * 4, cudaMemcpyDeviceToHost, st);
  cudaError_t err = cudaStreamSynchronize(st);
  if (err != cudaSuccess || (err = cudaGetLastError()) != cudaSuccess) {
    e.err = std::string("hived_events_kernel failed: ") + cudaGetErrorString(err);
    return HIVED_ERR_PLATFORM;
  }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, t->start, t->stop);
  e.lastKernelMs = ms;
  e.kernelMsTotal += ms;
  e.kernelLaunches += 1;
  e.poolOff = scal[0];
  e.poolEnd.assign(1, scal[0]);
  if (e.poolOff > poolCap) return HIVED_ERR_CAPACITY;
  memcpy(res, h + oRes, (size_t)n * sizeof(hived_result_t));
  const int64_t got = e.poolOff < window ? e.poolOff : window;
  if (got > 0) memcpy(pool, h + oPool, (size_t)got * 4);
  if (e.poolOff > window) cudaMemcpy(pool + window, (int32_t*)e.dPool.p + window, (size_t)(e.poolOff - window) * 4, cudaMemcpyDeviceToHost);
  return 0;
}

// ---- pool compaction after a VC-parallel run -------------------------------------------------------------
// Every CTA appended its results' leaf triples / victim pairs to its own pool slice; the ABI promises one pool in
// event order.  Three data-parallel kernels: per-block exclusive scan of the words each result owns, scan of
// the block sums, then one warp per result gathers its words to the canonical offset and patches the result.
constexpr int SCAN_T = 256, SCAN_PER = 4, SCAN_BLOCK = SCAN_T * SCAN_PER;

__device__ __forceinline__ int resultWords(const hived_result_t& r) {
  if (r.kind == HIVED_KIND_BIND && r.n_leaves > 0) return 3 * r.n_leaves;
  if (r.kind == HIVED_KIND_PREEMPT && r.n_victims > 0) return 2 * r.n_victims;
  return 0;
}

__global__ void __launch_bounds__(SCAN_T) pool_words_kernel(const hived_result_t* __restrict__ res, int n, int32_t* __restrict__ excl,
                                                            long long* __restrict__ blockSum) {
  __shared__ int warpSum[SCAN_T / 32];
  const int base = (blockIdx.x * SCAN_T + threadIdx.x) * SCAN_PER;
  int w[SCAN_PER], mine = 0;
#pragma unroll
  for (int k = 0; k < SCAN_PER; k++) { w[k] = base + k < n ? resultWords(res[base + k]) : 0; mine += w[k]; }
  int incl = mine;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) warpSum[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int v = lane < SCAN_T / 32 ? warpSum[lane] : 0, inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane < SCAN_T / 32) warpSum[lane] = inc - v;
    if (lane == SCAN_T / 32 - 1) blockSum[blockIdx.x] = inc;
  }
  __syncthreads();
  int run = warpSum[wid] + incl - mine;
#pragma unroll
  for (int k = 0; k < SCAN_PER; k++) { if (base + k < n) excl[base + k] = run; run += w[k]; }
}

__global__ void __launch_bounds__(1024) pool_block_scan_kernel(long long* blockSum, int nb) {
  // one CTA; nb is small (n / 1024): serial carry over 1024-wide tiles
  __shared__ long long part[32];
  __shared__ long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int b0 = 0; b0 <= nb; b0 += 1024) {  // entry nb receives the grand total
    int i = b0 + threadIdx.x;
    long long v = i < nb ? blockSum[i] : 0, incl = v;
    for (int o = 1; o < 32; o <<= 1) { long long t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) part[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      long long p = part[lane], inc = p;
      for (int o = 1; o < 32; o <<= 1) { long long t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      part[lane] = inc - p;
    }
    __syncthreads();
    long long exclv = carry + part[wid] + incl - v;
    if (i <= nb) blockSum[i] = exclv;
    __syncthreads();
    if (threadIdx.x == 1023) carry = exclv + v;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) pool_gather_kernel(hived_result_t* res, int n, const int32_t* __restrict__ excl,
                                                          const long long* __restrict__ blockExcl, const int32_t* __restrict__ src,
                                                          int32_t* __restrict__ dst) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n) return;
  hived_result_t& r = res[i];
  const int words = resultWords(r);
  if (words == 0) return;
  const long long off = blockExcl[i / SCAN_BLOCK] + excl[i];
  const bool bind = r.kind == HIVED_KIND_BIND;
  const int from = bind ? r.leaf_off : r.victim_off;
  for (int k = lane; k < words; k += 32) dst[off + k] = src[from + k];
  __syncwarp();
  if (lane == 0) {
    if (bind) { r.this_off = (int32_t)(off + (r.this_off - r.leaf_off)); r.leaf_off = (int32_t)off; }
    else r.victim_off = (int32_t)off;
  }
}

int bk_canonicalise(Engine& e, int n, long long* total) {
  *total = 0;
  if (n <= 0) return 0;
  CudaTimers* t = (CudaTimers*)e.stream;
  const int nb = (n + SCAN_BLOCK - 1) / SCAN_BLOCK;
  e.dScan.ensure((size_t)n * 4 + (size_t)(nb + 2) * 8 + 16);
  long long* blockSum = (long long*)e.dScan.p;              // [nb + 1], 8-byte aligned at the front
  int32_t* excl = (int32_t*)((char*)e.dScan.p + (size_t)(nb + 2) * 8);
  e.dPool2.ensure((size_t)(e.poolCapWords > 0 ? e.poolCapWords : 1) * 4);
  if (e.buffersFailed()) { e.err = "out of device memory for the pool compaction"; return HIVED_ERR_CAPACITY; }
  pool_words_kernel<<<nb, SCAN_T, 0, t->stream>>>((const hived_result_t*)e.dResults.p, n, excl, blockSum);
  pool_block_scan_kernel<<<1, 1024, 0, t->stream>>>(blockSum, nb);
  pool_gather_kernel<<<(int)(((long long)n * 32 + 255) / 256), 256, 0, t->stream>>>((hived_result_t*)e.dResults.p, n, excl, blockSum,
                                                                              (const int32_t*)e.dPool.p, (int32_t*)e.dPool2.p);
  long long tot = 0;
  cudaMemcpyAsync(&tot, blockSum + nb, 8, cudaMemcpyDeviceToHost, t->stream);
  cudaError_t err = cudaStreamSynchronize(t->stream);
  if (err != cudaSuccess || (err = cudaGetLastError()) != cudaSuccess) {
    e.err = std::string("pool compaction failed: ") + cudaGetErrorString(err);
    return HIVED_ERR_PLATFORM;
  }
  e.kernelLaunches += 3;
  *total = tot;
  return 0;
}

}  // namespace hived

extern "C" const char* hived_backend(void) { return "cuda-sm90a"; }
