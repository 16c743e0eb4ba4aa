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
#include <unordered_set>

#define HIVED_BK_LAUNCH_MANY 1  // the joint launch below
#define HIVED_BK_CONCURRENT 1   // concurrent contexts' own resident kernels and batches below
#define HIVED_BK_COPY_CTX 1     // hived_clone's copies on the clone's stream below
#include "hived_engine.hpp"
#include "hived_many.h"
#include "hived_seats.h"

namespace hived {

constexpr int NT = 512;  // threads per CTA (16 warps); the kernel needs the full register file of one SM

// scalars: the launch words of every CTA (CtaWords)
__global__ void __launch_bounds__(NT, 1)
hived_events_kernel(const hived_event_t* __restrict__ events, int n, hived_result_t* results,
                    const uint32_t* suggPool, const int32_t* aux, const int32_t* initLists, int nPinnedOrder, int nBad,
                    int32_t* pool, long long* scalars, const int32_t* own, const int32_t* ownOff) {
  runCta(g_hived_dev, &g_hived_sm, events, n, results, suggPool, aux, initLists, nPinnedOrder, nBad, pool, (CtaWords*)scalars, own,
         ownOff, blockIdx.x, gridDim.x);
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
  serveCta(g_hived_dev, slot, seq0, idleSpins, stageRes, dSugg, dAux, nPinnedOrder, nBad, pool);
}

static bool cudaOk(cudaError_t e, std::string& err, const char* what) {
  if (e == cudaSuccess) return true;
  err = std::string(what) + ": " + cudaGetErrorString(e);
  return false;
}

// A resident per-call kernel (bk_run_small): a non-blocking stream of its own, one request slot in mapped host memory
// and the device staging of the events it runs.
struct ServeChan {
  cudaStream_t stream = nullptr;
  cudaStream_t copyStream = nullptr;     // concurrent kernels: the pool words beyond the slot's window
  volatile int32_t* slotHost = nullptr;  // cudaHostAlloc(mapped)
  int32_t* slotDev = nullptr;
  hived_result_t* stageRes = nullptr;
  uint32_t* dSugg = nullptr;
  int32_t* dAux = nullptr;
  int32_t* pool = nullptr;
  long long poolCap = 0;
  int seq = 0;
  int conc = -1;         // -1: hived_serve_kernel on g_hived_dev; else the concurrent slot its hived_serve_conc_kernel reads
  bool alive = false;    // a serve kernel was launched and has not been seen to exit
  SeatLedger* seat = nullptr;      // hived_serve_kernel: the device's ledger while the kernel holds a seat there
  SeatLedger* slotSeat = nullptr;  // concurrent kernels: the seat held from creation to destruction
  long long served = 0, launches = 0;
  std::vector<void*> retired;  // concurrent batches: cudaMalloc'd staging replaced by pooled memory, freed at destroy
};

// ---- a concurrent context's batch (bk_batch_begin .. bk_batch_end) ------------------------------------------------
// In between, the calling thread's copies, staging allocations and launches for the context go to the stream of the
// context's resident kernel (stopped first) and synchronise with that stream only.  cudaMemcpy would run on the legacy
// default stream, which waits for every blocking stream (the turn-taking contexts' streams), and cudaFree may
// synchronise the whole device, which waits until every busy concurrent context's resident kernel has gone idle.
// Staging that grows inside a batch therefore comes from the stream-ordered allocator; the cudaMalloc'd buffer it
// replaces is kept until the context is destroyed.
static thread_local ServeChan* t_own = nullptr;
static std::mutex g_pooledMu;
static std::unordered_set<void*> g_pooled;  // every live cudaMallocAsync block of bk_alloc

void* bk_alloc(size_t bytes) {
  void* p = nullptr;
  if (t_own) {
    if (cudaMallocAsync(&p, bytes ? bytes : 1, t_own->stream) != cudaSuccess) return nullptr;
    std::lock_guard<std::mutex> lk(g_pooledMu);
    g_pooled.insert(p);
    return p;
  }
  if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  return p;
}
void bk_free(void* p) {
  if (!p) return;
  bool pooled;
  {
    std::lock_guard<std::mutex> lk(g_pooledMu);
    pooled = g_pooled.erase(p) > 0;
  }
  if (pooled && t_own) cudaFreeAsync(p, t_own->stream);
  else if (t_own) t_own->retired.push_back(p);
  else cudaFree(p);  // (for a pooled block: no implicit synchronisation; the context's last batch was synchronised)
}
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
static void copy(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind) {
  if (!bytes) return;
  if (!t_own) { noteCopy(cudaMemcpy(dst, src, bytes, kind)); return; }
  cudaError_t ce = cudaMemcpyAsync(dst, src, bytes, kind, t_own->stream);
  noteCopy(ce == cudaSuccess ? cudaStreamSynchronize(t_own->stream) : ce);
}
void bk_h2d(void* dst, const void* src, size_t bytes) { copy(dst, src, bytes, cudaMemcpyHostToDevice); }
void bk_d2h(void* dst, const void* src, size_t bytes) { copy(dst, src, bytes, cudaMemcpyDeviceToHost); }
void bk_d2d(void* dst, const void* src, size_t bytes) { copy(dst, src, bytes, cudaMemcpyDeviceToDevice); }
void bk_zero(void* dst, size_t bytes) {
  if (!bytes) return;
  if (!t_own) { noteCopy(cudaMemset(dst, 0, bytes)); return; }
  cudaError_t ce = cudaMemsetAsync(dst, 0, bytes, t_own->stream);
  noteCopy(ce == cudaSuccess ? cudaStreamSynchronize(t_own->stream) : ce);
}

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
  ServeChan serve;       // the resident kernel of the turn-taking path (g_hived_dev)
  bool disabled = false; // HIVED_NO_RESIDENT=1, or setting it up failed: one launch per call
  ServeChan* conc = nullptr;  // a concurrent context's own resident kernel (bk_open_concurrent); nullptr otherwise
};

static bool noResident() {
  const char* off = getenv("HIVED_NO_RESIDENT");
  return off && *off && *off != '0';
}

// ---- co-residency seats (hived_seats.h): one ledger per device, as many seats as CTAs of the program fit on it --------
static SeatLedger g_seats[64];
static SeatLedger& seatsOf(const Engine& e) {  // the context's device is current
  const int dv = e.deviceOrdinal >= 0 && e.deviceOrdinal < 64 ? e.deviceOrdinal : 0;
  const int fit = manyCoResident(e.deviceOrdinal);
  if (fit > 0) g_seats[dv].setCapacity(fit);  // (unset while it cannot be queried: every request is refused)
  return g_seats[dv];
}
static int seatError(Engine& e, int n) {
  char buf[160];
  snprintf(buf, sizeof buf, "cannot hold %d co-resident CTAs: the device fits %d (occupancy x SMs)", n, seatsOf(e).capacity());
  e.err = buf;
  return HIVED_ERR_PLATFORM;
}

// A resident kernel was seen to exit (or cannot be waited for any more): its seat, if it holds one, is free again.
static void serveLeft(ServeChan& c) {
  c.alive = false;
  if (c.seat) c.seat->release(1);
  c.seat = nullptr;
}

// Stop a resident kernel (if any) and wait until it has left.
static void serveStop(ServeChan& c) {
  if (!c.alive) return;
  volatile int32_t* s = c.slotHost;
  if (!s[SERVE_DONE_EXITED]) {
    s[SERVE_N] = 0;  // STOP
    __sync_synchronize();
    s[SERVE_SEQ] = ++c.seq;
  }
  cudaStreamSynchronize(c.stream);
  serveLeft(c);
}

// ---- whose Dev is in the constant bank (g_hived_dev, hived_core.h) of each device ---------------------------------
// One context per device at a time.  Every section that launches a kernel or talks to a resident one holds g_devMu
// (contexts of one process take turns on the GPU; a context by itself is single-threaded per the ABI), makes sure its
// own Dev is the one loaded, and leaves nothing of its own running except the resident per-call kernel — which the
// next owner stops before it overwrites the constant bank.  A concurrent context's own resident kernel
// (HIVED_OPT_CONCURRENT, below) reads another constant slot and is never stopped from here: only its own caller stops
// it (bk_quiesce), since another thread's stop would race with that caller's call in flight.
static std::recursive_mutex g_devMu;
static Engine* g_devOwner[64] = {nullptr};

// g_devMu held on behalf of the listed contexts: each one's turn counter (hived_bench_turns) counts the outermost hold
static thread_local int t_turnDepth = 0;
struct Turn {
  std::lock_guard<std::recursive_mutex> lk;
  Turn(Engine* const* es, int k) : lk(g_devMu) {
    if (t_turnDepth++ == 0)
      for (int y = 0; y < k; y++) es[y]->turns++;
  }
  explicit Turn(Engine& e) : lk(g_devMu) { if (t_turnDepth++ == 0) e.turns++; }
  ~Turn() { t_turnDepth--; }
};

static int ensureDevLoaded(Engine& e) {  // g_devMu held, the context's device current
  const int dv = e.deviceOrdinal >= 0 && e.deviceOrdinal < 64 ? e.deviceOrdinal : 0;
  if (g_devOwner[dv] == &e) return 0;
  if (g_devOwner[dv]) serveStop(((CudaTimers*)g_devOwner[dv]->stream)->serve);
  g_devOwner[dv] = nullptr;
  cudaError_t ce = cudaMemcpyToSymbol(g_hived_dev, &e.dev, sizeof(Dev));  // synchronous: nothing of ours is running
  if (ce != cudaSuccess) { e.err = std::string("cudaMemcpyToSymbol(g_hived_dev): ") + cudaGetErrorString(ce); return HIVED_ERR_PLATFORM; }
  g_devOwner[dv] = &e;
  return 0;
}
static void concClose(Engine& e);
void bk_forget(Engine& e) {  // the context is going away
  {
    Turn turn(e);
    for (auto& o : g_devOwner) if (o == &e) o = nullptr;
  }
  concClose(e);
}

// Stop the context's resident kernels (if any) and wait until they have left: before anything else launches on or
// writes to the scheduler state.  Called by the context's own caller, with the context's device current.
void bk_quiesce(Engine& e) {
  Turn turn(e);
  CudaTimers* t = (CudaTimers*)e.stream;
  if (!t) return;
  serveStop(t->serve);
  if (t->conc) serveStop(*t->conc);
}

// ---- concurrent contexts (HIVED_OPT_CONCURRENT) --------------------------------------------------------------------
// Each holds one of the device's HIVED_CONCURRENT_MAX slots from hived_create to hived_destroy: its Dev sits in constant
// slot s of the concurrent build (hived_cuda_conc.cu), copied once, and its per-call path runs on a resident kernel of
// its own (hived_serve_conc_kernel) through a request slot of its own, without g_devMu.
// Invariant: a slot's Dev is written only while no kernel that reads that slot runs (the slot is free: the previous
// holder's kernel was stopped before it gave the slot back), and the kernel that reads it is launched after the write
// has completed.  Writes to other slots — another context's creation, a joint launch's slots 0..k-1 — may happen while
// resident kernels run.  Taking a slot happens under g_devMu: a g_devMu holder that budgets for the slots in use (the
// joint launch's rounds) sees no new one appear before it has launched.  Each slot with a resident kernel holds one
// seat of the device's ledger from creation to destruction.
static std::mutex g_concMu;
static Engine* g_concSlot[64][HIVED_CONCURRENT_MAX] = {};

// Resident CTAs of concurrent kernels that may be live on the device at any moment (one per slot taken, whether its
// kernel runs now or not: another thread may launch it at any time).
static int concInUse(int dv) {
  std::lock_guard<std::mutex> lk(g_concMu);
  int n = 0;
  for (Engine* o : g_concSlot[dv]) n += o != nullptr;
  return n;
}

// Device staging of a resident kernel's channel; false if something could not be allocated.
static bool serveAlloc(const Engine& e, ServeChan& c) {
  void* h = nullptr;
  if (cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaHostAlloc(&h, (size_t)SERVE_SLOT_WORDS * 4, cudaHostAllocMapped) != cudaSuccess) return false;
  memset(h, 0, (size_t)SERVE_SLOT_WORDS * 4);
  c.slotHost = (volatile int32_t*)h;
  void* d = nullptr;
  if (cudaHostGetDevicePointer(&d, h, 0) != cudaSuccess) return false;
  c.slotDev = (int32_t*)d;
  c.poolCap = 3ll * e.dev.S.LS + 2 * 4096 + 64 > SERVE_POOL_WINDOW ? 3ll * e.dev.S.LS + 2 * 4096 + 64 : SERVE_POOL_WINDOW;
  c.poolCap *= SERVE_MAX_EVENTS;
  return cudaMalloc((void**)&c.stageRes, sizeof(hived_result_t) * SERVE_MAX_EVENTS) == cudaSuccess &&
         cudaMalloc((void**)&c.dSugg, (size_t)SERVE_SUGG_MAX * 4) == cudaSuccess &&
         cudaMalloc((void**)&c.dAux, (size_t)SERVE_AUX_MAX * 4) == cudaSuccess &&
         cudaMalloc((void**)&c.pool, (size_t)c.poolCap * 4) == cudaSuccess;
}

static void serveFree(ServeChan& c) {  // the kernel has left
  cudaFree(c.stageRes); cudaFree(c.dSugg); cudaFree(c.dAux); cudaFree(c.pool);
  for (void* p : c.retired) cudaFree(p);
  if (c.slotHost) cudaFreeHost((void*)c.slotHost);
  if (c.copyStream) cudaStreamDestroy(c.copyStream);
  if (c.stream) cudaStreamDestroy(c.stream);
}

// The largest cooperative grid of one context (launchProgram: one CTA per VC, at most 16).  A device keeps this many
// co-resident CTAs free of concurrent kernels, so that such a grid always fits beside them.
constexpr int COOP_CTAS_MAX = 16;

int bk_open_concurrent(Engine& e) {  // the end of hived_create: the device is current
  const int dv = e.deviceOrdinal >= 0 && e.deviceOrdinal < 64 ? e.deviceOrdinal : 0;
  const int fit = manyCoResident(e.deviceOrdinal);
  const int cap = fit - COOP_CTAS_MAX < HIVED_CONCURRENT_MAX ? fit - COOP_CTAS_MAX : HIVED_CONCURRENT_MAX;
  Turn turn(e);
  int slot = -1;
  {
    std::lock_guard<std::mutex> lk(g_concMu);
    int used = 0;
    for (int s = 0; s < HIVED_CONCURRENT_MAX; s++) {
      if (g_concSlot[dv][s]) used++;
      else if (slot < 0) slot = s;
    }
    if (used >= cap) {
      char buf[200];
      snprintf(buf, sizeof buf, "HIVED_OPT_CONCURRENT: all %d concurrent-context slots of device %d are taken "
               "(HIVED_CONCURRENT_MAX per device)", cap > 0 ? cap : 0, dv);
      e.err = buf;
      return HIVED_ERR_CAPACITY;
    }
    g_concSlot[dv][slot] = &e;
  }
  if (noResident()) return 0;  // the slot is held, but every call takes turns
  CudaTimers* t = (CudaTimers*)e.stream;
  ServeChan* c = new ServeChan();
  c->conc = slot;
  t->conc = c;
  if (!seatsOf(e).acquire(1)) return seatError(e, 1);
  c->slotSeat = &seatsOf(e);
  if (!serveAlloc(e, *c) || cudaStreamCreateWithFlags(&c->copyStream, cudaStreamNonBlocking) != cudaSuccess) {
    e.err = "out of device or pinned host memory for the concurrent context's resident kernel";
    return HIVED_ERR_CAPACITY;
  }
  cudaError_t ce = concLoadDev(e.dev, slot, c->stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(c->stream);
  if (ce != cudaSuccess) { e.err = std::string("copying the Dev into its concurrent slot: ") + cudaGetErrorString(ce); return HIVED_ERR_PLATFORM; }
  return 0;
}

static void concClose(Engine& e) {  // bk_quiesce has stopped the kernel
  CudaTimers* t = (CudaTimers*)e.stream;
  if (t && t->conc) {
    serveFree(*t->conc);
    if (t->conc->slotSeat) t->conc->slotSeat->release(1);
    delete t->conc;
    t->conc = nullptr;
  }
  std::lock_guard<std::mutex> lk(g_concMu);
  for (auto& dev : g_concSlot)
    for (Engine*& o : dev) if (o == &e) o = nullptr;
}

static_assert(NT / 32 <= MAX_WARPS, "the shared counters are sized for MAX_WARPS warps per CTA");

static int concLaunch(Engine& e, ServeChan& c, int n);

// The end of a launch queued on `st` for the contexts es[0..k) (its words' copy-back queued after t's stop event): wait
// for it, then every context's kernel time.  HIVED_ERR_PLATFORM with every context's err naming `kernel` if it failed.
static int launchDone(Engine* const* es, int k, CudaTimers* t, cudaStream_t st, const char* kernel) {
  cudaError_t err = cudaStreamSynchronize(st);
  if (err != cudaSuccess || (err = cudaGetLastError()) != cudaSuccess) {
    for (int y = 0; y < k; y++) es[y]->err = std::string(kernel) + " failed: " + cudaGetErrorString(err);
    return HIVED_ERR_PLATFORM;
  }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, t->start, t->stop);
  for (int y = 0; y < k; y++) {
    es[y]->lastKernelMs = ms;
    es[y]->kernelMsTotal += ms;
  }
  return 0;
}

// The context's stream and timing events, made by its first launch (or, for a clone, its first copy) with its device
// current; nullptr with e.err set if the stream cannot be created.
static CudaTimers* timersOf(Engine& e) {
  if (!e.stream) {
    // the kernel wants L1, not shared memory: ask for the smallest carveout that holds its ~18 KB of static smem
    cudaFuncSetAttribute(hived_events_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
    CudaTimers* t = new CudaTimers();
    if (!cudaOk(cudaStreamCreate(&t->stream), e.err, "cudaStreamCreate")) return nullptr;
    cudaEventCreate(&t->start);
    cudaEventCreate(&t->stop);
    e.stream = t;
  }
  return (CudaTimers*)e.stream;
}

int launchProgram(Engine& e, int n, bool withInit) {
  // a concurrent context's batch: its own stream, constant slot and seats, no turn
  if (t_own && e.stream && t_own == ((CudaTimers*)e.stream)->conc && !withInit && !e.mgMode) return concLaunch(e, *t_own, n);
  Turn turn(e);
  CudaTimers* t = timersOf(e);
  if (!t) return HIVED_ERR_NO_DEVICE;
  bk_quiesce(e);
  if (int rc = takeCopyError(e.err)) return rc;  // a staging copy of this batch (or of create()) failed
  if (int rc = ensureDevLoaded(e)) return rc;
  const int mgMode = withInit ? 0 : e.mgMode;
  const int C = withInit ? 1 : (mgMode == 3 ? 1 : e.launchCta);
  SeatHold seats(seatsOf(e), C);  // until the stream synchronise below has seen the kernels finish
  if (!seats.ok()) return seatError(e, C);
  if (mgMode == 3) {  // end of a multi-GPU partition run: the repair pass alone
    hived_repair_kernel<<<1, NT, 0, t->stream>>>();
    cudaError_t err = cudaStreamSynchronize(t->stream);
    if (err != cudaSuccess) { e.err = std::string("hived_repair_kernel failed: ") + cudaGetErrorString(err); return HIVED_ERR_PLATFORM; }
    e.kernelLaunches++;
    return 0;
  }
  CtaWords w[MAX_CTAS] = {};
  e.packCtaWords(w, C, withInit);
  cudaMemcpyAsync(e.dScalars.p, w, sizeof w, cudaMemcpyHostToDevice, t->stream);
  cudaEventRecord(t->start, t->stream);
  const hived_event_t* events = (const hived_event_t*)e.dEvents.p;
  hived_result_t* results = (hived_result_t*)e.dResults.p;
  const uint32_t* sugg = e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr;
  const int32_t* aux = e.hasAux ? (const int32_t*)e.dAux.p : nullptr;
  const int32_t* init = withInit ? (const int32_t*)e.dInit.p : nullptr;
  int32_t* pool = (int32_t*)e.dPool.p;
  long long* scalars = (long long*)e.dScalars.p;
  const int32_t* own = (C > 1 || mgMode) ? (const int32_t*)e.dOwn.p : nullptr;
  const int32_t* ownOff = own ? own + n : nullptr;
  const bool parallel = C > 1 && !mgMode;
  if (parallel) {
    // The CTAs of a VC-parallel batch wait for each other (ordered shared sections): launch them cooperatively, so
    // that the runtime guarantees that all of them are resident at the same time.
    void* args[] = {&events, &n, &results, &sugg, &aux, &init, &e.nPinnedOrder, &e.nBad, &pool, &scalars, &own, &ownOff};
    cudaError_t le = cudaLaunchCooperativeKernel((const void*)hived_events_kernel, dim3(C), dim3(NT), args, 0, t->stream);
    if (le != cudaSuccess) {
      e.err = std::string("cooperative launch of hived_events_kernel failed: ") + cudaGetErrorString(le);
      return HIVED_ERR_PLATFORM;
    }
    hived_repair_kernel<<<1, NT, 0, t->stream>>>();
  } else {
    hived_events_kernel<<<C, NT, 0, t->stream>>>(events, n, results, sugg, aux, init, e.nPinnedOrder, e.nBad, pool, scalars, own, ownOff);
  }
  cudaEventRecord(t->stop, t->stream);
  cudaMemcpyAsync(w, e.dScalars.p, sizeof w, cudaMemcpyDeviceToHost, t->stream);
  Engine* es[] = {&e};
  if (int rc = launchDone(es, 1, t, t->stream, "hived_events_kernel")) return rc;
  if (int rc = e.takeCtaWords(w, C, withInit, parallel ? 2 : 1)) { e.err = "initialisation panicked on the device"; return rc; }
  return 0;
}

// A concurrent context's staged batch (bk_batch_begin): the concurrent build's events kernel on the context's constant slot,
// one CTA per VC group, on the context's own stream.  No g_devMu, no g_hived_dev; the seats of its CTAs are held until
// the stream synchronise has seen the kernels finish.
static int concLaunch(Engine& e, ServeChan& c, int n) {
  CudaTimers* t = (CudaTimers*)e.stream;
  if (int rc = takeCopyError(e.err)) return rc;  // a staging copy of this batch failed
  const int C = e.launchCta;
  CtaWords w[MAX_CTAS] = {};
  e.packCtaWords(w, C, false);
  const ManySlot q{(const hived_event_t*)e.dEvents.p, (hived_result_t*)e.dResults.p,
                   e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, (int32_t*)e.dPool.p, (CtaWords*)e.dScalars.p,
                   C > 1 ? (const int32_t*)e.dOwn.p : nullptr, n, C, e.nPinnedOrder, e.nBad};
  SeatHold seats(seatsOf(e), C);
  if (!seats.ok()) return seatError(e, C);
  cudaMemcpyAsync(e.dScalars.p, w, sizeof w, cudaMemcpyHostToDevice, c.stream);
  cudaEventRecord(t->start, c.stream);
  cudaError_t err = concBatchLaunch(c.conc, q, c.stream);
  if (err != cudaSuccess) {
    cudaStreamSynchronize(c.stream);
    cudaGetLastError();
    e.err = std::string("launching hived_events_conc_kernel failed: ") + cudaGetErrorString(err);
    return HIVED_ERR_PLATFORM;
  }
  cudaEventRecord(t->stop, c.stream);
  cudaMemcpyAsync(w, e.dScalars.p, sizeof w, cudaMemcpyDeviceToHost, c.stream);
  Engine* es[] = {&e};
  if (int rc = launchDone(es, 1, t, c.stream, "hived_events_conc_kernel")) return rc;
  e.takeCtaWords(w, C, false, C > 1 ? 2 : 1);
  return 0;
}

bool bk_batch_begin(Engine& e) {
  CudaTimers* t = (CudaTimers*)e.stream;
  if (!t || !t->conc) return false;  // an ordinary context, or HIVED_NO_RESIDENT=1: the batch takes turns
  serveStop(*t->conc);               // only the context's own caller stops its kernel
  t_own = t->conc;
  return true;
}
void bk_batch_end(Engine&) { t_own = nullptr; }

// ---- hived_clone (include/hived_clone.h) ---------------------------------------------------------------------------
// The copies are queued on the clone's stream (copy engines; a peer copy when the clone lives on another device, which
// needs no peer access) and waited for once.  Ordering with the source: the caller holds `src`, so none of its calls is
// in flight.  Each of them ended either in a synchronisation of the stream that ran it (batches, joint launches, the
// per-call path without a resident kernel) or with the host observing the `done` word of a resident kernel, which the
// kernel stores after flushing its counters and __threadfence_system(): either way every write of src's last call is
// complete and visible to the copy engines.  A resident kernel of src that is still waiting for its next call writes
// no device state until it gets one, so it is left running, and src is not touched.  No turn: the copies run on the
// clone's own stream and read memory no other context writes.
int bk_copy_ctx(Engine& dst, const Engine& src, void* const* to, const void* const* from, const size_t* bytes, int n) {
  CudaTimers* t = timersOf(dst);  // dst's device is current (bk_init)
  if (!t) return HIVED_ERR_NO_DEVICE;
  if (int rc = takeCopyError(dst.err)) return rc;  // an upload of the static arrays failed
  cudaError_t ce = cudaSuccess;
  for (int i = 0; i < n && ce == cudaSuccess; i++) {
    if (!bytes[i]) continue;
    ce = dst.deviceOrdinal == src.deviceOrdinal
             ? cudaMemcpyAsync(to[i], from[i], bytes[i], cudaMemcpyDeviceToDevice, t->stream)
             : cudaMemcpyPeerAsync(to[i], dst.deviceOrdinal, from[i], src.deviceOrdinal, bytes[i], t->stream);
  }
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(t->stream);
  if (ce != cudaSuccess) {
    cudaGetLastError();
    dst.err = std::string("copying the source context's state failed: ") + cudaGetErrorString(ce);
    return HIVED_ERR_PLATFORM;
  }
  return 0;
}

// ---- joint launches (include/hived_multictx.h, hived_cuda_many.cu) ------------------------------------------------
// The staged batches of several contexts of one device run in one launch, each context on CTAs of its own, on the first
// context's stream.  g_hived_dev and its owner are not touched; but every resident per-call kernel of the device is
// stopped first — the participants' (they would write the same state) and the owner's (it holds an SM the joint launch
// may need to have all its CTAs resident).  Contexts whose CTAs do not fit on the device together go to further
// launches (rounds), greedily in list order.
int bk_launch_many(Engine* const* es, int k) {
  Turn turn(es, k);
  Engine& e0 = *es[0];
  const int dv = e0.deviceOrdinal >= 0 && e0.deviceOrdinal < 64 ? e0.deviceOrdinal : 0;
  for (int y = 0; y < k; y++) bk_quiesce(*es[y]);
  if (g_devOwner[dv]) serveStop(((CudaTimers*)g_devOwner[dv]->stream)->serve);
  auto fail = [&](const std::string& why) {
    for (int y = 0; y < k; y++) es[y]->err = why;
    return HIVED_ERR_PLATFORM;
  };
  std::string err;
  if (takeCopyError(err)) return fail(err);  // a staging copy of one of the batches failed
  // the concurrent contexts' resident CTAs may come and go during the launch (other threads): leave them one SM each
  const int fit = manyCoResident(e0.deviceOrdinal) - concInUse(dv);
  if (fit <= 0) return fail("joint launch: cannot query the co-resident CTA limit");
  CudaTimers* t = (CudaTimers*)e0.stream;
  std::vector<CtaWords> words((size_t)k * MAX_CTAS);
  ManyArgs a;
  const Dev* devs[HIVED_MANY_MAX];
  for (int y = 0; y < k; y++) {
    Engine& e = *es[y];
    const int C = e.launchCta;
    CtaWords* w = &words[(size_t)y * MAX_CTAS];
    e.packCtaWords(w, C, false);
    cudaMemcpyAsync(e.dScalars.p, w, MAX_CTAS * sizeof(CtaWords), cudaMemcpyHostToDevice, t->stream);
    a.slot[y] = ManySlot{(const hived_event_t*)e.dEvents.p, (hived_result_t*)e.dResults.p,
                         e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, (int32_t*)e.dPool.p, (CtaWords*)e.dScalars.p,
                         C > 1 ? (const int32_t*)e.dOwn.p : nullptr, e.stagedN, C, e.nPinnedOrder, e.nBad};
    devs[y] = &e.dev;
  }
  // rounds: the longest prefix of the rest whose (widest C) x (count) fits; they run one after another on one stream,
  // so the seats of the largest round cover them all
  int ends[HIVED_MANY_MAX], nRounds = 0, seatsNeeded = 0;
  for (int y0 = 0; y0 < k;) {
    int y1 = y0 + 1, cmax = a.slot[y0].C;
    while (y1 < k) {
      const int c = a.slot[y1].C > cmax ? a.slot[y1].C : cmax;
      if ((long long)c * (y1 - y0 + 1) > fit) break;
      cmax = c;
      y1++;
    }
    if (cmax * (y1 - y0) > seatsNeeded) seatsNeeded = cmax * (y1 - y0);
    ends[nRounds++] = y1;
    y0 = y1;
  }
  SeatHold seats(seatsOf(e0), seatsNeeded);  // until the stream synchronise below has seen the last round finish
  if (!seats.ok()) { seatError(e0, seatsNeeded); return fail(e0.err); }
  cudaEventRecord(t->start, t->stream);
  for (int i = 0, y0 = 0; i < nRounds; y0 = ends[i++]) {
    const int y1 = ends[i];
    ManyArgs r;
    for (int y = y0; y < y1; y++) r.slot[y - y0] = a.slot[y];
    cudaError_t le = manyLaunch(devs + y0, r, y1 - y0, t->stream);
    if (le != cudaSuccess) { cudaStreamSynchronize(t->stream); cudaGetLastError(); return fail(std::string("joint launch failed: ") + cudaGetErrorString(le)); }
  }
  cudaEventRecord(t->stop, t->stream);
  for (int y = 0; y < k; y++)
    cudaMemcpyAsync(&words[(size_t)y * MAX_CTAS], es[y]->dScalars.p, MAX_CTAS * sizeof(CtaWords), cudaMemcpyDeviceToHost, t->stream);
  if (int rc = launchDone(es, k, t, t->stream, "hived_events_many_kernel")) return rc;
  for (int y = 0; y < k; y++) es[y]->takeCtaWords(&words[(size_t)y * MAX_CTAS], es[y]->launchCta, false, es[y]->launchCta > 1 ? 2 : 1);
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
  if (t->serve.slotHost) return true;
  if (noResident() || !serveAlloc(e, t->serve)) { t->disabled = true; return false; }
  cudaFuncSetAttribute(hived_serve_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 10);
  return true;
}

// what the resident kernel's request slot holds
static bool serveTakes(int n, const uint32_t* suggPool, int64_t suggWords, const int32_t* aux, int64_t auxWords) {
  const bool hasSugg = suggPool != nullptr && suggWords > 0, hasAux = aux != nullptr && auxWords > 0;
  return n <= SERVE_MAX_EVENTS && !(hasSugg && suggWords > SERVE_SUGG_MAX) && !(hasAux && auxWords > SERVE_AUX_MAX);
}

// One call through a resident kernel's channel (serveTakes holds, the channel is set up).
static int serveCall(Engine& e, ServeChan& c, const hived_event_t* events, int n, const uint32_t* suggPool, int64_t suggWords,
                     const int32_t* aux, int64_t auxWords, hived_result_t* res, int32_t* pool, int64_t poolCap) {
  const bool hasSugg = suggPool != nullptr && suggWords > 0, hasAux = aux != nullptr && auxWords > 0;
  const long long cap = poolCap < c.poolCap ? poolCap : c.poolCap;
  e.notePriorities(events, n);
  e.setStaged(events, n, poolCap, hasSugg, hasAux);
  volatile int32_t* s = c.slotHost;
  int32_t* pay = (int32_t*)(s + SERVE_EV_OFF);
  memcpy(pay, events, (size_t)n * sizeof(hived_event_t));
  int32_t* hs = pay + SERVE_MAX_EVENTS * (int)(sizeof(hived_event_t) / 4);
  if (hasSugg) memcpy(hs, suggPool, (size_t)suggWords * 4);
  if (hasAux) memcpy(hs + (hasSugg ? suggWords : 0), aux, (size_t)auxWords * 4);
  s[SERVE_N] = n;
  s[SERVE_SUGG_WORDS] = hasSugg ? (int32_t)suggWords : 0;
  s[SERVE_AUX_WORDS] = hasAux ? (int32_t)auxWords : 0;
  s[SERVE_POOL_CAP] = (int32_t)cap;
  const int seq = ++c.seq;
  __sync_synchronize();
  s[SERVE_SEQ] = seq;
  auto launch = [&]() {
    s[SERVE_DONE_EXITED] = 0;
    __sync_synchronize();
    // 1500 polls over PCIe: the kernel leaves after 1.5-2 ms without a request on an H100
    // (profiles/micro/resident_idle_timeout.py)
    cudaError_t le = cudaSuccess;
    if (c.conc < 0) {
      // it stays resident after g_devMu is released: it holds a seat until it is seen to leave (serveLeft)
      if (!c.seat) {
        if (!seatsOf(e).acquire(1)) { seatError(e, 1); return false; }
        c.seat = &seatsOf(e);
      }
      hived_serve_kernel<<<1, NT, 0, c.stream>>>(c.slotDev, seq - 1, 1500, c.stageRes, c.dSugg, c.dAux, e.nPinnedOrder, e.nBad,
                                                 c.pool);
    } else
      le = concServeLaunch(c.conc, c.slotDev, seq - 1, 1500, c.stageRes, c.dSugg, c.dAux, e.nPinnedOrder, e.nBad, c.pool, c.stream);
    if (le != cudaSuccess) { e.err = std::string("launching hived_serve_conc_kernel failed: ") + cudaGetErrorString(le); return false; }
    c.alive = true;
    c.launches++;
    e.kernelLaunches++;
    return true;
  };
  if (!c.alive && !launch()) { serveLeft(c); return HIVED_ERR_PLATFORM; }
  // wait for `done`; a kernel that left just before the request arrived is replaced
  long long spins = 0;
  while (s[SERVE_DONE_SEQ] != seq) {
    if (s[SERVE_DONE_EXITED] && s[SERVE_DONE_SEQ] != seq) {
      cudaError_t err = cudaStreamSynchronize(c.stream);
      if (err != cudaSuccess) { e.err = std::string("hived_serve_kernel failed: ") + cudaGetErrorString(err); serveLeft(c); return HIVED_ERR_PLATFORM; }
      if (s[SERVE_DONE_SEQ] == seq) break;
      if (!launch()) { serveLeft(c); return HIVED_ERR_PLATFORM; }
    }
    if ((++spins & 0xfffff) == 0) {  // every ~million polls: is the kernel still healthy?
      cudaError_t err = cudaStreamQuery(c.stream);
      if (err != cudaSuccess && err != cudaErrorNotReady) {
        e.err = std::string("hived_serve_kernel failed: ") + cudaGetErrorString(err);
        serveLeft(c);
        return HIVED_ERR_PLATFORM;
      }
    }
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
  __sync_synchronize();
  c.served++;
  const long long used = (long long)(uint32_t)s[SERVE_DONE_POOL_LO] | ((long long)s[SERVE_DONE_POOL_HI] << 32);
  e.poolOff = used;
  e.poolEnd.assign(1, used);
  e.lastKernelMs = 0.f;
  if (used > cap) return HIVED_ERR_CAPACITY;
  memcpy(res, (const void*)(s + SERVE_RES_OFF), (size_t)n * sizeof(hived_result_t));
  const long long got = used < SERVE_POOL_WINDOW ? used : SERVE_POOL_WINDOW;
  if (got > 0) memcpy(pool, (const void*)(s + SERVE_RES_OFF + SERVE_MAX_EVENTS * (int)(sizeof(hived_result_t) / 4)), (size_t)got * 4);
  if (used > SERVE_POOL_WINDOW) {
    int32_t* dst = pool + SERVE_POOL_WINDOW;
    const int32_t* src = c.pool + SERVE_POOL_WINDOW;
    const size_t bytes = (size_t)(used - SERVE_POOL_WINDOW) * 4;
    if (c.conc < 0) {
      cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost);
    } else {  // a concurrent context synchronises with nothing but its own copy stream
      cudaError_t ce = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c.copyStream);
      if (ce == cudaSuccess) ce = cudaStreamSynchronize(c.copyStream);
      if (ce != cudaSuccess) { e.err = std::string("copying the pool words beyond the window: ") + cudaGetErrorString(ce); return HIVED_ERR_PLATFORM; }
    }
  }
  return 0;
}

int bk_run_small(Engine& e, const hived_event_t* events, int n, const uint32_t* suggPool, int64_t suggWords, const int32_t* aux,
                 int64_t auxWords, hived_result_t* res, int32_t* pool, int64_t poolCap) {
  if (!e.stream) return -1;  // the first launch (initialisation) creates the stream
  CudaTimers* t = (CudaTimers*)e.stream;
  const bool takes = serveTakes(n, suggPool, suggWords, aux, auxWords);
  // a concurrent context: its own resident kernel and constant slot, no g_devMu, no turn on g_hived_dev.  A call its
  // kernel does not take runs as a batch of its own (bk_batch_begin), except one with aux words (bind info over
  // SERVE_AUX_MAX, only ever a single hived_add_allocated_pod): the concurrent build's events kernel takes the joint
  // launch's ManySlot, which carries none, so that one takes turns.
  const bool hasAux = aux != nullptr && auxWords > 0;
  if (t->conc && takes) return serveCall(e, *t->conc, events, n, suggPool, suggWords, aux, auxWords, res, pool, poolCap);
  if (t->conc && !hasAux) return -1;
  Turn turn(e);
  if (t->conc) serveStop(*t->conc);  // the launch below writes the same state
  if (int rc = ensureDevLoaded(e)) return rc;
  if (!t->conc && takes && serveSetup(e, t))
    return serveCall(e, t->serve, events, n, suggPool, suggWords, aux, auxWords, res, pool, poolCap);
  static thread_local SmallStage stage;  // per host thread; the shim serialises calls per context anyway
  const bool hasSugg = suggPool != nullptr && suggWords > 0;
  const int64_t window = poolCap < SMALL_POOL_WINDOW ? poolCap : SMALL_POOL_WINDOW;
  const size_t oEv = 0, oScal = oEv + (size_t)n * sizeof(hived_event_t), oSugg = oScal + sizeof(CtaWords),
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
  e.setStaged(events, n, poolCap, hasSugg, hasAux);
  e.dEvents.ensure((size_t)n * sizeof(hived_event_t));
  e.dResults.ensure((size_t)n * sizeof(hived_result_t));
  e.dPool.ensure((size_t)(poolCap > 0 ? poolCap : 1) * 4);
  if (hasSugg) e.dSugg.ensure((size_t)suggWords * 4);
  if (hasAux) e.dAux.ensure((size_t)auxWords * 4);
  if (e.buffersFailed()) { e.err = "out of device memory while staging the call"; return HIVED_ERR_CAPACITY; }
  char* h = stage.host;
  memcpy(h + oEv, events, (size_t)n * sizeof(hived_event_t));
  CtaWords* w = (CtaWords*)(h + oScal);
  e.packCtaWords(w, 1, false);
  w->calm = 0;  // (prepare() did not judge these events: they take the general loop)
  if (hasSugg) memcpy(h + oSugg, suggPool, (size_t)suggWords * 4);
  if (hasAux) memcpy(h + oAux, aux, (size_t)auxWords * 4);
  cudaStream_t st = t->stream;
  cudaMemcpyAsync(e.dEvents.p, h + oEv, (size_t)n * sizeof(hived_event_t), cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(e.dScalars.p, w, sizeof(CtaWords), cudaMemcpyHostToDevice, st);
  if (hasSugg) cudaMemcpyAsync(e.dSugg.p, h + oSugg, (size_t)suggWords * 4, cudaMemcpyHostToDevice, st);
  if (hasAux) cudaMemcpyAsync(e.dAux.p, h + oAux, (size_t)auxWords * 4, cudaMemcpyHostToDevice, st);
  cudaEventRecord(t->start, st);
  hived_events_kernel<<<1, NT, 0, st>>>((const hived_event_t*)e.dEvents.p, n, (hived_result_t*)e.dResults.p,
                                        hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, hasAux ? (const int32_t*)e.dAux.p : nullptr,
                                        nullptr, e.nPinnedOrder, e.nBad, (int32_t*)e.dPool.p, (long long*)e.dScalars.p, nullptr, nullptr);
  cudaEventRecord(t->stop, st);
  cudaMemcpyAsync(w, e.dScalars.p, sizeof(CtaWords), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(h + oRes, e.dResults.p, (size_t)n * sizeof(hived_result_t), cudaMemcpyDeviceToHost, st);
  if (window > 0) cudaMemcpyAsync(h + oPool, e.dPool.p, (size_t)window * 4, cudaMemcpyDeviceToHost, st);
  Engine* es[] = {&e};
  if (int rc = launchDone(es, 1, t, st, "hived_events_kernel")) return rc;
  e.takeCtaWords(w, 1, false, 1);
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
  cudaStream_t st = t_own ? t_own->stream : t->stream;  // a concurrent context's batch: its own stream
  const int nb = (n + SCAN_BLOCK - 1) / SCAN_BLOCK;
  e.dScan.ensure((size_t)n * 4 + (size_t)(nb + 2) * 8 + 16);
  long long* blockSum = (long long*)e.dScan.p;              // [nb + 1], 8-byte aligned at the front
  int32_t* excl = (int32_t*)((char*)e.dScan.p + (size_t)(nb + 2) * 8);
  e.dPool2.ensure((size_t)(e.poolCapWords > 0 ? e.poolCapWords : 1) * 4);
  if (e.buffersFailed()) { e.err = "out of device memory for the pool compaction"; return HIVED_ERR_CAPACITY; }
  pool_words_kernel<<<nb, SCAN_T, 0, st>>>((const hived_result_t*)e.dResults.p, n, excl, blockSum);
  pool_block_scan_kernel<<<1, 1024, 0, st>>>(blockSum, nb);
  pool_gather_kernel<<<(int)(((long long)n * 32 + 255) / 256), 256, 0, st>>>((hived_result_t*)e.dResults.p, n, excl, blockSum,
                                                                              (const int32_t*)e.dPool.p, (int32_t*)e.dPool2.p);
  long long tot = 0;
  cudaMemcpyAsync(&tot, blockSum + nb, 8, cudaMemcpyDeviceToHost, st);
  cudaError_t err = cudaStreamSynchronize(st);
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
