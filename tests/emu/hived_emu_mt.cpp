// TEST / BENCH INFRASTRUCTURE ONLY — never built into, shipped with or loaded by the hivedscheduler_b200 package.
// The product's device program (csrc/hived_core.h) compiled for the HOST, one 1-lane "CTA" per host thread: the
// honest CPU comparator of bench.py ("cpu_flat": what the flat data structures and the algorithmic work of the
// device program give on CPU cores, as opposed to the faithful restatement of the Go reference in oracle/).
// VC-parallel batches run exactly as on the GPU — events routed to CTAs by virtual cluster, ordered shared
// sections through the progress words — with host atomics; HIVED_NCTA caps the number of threads.
#define HIVED_EMU 1
#define HIVED_EMU_MT 1
#include <cstdlib>
#include <cstring>
#include <thread>

#include "../../hivedscheduler_b200/csrc/hived_engine.hpp"

thread_local int hived::hv_tls_cta = 0;

namespace hived {
void* bk_alloc(size_t bytes) { return malloc(bytes ? bytes : 1); }
void bk_free(void* p) { free(p); }
void bk_h2d(void* dst, const void* src, size_t bytes) { memcpy(dst, src, bytes); }
void bk_d2h(void* dst, const void* src, size_t bytes) { memcpy(dst, src, bytes); }
void bk_d2d(void* dst, const void* src, size_t bytes) { memcpy(dst, src, bytes); }
void bk_zero(void* dst, size_t bytes) { memset(dst, 0, bytes); }
void bk_quiesce(Engine&) {}
void bk_forget(Engine&) {}
int bk_init(int&, std::string&) { return 0; }
void bk_use_device(int) {}
void bk_flush_l2() {}
int bk_run_small(Engine&, const hived_event_t*, int, const uint32_t*, int64_t, const int32_t*, int64_t, hived_result_t*, int32_t*,
                 int64_t) { return -1; }

static int resultWords(const hived_result_t& r) {
  if (r.kind == HIVED_KIND_BIND && r.n_leaves > 0) return 3 * r.n_leaves;
  if (r.kind == HIVED_KIND_PREEMPT && r.n_victims > 0) return 2 * r.n_victims;
  return 0;
}
int bk_canonicalise(Engine& e, int n, long long* total) {
  e.dPool2.ensure((size_t)(e.poolCapWords > 0 ? e.poolCapWords : 1) * 4);
  hived_result_t* res = (hived_result_t*)e.dResults.p;
  const int32_t* src = (const int32_t*)e.dPool.p;
  int32_t* dst = (int32_t*)e.dPool2.p;
  long long off = 0;
  for (int i = 0; i < n; i++) {
    hived_result_t& r = res[i];
    int words = resultWords(r);
    if (!words) continue;
    bool bind = r.kind == HIVED_KIND_BIND;
    int from = bind ? r.leaf_off : r.victim_off;
    memcpy(dst + off, src + from, (size_t)words * 4);
    if (bind) { r.this_off = (int32_t)(off + (r.this_off - r.leaf_off)); r.leaf_off = (int32_t)off; }
    else r.victim_off = (int32_t)off;
    off += words;
  }
  *total = off;
  return 0;
}

int launchProgram(Engine& e, int n, bool withInit) {
  const int C = withInit ? 1 : e.launchCta;
  const int mgMode = withInit ? 0 : e.mgMode;
  if (mgMode == 3) {
    hv_tls_cta = 0;
    Sm sm;
    memset((void*)&sm, 0, sizeof sm);
    Core core(e.dev, &sm, nullptr, 0, 1);
    core.repairSharedAncestors();
    e.kernelLaunches++;
    return 0;
  }
  std::vector<Sm> sms(C);
  memset((void*)sms.data(), 0, sizeof(Sm) * C);
  CtaWords w[MAX_CTAS] = {};
  e.packCtaWords(w, C, withInit);
  const int32_t* own = (C > 1 || mgMode) ? (const int32_t*)e.dOwn.p : nullptr;
  auto body = [&](int cta) {
    hv_tls_cta = cta;
    runCta(e.dev, &sms[cta], (const hived_event_t*)e.dEvents.p, n, (hived_result_t*)e.dResults.p,
           e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, e.hasAux ? (const int32_t*)e.dAux.p : nullptr,
           withInit ? (const int32_t*)e.dInit.p : nullptr, e.nPinnedOrder, e.nBad, (int32_t*)e.dPool.p, w, own,
           own ? own + n : nullptr, cta, C);
  };
  if (C == 1) {
    body(0);
  } else {
    std::vector<std::thread> th;
    for (int c = 0; c < C; c++) th.emplace_back(body, c);
    for (auto& t : th) t.join();
    hv_tls_cta = 0;
  }
  if (C > 1 && !mgMode) {
    Sm sm;
    memset((void*)&sm, 0, sizeof sm);
    Core core(e.dev, &sm, nullptr, 0, 1);
    core.repairSharedAncestors();
  }
  if (int rc = e.takeCtaWords(w, C, withInit, (C > 1 && !mgMode) ? 2 : 1)) { e.err = "initialisation panicked"; return rc; }
  return 0;
}
}  // namespace hived

extern "C" const char* hived_backend(void) { return "host-threads-emulation-of-device-program (test / bench only)"; }
