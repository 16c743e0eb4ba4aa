// TEST INFRASTRUCTURE ONLY — never built into, shipped with or loaded by the hivedscheduler_b200 package.
// The product's device program (csrc/hived_core.h) behind the same C ABI, executed by the functional SIMT
// emulator of simt_rt.h with the kernel's real geometry: 32-lane warps, a leader warp plus worker warps per
// CTA, one CTA per group of VCs with the ordered shared sections between them.  Complements hived_emu.cpp
// (1 lane: scheduling logic) by covering the warp-level code and the inter-CTA protocol on a box without a GPU.
#define HIVED_SIMT_EMU 1
#include <cstdlib>
#include <cstring>

#include "simt_rt.h"

#include "../../hivedscheduler_b200/csrc/hived_engine.hpp"

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
// host statement of the three pool-compaction kernels of hived_cuda.cu
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

struct LaunchArgs {
  Engine* e;
  int n;
  bool withInit;
  int C;
  Sm* sms;
  CtaWords* words;
  bool repair;
  int mgMode;
};

static void kernelEntry(void* p) {
  LaunchArgs& a = *(LaunchArgs*)p;
  Engine& e = *a.e;
  const int cta = simt::cta();
  Sm& sm = a.sms[cta];
  if (a.repair) {
    Core core(e.dev, &sm, nullptr, 0, 1);
    core.repairSharedAncestors();
    return;
  }
  const int32_t* own = (a.C > 1 || a.mgMode) ? (const int32_t*)e.dOwn.p : nullptr;
  runCta(e.dev, &sm, (const hived_event_t*)e.dEvents.p, a.n, (hived_result_t*)e.dResults.p,
         e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, e.hasAux ? (const int32_t*)e.dAux.p : nullptr,
         a.withInit ? (const int32_t*)e.dInit.p : nullptr, e.nPinnedOrder, e.nBad, (int32_t*)e.dPool.p, a.words, own,
         own ? own + a.n : nullptr, cta, a.C);
}

int launchProgram(Engine& e, int n, bool withInit) {
  static int NT = 0;
  if (!NT) { const char* env = getenv("HIVED_SIMT_NT"); NT = env ? atoi(env) : 96; if (NT < 32 || NT % 32 || NT > 32 * MAX_WARPS) NT = 96; }
  const int C = withInit ? 1 : e.launchCta;
  const int mgMode = withInit ? 0 : e.mgMode;
  std::vector<Sm> sms(C);
  memset((void*)sms.data(), 0, sizeof(Sm) * C);
  CtaWords w[MAX_CTAS] = {};
  if (mgMode == 3) {
    LaunchArgs r{&e, n, false, 1, sms.data(), w, true, 0};
    simt::launch(1, NT, kernelEntry, &r);
    e.kernelLaunches++;
    return 0;
  }
  e.packCtaWords(w, C, withInit);
  LaunchArgs a{&e, n, withInit, C, sms.data(), w, false, mgMode};
  simt::launch(C, NT, kernelEntry, &a);
  if (C > 1 && !mgMode) {
    LaunchArgs r{&e, n, false, 1, sms.data(), w, true, 0};
    simt::launch(1, NT, kernelEntry, &r);
  }
  if (int rc = e.takeCtaWords(w, C, withInit, (C > 1 && !mgMode) ? 2 : 1)) { e.err = "initialisation panicked"; return rc; }
  return 0;
}
}  // namespace hived

extern "C" const char* hived_backend(void) { return "simt-emulation-of-device-program (test only)"; }
