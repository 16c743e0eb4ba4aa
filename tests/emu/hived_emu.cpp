// TEST INFRASTRUCTURE ONLY — never built into, shipped with or loaded by the hivedscheduler_b200
// package.  Compiles the product's device program (csrc/hived_core.h) for the host as a
// 1-thread / 1-lane CTA (HIVED_EMU) behind the same C ABI, so that the kernel LOGIC can be
// parity-tested against the oracle in a container that has no GPU.  GPU tests (-m gpu) exercise
// the real sm_90a build; this file exists because GPU round trips are scarce during development.
#define HIVED_EMU 1
#include <cstdlib>
#include <cstring>

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
int bk_canonicalise(Engine&, int, long long*) { return HIVED_ERR_PLATFORM; }  // never reached: the emulation runs one CTA
int bk_run_small(Engine&, const hived_event_t*, int, const uint32_t*, int64_t, const int32_t*, int64_t, hived_result_t*, int32_t*,
                 int64_t) { return -1; }  // a CUDA staging optimisation: the emulation always takes the general path
int launchProgram(Engine& e, int n, bool withInit) {
  // the emulation runs ONE CTA: VC-parallel batches are exercised on the GPU only
  e.launchCta = 1;
  e.poolBase.assign(2, 0);
  e.poolBase[1] = withInit ? 0 : e.poolCapWords;
  static Sm sm;
  memset(&sm, 0, sizeof sm);
  sm.pool_off = 0;
  sm.lead_k = -1;
  Core core(e.dev, &sm, (int32_t*)e.dPool.p, withInit ? 0 : e.poolCapWords, 1);
  core.run((const hived_event_t*)e.dEvents.p, n, (hived_result_t*)e.dResults.p,
           e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, e.hasAux ? (const int32_t*)e.dAux.p : nullptr,
           withInit ? (const int32_t*)e.dInit.p : nullptr, e.nPinnedOrder, e.nBad, nullptr, n);
  e.poolOff = sm.pool_off;
  e.poolEnd.assign(1, sm.pool_off);
  e.kernelLaunches++;
  if (withInit && sm.panic) { e.err = "initialisation panicked"; return sm.panic; }
  return 0;
}
}  // namespace hived

extern "C" const char* hived_backend(void) { return "host-emulation-of-device-program (test only)"; }
