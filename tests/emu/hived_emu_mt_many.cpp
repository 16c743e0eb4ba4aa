// TEST INFRASTRUCTURE ONLY — the thread emulation of hived_emu_mt.cpp with a joint launch of its own
// (include/hived_multictx.h): every CTA of every listed context on a host thread of its own, all at the same time, each
// Core built on its own context's Dev, then the repair pass of the contexts that ran VC-parallel.  Exercises the
// staging, CTA routing, per-context fetch and error isolation of hived_process_events_many on a box without a GPU.
#define HIVED_BK_LAUNCH_MANY 1
#include "hived_emu_mt.cpp"

namespace hived {

int bk_launch_many(Engine* const* es, int k) {
  struct Ctx {
    Engine* e;
    int C;
    std::vector<Sm> sms;
    CtaWords w[MAX_CTAS];
  };
  std::vector<Ctx> cs;
  for (int y = 0; y < k; y++) {
    Ctx c{es[y], es[y]->launchCta, std::vector<Sm>(es[y]->launchCta), {}};
    memset((void*)c.sms.data(), 0, sizeof(Sm) * c.C);
    es[y]->packCtaWords(c.w, c.C, false);
    cs.push_back(std::move(c));
  }
  auto body = [](Ctx* c, int cta) {  // launchProgram's CTA body of an ordinary (not initialising, not partitioned) run
    Engine& e = *c->e;
    const int n = e.stagedN;
    hv_tls_cta = cta;
    const int32_t* own = c->C > 1 ? (const int32_t*)e.dOwn.p : nullptr;
    runCta(e.dev, &c->sms[cta], (const hived_event_t*)e.dEvents.p, n, (hived_result_t*)e.dResults.p,
           e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr, e.hasAux ? (const int32_t*)e.dAux.p : nullptr, nullptr, e.nPinnedOrder,
           e.nBad, (int32_t*)e.dPool.p, c->w, own, own ? own + n : nullptr, cta, c->C);
  };
  std::vector<std::thread> th;
  for (auto& c : cs)
    for (int cta = 0; cta < c.C; cta++) th.emplace_back(body, &c, cta);
  for (auto& t : th) t.join();
  hv_tls_cta = 0;
  for (auto& c : cs) {
    Engine& e = *c.e;
    if (c.C > 1) {
      Sm sm;
      memset((void*)&sm, 0, sizeof sm);
      Core core(e.dev, &sm, nullptr, 0, 1);
      core.repairSharedAncestors();
    }
    e.takeCtaWords(c.w, c.C, false, c.C > 1 ? 2 : 1);
  }
  return 0;
}

}  // namespace hived
