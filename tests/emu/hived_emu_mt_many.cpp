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
  };
  std::vector<Ctx> cs;
  for (int y = 0; y < k; y++) {
    Ctx c{es[y], es[y]->launchCta, std::vector<Sm>(es[y]->launchCta)};
    memset((void*)c.sms.data(), 0, sizeof(Sm) * c.C);
    cs.push_back(std::move(c));
  }
  auto body = [](Ctx* c, int cta) {  // launchProgram's CTA body of an ordinary (not initialising, not partitioned) run
    Engine& e = *c->e;
    const int n = e.stagedN;
    hv_tls_cta = cta;
    Sm& sm = c->sms[cta];
    sm.lead_k = -1;
    sm.pool_off = e.poolBase[cta];
    const int32_t* own = c->C > 1 ? (const int32_t*)e.dOwn.p : nullptr;
    const int32_t* ownOff = own ? own + n : nullptr;
    Core core(e.dev, &sm, (int32_t*)e.dPool.p, e.poolBase[cta + 1], c->C);
    core.run((const hived_event_t*)e.dEvents.p, n, (hived_result_t*)e.dResults.p, e.hasSugg ? (const uint32_t*)e.dSugg.p : nullptr,
             e.hasAux ? (const int32_t*)e.dAux.p : nullptr, nullptr, e.nPinnedOrder, e.nBad, own ? own + ownOff[cta] : nullptr,
             own ? ownOff[cta + 1] - ownOff[cta] : n);
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
    e.kernelLaunches += c.C > 1 ? 2 : 1;
    e.poolEnd.assign(c.C, 0);
    for (int cta = 0; cta < c.C; cta++) e.poolEnd[cta] = c.sms[cta].pool_off;
    e.poolOff = c.sms[0].pool_off;
  }
  return 0;
}

}  // namespace hived
