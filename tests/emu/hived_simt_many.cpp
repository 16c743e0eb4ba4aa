// TEST INFRASTRUCTURE ONLY — the SIMT emulation of hived_simt.cpp with a joint launch of its own
// (include/hived_multictx.h): one grid of (max C) x k CTAs as on the GPU (hived_cuda_many.cu), CTA (x, y) being CTA x
// of context y, each Core built on its own context's Dev, a CTA with x >= C_y leaving at once; then the repair pass of
// the contexts that ran VC-parallel.
#define HIVED_BK_LAUNCH_MANY 1
#include "hived_simt.cpp"

namespace hived {

struct ManyLaunch {
  std::vector<LaunchArgs> ctx;
  int cmax;
};

static void manyEntry(void* p) {
  ManyLaunch& m = *(ManyLaunch*)p;
  const int flat = simt::cta();
  simt::rt().cur->cta = flat % m.cmax;  // what the program sees as its CTA index (blockIdx.x)
  LaunchArgs& a = m.ctx[flat / m.cmax];
  if (flat % m.cmax >= a.C) return;
  kernelEntry(&a);
}

int bk_launch_many(Engine* const* es, int k) {
  const char* env = getenv("HIVED_SIMT_NT");  // the block size of launchProgram
  int NT = env ? atoi(env) : 96;
  if (NT < 32 || NT % 32 || NT > 32 * MAX_WARPS) NT = 96;
  std::vector<std::vector<Sm>> sms(k);
  std::vector<std::vector<long long>> scal(k, std::vector<long long>(MAX_CTAS * 4, 0));
  ManyLaunch m{{}, 1};
  for (int y = 0; y < k; y++) {
    Engine& e = *es[y];
    const int C = e.launchCta;
    sms[y].resize(C);
    memset((void*)sms[y].data(), 0, sizeof(Sm) * C);
    for (int c = 0; c < C; c++) { scal[y][c * 4 + 0] = e.poolBase[c]; scal[y][c * 4 + 1] = e.poolBase[c + 1]; }
    m.ctx.push_back(LaunchArgs{&e, e.stagedN, false, C, sms[y].data(), scal[y].data(), false, 0});
    if (C > m.cmax) m.cmax = C;
  }
  simt::launch(m.cmax * k, NT, manyEntry, &m);
  for (int y = 0; y < k; y++) {
    Engine& e = *es[y];
    const int C = e.launchCta;
    if (C > 1) {
      LaunchArgs r{&e, e.stagedN, false, 1, sms[y].data(), scal[y].data(), true, 0};
      simt::launch(1, NT, kernelEntry, &r);
    }
    e.kernelLaunches += C > 1 ? 2 : 1;
    e.poolEnd.assign(C, 0);
    for (int c = 0; c < C; c++) e.poolEnd[c] = scal[y][c * 4 + 0];
    e.poolOff = scal[y][0];
  }
  return 0;
}

}  // namespace hived
