// Drives hived_seats.h (the co-residency seat ledger) from many threads; prints "ok" or what went wrong (exit 1).
//   seat_ledger_stress <capacity> <threads> <requests per thread> <seed>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <random>
#include <thread>
#include <vector>

#include "../../hivedscheduler_b200/csrc/hived_seats.h"

using hived::SeatLedger;

static int fail(const char* what) {
  printf("FAIL: %s\n", what);
  return 1;
}

static void waitQueued(SeatLedger& l, int n) {
  while (l.queued() < n) std::this_thread::sleep_for(std::chrono::microseconds(50));
}

int main(int argc, char** argv) {
  if (argc != 5) return fail("usage");
  const int cap = atoi(argv[1]), nThreads = atoi(argv[2]), nReq = atoi(argv[3]);
  const unsigned seed = (unsigned)atoi(argv[4]);

  // 1. random requests from many threads: the seats held never exceed the capacity, and every request is served
  {
    SeatLedger l;
    l.setCapacity(cap);
    std::atomic<int> inUse{0}, peak{0}, served{0};
    std::atomic<bool> over{false};
    std::vector<std::thread> th;
    for (int t = 0; t < nThreads; t++)
      th.emplace_back([&, t] {
        std::mt19937 rng(seed * 7919u + t);
        for (int r = 0; r < nReq; r++) {
          const int n = 1 + (int)(rng() % (unsigned)cap);
          if (!l.acquire(n)) { over = true; return; }
          const int now = inUse += n;
          if (now > cap) over = true;
          int p = peak.load();
          while (now > p && !peak.compare_exchange_weak(p, now)) {}
          std::this_thread::sleep_for(std::chrono::microseconds(rng() % 200));
          inUse -= n;
          l.release(n);
          served++;
        }
      });
    for (auto& x : th) x.join();
    if (over) return fail("more seats held than the capacity, or a request within it refused");
    if (served != nThreads * nReq) return fail("not every request was served");
    if (l.held() != 0 || l.queued() != 0) return fail("seats or requests left over");
    printf("random: %d requests, peak %d of %d seats\n", (int)served, (int)peak, cap);
  }

  // 2. first come, first served: requests queued one after another are granted in that order, and a request for every
  //    seat is not overtaken by smaller ones queued after it
  {
    SeatLedger l;
    l.setCapacity(cap);
    if (!l.acquire(cap)) return fail("a request for every seat refused");
    std::mutex mu;
    std::vector<int> order;
    std::vector<std::thread> th;
    const int nBig = 4, nSmall = 6;
    // the big ones need more than half the seats each, the first and the last every seat: one holder at a time until
    // the last big one has recorded its grant, so the recorded order is the grant order
    for (int i = 0; i < nBig; i++) {
      th.emplace_back([&, i] {
        const int n = i == 0 || i == nBig - 1 ? cap : cap / 2 + 1;
        l.acquire(n);
        { std::lock_guard<std::mutex> g(mu); order.push_back(i); }
        std::this_thread::sleep_for(std::chrono::milliseconds(2));
        l.release(n);
      });
      waitQueued(l, i + 1);
    }
    for (int i = 0; i < nSmall; i++) {
      th.emplace_back([&, i] {
        l.acquire(1);
        { std::lock_guard<std::mutex> g(mu); order.push_back(100 + i); }
        l.release(1);
      });
      waitQueued(l, nBig + i + 1);
    }
    l.release(cap);
    for (auto& x : th) x.join();
    for (int i = 0; i < nBig; i++)
      if (order[i] != i) return fail("grants out of arrival order");
    if ((int)order.size() != nBig + nSmall) return fail("not every queued request was served");
    printf("fifo: %d grants in arrival order\n", nBig);
  }

  // 3. a request larger than the device is refused at once and takes nothing; so is any request before the capacity is
  //    known
  {
    SeatLedger l;
    if (l.acquire(1)) return fail("a request granted before the capacity was set");
    l.setCapacity(cap);
    l.setCapacity(cap + 100);
    if (l.capacity() != cap) return fail("the capacity changed after it was set");
    if (l.acquire(cap + 1)) return fail("an oversized request granted");
    if (l.held() != 0 || l.queued() != 0) return fail("a refused request left something behind");
    hived::SeatHold h(l, cap);
    if (!h.ok() || l.held() != cap) return fail("SeatHold did not take its seats");
  }
  printf("ok\n");
  return 0;
}
