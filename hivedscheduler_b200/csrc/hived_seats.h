// Co-residency seats of one device (host only; DESIGN.md §4 "Concurrent batches").
//
// A cooperative grid whose CTAs are not all resident at the same time waits forever, and so does a resident per-call
// kernel that is never asked to stop.  Every kernel of the library that may wait for something other than its own CTAs'
// work (a cooperative grid, a resident kernel) therefore holds one seat per CTA while it may be on the device, and a
// device has as many seats as CTAs of the program fit on it at once.  Then
//   resident kernels + cooperative grids of running batches + the grid of the g_devMu holder <= seats
// holds at every moment, and every such grid is co-resident.
//
// Requests are served whole and in arrival order (tickets), so that a 16-CTA request is not starved by a stream of
// smaller ones; a request larger than the device is refused instead of queued.
#pragma once
#include <condition_variable>
#include <cstdint>
#include <mutex>

namespace hived {

class SeatLedger {
 public:
  // the seats of the device; the first call fixes them (later calls with another value change nothing)
  void setCapacity(int seats) {
    std::lock_guard<std::mutex> lk(mu_);
    if (cap_ < 0) cap_ = seats;
  }
  int capacity() {
    std::lock_guard<std::mutex> lk(mu_);
    return cap_;
  }
  // Blocks until n seats are free and every earlier request has been served, then takes them.  false (nothing taken)
  // when n exceeds the capacity, or the capacity has not been set.
  bool acquire(int n) {
    std::unique_lock<std::mutex> lk(mu_);
    if (n < 0 || cap_ < 0 || n > cap_) return false;
    const uint64_t ticket = next_++;
    cv_.wait(lk, [&] { return serving_ == ticket && held_ + n <= cap_; });
    held_ += n;
    serving_++;
    lk.unlock();
    cv_.notify_all();  // the next ticket may fit as well
    return true;
  }
  void release(int n) {
    {
      std::lock_guard<std::mutex> lk(mu_);
      held_ -= n;
    }
    cv_.notify_all();
  }
  int held() {
    std::lock_guard<std::mutex> lk(mu_);
    return held_;
  }
  int queued() {  // requests waiting for their seats
    std::lock_guard<std::mutex> lk(mu_);
    return (int)(next_ - serving_);
  }

 private:
  std::mutex mu_;
  std::condition_variable cv_;
  int cap_ = -1, held_ = 0;
  uint64_t next_ = 0, serving_ = 0;
};

// Seats held for one launch: released when the holder goes out of scope (the error paths included).
class SeatHold {
 public:
  SeatHold(SeatLedger& l, int n) : l_(l), n_(l.acquire(n) ? n : -1) {}
  ~SeatHold() { if (n_ > 0) l_.release(n_); }
  bool ok() const { return n_ >= 0; }
  SeatHold(const SeatHold&) = delete;
  SeatHold& operator=(const SeatHold&) = delete;

 private:
  SeatLedger& l_;
  int n_;
};

}  // namespace hived
