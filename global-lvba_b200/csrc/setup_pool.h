// setup_pool.h — host threads for the set-up loops of the one-shot calls (plain C++, no CUDA): parallel_chunks().
#pragma once
#include <pthread.h>

#include <algorithm>
#include <condition_variable>
#include <cstdint>
#include <functional>
#include <mutex>
#include <new>
#include <thread>
#include <vector>

namespace lvba {

constexpr int kMaxSetupThreads = 8;      // the most threads of a parallel_chunks region (its `worker` is below this)

// fn(begin, end, worker) over [0, n) split into contiguous chunks on up to 8 threads.  The set-up of a one-shot call
// (validation, envelope structure, gathers) is a few milliseconds of host loops next to ~15 ms of device work, and a call has
// several of them: the helpers are a PERSISTENT pool (created on first use, parked on a condition variable between regions) —
// spawning and joining seven std::threads per region cost more than most of the loops they ran (0.1-0.4 ms per region).
// One region at a time: a second caller (or a nested region) runs its loop inline.
class SetupPool {
 public:
  static SetupPool& get() { static SetupPool p; return p; }
  SetupPool() { pthread_atfork(nullptr, nullptr, &SetupPool::after_fork_in_child); }
  // job(w) for w = 0 .. nt-1: w = 0 on the calling thread, the others on the pool's workers; returns when all are done
  template <class Job>
  void run(int nt, const Job& job) {
    if (nt <= 1 || in_job()) { for (int w = 0; w < nt; ++w) job(w); return; }      // nested region: inline
    std::unique_lock<std::mutex> region(region_mu_, std::try_to_lock);
    if (!region.owns_lock()) { for (int w = 0; w < nt; ++w) job(w); return; }        // another caller's region is running: inline
    const std::function<void(int)> f = [&job](int w) { in_job() = true; job(w); in_job() = false; };
    {
      std::lock_guard<std::mutex> lk(mu_);
      while ((int)workers_.size() < nt - 1) { const int w = (int)workers_.size() + 1; workers_.emplace_back([this, w] { worker(w); }); }
      job_ = &f; nt_ = nt; pending_ = nt - 1; ++gen_;
    }
    go_.notify_all();
    f(0);
    std::unique_lock<std::mutex> lk(mu_);
    done_.wait(lk, [&] { return pending_ == 0; });
    job_ = nullptr;
  }
  ~SetupPool() {
    { std::lock_guard<std::mutex> lk(mu_); stop_ = true; }
    go_.notify_all();
    for (auto& t : workers_) t.join();
  }

 private:
  static bool& in_job() { static thread_local bool b = false; return b; }
  // a forked child has none of the parent's threads: forget them (the objects are leaked on purpose — destroying a joinable
  // std::thread terminates) and start from fresh synchronisation objects
  static void after_fork_in_child() {
    SetupPool& p = get();
    new (&p.workers_) std::vector<std::thread>();
    new (&p.region_mu_) std::mutex(); new (&p.mu_) std::mutex();
    new (&p.go_) std::condition_variable(); new (&p.done_) std::condition_variable();
    p.job_ = nullptr; p.nt_ = 0; p.pending_ = 0; p.stop_ = false;
  }
  void worker(int w) {
    long seen = 0;
    std::unique_lock<std::mutex> lk(mu_);
    for (;;) {
      go_.wait(lk, [&] { return stop_ || gen_ != seen; });
      if (stop_) return;
      seen = gen_;
      if (w >= nt_) continue;                          // this region uses fewer threads
      const std::function<void(int)>* j = job_;
      lk.unlock();
      (*j)(w);
      lk.lock();
      if (--pending_ == 0) done_.notify_one();
    }
  }
  std::mutex region_mu_, mu_;
  std::condition_variable go_, done_;
  std::vector<std::thread> workers_;
  const std::function<void(int)>* job_ = nullptr;
  long gen_ = 0;
  int nt_ = 0, pending_ = 0;
  bool stop_ = false;
};
template <class Fn>
inline void parallel_chunks(int64_t n, int64_t min_chunk, Fn fn) {
  unsigned hw = std::thread::hardware_concurrency();
  int nt = (int)std::min<int64_t>(std::min<unsigned>(hw ? hw : 1u, (unsigned)kMaxSetupThreads), std::max<int64_t>(1, n / std::max<int64_t>(min_chunk, 1)));
  if (nt <= 1) { fn((int64_t)0, n, 0); return; }
  SetupPool::get().run(nt, [&](int w) { fn(n * w / nt, n * (w + 1) / nt, w); });
}

}  // namespace lvba
