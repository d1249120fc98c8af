// seaweedfs_b200/csrc/io_pool.h — a small blocking fork-join pool for host-side work that the GPU cannot do:
// the k preads / k+m pwrites of a stripe in the file pipeline (ec_files.cc) and the bounce copies between
// pageable caller memory and the pinned staging ring at the Encoder seam (host_seam.cc).  No GF arithmetic
// ever runs here.  tests/test_iopool.py compiles this class on its own under ThreadSanitizer and AddressSanitizer.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

namespace swec {

// A few I/O threads shared by the reader and the writer side: every shard file is independent, so
// the k preads of a stripe (and the k+m pwrites of a finished one) run concurrently.  One thread
// doing them serially tops out near 1.5 GB/s even on RAM-backed files.
//
// spin_us > 0 (the Encoder seam's copy crew): idle workers and the submitting thread poll for up to that long
// before they sleep on the condition variable.  A condvar wake-up costs 50-100 us on a busy (or cgroup-throttled)
// host — more than the whole DMA of a 256 KiB-per-shard Encode call — so back-to-back calls must find the crew awake.
class IoPool {
  public:
    explicit IoPool(size_t n, unsigned spin_us = 0) : spin_us_(spin_us) {
        for (size_t i = 0; i < n; i++) threads_.emplace_back([this] { loop(); });
    }
    ~IoPool() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_.store(true);
        }
        cv_.notify_all();
        for (auto& t : threads_) t.join();
    }
    // run fn(0..n-1) across the pool (the caller takes a share too); returns the first non-zero result
    int parallel_for(int n, const std::function<int(int)>& fn) {
        if (n <= 0) return 0;
        Batch b;  // lives on this stack frame: nobody may touch it once finished == n has been observed UNDER THE LOCK
        b.fn = &fn;
        b.n = n;
        std::unique_lock<std::mutex> lk(mu_);
        batches_.push_back(&b);
        unclaimed_.fetch_add(n, std::memory_order_release);
        if (sleepers_ > 0) cv_.notify_all();
        work(&b, lk);
        if (spin_us_ && b.finished.load(std::memory_order_acquire) < n) {
            lk.unlock();
            const auto t0 = std::chrono::steady_clock::now();
            while (b.finished.load(std::memory_order_acquire) < n && !spun_out(t0, 20u * spin_us_)) relax();
            lk.lock();  // a worker that has just counted the last task still holds the lock while it notifies
        }
        b.done_cv.wait(lk, [&] { return b.finished.load(std::memory_order_relaxed) == b.n; });
        batches_.erase(std::find(batches_.begin(), batches_.end(), &b));
        return b.rc;
    }

  private:
    struct Batch {
        const std::function<int(int)>* fn = nullptr;
        int n = 0, next = 0, rc = 0;
        std::atomic<int> finished{0};
        std::condition_variable done_cv;
    };
    static void relax() {
#if defined(__x86_64__) || defined(__i386__)
        __builtin_ia32_pause();
#endif
    }
    static bool spun_out(std::chrono::steady_clock::time_point t0, unsigned us) {
        return std::chrono::steady_clock::now() - t0 > std::chrono::microseconds(us);
    }
    // Called and returns with mu_ held.  A batch is only dereferenced while the lock has been held
    // continuously since we last saw it unfinished (its owner cannot return without the lock).
    void work(Batch* b, std::unique_lock<std::mutex>& lk) {
        while (b->next < b->n) {
            const int i = b->next++;
            unclaimed_.fetch_sub(1, std::memory_order_relaxed);
            const std::function<int(int)>* fn = b->fn;
            lk.unlock();
            const int rc = (*fn)(i);
            lk.lock();
            if (rc && !b->rc) b->rc = rc;
            if (b->finished.fetch_add(1, std::memory_order_release) + 1 == b->n) {
                b->done_cv.notify_all();
                return;  // the owner may destroy the batch as soon as we release the lock
            }
        }
    }
    Batch* find_work() {  // mu_ held
        for (Batch* x : batches_)
            if (x->next < x->n) return x;
        return nullptr;
    }
    void loop() {
        std::unique_lock<std::mutex> lk(mu_);
        for (;;) {
            if (stop_.load()) return;
            if (Batch* b = find_work()) {
                work(b, lk);
                continue;
            }
            if (spin_us_) {  // stay awake for a while: the next call of a back-to-back caller is microseconds away
                lk.unlock();
                const auto t0 = std::chrono::steady_clock::now();
                bool timed_out = false;
                while (unclaimed_.load(std::memory_order_acquire) <= 0 && !stop_.load(std::memory_order_relaxed)) {
                    if (spun_out(t0, spin_us_)) {
                        timed_out = true;
                        break;
                    }
                    relax();
                }
                lk.lock();
                if (!timed_out) continue;
            }
            sleepers_++;
            cv_.wait(lk, [&] { return stop_.load() || find_work() != nullptr; });
            sleepers_--;
        }
    }
    std::vector<std::thread> threads_;
    std::deque<Batch*> batches_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::atomic<bool> stop_{false};
    std::atomic<int> unclaimed_{0};  // tasks nobody has started yet, over all batches (the spinners' signal)
    int sleepers_ = 0;               // workers blocked in cv_.wait (mu_ held to touch it)
    const unsigned spin_us_;
};

// ---- end of IoPool

}  // namespace swec
