// coalesce.h -- the request queue behind pb_search (DESIGN.md 4m): concurrent single-query callers of one handle are
// merged into shared batches, group-commit style.  No thread is created: the caller at the head of the queue becomes
// the leader of the next batch, runs it through the callable it was given and wakes the callers that rode along.
// Nothing here knows CUDA or pb_index, so the queue is tested on its own (tests/test_coalesce_cpu.py).
//
// Lock order: `mu` is a leaf.  It is never held while a batch runs, so the callable may take any lock it likes.
#ifndef PB_COALESCE_H
#define PB_COALESCE_H

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <string>
#include <vector>

namespace pbq {

struct Config {
    int max_queries = 1;   // largest merged batch; <= 1: the queue is off
    int max_wait_us = 0;   // how long a leader with a short batch waits for company; 0 = never
    int max_inflight = 2;  // merged batches that may run at once
};

struct Counters {  // pb_coalesce_stats, field for field
    int64_t n_requests = 0, n_batches = 0, n_bypassed = 0, n_refused = 0, n_rerun_alone = 0, max_batch = 0;
    int64_t batch_hist[8] = {};  // batches of 1, 2, 3-4, 5-8, 9-16, 17-32, 33-64, > 64
    int64_t queue_wait_us = 0;
};

// One caller's request.  The caller derives its payload from it, keeps it on its stack and blocks in submit() until
// the request is done; the batch callable fills the payload's results.
struct Request {
    int status = 0;
    std::string error;  // message of a non-zero status
    // the queue's own fields (under Queue::mu)
    Request *next = nullptr;
    bool done = false;
    std::chrono::steady_clock::time_point enqueued;
    std::condition_variable cv;  // "you are done" or "you are the head and a batch may start"
};

// Run is callable as int(Request *const *reqs, size_t n, std::string &err): run the n requests as one batch, fill
// their results, return 0; or return a status with its message in err and leave the results alone.
template <class Run> class Queue {
public:
    // fatal_status: a merged batch that returns it fails every member (a device error); any other failure of a batch
    // of several re-runs the members alone, in order, and each gets the status of its own run.
    Queue(Run run, int fatal_status) : run_(run), fatal_(fatal_status) {}

    void configure(const Config &c) {
        std::lock_guard<std::mutex> g(mu_);
        cfg_ = c;
    }
    bool enabled() {
        std::lock_guard<std::mutex> g(mu_);
        return cfg_.max_queries > 1;
    }
    void count_bypassed() { bypassed_.fetch_add(1, std::memory_order_relaxed); }
    void count_refused() { refused_.fetch_add(1, std::memory_order_relaxed); }
    Counters counters(bool reset) {
        std::lock_guard<std::mutex> g(mu_);
        Counters c = st_;
        c.n_bypassed = reset ? bypassed_.exchange(0) : bypassed_.load();
        c.n_refused = reset ? refused_.exchange(0) : refused_.load();
        if (reset) st_ = Counters();
        return c;
    }

    // Blocks until r is done; r.status / r.error and the payload hold its result.
    void submit(Request &r) {
        std::unique_lock<std::mutex> lk(mu_);
        r.enqueued = std::chrono::steady_clock::now();
        r.next = nullptr;
        r.done = false;
        (tail_ ? tail_->next : head_) = &r;
        tail_ = &r;
        ++st_.n_requests;
        if (gathering_) fill_cv_.notify_one();
        // a leader that is still gathering takes the new arrivals, so nobody else starts a batch meanwhile
        while (!r.done && !(head_ == &r && !gathering_ && inflight_ < std::max(cfg_.max_inflight, 1))) r.cv.wait(lk);
        if (!r.done) lead(lk);
    }

private:
    void take(std::vector<Request *> &batch, size_t cap) {
        while (head_ && batch.size() < cap) {
            batch.push_back(head_);
            head_ = head_->next;
        }
        if (!head_) tail_ = nullptr;
    }
    void wake_head() {
        if (head_ && !gathering_ && inflight_ < std::max(cfg_.max_inflight, 1)) head_->cv.notify_one();
    }

    // the caller is the head of the queue and holds the lock
    void lead(std::unique_lock<std::mutex> &lk) {
        ++inflight_;
        const size_t cap = (size_t)std::max(cfg_.max_queries, 1);
        std::vector<Request *> batch;
        if (!spare_.empty()) {
            batch.swap(spare_.back());
            spare_.pop_back();
        }
        batch.clear();
        take(batch, cap);
        if (cfg_.max_wait_us > 0 && batch.size() < cap) {
            const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(cfg_.max_wait_us);
            gathering_ = true;
            while (batch.size() < cap && fill_cv_.wait_until(lk, deadline) != std::cv_status::timeout) take(batch, cap);
            take(batch, cap);
            gathering_ = false;
        }
        const auto start = std::chrono::steady_clock::now();
        for (Request *m : batch)
            st_.queue_wait_us += std::chrono::duration_cast<std::chrono::microseconds>(start - m->enqueued).count();
        const size_t n = batch.size();
        ++st_.n_batches;
        st_.max_batch = std::max<int64_t>(st_.max_batch, (int64_t)n);
        int bucket = 0;
        while (bucket < 7 && ((size_t)1 << bucket) < n) ++bucket;
        ++st_.batch_hist[bucket];
        wake_head();  // another batch may start while this one runs
        lk.unlock();

        std::string err;
        int st = run_(batch.data(), n, err);
        size_t rerun = 0;
        if (st != 0 && st != fatal_ && n > 1) {
            rerun = n;
            for (Request *m : batch) {
                m->error.clear();
                m->status = run_(&m, 1, m->error);
            }
        } else {
            for (Request *m : batch) {
                m->status = st;
                if (st != 0) m->error = err;
            }
        }

        lk.lock();
        st_.n_rerun_alone += (int64_t)rerun;
        for (Request *m : batch) {  // notified under the lock: a follower returns, and its Request dies, only after it
            m->done = true;
            m->cv.notify_one();
        }
        batch.clear();
        spare_.push_back(std::move(batch));
        --inflight_;
        wake_head();
    }

    Run run_;
    const int fatal_;
    std::mutex mu_;
    std::condition_variable fill_cv_;  // a gathering leader waits here for arrivals
    Config cfg_;
    Counters st_;
    std::atomic<int64_t> bypassed_{0}, refused_{0};
    Request *head_ = nullptr, *tail_ = nullptr;
    int inflight_ = 0;
    bool gathering_ = false;
    std::vector<std::vector<Request *>> spare_;  // member lists of finished batches, reused
};

}  // namespace pbq
#endif
