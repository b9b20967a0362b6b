// deployment.cpp -- an index directory doc-sharded over several devices of this process behind one pb_index handle
// (pb_index_load_devices, DESIGN.md 4o).  Host code only: the ranks are ordinary handles of pb_index_load_range_flags
// joined in a pb_shard_group, and every rank is driven through the public entry points.
//
// Threads: rank 0 runs on the caller's thread, so its thread-local pb_last_error and pb_last_* stats are the caller's;
// ranks 1..n-1 each have a persistent worker created at load and joined at close.  Order: every collective holds `mu`
// for the whole call, so concurrent callers, the coalescer's batches and mutations reach every rank in one order.
// Layout: mutations also hold `layout` alone; the accessors read it shared, so they (and pb_search's check of a request
// before it is queued) wait for a mutation, as on one handle, but never for a search.
#include "engine_internal.h"

#include <algorithm>
#include <cstdio>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <thread>

namespace {

struct SearchScratch {  // one rank's copy of a search's outputs (ranks >= 1)
    std::vector<int64_t> ids;
    std::vector<float> scores;
    std::vector<int32_t> counts;
};

}  // namespace

struct Deployment : Group {
    std::vector<pb_index *> ranks;
    std::vector<int> devices;
    pb_shard_group *group = nullptr;
    std::vector<std::unique_ptr<RankWorker>> workers;  // [world]; workers[0] is empty (rank 0 runs on the caller)
    std::mutex mu;                  // one collective at a time; also one job at a time for the rank threads
    std::shared_mutex layout;       // the ranks' ranges and totals: held alone by mutations (inside mu), shared by readers
    std::vector<SearchScratch> scratch;  // under mu

    int world() const { return (int)ranks.size(); }

    // job(r) for every rank at once, whose result is one status: the lowest failing rank's, where with skip_comm a rank
    // reporting PB_ERR_COMM (a peer's failure seen through the group) gives way to a rank with a failure of its own.
    // That rank's message becomes the caller's.
    pb_status run_one(const Job &job, bool skip_comm = true) {
        std::vector<pb_status> st;
        std::vector<std::string> err;
        run_slots(world(), job, workers.data() + 1, st, err);
        int pick = -1;
        for (int r = 0; r < world() && pick < 0; ++r)
            if (st[r] != PB_OK && !(skip_comm && st[r] == PB_ERR_COMM)) pick = r;
        for (int r = 0; r < world() && pick < 0; ++r)
            if (st[r] != PB_OK) pick = r;
        if (pick < 0) return PB_OK;
        // A sharded collective gives every rank the failing rank's status; the others' text only names that rank, so
        // the caller gets the failing rank's own message
        int named = -1;
        if (sscanf(err[pick].c_str(), "rank %d of the group failed", &named) == 1 && named >= 0 && named < world() &&
            st[named] == st[pick])
            pick = named;
        return pb_fail(st[pick], "%s", err[pick].c_str());
    }

    // each rank's global range [base[r], base[r + 1]): rank r starts where its handle's doc_id_base says
    pb_status bounds(std::vector<int64_t> &base) {
        base.assign((size_t)world() + 1, 0);
        for (int r = 0; r < world(); ++r) {
            int32_t w = 0;
            int64_t b[2];
            pb_status s = pb_index_shard_layout(ranks[r], &w, b, nullptr);
            if (s != PB_OK) return s;
            base[r] = b[0];
            base[r + 1] = b[1];
        }
        return PB_OK;
    }

    // A resize's new layout: next[r] becomes rank r of g, on devs[r].  The threads and scratch follow the world: worker
    // r serves slot r, so the workers of the slots both worlds have stay, and those of the slots it loses are joined.
    // Under mu and layout, with no collective running; cannot fail.
    void reform(std::vector<pb_index *> next, std::vector<int> devs, pb_shard_group *g) {
        for (size_t r = 0; r < next.size(); ++r) pb_index_group_move(next[r], g, (int)r);  // r < g's world: succeeds
        ranks = std::move(next);
        devices = std::move(devs);
        group = g;
        workers.resize((size_t)world());
        for (int r = 1; r < world(); ++r)
            if (!workers[r]) workers[r].reset(new RankWorker(r));
        scratch.resize((size_t)world());
    }

    // joins the loaded ranks in the group and makes the handle; on failure the caller deletes this
    pb_status finish(pb_index **out) {
        for (int r = 0; r < world(); ++r) {
            pb_status s = pb_index_group_join(ranks[r], group, r);
            if (s != PB_OK) return s;
        }
        *out = pb_index_new_group(this, ranks[0]);
        return PB_OK;
    }

    // stops and joins the threads, closes the ranks, destroys the group
    ~Deployment() override {
        workers.clear();  // joins the threads
        for (pb_index *ix : ranks) pb_index_close(ix);
        pb_shard_group_destroy(group);
    }

    const char *kind() const override { return "a multi-device handle (pb_index_load_devices)"; }
    Deployment *as_deployment() override { return this; }
    pb_index *member(int r) override { return ranks[r]; }
    int size() override { return world(); }
    void totals(long long *D, long long *N) override;
    pb_status memory(int64_t *device_bytes, int64_t *host_bytes) override;
    pb_status shard_layout(int32_t *out_world, int64_t *out_bounds, int32_t *out_devices) override;
    pb_status append(pb_codec *codec, const float *embeddings, const int64_t *codes, const uint8_t *residuals,
                     const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space, const char *index_dir,
                     int64_t batch_size, int64_t *out_first_doc_id) override;
    pb_status del(const int64_t *doc_ids, int64_t n_ids, const char *index_dir, int64_t *out_deleted) override;
    pb_status rebalance(const int64_t *bounds, int64_t *out_bounds) override;
    pb_status decompress(const int64_t *doc_ids, int64_t n_docs, float *out_embeddings, int64_t *out_lengths) override;
    pb_status exhaustive(const float *queries, const int64_t *q_off, int64_t n_queries, float *out_scores) override;
    // each addresses one rank's handle
    pb_status reserve(int64_t, int64_t) override {
        return refuse("pb_index_reserve (reserve a rank's capacity before it joins a group)");
    }
    pb_status export_ivf(int64_t *, int32_t *, int64_t *) override { return refuse("pb_index_export_ivf"); }
    pb_status last_delete_ms(float *) override { return refuse("pb_last_delete_ms"); }
    // the ranks as they are: a resize waits for these, a search does not
    void each(const std::function<void(pb_index *)> &call) override {
        std::shared_lock<std::shared_mutex> g(layout);
        for (pb_index *ix : ranks) call(ix);
    }
    pb_status in_turn(bool, const std::function<pb_status(pb_index *)> &call) override;
    pb_status one(int64_t, const std::function<pb_status(pb_index *)> &call) override {
        std::shared_lock<std::shared_mutex> g(layout);
        return call(ranks[0]);
    }
};

extern "C" pb_status pb_index_load_devices(const char *index_dir, const int32_t *devices, int32_t n_devices,
                                           int32_t flags, pb_index **out) {
    if (!index_dir || !devices || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_devices < 1 || n_devices > 64)
        return pb_fail(PB_ERR_INVALID, "n_devices %d outside [1, 64] (the shard group's limit)", (int)n_devices);
    const int n = pb_device_count();
    if (n == 0) return pb_fail(PB_ERR_CUDA, "no CUDA device available; libplaid_b200 has no CPU fallback");
    for (int r = 0; r < n_devices; ++r)
        if (devices[r] < 0 || devices[r] >= n)
            return pb_fail(PB_ERR_INVALID, "devices[%d] = %d out of range (have %d)", r, (int)devices[r], n);
    std::vector<int64_t> b((size_t)n_devices + 1);
    pb_status s = pb_index_dir_shard_bounds(index_dir, n_devices, b.data());
    if (s != PB_OK) return s;

    std::unique_ptr<Deployment> d(new Deployment());
    d->devices.assign(devices, devices + n_devices);
    d->ranks.assign((size_t)n_devices, nullptr);
    d->scratch.resize((size_t)n_devices);
    if ((s = pb_shard_group_create(n_devices, &d->group)) != PB_OK) return s;
    d->workers.resize((size_t)n_devices);
    for (int r = 1; r < n_devices; ++r) d->workers[r].reset(new RankWorker(r));
    // the ranks load concurrently; the lowest failing rank's status and message, and nothing left behind
    s = d->run_one([&](int r) {
        return pb_index_load_range_flags(index_dir, devices[r], b[r], b[r + 1], flags, &d->ranks[r]);
    }, false);
    d->ranks.erase(std::remove(d->ranks.begin(), d->ranks.end(), nullptr), d->ranks.end());
    if (s != PB_OK) return s;  // ~Deployment closes the ranks that loaded
    if ((s = d->finish(out)) != PB_OK) return s;
    d.release();
    return PB_OK;
}

pb_status pb_dep_assemble(std::vector<pb_index *> ranks, const std::vector<int> &devices, pb_index **out) {
    const int n = (int)ranks.size();
    std::unique_ptr<Deployment> d(new Deployment());
    d->ranks = std::move(ranks);  // closed by ~Deployment on failure
    d->devices = devices;
    d->scratch.resize((size_t)n);
    pb_status s = pb_shard_group_create(n, &d->group);
    if (s != PB_OK) return s;
    d->workers.resize((size_t)n);
    for (int r = 1; r < n; ++r) d->workers[r].reset(new RankWorker(r));
    if ((s = d->finish(out)) != PB_OK) return s;
    d.release();
    return PB_OK;
}

pb_status pb_dep_search(Deployment *d, int64_t n_queries, int64_t stride, int64_t *out_ids, float *out_scores,
                        int32_t *out_counts,
                        const std::function<pb_status(pb_index *, int64_t *, float *, int32_t *)> &call) {
    std::lock_guard<std::mutex> g(d->mu);
    const size_t rows = (size_t)std::max<int64_t>(n_queries, 0), cells = rows * (size_t)std::max<int64_t>(stride, 0);
    for (int r = 1; r < d->world(); ++r) {
        SearchScratch &s = d->scratch[r];
        s.ids.resize(std::max<size_t>(cells, 1)), s.scores.resize(std::max<size_t>(cells, 1));
        s.counts.resize(std::max<size_t>(rows, 1));
    }
    return d->run_one([&](int r) {
        if (r == 0) return call(d->ranks[0], out_ids, out_scores, out_counts);
        SearchScratch &s = d->scratch[r];
        return call(d->ranks[r], out_ids ? s.ids.data() : nullptr, out_scores ? s.scores.data() : nullptr,
                    out_counts ? s.counts.data() : nullptr);
    });
}

void Deployment::totals(long long *D, long long *N) {
    std::shared_lock<std::shared_mutex> g(layout);
    *D = *N = 0;
    for (pb_index *ix : ranks) {
        *D += pb_index_num_documents(ix);
        *N += pb_index_num_embeddings(ix);
    }
}

pb_status Deployment::memory(int64_t *device_bytes, int64_t *host_bytes) {
    std::shared_lock<std::shared_mutex> g(layout);
    int64_t dev = 0, host = 0;
    for (pb_index *ix : ranks) {
        int64_t a = 0, b = 0;
        pb_status s = pb_index_memory(ix, &a, &b);
        if (s != PB_OK) return s;
        dev += a, host += b;
    }
    if (device_bytes) *device_bytes = dev;
    if (host_bytes) *host_bytes = host;
    return PB_OK;
}

pb_status Deployment::shard_layout(int32_t *out_world, int64_t *out_bounds, int32_t *out_devices) {
    std::shared_lock<std::shared_mutex> g(layout);
    std::vector<int64_t> base;
    pb_status s = bounds(base);
    if (s != PB_OK) return s;
    *out_world = world();
    if (out_bounds) std::copy(base.begin(), base.end(), out_bounds);
    if (out_devices) std::copy(devices.begin(), devices.end(), out_devices);
    return PB_OK;
}

// Each id goes to the rank holding it, in input order; the ranks run in parallel and write disjoint rows of the output
pb_status Deployment::decompress(const int64_t *doc_ids, int64_t n_docs, float *out_embeddings, int64_t *out_lengths) {
    if ((!doc_ids && n_docs) || !out_lengths) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_docs <= 0) return PB_OK;
    std::lock_guard<std::mutex> g(mu);  // the rank threads; mutations, which move the ranges, wait
    std::vector<int64_t> base;
    pb_status s = bounds(base);
    if (s != PB_OK) return s;
    const int W = world();
    std::vector<std::vector<int64_t>> ids((size_t)W), pos((size_t)W), lens((size_t)W);
    for (int64_t i = 0; i < n_docs; ++i) {
        out_lengths[i] = 0;  // an id no rank holds: length 0, as on one handle
        const int64_t id = doc_ids[i];
        if (id < base[0] || id >= base[W]) continue;
        const int r = (int)(std::upper_bound(base.begin(), base.end(), id) - base.begin()) - 1;  // skips empty ranks
        ids[r].push_back(id);
        pos[r].push_back(i);
    }
    s = run_one([&](int r) {
        lens[r].assign(ids[r].size(), 0);
        return ids[r].empty() ? PB_OK
                              : pb_decompress_documents(ranks[r], ids[r].data(), (int64_t)ids[r].size(), nullptr,
                                                        lens[r].data());
    }, false);
    if (s != PB_OK) return s;
    for (int r = 0; r < W; ++r)
        for (size_t j = 0; j < pos[r].size(); ++j) out_lengths[pos[r][j]] = lens[r][j];
    if (!out_embeddings) return PB_OK;
    std::vector<int64_t> start((size_t)n_docs + 1, 0);  // row of each input id in the output
    for (int64_t i = 0; i < n_docs; ++i) start[i + 1] = start[i] + out_lengths[i];
    const size_t dim = (size_t)pb_index_embedding_dim(ranks[0]);
    return run_one([&](int r) {
        int64_t rows = 0;
        for (int64_t l : lens[r]) rows += l;
        if (rows == 0) return PB_OK;
        std::vector<float> buf((size_t)rows * dim);
        std::vector<int64_t> got(ids[r].size());
        pb_status st = pb_decompress_documents(ranks[r], ids[r].data(), (int64_t)ids[r].size(), buf.data(), got.data());
        if (st != PB_OK) return st;
        const float *src = buf.data();
        for (size_t j = 0; j < pos[r].size(); ++j) {
            std::copy(src, src + (size_t)got[j] * dim, out_embeddings + (size_t)start[pos[r][j]] * dim);
            src += (size_t)got[j] * dim;
        }
        return PB_OK;
    }, false);
}

// Rank r fills columns [base[r], base[r + 1]) of each D_total-wide row
pb_status Deployment::exhaustive(const float *queries, const int64_t *q_off, int64_t n_queries, float *out_scores) {
    if ((!queries && n_queries) || !q_off || (!out_scores && n_queries)) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_queries <= 0) return PB_OK;
    std::lock_guard<std::mutex> g(mu);  // the rank threads; mutations, which move the ranges, wait
    std::vector<int64_t> base;
    pb_status s = bounds(base);
    if (s != PB_OK) return s;
    const size_t D = (size_t)(base[world()] - base[0]);
    return run_one([&](int r) {
        const size_t Dr = (size_t)(base[r + 1] - base[r]), c0 = (size_t)(base[r] - base[0]);
        if (Dr == 0) return PB_OK;
        std::vector<float> buf((size_t)n_queries * Dr);
        pb_status st = pb_exhaustive_scores(ranks[r], queries, q_off, n_queries, buf.data());
        if (st != PB_OK) return st;
        for (int64_t q = 0; q < n_queries; ++q)
            std::copy(buf.data() + (size_t)q * Dr, buf.data() + (size_t)(q + 1) * Dr, out_scores + (size_t)q * D + c0);
        return PB_OK;
    }, false);
}

pb_status Deployment::del(const int64_t *doc_ids, int64_t n_ids, const char *index_dir, int64_t *out_deleted) {
    std::lock_guard<std::mutex> g(mu);
    std::unique_lock<std::shared_mutex> l(layout);
    std::vector<int64_t> n((size_t)world(), 0);
    pb_status s = run_one([&](int r) {
        return pb_index_delete_sharded(ranks[r], doc_ids, n_ids, index_dir, &n[r]);
    });
    if (out_deleted) *out_deleted = s == PB_OK ? n[0] : 0;
    return s;
}

pb_status Deployment::in_turn(bool, const std::function<pb_status(pb_index *)> &call) {
    std::shared_lock<std::shared_mutex> g(layout);
    for (int r = 0; r < world(); ++r)
        if (pb_status s = call(ranks[r])) {
            const std::string e = pb_last_error();
            return world() == 1 ? s : pb_fail(s, "rank %d: %s", r, e.c_str());
        }
    return PB_OK;
}

// Only the last rank receives the codec and the documents: an append goes to the end of the deployment
pb_status Deployment::append(pb_codec *codec, const float *embeddings, const int64_t *codes, const uint8_t *residuals,
                             const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space, const char *index_dir,
                             int64_t batch_size, int64_t *out_first_doc_id) {
    std::lock_guard<std::mutex> g(mu);
    std::unique_lock<std::shared_mutex> l(layout);
    const int last = world() - 1;
    std::vector<int64_t> first((size_t)world(), 0);
    pb_status s = run_one([&](int r) {
        pb_index *ix = ranks[r];
        const bool mine = r == last;
        if (codec)
            return pb_index_append_sharded(ix, mine ? codec : nullptr, mine ? embeddings : nullptr, doc_lengths, n_docs,
                                           memory_space, index_dir, batch_size, &first[r]);
        return pb_index_append_encoded_sharded(ix, mine ? codes : nullptr, mine ? residuals : nullptr, doc_lengths,
                                               n_docs, memory_space, &first[r]);
    });
    if (s == PB_OK && out_first_doc_id) *out_first_doc_id = first[0];
    return s;
}

pb_status Deployment::rebalance(const int64_t *bounds, int64_t *out_bounds) {
    std::lock_guard<std::mutex> g(mu);
    std::unique_lock<std::shared_mutex> l(layout);
    const size_t W1 = (size_t)world() + 1;
    std::vector<std::vector<int64_t>> got((size_t)world(), std::vector<int64_t>(W1, 0));
    pb_status s = run_one([&](int r) { return pb_index_rebalance_sharded(ranks[r], bounds, got[r].data()); });
    if (s == PB_OK && out_bounds) std::copy(got[0].begin(), got[0].end(), out_bounds);
    return s;
}

// bounds [W + 1] (host) tile [0, D): non-decreasing from 0 to D
static pb_status check_tiling(const int64_t *b, int W, long long D) {
    bool ok = b[0] == 0 && b[W] == D;
    for (int r = 0; r < W; ++r) ok = ok && b[r] <= b[r + 1];
    if (ok) return PB_OK;
    return pb_fail(PB_ERR_INVALID, "bounds must be non-decreasing from 0 to D_total = %lld over the %d ranks of the new "
                   "world", D, W);
}

// New ranks open empty after the last one, every rank moves to a group of the new world, and the rebalance moves the
// documents.  If the rebalance fails every rank is as it was: the old ranks go back to their group (never used in the
// meantime, so whole) and the new ones are closed.
pb_status pb_dep_add_devices(Deployment *d, const int32_t *devices, int32_t n, const int64_t *bounds, int64_t *out_bounds) {
    std::lock_guard<std::mutex> g(d->mu);
    std::unique_lock<std::shared_mutex> l(d->layout);
    const int W = d->world();
    if (n < 1 || W + n > 64)
        return pb_fail(PB_ERR_INVALID, "adding %d ranks to %d: the new world must be in [%d, 64] (the shard group's limit)",
                       (int)n, W, W + 1);
    const int have = pb_device_count();
    for (int i = 0; i < n; ++i)
        if (devices[i] < 0 || devices[i] >= have)
            return pb_fail(PB_ERR_INVALID, "devices[%d] = %d out of range (have %d)", i, (int)devices[i], have);
    const int W1 = W + n;
    std::vector<int64_t> base;
    pb_status s = d->bounds(base);
    if (s == PB_OK && bounds) s = check_tiling(bounds, W1, base[W]);
    if (s != PB_OK) return s;
    std::vector<pb_index *> prev = d->ranks, next = d->ranks;
    std::vector<int> prev_dev = d->devices, devs = d->devices;
    auto drop = [&] {
        for (int r = W; r < (int)next.size(); ++r) pb_index_close(next[r]);
    };
    for (int i = 0; i < n && s == PB_OK; ++i) {
        pb_index *e = nullptr;
        s = pb_index_clone_empty(d->ranks[0], devices[i], base[W], &e);
        if (s == PB_OK) next.push_back(e), devs.push_back(devices[i]);
    }
    pb_shard_group *g1 = nullptr;
    if (s == PB_OK) s = pb_shard_group_create(W1, &g1);
    if (s != PB_OK) {
        drop();
        return s;
    }
    pb_shard_group *g0 = d->group;
    d->reform(next, devs, g1);
    std::vector<std::vector<int64_t>> got((size_t)W1, std::vector<int64_t>((size_t)W1 + 1, 0));
    s = d->run_one([&](int r) { return pb_index_rebalance_sharded(d->ranks[r], bounds, got[r].data()); });
    if (s != PB_OK) {
        const std::string e = pb_last_error();
        d->reform(prev, prev_dev, g0);
        drop();
        pb_shard_group_destroy(g1);
        return pb_fail(s, "%s", e.c_str());
    }
    pb_shard_group_destroy(g0);
    if (out_bounds) std::copy(got[0].begin(), got[0].end(), out_bounds);
    return PB_OK;
}

// The rebalance runs over the current group, the leaving ranks taking empty ranges at their positions; then they are
// closed and the others move, in their order, to a group of the new world (created first, so that nothing can fail
// after the documents have moved).  If the rebalance fails every rank is as it was.
pb_status pb_dep_remove_ranks(Deployment *d, pb_index *handle, const int32_t *ranks, int32_t n, const int64_t *bounds,
                              int64_t *out_bounds) {
    std::lock_guard<std::mutex> g(d->mu);
    std::unique_lock<std::shared_mutex> l(d->layout);
    const int W = d->world();
    if (n < 1 || n >= W)
        return pb_fail(PB_ERR_INVALID, "removing %d of %d ranks: at least one must leave and one stay", (int)n, W);
    std::vector<uint8_t> stays((size_t)W, 1);
    for (int i = 0; i < n; ++i) {
        const int r = ranks[i];
        if (r < 0 || r >= W) return pb_fail(PB_ERR_INVALID, "ranks[%d] = %d outside [0, %d)", i, r, W);
        if (!stays[r]) return pb_fail(PB_ERR_INVALID, "rank %d is listed twice", r);
        stays[r] = 0;
    }
    const int W1 = W - n;
    std::vector<int64_t> base, b;
    pb_status s = d->bounds(base);
    if (s == PB_OK && bounds) s = check_tiling(bounds, W1, base[W]);
    if (s != PB_OK) return s;
    if (bounds) {  // over the old world: a leaving rank gets the empty range where the next staying rank starts
        b.assign((size_t)W + 1, base[W]);
        for (int r = 0, j = 0; r < W; ++r) {
            b[r] = bounds[j];
            j += stays[r];
        }
    }
    pb_shard_group *g1 = nullptr;
    if ((s = pb_shard_group_create(W1, &g1)) != PB_OK) return s;
    std::vector<std::vector<int64_t>> got((size_t)W, std::vector<int64_t>((size_t)W + 1, 0));
    s = d->run_one([&](int r) {
        return pb_index_rebalance_shares(d->ranks[r], bounds ? b.data() : nullptr, bounds ? nullptr : stays.data(),
                                         got[r].data());
    });
    if (s != PB_OK) {
        pb_shard_group_destroy(g1);
        return s;
    }
    std::vector<pb_index *> next, gone;
    std::vector<int> devs;
    for (int r = 0; r < W; ++r) {
        (stays[r] ? next : gone).push_back(d->ranks[r]);
        if (stays[r]) devs.push_back(d->devices[r]);
    }
    pb_shard_group *g0 = d->group;
    d->reform(next, devs, g1);
    for (pb_index *x : gone) pb_index_close(x);
    pb_shard_group_destroy(g0);
    pb_index_deployment_rank0(handle, d->ranks[0]);
    if (out_bounds) {
        for (int r = 0, j = 0; r < W; ++r)
            if (stays[r]) out_bounds[j++] = got[0][r];
        out_bounds[W1] = base[W];
    }
    return PB_OK;
}
