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

struct Deployment {
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

    // joins the loaded ranks in the group and makes the handle; on failure the caller deletes this
    pb_status finish(pb_index **out) {
        for (int r = 0; r < world(); ++r) {
            pb_status s = pb_index_group_join(ranks[r], group, r);
            if (s != PB_OK) return s;
        }
        *out = pb_index_new_deployment(this, ranks[0]);
        return PB_OK;
    }

    ~Deployment() {
        workers.clear();  // joins the threads
        for (pb_index *ix : ranks) pb_index_close(ix);
        pb_shard_group_destroy(group);
    }
};

pb_index *pb_dep_rank(Deployment *d, int r) { return d->ranks[r]; }
void pb_dep_close(Deployment *d) { delete d; }

void pb_dep_each(Deployment *d, const std::function<void(pb_index *)> &call) {
    for (pb_index *ix : d->ranks) call(ix);
}

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

pb_status pb_dep_totals(Deployment *d, long long *D, long long *N) {
    std::shared_lock<std::shared_mutex> g(d->layout);
    *D = *N = 0;
    for (pb_index *ix : d->ranks) {
        *D += pb_index_num_documents(ix);
        *N += pb_index_num_embeddings(ix);
    }
    return PB_OK;
}

pb_status pb_dep_memory(Deployment *d, int64_t *device_bytes, int64_t *host_bytes) {
    std::shared_lock<std::shared_mutex> g(d->layout);
    int64_t dev = 0, host = 0;
    for (pb_index *ix : d->ranks) {
        int64_t a = 0, b = 0;
        pb_status s = pb_index_memory(ix, &a, &b);
        if (s != PB_OK) return s;
        dev += a, host += b;
    }
    if (device_bytes) *device_bytes = dev;
    if (host_bytes) *host_bytes = host;
    return PB_OK;
}

pb_status pb_dep_layout(Deployment *d, int32_t *out_world, int64_t *out_bounds, int32_t *out_devices) {
    std::shared_lock<std::shared_mutex> g(d->layout);
    std::vector<int64_t> base;
    pb_status s = d->bounds(base);
    if (s != PB_OK) return s;
    *out_world = d->world();
    if (out_bounds) std::copy(base.begin(), base.end(), out_bounds);
    if (out_devices) std::copy(d->devices.begin(), d->devices.end(), out_devices);
    return PB_OK;
}

// Each id goes to the rank holding it, in input order; the ranks run in parallel and write disjoint rows of the output
pb_status pb_dep_decompress(Deployment *d, const int64_t *doc_ids, int64_t n_docs, float *out_embeddings,
                            int64_t *out_lengths) {
    if ((!doc_ids && n_docs) || !out_lengths) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_docs <= 0) return PB_OK;
    std::lock_guard<std::mutex> g(d->mu);  // the rank threads; mutations, which move the ranges, wait
    std::vector<int64_t> base;
    pb_status s = d->bounds(base);
    if (s != PB_OK) return s;
    const int W = d->world();
    std::vector<std::vector<int64_t>> ids((size_t)W), pos((size_t)W), lens((size_t)W);
    for (int64_t i = 0; i < n_docs; ++i) {
        out_lengths[i] = 0;  // an id no rank holds: length 0, as on one handle
        const int64_t id = doc_ids[i];
        if (id < base[0] || id >= base[W]) continue;
        const int r = (int)(std::upper_bound(base.begin(), base.end(), id) - base.begin()) - 1;  // skips empty ranks
        ids[r].push_back(id);
        pos[r].push_back(i);
    }
    s = d->run_one([&](int r) {
        lens[r].assign(ids[r].size(), 0);
        return ids[r].empty() ? PB_OK
                              : pb_decompress_documents(d->ranks[r], ids[r].data(), (int64_t)ids[r].size(), nullptr,
                                                        lens[r].data());
    }, false);
    if (s != PB_OK) return s;
    for (int r = 0; r < W; ++r)
        for (size_t j = 0; j < pos[r].size(); ++j) out_lengths[pos[r][j]] = lens[r][j];
    if (!out_embeddings) return PB_OK;
    std::vector<int64_t> start((size_t)n_docs + 1, 0);  // row of each input id in the output
    for (int64_t i = 0; i < n_docs; ++i) start[i + 1] = start[i] + out_lengths[i];
    const size_t dim = (size_t)pb_index_embedding_dim(d->ranks[0]);
    return d->run_one([&](int r) {
        int64_t rows = 0;
        for (int64_t l : lens[r]) rows += l;
        if (rows == 0) return PB_OK;
        std::vector<float> buf((size_t)rows * dim);
        std::vector<int64_t> got(ids[r].size());
        pb_status st = pb_decompress_documents(d->ranks[r], ids[r].data(), (int64_t)ids[r].size(), buf.data(), got.data());
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
pb_status pb_dep_exhaustive(Deployment *d, const float *queries, const int64_t *q_off, int64_t n_queries,
                            float *out_scores) {
    if ((!queries && n_queries) || !q_off || (!out_scores && n_queries)) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_queries <= 0) return PB_OK;
    std::lock_guard<std::mutex> g(d->mu);  // the rank threads; mutations, which move the ranges, wait
    std::vector<int64_t> base;
    pb_status s = d->bounds(base);
    if (s != PB_OK) return s;
    const size_t D = (size_t)(base[d->world()] - base[0]);
    return d->run_one([&](int r) {
        const size_t Dr = (size_t)(base[r + 1] - base[r]), c0 = (size_t)(base[r] - base[0]);
        if (Dr == 0) return PB_OK;
        std::vector<float> buf((size_t)n_queries * Dr);
        pb_status st = pb_exhaustive_scores(d->ranks[r], queries, q_off, n_queries, buf.data());
        if (st != PB_OK) return st;
        for (int64_t q = 0; q < n_queries; ++q)
            std::copy(buf.data() + (size_t)q * Dr, buf.data() + (size_t)(q + 1) * Dr, out_scores + (size_t)q * D + c0);
        return PB_OK;
    }, false);
}

pb_status pb_dep_delete(Deployment *d, const int64_t *doc_ids, int64_t n_ids, const char *index_dir, int64_t *out_deleted) {
    std::lock_guard<std::mutex> g(d->mu);
    std::unique_lock<std::shared_mutex> l(d->layout);
    std::vector<int64_t> n((size_t)d->world(), 0);
    pb_status s = d->run_one([&](int r) {
        return pb_index_delete_sharded(d->ranks[r], doc_ids, n_ids, index_dir, &n[r]);
    });
    if (out_deleted) *out_deleted = s == PB_OK ? n[0] : 0;
    return s;
}

// Only the last rank receives the codec and the documents: an append goes to the end of the deployment
pb_status pb_dep_append(Deployment *d, pb_codec *codec, const float *embeddings, const int64_t *codes,
                        const uint8_t *residuals, const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space,
                        const char *index_dir, int64_t batch_size, int64_t *out_first_doc_id) {
    std::lock_guard<std::mutex> g(d->mu);
    std::unique_lock<std::shared_mutex> l(d->layout);
    const int last = d->world() - 1;
    std::vector<int64_t> first((size_t)d->world(), 0);
    pb_status s = d->run_one([&](int r) {
        pb_index *ix = d->ranks[r];
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

pb_status pb_dep_rebalance(Deployment *d, const int64_t *bounds, int64_t *out_bounds) {
    std::lock_guard<std::mutex> g(d->mu);
    std::unique_lock<std::shared_mutex> l(d->layout);
    const size_t W1 = (size_t)d->world() + 1;
    std::vector<std::vector<int64_t>> got((size_t)d->world(), std::vector<int64_t>(W1, 0));
    pb_status s = d->run_one([&](int r) { return pb_index_rebalance_sharded(d->ranks[r], bounds, got[r].data()); });
    if (s == PB_OK && out_bounds) std::copy(got[0].begin(), got[0].end(), out_bounds);
    return s;
}
