// replicas.cpp -- an index directory replicated over several devices of this process behind one pb_index handle
// (pb_index_load_replicas, DESIGN.md 4q).  Host code only: each replica is an ordinary handle (S = 1) or a deployment of
// pb_index_load_devices (S > 1), driven through the public entry points.
//
// Routing: a call of n queries is cut into k = min(R, ceil(n / SLICE_MIN)) contiguous slices, each served by one of the
// k least-loaded replicas (queries in flight; ties to the lowest index).  Slice 0 runs on the caller's thread; the others
// on a crew of helper threads taken from the set's pool, so that concurrent callers each cut their own call.
// Consistency: routed calls hold `rw` shared, mutations alone (with `gate` first, so that a stream of searches cannot
// starve a mutation): a search sees every replica before a mutation or every replica after it.
// Resizes (DESIGN §4u): mutations, row-cache changes and resizes also take `change` first, one at a time, so that an
// add copies replica 0 while searches go on and no mutation can come between its copies; the member list, the devices
// and the routing counters change under `rw` alone and `mu`, where every reader of them looks.
#include "engine_internal.h"

#include <algorithm>
#include <memory>
#include <mutex>
#include <numeric>
#include <shared_mutex>

namespace {

// The fewest queries a slice gets: below it a slice's fixed cost (its own sub-batch, score table and transfers) outweighs
// what another replica adds (DESIGN §4q)
constexpr int64_t SLICE_MIN = 32;

// Idle crews a set keeps: more concurrent cut calls than this create their crews for the call
constexpr size_t MAX_IDLE_CREWS = 2;

struct Crew {  // helper threads of one routed call: slices 1..R-1
    std::vector<std::unique_ptr<RankWorker>> w;
};

}  // namespace

struct Replicas : Group {
    int S = 1;
    std::vector<pb_index *> members;  // [R]: plain handles (S = 1) or deployments (S > 1)
    std::vector<int> devices;         // [R * S]
    std::mutex change;  // one mutation, row-cache change or resize at a time; taken before gate
    std::mutex gate;
    std::shared_mutex rw;
    std::mutex mu;  // the counters and the crews; R changes under it too (pb_rep_sized)
    std::vector<int64_t> inflight, calls, queries;
    std::vector<std::unique_ptr<Crew>> crews;

    int R() const { return (int)members.size(); }
    std::shared_lock<std::shared_mutex> read_lock() {
        { std::lock_guard<std::mutex> g(gate); }
        return std::shared_lock<std::shared_mutex>(rw);
    }
    // the share.size() least-loaded replicas, ties to the lowest index; each takes its share of queries
    std::vector<int> pick(const std::vector<int64_t> &share) {
        std::lock_guard<std::mutex> g(mu);
        std::vector<int> order((size_t)R());
        std::iota(order.begin(), order.end(), 0);
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return inflight[a] < inflight[b]; });
        order.resize(share.size());
        for (size_t i = 0; i < share.size(); ++i) {
            inflight[order[i]] += share[i];
            calls[order[i]] += 1;
            queries[order[i]] += share[i];
        }
        return order;
    }
    void done(const std::vector<int> &who, const std::vector<int64_t> &share) {
        std::lock_guard<std::mutex> g(mu);
        for (size_t i = 0; i < who.size(); ++i) inflight[who[i]] -= share[i];
    }
    std::unique_ptr<Crew> take_crew() {
        {
            std::lock_guard<std::mutex> g(mu);
            if (!crews.empty()) {
                std::unique_ptr<Crew> c = std::move(crews.back());
                crews.pop_back();
                return c;
            }
        }
        std::unique_ptr<Crew> c(new Crew());
        for (int i = 1; i < R(); ++i) c->w.emplace_back(new RankWorker(i));
        return c;
    }
    // at most MAX_IDLE_CREWS crews stay for later calls; a crew beyond them, or of another R, is joined here
    void give_crew(std::unique_ptr<Crew> c) {
        std::unique_lock<std::mutex> g(mu);
        if (crews.size() < MAX_IDLE_CREWS && (int)c->w.size() == R() - 1) crews.push_back(std::move(c));
        g.unlock();
        c.reset();
    }
    // op(member, g) on every replica at once, slice-thread style (replica 0 on the caller's thread); the lowest failing
    // replica's status and message.  With a vote (S > 1 mutations) the replicas' ranks take it together.
    pb_status at_once(const std::function<pb_status(pb_index *, int)> &op, RepVote *vote = nullptr) {
        for (int g = 0; g < R() && vote; ++g) pb_index_set_rep_vote(members[g], vote, g);
        std::unique_ptr<Crew> crew = take_crew();
        std::vector<pb_status> st;
        std::vector<std::string> err;
        run_slots(R(), [&](int g) { return op(members[g], g); }, crew->w.data(), st, err);
        give_crew(std::move(crew));
        for (int g = 0; g < R() && vote; ++g) pb_index_set_rep_vote(members[g], nullptr, 0);
        for (int g = 0; g < R(); ++g)
            if (st[g] != PB_OK)
                return g == 0 ? pb_fail(st[0], "%s", err[0].c_str())
                              : pb_fail(st[g], "replica %d: %s", g, err[g].c_str());
        return PB_OK;
    }
    // at_once() of a mutation on deployments, with the vote that makes it commit on every replica or on none
    pb_status voted(bool with_dir, bool share_rows, const std::function<pb_status(pb_index *, int)> &op) {
        std::unique_ptr<RepVote, void (*)(RepVote *)> v(pb_rep_vote_new(R() * S, with_dir, share_rows), pb_rep_vote_free);
        return at_once(op, v.get());
    }
    // joins the threads, closes the replicas
    ~Replicas() override {
        crews.clear();  // joins the threads
        for (pb_index *m : members)
            if (m) pb_index_close(m);
    }

    const char *kind() const override { return "a replica set (pb_index_load_replicas)"; }
    Replicas *as_replicas() override { return this; }
    pb_index *member(int g) override { return members[g]; }  // the caller holds rw or change
    pb_status first(const std::function<pb_status(pb_index *)> &call) override {
        auto rd = read_lock();
        return call(members[0]);
    }
    // what every replica holds, from replica 0
    void totals(long long *D, long long *N) override {
        first([&](pb_index *m) { return pb_index_totals(m, D, N), PB_OK; });
    }
    pb_status shard_layout(int32_t *out_world, int64_t *out_bounds, int32_t *out_devices) override {
        return first([&](pb_index *m) { return pb_index_shard_layout(m, out_world, out_bounds, out_devices); });
    }
    pb_status last_delete_ms(float *out_ms) override {
        return first([&](pb_index *m) { return pb_last_delete_ms(m, out_ms); });  // the set's last delete ran there too
    }
    pb_status memory(int64_t *device_bytes, int64_t *host_bytes) override;
    // the mutations, under the set's writer lock
    pb_status append(pb_codec *codec, const float *embeddings, const int64_t *codes, const uint8_t *residuals,
                     const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space, const char *index_dir,
                     int64_t batch_size, int64_t *out_first_doc_id) override;
    pb_status del(const int64_t *doc_ids, int64_t n_ids, const char *index_dir, int64_t *out_deleted) override;
    pb_status rebalance(const int64_t *bounds, int64_t *out_bounds) override;
    pb_status reserve(int64_t num_documents, int64_t num_embeddings) override;
    // the readers of one whole copy, on the least-loaded replica
    pb_status decompress(const int64_t *doc_ids, int64_t n_docs, float *out_embeddings, int64_t *out_lengths) override {
        return one(0, [&](pb_index *m) { return pb_decompress_documents(m, doc_ids, n_docs, out_embeddings, out_lengths); });
    }
    pb_status exhaustive(const float *queries, const int64_t *q_off, int64_t n_queries, float *out_scores) override {
        return one(0, [&](pb_index *m) { return pb_exhaustive_scores(m, queries, q_off, n_queries, out_scores); });
    }
    pb_status export_ivf(int64_t *out_ivf, int32_t *out_lengths, int64_t *out_total) override {
        return one(0, [&](pb_index *m) { return pb_index_export_ivf(m, out_ivf, out_lengths, out_total); });
    }
    // the replicas as they are: a resize publishes under the writer lock and gives new replicas replica 0's switches
    void each(const std::function<void(pb_index *)> &call) override {
        auto rd = read_lock();
        for (pb_index *m : members) call(m);
    }
    pb_status in_turn(bool writer, const std::function<pb_status(pb_index *)> &call) override;
    pb_status one(int64_t n, const std::function<pb_status(pb_index *)> &call) override;
};

// One replica copied from m0 (a plain handle, or a deployment of S ranks) onto devices dv[0 .. S-1], device to device:
// a pb_index_clone of each of its ranks, joined as a deployment when S > 1
static pb_status copy_replica(pb_index *m0, int S, const int32_t *dv, pb_index **out) {
    if (S == 1) return pb_index_clone(m0, dv[0], out);
    std::vector<pb_index *> ranks;
    for (int r = 0; r < S; ++r) {
        pb_index *c = nullptr;
        const pb_status st = pb_index_clone(pb_rank_of(m0, r), dv[r], &c);
        if (st != PB_OK) {
            for (pb_index *x : ranks) pb_index_close(x);
            return st;
        }
        ranks.push_back(c);
    }
    return pb_dep_assemble(ranks, std::vector<int>(dv, dv + S), out);
}

// n replicas copied from m0 concurrently, one library thread per replica (the caller's current device stays as it
// was), copy i onto devices[i*S .. i*S + S-1].  On failure the lowest failing copy's status and message, and every
// copy made is closed.
static pb_status copy_replicas(pb_index *m0, int S, const int32_t *devices, int n, std::vector<pb_index *> &out) {
    out.assign((size_t)n, nullptr);
    const Job copy = [&](int i) { return copy_replica(m0, S, devices + (size_t)i * S, &out[i]); };
    std::vector<std::unique_ptr<RankWorker>> w;
    for (int i = 0; i < n; ++i) w.emplace_back(new RankWorker(i));
    for (auto &x : w) x->submit(copy);
    for (auto &x : w) x->wait();
    for (auto &x : w)
        if (x->status != PB_OK) {
            for (pb_index *c : out) pb_index_close(c);  // null for the copies that failed
            out.clear();
            return pb_fail(x->status, "%s", x->error.c_str());
        }
    return PB_OK;
}

extern "C" pb_status pb_index_load_replicas(const char *index_dir, const int32_t *devices, int32_t n_devices,
                                            int32_t n_shards, int32_t flags, pb_index **out) {
    if (!index_dir || !devices || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_shards < 1) return pb_fail(PB_ERR_INVALID, "n_shards %d < 1", (int)n_shards);
    if (n_devices < 1 || n_devices % n_shards != 0)
        return pb_fail(PB_ERR_INVALID, "n_devices %d is not a positive multiple of n_shards %d", (int)n_devices,
                       (int)n_shards);
    if (n_devices > PB_MAX_MEMBERS) return pb_fail(PB_ERR_INVALID, "n_devices %d above 64 members", (int)n_devices);
    const int n = pb_device_count();
    if (n == 0) return pb_fail(PB_ERR_CUDA, "no CUDA device available; libplaid_b200 has no CPU fallback");
    for (int i = 0; i < n_devices; ++i)
        if (devices[i] < 0 || devices[i] >= n)
            return pb_fail(PB_ERR_INVALID, "devices[%d] = %d out of range (have %d)", i, (int)devices[i], n);
    *out = nullptr;
    const int R = n_devices / n_shards, S = n_shards;
    std::unique_ptr<Replicas> rs(new Replicas());
    rs->S = S;
    rs->devices.assign(devices, devices + n_devices);
    rs->members.assign((size_t)R, nullptr);
    rs->inflight.assign((size_t)R, 0), rs->calls.assign((size_t)R, 0), rs->queries.assign((size_t)R, 0);
    // replica 0 from the directory
    pb_status s = S == 1 ? pb_index_load_range_flags(index_dir, devices[0], 0, -1, flags, &rs->members[0])
                         : pb_index_load_devices(index_dir, devices, S, flags, &rs->members[0]);
    if (s != PB_OK) return s;
    pb_index *m0 = rs->members[0];
    std::vector<pb_index *> copies;
    if ((s = copy_replicas(m0, S, devices + S, R - 1, copies)) != PB_OK) return s;
    std::copy(copies.begin(), copies.end(), rs->members.begin() + 1);
    *out = pb_index_new_group(rs.get(), m0);
    rs.release();
    return PB_OK;
}

pb_status pb_rep_search(Replicas *rs, int64_t n, const std::function<pb_status(pb_index *, int64_t, int64_t, int)> &call) {
    auto rd = rs->read_lock();
    const int k = (int)std::max<int64_t>(1, std::min<int64_t>(rs->R(), (n + SLICE_MIN - 1) / SLICE_MIN));
    std::vector<int64_t> b((size_t)k + 1), share((size_t)k);
    for (int i = 0; i <= k; ++i) b[i] = n * i / k;
    for (int i = 0; i < k; ++i) share[i] = b[i + 1] - b[i];
    const std::vector<int> who = rs->pick(share);
    std::unique_ptr<Crew> crew;
    if (k > 1) crew = rs->take_crew();
    std::vector<pb_status> st;
    std::vector<std::string> err;
    run_slots(k, [&](int i) { return call(rs->members[who[i]], b[i], b[i + 1], i); }, crew ? crew->w.data() : nullptr,
              st, err);
    if (crew) rs->give_crew(std::move(crew));
    rs->done(who, share);
    for (int i = 0; i < k; ++i)
        if (st[i] != PB_OK) return pb_fail(st[i], "%s", err[i].c_str());
    return PB_OK;
}

pb_status Replicas::one(int64_t n, const std::function<pb_status(pb_index *)> &call) {
    auto rd = read_lock();
    const std::vector<int64_t> share(1, std::max<int64_t>(n, 0));
    const std::vector<int> who = pick(share);
    const pb_status st = call(members[who[0]]);
    done(who, share);
    return st;
}

// device bytes over every member; host bytes once: every replica reads replica 0's pinned arrays
pb_status Replicas::memory(int64_t *device_bytes, int64_t *host_bytes) {
    auto rd = read_lock();
    int64_t dev = 0, host = 0;
    for (int g = 0; g < R(); ++g) {
        int64_t a = 0, h = 0;
        pb_status s = pb_index_memory(members[g], &a, &h);
        if (s != PB_OK) return s;
        dev += a;
        if (g == 0) host = h;
    }
    if (device_bytes) *device_bytes = dev;
    if (host_bytes) *host_bytes = host;
    return PB_OK;
}

// A mutable host-tier set: replica 0 grows and rewrites the row stores every replica reads, so no replica may have
// work in flight when a mutation starts (the set's writer lock keeps new work out until it ends)
static pb_status quiesce(Replicas *rs) {
    if (!pb_host_rows_shared(rs->members[0])) return PB_OK;
    for (pb_index *m : rs->members)
        if (pb_status s = pb_sync_devices(m)) return s;
    return PB_OK;
}

pb_status Replicas::del(const int64_t *doc_ids, int64_t n_ids, const char *index_dir, int64_t *out_deleted) {
    std::lock_guard<std::mutex> c(change);
    std::lock_guard<std::mutex> g(gate);
    std::unique_lock<std::shared_mutex> wr(rw);
    if (pb_status s = quiesce(this)) return s;
    if (S == 1) return pb_members_delete(members, doc_ids, n_ids, index_dir, out_deleted);
    // replica 0 writes the directory
    return voted(index_dir != nullptr, false, [&](pb_index *m, int r) {
        int64_t d = 0;
        const pb_status s = pb_index_delete(m, doc_ids, n_ids, r == 0 ? index_dir : nullptr, &d);
        if (r == 0 && out_deleted) *out_deleted = d;
        return s;
    });
}

pb_status Replicas::append(pb_codec *codec, const float *embeddings, const int64_t *codes, const uint8_t *residuals,
                           const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space, const char *index_dir,
                           int64_t batch_size, int64_t *out_first_doc_id) {
    std::lock_guard<std::mutex> c(change);
    std::lock_guard<std::mutex> g(gate);
    std::unique_lock<std::shared_mutex> wr(rw);
    if (pb_status s = quiesce(this)) return s;
    if (S == 1)
        return pb_members_append(members, codec, embeddings, codes, residuals, doc_lengths, n_docs, memory_space,
                                 index_dir, batch_size, out_first_doc_id);
    // with a codec replica 0's last rank encodes and writes the directory; the other replicas append its rows.  On a
    // mutable host tier they also wait for it without a codec: its prepare writes the rows they read
    return voted(index_dir != nullptr, codec != nullptr || pb_host_rows_shared(members[0]),
                     [&](pb_index *m, int r) -> pb_status {
        if (r == 0)
            return codec ? pb_index_append(m, codec, embeddings, doc_lengths, n_docs, memory_space, index_dir, batch_size,
                                           out_first_doc_id)
                         : pb_index_append_encoded(m, codes, residuals, doc_lengths, n_docs, memory_space,
                                                   out_first_doc_id);
        return pb_index_append_encoded(m, codes, residuals, doc_lengths, n_docs, memory_space, nullptr);
    });
}

// Capacity only: a replica that reserved before another failed keeps it, and no result depends on it
pb_status Replicas::reserve(int64_t num_documents, int64_t num_embeddings) {
    std::lock_guard<std::mutex> c(change);
    std::lock_guard<std::mutex> g(gate);
    std::unique_lock<std::shared_mutex> wr(rw);
    if (pb_status s = quiesce(this)) return s;
    return at_once([&](pb_index *m, int) { return pb_index_reserve(m, num_documents, num_embeddings); });
}

pb_status Replicas::rebalance(const int64_t *bounds, int64_t *out_bounds) {
    std::lock_guard<std::mutex> c(change);
    std::lock_guard<std::mutex> g(gate);
    std::unique_lock<std::shared_mutex> wr(rw);
    return voted(false, false, [&](pb_index *m, int r) {
        return pb_index_rebalance_sharded(m, bounds, r == 0 ? out_bounds : nullptr);
    });
}

pb_status Replicas::in_turn(bool writer, const std::function<pb_status(pb_index *)> &call) {
    std::unique_lock<std::mutex> c(change, std::defer_lock);
    if (writer) c.lock();
    std::unique_lock<std::mutex> g(gate);
    std::unique_lock<std::shared_mutex> wr(rw, std::defer_lock);
    std::shared_lock<std::shared_mutex> rd(rw, std::defer_lock);
    if (writer) wr.lock();
    else g.unlock(), rd.lock();
    for (int i = 0; i < R(); ++i)
        if (pb_status s = call(members[i])) {
            const std::string e = pb_last_error();
            return i == 0 ? s : pb_fail(s, "replica %d: %s", i, e.c_str());
        }
    return PB_OK;
}

extern "C" pb_status pb_index_replica_layout(const pb_index *ix, int32_t *out_replicas, int32_t *out_shards,
                                             int32_t *out_devices) {
    if (!ix || !out_replicas || !out_shards) return pb_fail(PB_ERR_INVALID, "null argument");
    Replicas *rs = pb_replicas_of(ix);
    if (!rs) {  // any other handle is one replica of its own ranks
        int32_t world = 0;
        std::vector<int32_t> dev(64);
        pb_status s = pb_index_shard_layout(ix, &world, nullptr, dev.data());
        if (s != PB_OK) return s;
        *out_replicas = 1, *out_shards = world;
        if (out_devices) std::copy(dev.begin(), dev.begin() + world, out_devices);
        return PB_OK;
    }
    auto rd = rs->read_lock();
    *out_replicas = rs->R(), *out_shards = rs->S;
    if (out_devices) std::copy(rs->devices.begin(), rs->devices.end(), out_devices);
    return PB_OK;
}

extern "C" pb_status pb_index_replica_stats(pb_index *ix, int64_t *out_calls, int64_t *out_queries, int32_t reset) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    Replicas *rs = pb_replicas_of(ix);
    if (!rs) return pb_fail(PB_ERR_INVALID, "not a replica set (pb_index_load_replicas)");
    std::lock_guard<std::mutex> g(rs->mu);
    if (out_calls) std::copy(rs->calls.begin(), rs->calls.end(), out_calls);
    if (out_queries) std::copy(rs->queries.begin(), rs->queries.end(), out_queries);
    if (reset) std::fill(rs->calls.begin(), rs->calls.end(), 0), std::fill(rs->queries.begin(), rs->queries.end(), 0);
    return PB_OK;
}

void pb_rep_sized(Replicas *rs, const std::function<void(int)> &call) {
    std::lock_guard<std::mutex> g(rs->mu);
    call(rs->R());
}

// The set after a resize: next[g] becomes replica g with its devices, counters (a new replica's at 0) and the handle's
// coalescing limit follow, and the idle crews (R - 1 helpers each) are handed back to be joined after the locks.  Under
// change, gate and rw alone; cannot fail.
static std::vector<std::unique_ptr<Crew>> publish(Replicas *rs, pb_index *handle, std::vector<pb_index *> next,
                                                  std::vector<int> devs, const std::vector<int> &from) {
    std::lock_guard<std::mutex> g(rs->mu);
    std::vector<int64_t> inflight, calls, queries;
    for (int f : from) {
        inflight.push_back(f < 0 ? 0 : rs->inflight[f]);
        calls.push_back(f < 0 ? 0 : rs->calls[f]);
        queries.push_back(f < 0 ? 0 : rs->queries[f]);
    }
    const bool first_changed = next[0] != rs->members[0];
    rs->members = std::move(next);
    rs->devices = std::move(devs);
    rs->inflight.swap(inflight), rs->calls.swap(calls), rs->queries.swap(queries);
    if (first_changed) pb_index_deployment_rank0(handle, rs->members[0]);
    pb_index_apply_coalescing(handle, rs->R());
    std::vector<std::unique_ptr<Crew>> idle;
    idle.swap(rs->crews);
    return idle;
}

// Replica 0 is copied while the set serves: only `change` is held, so searches and readers go on and mutations wait.
// The copies then join the rotation at once, under the writer lock, with the switches replica 0 has then.
pb_status pb_rep_add(Replicas *rs, pb_index *handle, const int32_t *devices, int32_t n) {
    std::lock_guard<std::mutex> c(rs->change);
    const int S = rs->S, R = rs->R();
    if (n < 1 || n % S != 0)
        return pb_fail(PB_ERR_INVALID, "n_devices %d is not a positive multiple of the set's %d shards", (int)n, S);
    if (R * S + n > PB_MAX_MEMBERS)
        return pb_fail(PB_ERR_INVALID, "%d devices in all: above 64 members", R * S + (int)n);
    const int have = pb_device_count();
    for (int i = 0; i < n; ++i)
        if (devices[i] < 0 || devices[i] >= have)
            return pb_fail(PB_ERR_INVALID, "devices[%d] = %d out of range (have %d)", i, (int)devices[i], have);
    pb_index *m0 = rs->members[0];
    // the copies run on streams of their own: replica 0's device work of earlier mutations ends first
    pb_status s = pb_sync_devices(m0);
    std::vector<pb_index *> copies;
    if (s == PB_OK) s = copy_replicas(m0, S, devices, n / S, copies);
    if (s != PB_OK) return s;
    std::vector<std::unique_ptr<Crew>> idle;
    {
        std::lock_guard<std::mutex> g(rs->gate);
        std::unique_lock<std::shared_mutex> wr(rs->rw);
        for (pb_index *x : copies) pb_index_copy_switches(x, m0);  // a pb_set_* call may have come during the copy
        std::vector<pb_index *> next = rs->members;
        next.insert(next.end(), copies.begin(), copies.end());
        std::vector<int> devs = rs->devices;
        devs.insert(devs.end(), devices, devices + n);
        std::vector<int> from((size_t)(R + n / S), -1);
        std::iota(from.begin(), from.begin() + R, 0);
        idle = publish(rs, handle, std::move(next), std::move(devs), from);
    }
    return PB_OK;  // idle joins its threads here, after the locks
}

// The leaving replicas are taken out under the writer lock, which waits for the routed calls and merged batches that
// hold the set; they are closed after it.  Requests still queued run on the replicas that stay.
pb_status pb_rep_remove(Replicas *rs, pb_index *handle, const int32_t *which, int32_t n) {
    std::lock_guard<std::mutex> c(rs->change);
    const int R = rs->R(), S = rs->S;
    if (n < 1 || n >= R)
        return pb_fail(PB_ERR_INVALID, "removing %d of %d replicas: at least one must leave and one stay", (int)n, R);
    std::vector<uint8_t> stays((size_t)R, 1);
    for (int i = 0; i < n; ++i) {
        const int g = which[i];
        if (g < 0 || g >= R) return pb_fail(PB_ERR_INVALID, "replicas[%d] = %d outside [0, %d)", i, g, R);
        if (!stays[g]) return pb_fail(PB_ERR_INVALID, "replica %d is listed twice", g);
        stays[g] = 0;
    }
    std::vector<pb_index *> gone;
    std::vector<std::unique_ptr<Crew>> idle;
    {
        std::lock_guard<std::mutex> g(rs->gate);
        std::unique_lock<std::shared_mutex> wr(rs->rw);
        std::vector<pb_index *> next;
        std::vector<int> devs, from;
        for (int g = 0; g < R; ++g) {
            if (!stays[g]) {
                gone.push_back(rs->members[g]);
                continue;
            }
            next.push_back(rs->members[g]);
            devs.insert(devs.end(), rs->devices.begin() + (size_t)g * S, rs->devices.begin() + (size_t)(g + 1) * S);
            from.push_back(g);
        }
        idle = publish(rs, handle, std::move(next), std::move(devs), from);
    }
    idle.clear();  // joins the threads
    for (pb_index *m : gone) pb_index_close(m);  // a host-tier store stays with the replicas that share it
    return PB_OK;
}
