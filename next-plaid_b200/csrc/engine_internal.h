// engine_internal.h -- C++-side entry points shared between engine.cu, loader.cpp, builder.cpp and deployment.cpp (not
// exported).
#pragma once
#include "../../include/plaid_b200.h"

#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

pb_status pb_fail(pb_status s, const char *fmt, ...);

using Job = std::function<pb_status(int rank)>;

// A library thread of a deployment's rank, a replica set's slice or a search lane: waits for a job, runs it, records
// its status and pb_last_error() text
struct RankWorker {
    int rank;
    std::thread th;
    std::mutex m;
    std::condition_variable cv;
    const Job *job = nullptr;
    bool done = false, quit = false;
    pb_status status = PB_OK;
    std::string error;
    explicit RankWorker(int r) : rank(r) {
        th = std::thread([this] {
            std::unique_lock<std::mutex> lk(m);
            for (;;) {
                cv.wait(lk, [this] { return job || quit; });
                if (quit) return;
                const Job *j = job;
                lk.unlock();
                const pb_status s = (*j)(rank);
                std::string e = s == PB_OK ? std::string() : std::string(pb_last_error());
                lk.lock();
                status = s, error = std::move(e);
                job = nullptr;
                done = true;
                cv.notify_all();
            }
        });
    }
    void submit(const Job &j) {
        std::lock_guard<std::mutex> lk(m);
        job = &j;
        done = false;
        cv.notify_all();
    }
    void wait() {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [this] { return done; });
    }
    ~RankWorker() {
        {
            std::lock_guard<std::mutex> lk(m);
            quit = true;
            cv.notify_all();
        }
        if (th.joinable()) th.join();
    }
};

// job(i) for slots 0..k-1 at once: slot 0 on the caller's thread, slot i >= 1 on helpers[i - 1], a RankWorker of rank
// i.  st[i] is slot i's status and err[i] its pb_last_error() text when it failed; the caller picks the one it reports.
inline void run_slots(int k, const Job &job, const std::unique_ptr<RankWorker> *helpers, std::vector<pb_status> &st,
                      std::vector<std::string> &err) {
    st.assign((size_t)k, PB_OK);
    err.assign((size_t)k, std::string());
    for (int i = 1; i < k; ++i) helpers[i - 1]->submit(job);
    st[0] = job(0);
    if (st[0] != PB_OK) err[0] = pb_last_error();
    for (int i = 1; i < k; ++i) {
        helpers[i - 1]->wait();
        st[i] = helpers[i - 1]->status;
        err[i] = helpers[i - 1]->error;
    }
}

// A handle that holds no documents and stands for other handles, its members: a deployment (pb_index_load_devices,
// deployment.cpp, DESIGN §4o) for the ranks of a doc-sharded index in one process, driven by the library's own
// threads; a replica set (pb_index_load_replicas, replicas.cpp, DESIGN §4q) for R full copies of an index, each a plain
// handle or a deployment.  The members are driven through the public entry points.  Such a handle's pb_index owns its
// Group; the entry points of engine.cu check their arguments and hand the call to it.
struct Deployment;
struct Replicas;
struct Group {
    virtual ~Group() = default;
    // what the handle is called in a refusal
    virtual const char *kind() const = 0;
    pb_status refuse(const char *call) const {
        return pb_fail(PB_ERR_UNSUPPORTED, "%s on %s is not supported", call, kind());
    }
    // the concrete group, for the calls only one kind serves (search, resize); null for the other kind
    virtual Deployment *as_deployment() { return nullptr; }
    virtual Replicas *as_replicas() { return nullptr; }
    // member i's handle, unlocked: only for a group whose members cannot change (a replica set, or a deployment that is
    // a replica set's member and so refuses pb_index_add_devices / pb_index_remove_ranks); elsewhere one() or in_turn()
    virtual pb_index *member(int i) = 0;
    virtual int size() = 0;
    // the whole index's documents and tokens, read together
    virtual void totals(long long *D, long long *N) = 0;
    virtual pb_status memory(int64_t *device_bytes, int64_t *host_bytes) = 0;
    virtual pb_status shard_layout(int32_t *out_world, int64_t *out_bounds, int32_t *out_devices) = 0;
    // pb_index_append (codec != null) or pb_index_append_encoded
    virtual pb_status append(pb_codec *codec, const float *embeddings, const int64_t *codes, const uint8_t *residuals,
                             const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space, const char *index_dir,
                             int64_t batch_size, int64_t *out_first_doc_id) = 0;
    virtual pb_status del(const int64_t *doc_ids, int64_t n_ids, const char *index_dir, int64_t *out_deleted) = 0;
    virtual pb_status rebalance(const int64_t *bounds, int64_t *out_bounds) = 0;
    virtual pb_status reserve(int64_t num_documents, int64_t num_embeddings) = 0;
    virtual pb_status decompress(const int64_t *doc_ids, int64_t n_docs, float *out_embeddings, int64_t *out_lengths) = 0;
    virtual pb_status exhaustive(const float *queries, const int64_t *q_off, int64_t n_queries, float *out_scores) = 0;
    virtual pb_status export_ivf(int64_t *out_ivf, int32_t *out_lengths, int64_t *out_total) = 0;
    virtual pb_status last_delete_ms(float *out_ms) = 0;
    // call(m) on every member's handle, on the caller's thread, outside the group's collectives (the pb_set_* switches)
    virtual void each(const std::function<void(pb_index *)> &call) = 0;
    // call(m) on every member in turn, the lowest member's failure first, as a writer or a reader of the group (the row
    // cache's entry points)
    virtual pb_status in_turn(bool writer, const std::function<pb_status(pb_index *)> &call) = 0;
    // call(m) on one member, on the caller's thread, for a whole request of n queries (a merged batch, a reader)
    virtual pb_status one(int64_t n_queries, const std::function<pb_status(pb_index *)> &call) = 0;
};
// A group's handle, owning g: K, dim, nbits and device copied from g's first member (pb_index_deployment_rank0); the
// PB_COALESCE* defaults applied
pb_index *pb_index_new_group(Group *g, const pb_index *first);
// the handle's fields taken from rank 0 again, after a resize gave it another rank 0
void pb_index_deployment_rank0(pb_index *ix, const pb_index *rank0);
// A search collective: call(m, ids, scores, counts) on every rank at once, rank 0 with the caller's outputs and the
// others with scratch outputs of n_queries rows of `stride` (null where the caller's is null)
pb_status pb_dep_search(Deployment *d, int64_t n_queries, int64_t stride, int64_t *out_ids, float *out_scores,
                        int32_t *out_counts,
                        const std::function<pb_status(pb_index *, int64_t *, float *, int32_t *)> &call);
// pb_index_add_devices / pb_index_remove_ranks after the handle's checks.  `handle` is the deployment's own: its rank-0
// fields follow a new rank 0.
pb_status pb_dep_add_devices(Deployment *d, const int32_t *devices, int32_t n, const int64_t *bounds, int64_t *out_bounds);
pb_status pb_dep_remove_ranks(Deployment *d, pb_index *handle, const int32_t *ranks, int32_t n, const int64_t *bounds,
                              int64_t *out_bounds);
// A deployment of ranks already loaded (ranks[r] on devices[r], not yet in a group): joins them in a new group and
// returns its handle.  On failure the ranks are closed.
pb_status pb_dep_assemble(std::vector<pb_index *> ranks, const std::vector<int> &devices, pb_index **out);
// A routed search of n queries: cut into contiguous slices [b0, b1), each run by call(member, b0, b1, slice) on one of
// the least-loaded replicas, slice 0 on the caller's thread.  Returns the lowest failing slice's status.
pb_status pb_rep_search(Replicas *rs, int64_t n_queries,
                        const std::function<pb_status(pb_index *, int64_t, int64_t, int)> &call);

// A copy of a plain handle (or one rank of a deployment, outside its group) on `device`: every array, derived ones
// included, copied device to device; a host-tier handle shares src's pinned residuals.  The copy's device-dependent
// scalars are its own.
pb_status pb_index_clone(const pb_index *src, int device, pb_index **out);
// An empty rank on `device` opened from a peer src (a handle of the same index, one deployment rank): src's centroids,
// bucket weights and search switches copied, no documents, global ids from doc_id_base.  It equals pb_index_load_range
// of an empty range at doc_id_base -- scalars, arrays and pb_index_memory -- and reads no file.  As such a load it holds
// no tensor-core centroid operands: they are built when its first tokens arrive.  PB_ERR_UNSUPPORTED when src is
// host-tier or uses the caller's residual array (a deployment's ranks cannot move their documents then).
pb_status pb_index_clone_empty(const pb_index *src, int device, long long doc_id_base, pb_index **out);
// A rank of an in-process group leaves it and joins g as `rank`; no collective of either group may be running
pb_status pb_index_group_move(pb_index *ix, pb_shard_group *g, int rank);
// pb_index_rebalance_sharded on one rank of a group, where shares [world] (null: every rank) says which ranks take a
// share of the token-balanced split when bounds is null: the others get empty ranges at their positions (a rank that
// leaves its deployment).  Every rank passes the same shares.
pb_status pb_index_rebalance_shares(pb_index *ix, const int64_t *bounds, const uint8_t *shares, int64_t *out_bounds);
// Appends and deletes on plain handles that hold the same documents, as one: every member prepares, the directory is
// written once, then every member commits.  An append with a codec encodes on members[0] only; the others take its
// encoded rows.
pb_status pb_members_append(const std::vector<pb_index *> &members, pb_codec *codec, const float *embeddings,
                            const int64_t *codes, const uint8_t *residuals, const int64_t *doc_lengths, int64_t n_docs,
                            int32_t space, const char *index_dir, int64_t batch_size, int64_t *out_first);
pb_status pb_members_delete(const std::vector<pb_index *> &members, const int64_t *doc_ids, int64_t n_ids,
                            const char *index_dir, int64_t *out_deleted);
// The vote a set's replicas take together on a mutation, so that it commits on every replica or on none (engine.cu):
// for `ranks` ranks in all; with_dir: replica 0 writes the directory; share_rows: an append with a codec, which replica
// 0 encodes for every replica.  Set on every rank of replica g's handle for the mutation (null clears it).
struct RepVote;
RepVote *pb_rep_vote_new(int ranks, bool with_dir, bool share_rows);
void pb_rep_vote_free(RepVote *v);
void pb_index_set_rep_vote(pb_index *member, RepVote *v, int replica);
// the set behind a handle (null for any other handle); rank r of a deployment's handle (the handle itself otherwise)
Replicas *pb_replicas_of(const pb_index *ix);
pb_index *pb_rank_of(pb_index *ix, int r);
// a handle's documents and tokens, read together
void pb_index_totals(const pb_index *ix, long long *D, long long *N);
// a mutable host-tier handle or deployment: the replicas of a set write one shared row store, through replica 0 only
bool pb_host_rows_shared(pb_index *ix);
// cudaDeviceSynchronize on the device of ix, or of each of its ranks
pb_status pb_sync_devices(pb_index *ix);
// pb_index_open without the per-token arrays; follow with pb_index_upload_tokens per chunk.
pb_status pb_index_open_begin(const pb_index_desc *d, pb_index **out);
pb_status pb_index_upload_tokens(pb_index *ix, long long tok_off, const int64_t *codes, const uint8_t *residuals,
                                 long long n, int space);
// call once after the last pb_index_upload_tokens
pb_status pb_index_finalize(pb_index *ix);
// For a handle begun without an inverted file: the part of a directory's inverted file (host ivf.npy <i8 [total],
// ivf_lengths [K], global ids, all checked against [0, limit)) that lies in docs [b, e), each list filtered in file
// order with ids minus b, instead of the one pb_index_finalize would build from the codes.
pb_status pb_index_upload_ivf_range(pb_index *ix, const int64_t *ivf, const int32_t *lengths, long long total,
                                    long long limit, long long b, long long e);
// The inverted file of a directory after a change, from its ivf.npy (host, as above, ids in [0, D)) to the host, i64
// global ids: with a deleted set (device bits / word_pre over the D docs) deleted ids leave the lists and survivors are
// renumbered (delete.rs:196-237); with the sorted (centroid << 32 | doc) device keys of m appended docs each list is
// followed by its new pairs as ids D + doc (update.rs:1000-1067).
pb_status pb_index_patch_ivf(pb_index *ix, const int64_t *file_ivf, const int32_t *file_lengths, long long total, long long D,
                             const uint32_t *bits, const long long *word_pre, const uint64_t *keys, long long m,
                             std::vector<int64_t> &ivf, std::vector<int32_t> &lengths);
// pb_index_patch_ivf on the directory's ivf.npy / ivf_lengths.npy as they are on disk
pb_status pb_dir_patch_ivf(pb_index *ix, const char *index_dir, long long D, const uint32_t *bits, const long long *word_pre,
                           const uint64_t *keys, long long m, std::vector<int64_t> &ivf, std::vector<int32_t> &lengths);

// The index directory, as the loader reads it: a whole file; a number of a flat JSON object; a doclens.{i}.json list;
// the chunk file pair {i}.codes.npy <i8 [n_tokens] / {i}.residuals.npy u1 [n_tokens][packed].
pb_status pb_read_text(const std::string &path, std::string &out);
bool pb_json_number(const std::string &j, const char *key, double &out);
pb_status pb_read_doclens(const std::string &path, std::vector<int64_t> &out);
pb_status pb_read_chunk(const std::string &dir, long long chunk, long long n_tokens, long long packed,
                        std::vector<int64_t> &codes, std::vector<uint8_t> &residuals);
// a 2-D <f4 NPY file (embeddings.npy, buffer.npy)
pb_status pb_read_npy_f32(const std::string &path, long long &rows, long long &cols, std::vector<float> &out);

// update_index's file changes (update.rs:794-1117, update_threshold = false) for n_docs documents appended to the
// index in index_dir, which holds old_D documents: chunk files in batches of batch_size docs (the first merged into a
// last chunk of < 2000 docs), the merged inverted file ivf / ivf_lengths (global ids), metadata.json, and removal of
// the merged_* caches.  codes i64 [sum doc_lengths], residuals packed [sum doc_lengths][dim*nbits/8].
pb_status pb_dir_append(const char *index_dir, long long old_D, long long K, int dim, int nbits, long long batch_size,
                        const int64_t *codes, const uint8_t *residuals, const int64_t *doc_lengths, long long n_docs,
                        const int64_t *ivf, long long ivf_total, const int32_t *ivf_lengths);

// Index build (builder.cpp).  The first `take` entries of a seeded Fisher-Yates shuffle of 0..n-1 (splitmix64): the
// sample plan of pb_create_index.
std::vector<long long> shuffled_prefix(long long n, long long take, uint64_t seed);
// NPY v1.0 files: a whole file; a file of `bytes` payload bytes whose payload is written later, in pieces (byte offset
// into the payload), by any process
pb_status write_npy(const std::string &path, const char *descr, const std::vector<long long> &shape, const void *data,
                    size_t bytes);
pb_status write_text(const std::string &path, const std::string &txt);
struct NpyPiece {
    size_t offset, bytes;
    const char *src;
};
pb_status npy_create(const std::string &path, const char *descr, const std::vector<long long> &shape, size_t bytes);
pb_status npy_put(const std::string &path, const char *descr, const std::vector<long long> &shape,
                  const std::vector<NpyPiece> &pieces);
// chunk c's four files: n tokens starting at token t0 of the index, its n_docs documents' lengths
pb_status pb_write_chunk(const std::string &dir, long long c, const int64_t *codes, const uint8_t *residuals, long long n,
                         int packed, const int64_t *doc_lengths, long long n_docs, long long t0);
// centroids.npy, bucket_cutoffs.npy, bucket_weights.npy, avg_residual.npy, cluster_threshold.npy, plan.json
pb_status pb_write_codec_files(const std::string &dir, long long K, int dim, int nbits, const float *centroids,
                               const float *cutoffs, const float *weights, const float *avg_res, float threshold,
                               long long n_chunks);
// metadata.json of a new index of D documents and N tokens
pb_status pb_write_create_meta(const std::string &dir, long long n_chunks, int nbits, long long K, long long N, long long D,
                               int dim);
// the directory check of a collective build: rank 0 creates index_dir and a token file in it, the other ranks check
// that they read the same token (PB_ERR_IO otherwise), rank 0 removes the file
pb_status pb_dir_token_put(const char *index_dir, long long token);
pb_status pb_dir_token_check(const char *index_dir, long long token);
void pb_dir_token_drop(const char *index_dir);
// pb_create_index after its argument checks: pb_create_index_sharded over a group of one on params->device
pb_status pb_create_local(const float *embeddings, const int64_t *doc_lengths, int64_t n_docs, int32_t dim,
                          const pb_create_params *params, const char *index_dir, pb_index **out_index);

// PB_ERR_INVALID (PB_ERR_IO when unreadable) unless the directory's metadata.json holds D documents and nbits
pb_status pb_dir_check_documents(const char *index_dir, int nbits, long long D);

// delete_from_index's file changes (delete.rs:66-273) for the documents whose bit is set in `deleted` (one bit per doc
// of the old_D the directory holds): filtered chunk files and chunk metadata for every chunk with a deleted doc, the
// filtered inverted file ivf / ivf_lengths, metadata.json, removal of the merged_* caches, and the filtering of
// embeddings.npy / buffer.npy (clean_embeddings_files, delete.rs:286-398).
pb_status pb_dir_delete(const char *index_dir, long long old_D, long long K, int dim, int nbits, const uint32_t *deleted,
                        const int64_t *ivf, long long ivf_total, const int32_t *ivf_lengths);
