// engine.cu -- host side of libplaid_b200: the device-resident index (what MmapIndex holds after
// load, index.rs:995-1016), the search pipeline that replaces search::search_many_mmap
// (search.rs:643) and the C-ABI of include/plaid_b200.h.  No CPU fallback anywhere: every entry
// point needs an sm_90 (H100) device.
#include "coalesce.h"
#include "engine_internal.h"
#include "kernels.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <functional>
#include <map>
#include <tuple>
#include <thread>
#include <type_traits>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <vector>

#include <dlfcn.h>

// ------------------------------------------------------------------------------------------
// NCCL, bound at run time (dlopen) so single-GPU hosts need no libnccl.  Only the doc-sharded path
// (pb_index_comm_init) touches it.  Types restated from nccl.h 2.27 (stable ABI since 2.x).
// ------------------------------------------------------------------------------------------
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { PB_NCCL_UINT8 = 1, PB_NCCL_UINT64 = 5, PB_NCCL_FLOAT32 = 7, PB_NCCL_SUM = 0 };
struct NcclApi {
    void *h = nullptr;
    int (*GetUniqueId)(ncclUniqueId *) = nullptr;
    int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    // point-to-point, bound when present: only pb_index_rebalance_sharded needs them, so load() does not require them
    int (*Send)(const void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*Recv)(void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    bool has_p2p() const { return Send && Recv && GroupStart && GroupEnd; }
    bool load() {
        if (h) return true;
        const char *names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (h) break;
        }
        if (!h) return false;
        GetUniqueId = (int (*)(ncclUniqueId *))dlsym(h, "ncclGetUniqueId");
        CommInitRank = (int (*)(ncclComm_t *, int, ncclUniqueId, int))dlsym(h, "ncclCommInitRank");
        CommDestroy = (int (*)(ncclComm_t))dlsym(h, "ncclCommDestroy");
        AllGather = (int (*)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t))dlsym(h, "ncclAllGather");
        AllReduce = (int (*)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(h, "ncclAllReduce");
        GetErrorString = (const char *(*)(int))dlsym(h, "ncclGetErrorString");
        Send = (int (*)(const void *, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(h, "ncclSend");
        Recv = (int (*)(void *, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(h, "ncclRecv");
        GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
        GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
        return GetUniqueId && CommInitRank && CommDestroy && AllGather && AllReduce && GetErrorString;
    }
};
static NcclApi g_nccl;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;

pb_status pb_fail(pb_status s, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return s;
}

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return pb_fail(PB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_),   \
                           __FILE__, __LINE__);                                                    \
    } while (0)
#define CKN(call)                                                                                  \
    do {                                                                                           \
        int r_ = (call);                                                                           \
        if (r_ != 0) return pb_fail(PB_ERR_COMM, "%s failed: %s", #call, g_nccl.GetErrorString(r_)); \
    } while (0)
#define CKS(expr)                                                                                  \
    do {                                                                                           \
        pb_status s_ = (expr);                                                                     \
        if (s_ != PB_OK) return s_;                                                                \
    } while (0)

// CUDA-event pair around the main kernel of a stage (profiling mode only); read after the sub-batch's synchronize
#define KEV_BEGIN(k)                                                                               \
    do {                                                                                           \
        if (ix->profiling) CK(cudaEventRecord(ws.kev[2 * (k)], ws.stream));                        \
    } while (0)
#define KEV_END(k)                                                                                 \
    do {                                                                                           \
        if (ix->profiling) {                                                                       \
            CK(cudaEventRecord(ws.kev[2 * (k) + 1], ws.stream));                                   \
            g_stats.kernel_seen[k] = true;                                                         \
        }                                                                                          \
    } while (0)

extern "C" const char *pb_last_error(void) { return g_err.c_str(); }
extern "C" const char *pb_version(void) { return "plaid_b200 0.1 (sm_90a)"; }

extern "C" int32_t pb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

static pb_status check_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return pb_fail(PB_ERR_CUDA, "no CUDA device available (%s); libplaid_b200 has no CPU fallback",
                       e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= n) return pb_fail(PB_ERR_INVALID, "device %d out of range (have %d)", device, n);
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, device));
    if (p.major != 9 || p.minor != 0)
        return pb_fail(PB_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only", device, p.major,
                       p.minor);
    CK(cudaSetDevice(device));
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// device buffers
// ------------------------------------------------------------------------------------------
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    bool zero_on_grow = false;
    bool owned = true;
    void adopt(void *ptr, size_t bytes) {  // caller-owned device memory, used in place
        if (p && owned) cudaFree(p);
        p = ptr;
        cap = bytes;
        owned = false;
    }
    pb_status ensure(size_t bytes) {
        if (bytes <= cap) return PB_OK;
        if (p && owned) cudaFree(p);
        owned = true;
        p = nullptr;
        cap = 0;
        size_t want = bytes + (bytes >> 3) + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return pb_fail(PB_ERR_NOMEM, "cudaMalloc(%zu bytes) failed: %s", want, cudaGetErrorString(e));
        }
        cap = want;
        if (zero_on_grow) {
            e = cudaMemset(p, 0, want);
            if (e != cudaSuccess) return pb_fail(PB_ERR_CUDA, "cudaMemset failed: %s", cudaGetErrorString(e));
        }
        return PB_OK;
    }
    // Capacity for `bytes` that keeps the first `keep` bytes: a new allocation of max(bytes, 1.5 x the old capacity)
    // (exactly `bytes` when !geometric) and one device-to-device copy.  On failure the old buffer is untouched.
    pb_status grow(size_t bytes, size_t keep, bool geometric = true) {
        if (bytes <= cap) return PB_OK;
        if (p && !owned) return pb_fail(PB_ERR_UNSUPPORTED, "caller-owned device memory cannot grow");
        const size_t want = geometric ? std::max(bytes, cap + cap / 2) : bytes;
        void *q = nullptr;
        cudaError_t e = cudaMalloc(&q, want);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return pb_fail(PB_ERR_NOMEM, "cudaMalloc(%zu bytes) failed: %s", want, cudaGetErrorString(e));
        }
        if (keep && p) {
            e = cudaMemcpy(q, p, std::min(keep, cap), cudaMemcpyDeviceToDevice);
            if (e != cudaSuccess) {
                cudaFree(q);
                return pb_fail(PB_ERR_CUDA, "cudaMemcpy failed: %s", cudaGetErrorString(e));
            }
        }
        if (p) cudaFree(p);
        p = q;
        cap = want;
        owned = true;
        return PB_OK;
    }
    void swap(DevBuf &o) {
        std::swap(p, o.p);
        std::swap(cap, o.cap);
        std::swap(zero_on_grow, o.zero_on_grow);
        std::swap(owned, o.owned);
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
    ~DevBuf() {
        if (p && owned) cudaFree(p);
    }
};

struct HostBuf {  // pinned
    void *p = nullptr;
    size_t cap = 0;
    pb_status ensure(size_t bytes) {
        if (bytes <= cap) return PB_OK;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMallocHost(&p, bytes + 256);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return pb_fail(PB_ERR_NOMEM, "cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e));
        }
        cap = bytes + 256;
        return PB_OK;
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
    ~HostBuf() {
        if (p) cudaFreeHost(p);
    }
};

// One pinned, mapped and portable host allocation of n bytes
static pb_status pinned_segment(size_t n, std::shared_ptr<uint8_t> &out) {
    void *h = nullptr;
    cudaError_t e = cudaHostAlloc(&h, n, cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return pb_fail(PB_ERR_NOMEM, "cudaHostAlloc(%zu bytes, mapped) failed: %s", n, cudaGetErrorString(e));
    }
    out.reset(static_cast<uint8_t *>(h), [](uint8_t *q) { cudaFreeHost(q); });
    return PB_OK;
}

// The packed residuals of a PB_OPEN_HOST_RESIDUALS handle (DESIGN.md 4r): segments of 2^shift bytes, each one pinned
// host allocation; byte b of the row array is at seg[b >> shift] + (b & (2^shift - 1)).  An open makes the last segment
// exactly as long as the rows need; the first growth replaces it by a full one (a copy of at most one segment), and
// later growths only add segments.  The replicas of a set share one store, freed with the last of them; each reads it
// through its own device table of the segments' mapped addresses (HostTier).  mu serialises growths.
struct HostRows {
    int shift = 28;
    std::vector<std::shared_ptr<uint8_t>> seg;
    size_t bytes = 0;             // pinned bytes held: the capacity, since only the last segment can be short
    unsigned long long gen = 0;   // changes whenever a segment's address does
    std::mutex mu;
    size_t seg_bytes() const { return (size_t)1 << shift; }
    pb_status open(size_t n) {
        for (size_t o = 0; o < n; o += seg_bytes()) {
            seg.emplace_back();
            CKS(pinned_segment(std::min(seg_bytes(), n - o), seg.back()));
            bytes += std::min(seg_bytes(), n - o);
        }
        ++gen;
        return PB_OK;
    }
    // capacity for `want` bytes; every allocation before the first change, so a failure changes nothing
    pb_status grow(size_t want) {
        if (want <= bytes) return PB_OK;
        const size_t S = seg_bytes(), tail = bytes & (S - 1), need = (want + S - 1) / S;
        std::shared_ptr<uint8_t> full;
        if (tail) CKS(pinned_segment(S, full));
        std::vector<std::shared_ptr<uint8_t>> add(need - seg.size());
        for (auto &x : add) CKS(pinned_segment(S, x));
        if (tail) {
            memcpy(full.get(), seg.back().get(), tail);
            seg.back() = std::move(full);
        }
        for (auto &x : add) seg.push_back(std::move(x));
        bytes = seg.size() * S;
        ++gen;
        return PB_OK;
    }
    // f(host address, offset into the range, length) for each segment piece of bytes [b, b + n)
    template <class F> pb_status pieces(size_t b, size_t n, F &&f) const {
        for (size_t done = 0; done < n;) {
            const size_t o = (b + done) & (seg_bytes() - 1), m = std::min(n - done, seg_bytes() - o);
            CKS(f(seg[(b + done) >> shift].get() + o, done, m));
            done += m;
        }
        return PB_OK;
    }
    // bytes [b, b + n) from src (host or device memory), or to dst (host memory)
    pb_status write(size_t b, const uint8_t *src, size_t n, int space) const {
        return pieces(b, n, [&](uint8_t *h, size_t o, size_t m) -> pb_status {
            if (space == PB_MEM_DEVICE) CK(cudaMemcpy(h, src + o, m, cudaMemcpyDeviceToHost));
            else memcpy(h, src + o, m);
            return PB_OK;
        });
    }
    pb_status read(size_t b, uint8_t *dst, size_t n) const {
        return pieces(b, n, [&](uint8_t *h, size_t o, size_t m) -> pb_status {
            memcpy(dst + o, h, m);
            return PB_OK;
        });
    }
    // bytes [b, b + n) to device memory, one copy per piece on st
    pb_status to_device(size_t b, uint8_t *dst, size_t n, cudaStream_t st) const {
        return pieces(b, n, [&](uint8_t *h, size_t o, size_t m) -> pb_status {
            CK(cudaMemcpyAsync(dst + o, h, m, cudaMemcpyHostToDevice, st));
            return PB_OK;
        });
    }
};

// One handle's view of its host rows: the store, and the store's segment table as this handle's device reads it
struct HostTier {
    std::shared_ptr<HostRows> rows;
    DevBuf table;                        // [segments] mapped addresses on the handle's device
    unsigned long long table_gen = ~0ull;
    // the table after a change of the store's segments (the current device is the handle's)
    pb_status sync() {
        if (!rows || table_gen == rows->gen) return PB_OK;
        std::vector<const uint8_t *> a(rows->seg.size());
        for (size_t k = 0; k < a.size(); ++k) {
            void *d = nullptr;
            CK(cudaHostGetDevicePointer(&d, rows->seg[k].get(), 0));
            a[k] = static_cast<const uint8_t *>(d);
        }
        CKS(table.ensure(std::max<size_t>(a.size() * 8, 16)));
        if (!a.empty()) CK(cudaMemcpy(table.p, a.data(), a.size() * 8, cudaMemcpyHostToDevice));
        table_gen = rows->gen;
        return PB_OK;
    }
    // capacity for `want` bytes, and this handle's table to match
    pb_status grow(size_t want) {
        std::lock_guard<std::mutex> g(rows->mu);
        CKS(rows->grow(want));
        return sync();
    }
    SegRows dev() const { return SegRows{table.as<const uint8_t *const>(), rows->shift}; }
};

// ------------------------------------------------------------------------------------------
// Cross-rank exchanges.  A rank reaches its peers over NCCL (one process per GPU) or through an in-process shard group:
// ONE process drives several shards from several host threads (any mix of devices, including all shards on one GPU --
// which is how the sharded paths run under `pytest -m gpu` on a single-GPU box).  ShardComm is one rank's end of
// either; the search, the sharded update, the rebalance and the data-parallel k-means see only its collectives.
// ------------------------------------------------------------------------------------------
struct pb_shard_group {
    int world = 0;
    std::mutex mu;
    std::condition_variable cv;
    int arrived = 0;
    unsigned long long gen = 0;
    bool broken = false, failing = false;
    std::vector<const void *const *> table;  // per rank: the device pointers it sends, [destination][item]
    std::vector<int> dev;
    // false = a peer failed or did not arrive within the timeout; the group stays broken.  unbounded: wait for the
    // peers however long they take (a peer that fails still breaks the group), for a peer known to be busy.  ok =
    // false: this rank failed; the group breaks once every rank has arrived, and every rank returns false
    bool barrier(bool unbounded = false, bool ok = true) {
        std::unique_lock<std::mutex> g(mu);
        if (broken) return false;
        const unsigned long long my = gen;
        failing = failing || !ok;
        if (++arrived == world) {
            arrived = 0;
            ++gen;
            broken = failing;
            cv.notify_all();
            return !broken;
        }
        auto done = [&] { return gen != my || broken; };
        if (unbounded) cv.wait(g, done);
        else if (!cv.wait_for(g, std::chrono::seconds(60), done)) broken = true;
        if (broken) cv.notify_all();
        return !broken;
    }
    void fail() {
        std::lock_guard<std::mutex> g(mu);
        broken = true;
        cv.notify_all();
    }
};

struct ShardComm {
    int rank = 0, world = 1, device = 0;
    ncclComm_t nccl = nullptr;        // owned
    pb_shard_group *group = nullptr;  // or a member of this group
    ShardComm() = default;
    ShardComm(const ShardComm &) = delete;  // the NCCL communicator is destroyed once
    ShardComm &operator=(const ShardComm &) = delete;
    ~ShardComm() {
        if (nccl) g_nccl.CommDestroy(nccl);
    }

    // world 1 is a group of one and needs no NCCL
    pb_status init_nccl(const uint8_t *id128, int r, int w, int dev) {
        if (w < 1 || r < 0 || r >= w) return pb_fail(PB_ERR_INVALID, "bad rank %d / world %d", r, w);
        if (joined()) return pb_fail(PB_ERR_INVALID, "communicator already initialised");
        if (w > 1) {
            if (!g_nccl.load()) return pb_fail(PB_ERR_COMM, "libnccl.so.2 not found (%s)", dlerror());
            CK(cudaSetDevice(dev));
            ncclUniqueId id;
            memcpy(id.internal, id128, 128);
            CKN(g_nccl.CommInitRank(&nccl, w, id, r));
        }
        rank = r, world = w, device = dev;
        return PB_OK;
    }
    pb_status join(pb_shard_group *g, int r, int dev) {
        if (r < 0 || r >= g->world) return pb_fail(PB_ERR_INVALID, "bad rank %d / world %d", r, g->world);
        if (joined()) return pb_fail(PB_ERR_INVALID, "communicator already initialised");
        std::lock_guard<std::mutex> lk(g->mu);
        g->dev[r] = dev;
        group = g, rank = r, world = g->world, device = dev;
        return PB_OK;
    }
    bool joined() const { return nccl || group; }
    // an in-process rank leaves its group, so that it can join another (a deployment changing its number of ranks).
    // No collective of the group may be running.  An NCCL communicator stays as it is.
    void leave() {
        if (!nccl) group = nullptr, rank = 0, world = 1;
    }
    // the peers must not wait for a rank that gave up: breaks an in-process group (NCCL keeps no such state)
    void fail() {
        if (group) group->fail();
    }
    // exchange() over NCCL needs its optional point-to-point symbols
    bool has_p2p() const { return !nccl || g_nccl.has_p2p(); }

    // every rank's `words` 64-bit words at `send`, into `recv` in rank order.  unbounded: the in-process group waits
    // for late peers without its 60 s timeout (NCCL waits either way)
    pb_status allgather(cudaStream_t stream, const void *send, void *recv, size_t words, bool unbounded = false) {
        if (nccl) {
            CKN(g_nccl.AllGather(send, recv, words, PB_NCCL_UINT64, nccl, stream));
            return PB_OK;
        }
        return gather(stream, send, recv, words * 8, unbounded);
    }

    // in-place sum of `count` floats over the ranks, synchronized; the result is bit-identical on every rank (the
    // in-process group gathers every rank's buffer into `stage` and sums it in rank order)
    pb_status allreduce_sum(cudaStream_t stream, float *buf, size_t count, DevBuf &stage) {
        if (world == 1) return PB_OK;
        if (nccl) {
            CKN(g_nccl.AllReduce(buf, buf, count, PB_NCCL_FLOAT32, PB_NCCL_SUM, nccl, stream));
            CK(cudaStreamSynchronize(stream));
            return PB_OK;
        }
        CKS(stage.ensure((size_t)world * count * 4));
        CKS(gather(stream, buf, stage.p, count * 4, false));
        k_sum_ranks<<<stage.cap ? 296 : 1, 256, 0, stream>>>(stage.as<float>(), world, (long long)count, buf);
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(stream));
        return PB_OK;
    }

    // `items` pieces between every pair of ranks, synchronized: send_* are [destination][item], recv_* [source][item],
    // and a piece's sizes agree at both ends.  Waits for late peers.  NCCL: my own piece by a device copy, the others
    // by send / receive pairs in one group (has_p2p() must hold)
    pb_status exchange(cudaStream_t stream, int items, const void *const *send_ptrs, const size_t *send_bytes,
                       void *const *recv_ptrs, const size_t *recv_bytes) {
        if (!nccl) return pull(stream, items, send_ptrs, recv_ptrs, recv_bytes, true, true);
        for (int it = 0; it < items; ++it) {
            const size_t i = (size_t)rank * items + it;
            if (recv_bytes[i])
                CK(cudaMemcpyAsync(recv_ptrs[i], send_ptrs[i], recv_bytes[i], cudaMemcpyDeviceToDevice, stream));
        }
        int res = g_nccl.GroupStart();
        for (int r = 0; r < world && res == 0; ++r)
            for (int it = 0; r != rank && it < items && res == 0; ++it) {
                const size_t i = (size_t)r * items + it;
                if (send_bytes[i]) res = g_nccl.Send(send_ptrs[i], send_bytes[i], PB_NCCL_UINT8, r, nccl, stream);
            }
        for (int s = 0; s < world && res == 0; ++s)
            for (int it = 0; s != rank && it < items && res == 0; ++it) {
                const size_t i = (size_t)s * items + it;
                if (recv_bytes[i]) res = g_nccl.Recv(recv_ptrs[i], recv_bytes[i], PB_NCCL_UINT8, s, nccl, stream);
            }
        const int end = g_nccl.GroupEnd();
        if (res == 0) res = end;
        if (res != 0) return pb_fail(PB_ERR_COMM, "rebalance transfer failed: %s", g_nccl.GetErrorString(res));
        CK(cudaStreamSynchronize(stream));
        return PB_OK;
    }

  private:
    // The in-process protocol of every collective: publish my table of send pointers ([destination][item]), a barrier,
    // pull my pieces (recv / bytes [source][item]) from each source by peer copies, and a second barrier, after which
    // the sources may reuse their tables and buffers.  A rank whose CUDA work fails still takes both barriers, so that
    // no rank leaves while a peer reads its table or buffers; the barrier it fails at fails every rank and breaks the
    // group, unless keep_group (the caller reports the error to its peers itself).  A CUDA error returns PB_ERR_CUDA, a
    // broken or timed-out barrier PB_ERR_COMM.
    pb_status pull(cudaStream_t stream, int items, const void *const *send, void *const *recv, const size_t *bytes,
                   bool unbounded, bool keep_group) {
        if (!group) return pb_fail(PB_ERR_COMM, "sharded handle without a transport");
        cudaError_t e = cudaStreamSynchronize(stream);  // my send buffers are complete
        group->table[rank] = send;
        bool ok = group->barrier(unbounded, e == cudaSuccess || keep_group);
        for (int s = 0; s < world && ok && e == cudaSuccess; ++s)
            for (int it = 0; it < items && e == cudaSuccess; ++it) {
                const size_t i = (size_t)s * items + it;
                if (bytes[i])
                    e = cudaMemcpyPeerAsync(recv[i], device, group->table[s][(size_t)rank * items + it], group->dev[s],
                                            bytes[i], stream);
            }
        if (ok && e == cudaSuccess) e = cudaStreamSynchronize(stream);
        ok = ok && group->barrier(unbounded, e == cudaSuccess || keep_group);
        if (e != cudaSuccess) return pb_fail(PB_ERR_CUDA, "shard group exchange failed: %s", cudaGetErrorString(e));
        if (!ok) return pb_fail(PB_ERR_COMM, "shard group: a peer failed or timed out");
        return PB_OK;
    }
    // an all-gather of `bytes` per rank: every destination's entry is the one send buffer
    pb_status gather(cudaStream_t stream, const void *send, void *recv, size_t bytes, bool unbounded) {
        const std::vector<const void *> table((size_t)world, send);
        std::vector<void *> dst((size_t)world);
        for (int s = 0; s < world; ++s) dst[s] = static_cast<char *>(recv) + (size_t)s * bytes;
        const std::vector<size_t> n((size_t)world, bytes);
        return pull(stream, 1, table.data(), dst.data(), n.data(), unbounded, false);
    }
};

// per-call scratch; a pool of these makes pb_search_batch re-entrant on one handle
struct Workspace {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[PB_STAGE_COUNT + 1] = {};
    cudaEvent_t kev[2 * PB_KERNEL_COUNT] = {};  // begin / end around the main kernel of a stage
    cudaEvent_t call_ev[2] = {};                // around a whole search call
    DevBuf Q, qoff, ST, partial, sel, cells, ncells, bitmap, cand, ncand, approx, keys, kept, nkept, tokp, maxkey,
        exact, fkeys, oids, oscores, ocounts, subset, subset_bits, elig, list, counters, lkeys, ST16, qrange, qflag, lsum, cand2, ncand2,  cellbits,
        gkeys, krank, payload, gfkeys, gpayload, cmax16, tau16, plist, pcount, Qi, Qh16t, Ql16t, ST16b, k1diag, k1rows, ulist, nulist, est, kept2, krank2, nkept2, tokp2, ktok2, qnmax, qexp, qrange_tc, mslot, slicecnt, rcmax, rcpairs, rcn, cellflags, estkey, srcrank, xpairs, xnpairs, needexact, gbase, fdiag,
        a5floor, a5live, a5n1, a5n12, a5theta, smax, tdlive, tdcmax, tdiag;
    // subsets: the call's ids, its rows' spans, the passes' per-query rows and n, the all-eligible lists' lengths, the
    // eligible counts, and the doc-sharded exchanges (plan record, every rank's eligibility rows)
    DevBuf subspan, qsub, listn, eligcnt, xrec, xall, gelig;
    // host tier: the staged rows of the kept docs (residuals, codes, 1 / |v|), their slot offsets and slot list
    DevBuf s_res, s_codes, s_inv, soff, kept_s;
    DevBuf rc_hits;  // with a row cache: the slots staged from it and their bytes, this pass
    cudaEvent_t sev[2] = {};  // around the staging kernels
    HostBuf hq, hres, hcounts;
    pb_status init() {
        CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        for (auto &e : ev) CK(cudaEventCreate(&e));
        for (auto &e : kev) CK(cudaEventCreate(&e));
        for (auto &e : call_ev) CK(cudaEventCreate(&e));
        for (auto &e : sev) CK(cudaEventCreate(&e));
        bitmap.zero_on_grow = true;
        maxkey.zero_on_grow = true;
        subset_bits.zero_on_grow = true;
        elig.zero_on_grow = true;
        cellbits.zero_on_grow = true;
        rcmax.zero_on_grow = true;
        return PB_OK;
    }
    ~Workspace() {
        for (auto &e : ev)
            if (e) cudaEventDestroy(e);
        for (auto &e : kev)
            if (e) cudaEventDestroy(e);
        for (auto &e : call_ev)
            if (e) cudaEventDestroy(e);
        for (auto &e : sev)
            if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
    }
};

struct Stats {
    float ms[PB_STAGE_COUNT] = {};
    float kernel_ms[PB_KERNEL_COUNT] = {};
    bool kernel_seen[PB_KERNEL_COUNT] = {};
    float call_ms = 0.f;
    int launches[PB_STAGE_COUNT] = {};
    pb_work_counters work = {};
    long long staged_docs = 0, staged_bytes = 0;  // host tier: pb_last_staging_stats
    float staging_ms = 0.f;
};
static thread_local Stats g_stats;
static thread_local int g_budget_div = 1;  // lanes of the current call share the workspace budget

// pb_search's request queue (coalesce.h, DESIGN.md 4m) runs a merged batch through this: run_coalesced, below the
// search entry points
struct CoalescedRun {
    pb_index *ix;
    int operator()(pbq::Request *const *reqs, size_t n, std::string &err) const;
};
struct GatherBuf {  // host scratch of one merged batch: the arguments of its pb_search_batch_params call
    std::vector<float> queries, scores;
    std::vector<int64_t> q_off, sub_off, sub_ids, ids;
    std::vector<pb_search_params> params;
    std::vector<uint8_t> has_sub;
    std::vector<int32_t> counts;
};

// The totals of an index's documents.  Open derives them; append, delete and rebalance prepare new ones and publish
// them in one place (publish), so that the handle equals a fresh open of its documents.
struct DocTotals {
    long long D = 0, N = 0, ivf_len = 0, n_ucodes = 0;
    int max_doclen = 0;
    float vmin = 0.0f;  // smallest pre-normalisation token norm |c + w| over the index (error bound of the filter)
    float wmax = 0.0f;  // largest residual norm |w| over the index (same)
};

// The arrays derived from an index's documents, with their totals
struct DocArrays : DocTotals {
    DevBuf codes, residuals, doc_off, ucodes, udoc_off, ivf, ivf_off;
    DevBuf tok_inv_norm;               // [N] 1 / |c + w| for the linear estimate (k_maxsim_tc)
    DevBuf ivf_spare, ivf_off_spare;   // the other half of the inverted file's ping-pong: append / delete write into it
    // host tier with a row cache (pb_index_set_row_cache, DESIGN.md 4s): [D] i64 token offset of each doc's rows in the
    // cache or -1, and [D] u32 how often search staging kept each doc since the last fill by counts; empty otherwise
    DevBuf cache_off, kept_count;
    // every buffer, in one list (the memory count and the rebalance's swap walk it)
    template <class A> static auto buffers(A &a) {
        return std::array{&a.codes, &a.residuals, &a.doc_off, &a.ucodes, &a.udoc_off, &a.ivf,
                          &a.ivf_off, &a.tok_inv_norm, &a.ivf_spare, &a.ivf_off_spare, &a.cache_off, &a.kept_count};
    }
};

// The rest of a host-tier handle's row cache: the rows, the budget they fit, what they hold, and the search staging
// counters since the last reset.  The map and the counts are per-doc arrays (DocArrays).
struct RowCacheState {
    size_t budget = 0;       // 0: off, and cache_off / kept_count are empty
    DevBuf rows;             // the cached docs' packed rows, each doc's at a token offset
    long long docs = 0, bytes = 0, dead = 0;  // live cached docs and their row bytes; bytes of docs deleted since the fill
    float fill_ms = 0.f;
    std::atomic<long long> staged{0}, hit_docs{0}, hit_bytes{0};
    std::mutex fill_mu;      // one pb_index_set_row_cache / pb_index_fill_row_cache at a time
};

// A handle's switches of the search pipeline and the delete: defaults, the environment at open (pb_index_finalize), the
// pb_set_* calls.  A copy of a handle (pb_index_clone, pb_index_clone_empty) takes its source's.
struct Switches {
    bool fast_approx = true;   // two-pass approximate stage (exact cut either way)
    bool k1_tc = true;         // a2 on the tensor cores (k_scores16_tc) with its certified consumers: the default;
                               // PB_K1_TC=0 keeps every sub-batch on the exact fp32 kernel (the device-gated fallback)
    int k1_margin = 1;         // E: code units an estimate-built 16-bit code may differ from the exact one (PB_K1_TC_E widens it)
    bool k1_diag = false;      // also run the exact table and report the largest code difference (PB_K1_TC_DIAG=1)
    bool table_diag = false;   // PB_TABLE_DIAG=1: rerun k_chunkmax16 and k_a5_live on the tensor-core table and count the
                               // words the fused chunk maxima and live bits differ in
    int approx_grid = 8;       // k_approx16 CTAs per SM and query (PB_APPROX_GRID)
    bool a5_prune = true;      // bound the first pass from the live score-table rows (PB_A5_PRUNE=0: dense first pass)
    long long a5_live = -1;    // live rows aimed at per query token (PB_A5_LIVE; -1: K / 512)
    float a5_m1 = 1.25f;       // round 1 of the pruned first pass keeps the M1 = a5_m1 * M best bounds (PB_A5_M1, >= 1)
    int a5_waves = 8;          // k_a5_bound's grid in waves of resident CTAs, over the batch (PB_A5_WAVES)
    bool probe16 = true;       // a3 threshold-first selection on the 16-bit table (PB_PROBE16=0: per-lane lists only)
    bool fast_exact = true;    // tensor-core certified filter in front of the exact stage (same results either way)
    bool filter_diag = false;  // PB_FILTER_DIAG=1: score every kept doc exactly and measure the filter's estimate against it
    bool pair_exact = true;    // exact stage on the (token, query token) pairs that can hold a maximum (PB_PAIR_EXACT=0: k_exact)
    int ws_grid = 8;           // k_maxsim_tc CTAs per SM across the batch (PB_WS_GRID)
    int ws_grid2 = 8;          // the same for its pass 2 over the filter's survivors (PB_WS_GRID2; 1: 0.54, 2: 0.43, 4 and 8: 0.40 ms)
    int lanes = 1;             // slices of a batch searched concurrently, each on its own stream (pb_set_lanes / PB_LANES; 1 = off)
    bool profiling = false;
    size_t st_budget = (size_t)8 << 30;  // workspace budget of one search call (PB_WS_BUDGET_MB)
    long long delete_window = 1ll << 22;   // tokens per compaction window of pb_index_delete (PB_DELETE_WINDOW_TOKENS)
};

struct pb_index : DocArrays, Switches {
    int device = 0;
    int dim = 0, nbits = 0, packed = 0;
    long long K = 0, doc_id_base = 0;
    int sm_count = 132;
    DevBuf centroids, w_rev;
    bool host_tier = false;    // PB_OPEN_HOST_RESIDUALS: `residuals` stays empty, the rows live in host.rows
    bool host_mutable = false; // PB_OPEN_HOST_MUTABLE: appends and deletes write the host rows
    HostTier host;
    RowCacheState rc;
    unsigned long long doc_gen = 0;  // changes with every publish: a fill built out of place checks it before its swap
    bool build_ivf = false;    // no inverted file was given: built from the codes at finalize (index.rs:850-873)
    float cmax = 1.0f;         // largest centroid L2 norm (range of the 16-bit score table)
    int cent_exp = 0;          // centroids enter the tensor-core operands scaled by 2^cent_exp (max norm in [1, 2))
    DevBuf cent_h16t, cent_l16t;  // its centroid operands: fp16 hi / lo, MMA tile order
    std::mutex lane_mu;        // one laned call at a time per handle (a second concurrent caller runs un-laned)
    std::vector<std::unique_ptr<RankWorker>> lane_workers;  // lane_workers[l - 1] runs lane l
    std::mutex mu;
    std::vector<std::unique_ptr<Workspace>> pool;
    // pb_search: concurrent single-query callers merged into shared batches (pb_index_set_coalescing; off by default)
    pbq::Queue<CoalescedRun> coalescer{CoalescedRun{this}, PB_ERR_CUDA};
    std::atomic<bool> coalesce_on{false};
    pbq::Config coalesce_cfg;  // as the caller set it: a replica set's max_inflight is per replica
    std::vector<std::unique_ptr<GatherBuf>> gather_pool;  // under mu
    float delete_ms[3] = {0.f, 0.f, 0.f};  // last pb_index_delete with profiling on: compaction, inverted file, norms
    // Readers (searches, stage entry points, accessors) share the arrays; pb_index_append / pb_index_reserve hold them
    // alone.  A writer also holds `gate`, which every reader passes first: pthread rwlocks prefer readers, so without
    // it a steady stream of searches could keep an append waiting forever.
    mutable std::mutex gate;
    mutable std::shared_mutex rw;
    std::shared_lock<std::shared_mutex> read_lock() const {
        { std::lock_guard<std::mutex> g(gate); }
        return std::shared_lock<std::shared_mutex>(rw);
    }
    // pb_index_load_devices / pb_index_load_replicas: this handle holds no documents and stands for the members of
    // `group` (deployment.cpp, replicas.cpp)
    std::unique_ptr<Group> group;
    // a rank of a replica of such a set, during one of its mutations: the vote it takes with the other replicas
    RepVote *rep_vote = nullptr;
    int rep_index = 0;
    // doc-sharded deployment (pb_index_comm_init / pb_index_group_join).  Declared last, so destroyed first: an NCCL
    // communicator goes before the workspace streams it ran on
    ShardComm comm;
};

// A workspace of the handle's pool for one call.  It goes back to the pool only after a call that ran to completion
// (done): its scratch invariants (cleared bitmaps, zeroed maxima) are restored by the kernels themselves, so a call
// that fails half way must not hand its buffers to the next caller; its workspace is synchronized and dropped.
struct WorkspaceLease {
    pb_index *ix;
    std::unique_ptr<Workspace> ws;
    bool done = false;
    pb_status acquire() {
        {
            std::lock_guard<std::mutex> g(ix->mu);
            if (!ix->pool.empty()) {
                ws = std::move(ix->pool.back());
                ix->pool.pop_back();
                return PB_OK;
            }
        }
        ws.reset(new Workspace());
        return ws->init();
    }
    ~WorkspaceLease() {
        if (!ws) return;
        if (done) {
            std::lock_guard<std::mutex> g(ix->mu);
            ix->pool.push_back(std::move(ws));
        } else {
            cudaStreamSynchronize(ws->stream);
        }
    }
};

// a non-blocking stream of one collective call, destroyed with it
struct OwnedStream {
    cudaStream_t s = nullptr;
    ~OwnedStream() {
        if (s) cudaStreamDestroy(s);
    }
};

// ------------------------------------------------------------------------------------------
// DIM dispatch.  The embedding widths are listed here and nowhere else:
//   BuiltDims  every DIM-templated kernel is instantiated for these (a handle, codec or k-means of another dim is
//              refused with PB_ERR_UNSUPPORTED);
//   TcDims     the tensor-core paths run at these: a2 on wgmma (k_scores16_tc), the MaxSim filter (k_maxsim_tc,
//              k_pair_exact, the token norms it needs) and the tensor-core assignment (k_assign_tc).  A multiple of 16
//              (wgmma K = 16) whose error bound k1_err_codes keeps E = 1; 32 and 256 stay on the fp32 kernels.
// dispatch(d, f) calls f(std::integral_constant<int, d>) for a listed d and fails for any other: no switch falls through
// to another width's kernel.
// ------------------------------------------------------------------------------------------
template <int... Ds> struct DimSet {
    static bool has(int d) { return ((d == Ds) || ...); }
    static pb_status check(int d) {
        if (has(d)) return PB_OK;
        std::string list;
        ((list += (list.empty() ? "" : "/") + std::to_string(Ds)), ...);
        return pb_fail(PB_ERR_UNSUPPORTED, "embedding_dim %d not built (%s)", d, list.c_str());
    }
    template <class F> static pb_status dispatch(int d, F &&f) {
        pb_status s = PB_OK;
        const bool hit = ((d == Ds ? (s = f(std::integral_constant<int, Ds>()), true) : false) || ...);
        return hit ? s : check(d);
    }
};
using BuiltDims = DimSet<32, 48, 64, 96, 128, 256>;
using TcDims = DimSet<48, 64, 96, 128>;

// the statements after `dim` with DIM bound to the handle's width, for every built width
#define PB_DIM_SWITCH(dim, ...)                                                                                        \
    CKS(BuiltDims::dispatch(dim, [&](auto dim_c) -> pb_status {                                                        \
        constexpr int DIM = decltype(dim_c)::value;                                                                    \
        __VA_ARGS__;                                                                                                   \
        return PB_OK;                                                                                                  \
    }))

// QS: query tokens per score-table row.  Up to 32 tokens: rounded up to 8 (rows of at most 64 bytes); beyond: to a
// multiple of 64, so that a row is whole 128-byte lines (a 96-byte row straddles lines and costs the first approximate
// pass extra L2 requests)
static int query_row_tokens(int nq_max) {
    return nq_max <= 32 ? std::max(8, (nq_max + 7) & ~7) : ((nq_max + 63) & ~63);
}

static size_t smem_scores(int dim) { return (size_t)(PB_TOK_TILE + 2 * PB_Q_TILE) * (dim + 4) * sizeof(float); }
static size_t smem_exact(int dim, int packed) {
    return (size_t)(PB_TOK_TILE + PB_Q_TILE) * (dim + 4) * sizeof(float) + PB_Q_TILE * 129 * sizeof(float) +
           PB_TOK_TILE * sizeof(int) + 256 * sizeof(float) + (size_t)PB_TOK_TILE * packed;
}

template <class Kern> static pb_status set_smem(Kern k, size_t bytes) {
    // a kernel's static shared memory counts towards the 48 KB a launch may use without opting in.  The opt-in only
    // grows: lanes launch one kernel with different sizes from several threads, and a smaller value set between another
    // lane's setting and its launch would fail that launch
    if (bytes <= 40 * 1024) return PB_OK;
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, size_t> opted;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> g(mu);
    size_t &cur = opted[{dev, (const void *)k}];
    if (bytes > cur) {
        CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        cur = bytes;
    }
    return PB_OK;
}

// CTAs of a kernel that fit one SM at this block size and dynamic shared memory (at least 1), asked of the runtime
// once per (device, kernel, threads, bytes)
template <class Kern> static pb_status resident_ctas(Kern k, int threads, size_t smem, int *out) {
    static std::mutex mu;
    static std::map<std::tuple<int, const void *, int, size_t>, int> known;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> g(mu);
    const auto key = std::make_tuple(dev, (const void *)k, threads, smem);
    auto it = known.find(key);
    if (it == known.end()) {
        int n = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k, threads, smem));
        it = known.emplace(key, std::max(1, n)).first;
    }
    *out = it->second;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// index open / close
// ------------------------------------------------------------------------------------------
static unsigned bitrev_n(unsigned v, int nbits) {
    unsigned r = 0;
    for (int k = 0; k < nbits; ++k)
        if (v & (1u << k)) r |= 1u << (nbits - 1 - k);
    return r;
}

template <class T>
static pb_status fetch_host(std::vector<T> &dst, const T *src, size_t n, int space) {
    dst.resize(n);
    if (n == 0) return PB_OK;
    if (space == PB_MEM_DEVICE) CK(cudaMemcpy(dst.data(), src, n * sizeof(T), cudaMemcpyDeviceToHost));
    else memcpy(dst.data(), src, n * sizeof(T));
    return PB_OK;
}

static pb_status upload(DevBuf &dst, const void *src, size_t bytes, int space) {
    CKS(dst.ensure(std::max<size_t>(bytes, 16)));
    if (bytes == 0) return PB_OK;
    CK(cudaMemcpy(dst.p, src, bytes, space == PB_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    return PB_OK;
}

// i64 -> u32 with a range check, streamed through a bounded staging buffer, into dst[dst_off..]
static pb_status upload_narrow(DevBuf &dst, long long dst_off, const int64_t *src, long long n, long long limit,
                               int space, const char *what) {
    if (n == 0) return PB_OK;
    DevBuf bad;
    CKS(bad.ensure(16));
    CK(cudaMemset(bad.p, 0, 4));
    const long long chunk = 1ll << 26;  // 64M elements = 512 MiB of i64
    DevBuf stage;
    if (space == PB_MEM_HOST) CKS(stage.ensure((size_t)std::min(n, chunk) * 8));
    for (long long o = 0; o < n; o += chunk) {
        long long m = std::min(chunk, n - o);
        const long long *in = reinterpret_cast<const long long *>(src) + o;
        if (space == PB_MEM_HOST) {
            CK(cudaMemcpy(stage.p, in, (size_t)m * 8, cudaMemcpyHostToDevice));
            in = stage.as<long long>();
        }
        k_narrow_i64_u32<<<1184, 256>>>(in, dst.as<uint32_t>() + dst_off + o, m, limit, bad.as<int>());
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
    }
    int hbad = 0;
    CK(cudaMemcpy(&hbad, bad.p, 4, cudaMemcpyDeviceToHost));
    if (hbad) return pb_fail(PB_ERR_INVALID, "%s contains a value outside [0, %lld)", what, limit);
    return PB_OK;
}

// out[i] = in[0] + .. + in[i - 1] for i < n
static pb_status exclusive_sum(const long long *in, long long *out, long long n, DevBuf &tmp) {
    size_t tb = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, n));
    CKS(tmp.ensure(tb + 16));
    CK(cub::DeviceScan::ExclusiveSum(tmp.p, tb, in, out, n));
    return PB_OK;
}

// An inverted file computed from a directory's ivf.npy (host, total entries, lengths [K], global ids) into (out, out_off,
// *out_len): every list filtered to docs [b, e) in file order, ids minus b.  With a deleted set (bits, word_pre over
// the directory's docs, b = 0) its ids leave the lists too and survivors are renumbered (delete.rs:196-237); with
// the sorted (centroid, doc) keys of m appended docs, each list is followed by its new pairs as ids limit + doc
// (update.rs:1000-1067).  The file goes through a staging buffer of at most 2^26 entries (PB_LOAD_IVF_SLAB sets
// another size): a count pass, then the write pass into the exactly sized output, which copies the file a second time
// when it is more than one slab.  Any entry outside [0, limit) fails.
static pb_status ivf_from_file(pb_index *ix, const int64_t *ivf, const int32_t *lengths, long long total, long long limit,
                               long long b, long long e, const uint32_t *bits, const long long *word_pre, const u64 *keys,
                               long long m_keys, DevBuf &out, DevBuf &out_off, long long *out_len) {
    CK(cudaSetDevice(ix->device));
    const long long K = ix->K;
    std::vector<long long> foff((size_t)K + 1, 0);
    for (long long i = 0; i < K; ++i) {
        if (lengths[i] < 0) return pb_fail(PB_ERR_INVALID, "ivf_lengths[%lld] < 0", i);
        foff[i + 1] = foff[i] + lengths[i];
    }
    long long slab = 1ll << 26;  // 64M entries = 512 MiB of i64, as upload_narrow
    if (const char *v = getenv("PB_LOAD_IVF_SLAB")) slab = std::max(1ll, atoll(v));  // entries per slab
    const int grid = ix->sm_count * 8;
    DevBuf doff, cnt, stage, bad, tmp;
    CKS(upload(doff, foff.data(), foff.size() * 8, PB_MEM_HOST));
    CKS(cnt.ensure((size_t)(K + 1) * 8));
    CK(cudaMemset(cnt.p, 0, (size_t)(K + 1) * 8));
    CKS(stage.ensure(std::max<size_t>((size_t)std::min(total, slab) * 8, 16)));
    CKS(bad.ensure(16));
    CK(cudaMemset(bad.p, 0, 4));
    // slab [o, o + m) overlaps the lists c0 <= c < c1: c0 the last list starting at or before o, c1 the first at or after o + m
    auto lists = [&](long long o, long long m, long long &c0, long long &c1) {
        c0 = std::upper_bound(foff.begin(), foff.end(), o) - foff.begin() - 1;
        c1 = std::lower_bound(foff.begin(), foff.end(), o + m) - foff.begin();
    };
    // the kept entries of slab [o, o + m) at their lists' cursors
    DevBuf cur;
    CKS(cur.ensure((size_t)(K + 1) * 8));
    auto write = [&](long long o, long long m, long long c0, long long c1) -> pb_status {
        k_ivf_range_write<<<grid, 256>>>(stage.as<long long>(), o, m, doff.as<long long>(), c0, c1, b, e, bits, word_pre,
                                         cur.as<long long>(), out.as<uint32_t>());
        CK(cudaGetLastError());
        return PB_OK;
    };
    // When every valid entry is kept the offsets are the file's (shifted by the new pairs before each list), and each
    // slab is written as soon as it is counted, so the file is copied once.  Otherwise the write pass waits for the
    // scan of all the counts.
    const bool whole = b == 0 && e >= limit && !bits;
    CKS(out_off.ensure((size_t)(K + 1) * 8));
    if (whole) {
        if (m_keys > 0) {  // new_off[c] = file_off[c] + new pairs of the centroids below c
            CKS(tmp.ensure((size_t)(K + 1) * 8));
            k_ivf_offsets<<<(unsigned)((K + 256) / 256), 256>>>(keys, m_keys, K, tmp.as<long long>());
            CK(cudaGetLastError());
            std::vector<long long> before((size_t)K + 1);
            CK(cudaMemcpy(before.data(), tmp.p, before.size() * 8, cudaMemcpyDeviceToHost));
            for (long long c = 0; c <= K; ++c) before[c] += foff[c];
            CK(cudaMemcpy(out_off.p, before.data(), before.size() * 8, cudaMemcpyHostToDevice));
        } else {
            CK(cudaMemcpy(out_off.p, doff.p, (size_t)(K + 1) * 8, cudaMemcpyDeviceToDevice));
        }
        CK(cudaMemcpy(cur.p, out_off.p, (size_t)(K + 1) * 8, cudaMemcpyDeviceToDevice));
        *out_len = total + std::max(m_keys, 0ll);
        CKS(out.ensure(std::max<size_t>((size_t)*out_len * 4, 16)));
    }
    for (long long o = 0; o < total; o += slab) {
        const long long m = std::min(slab, total - o);
        long long c0, c1;
        lists(o, m, c0, c1);
        CK(cudaMemcpy(stage.p, ivf + o, (size_t)m * 8, cudaMemcpyHostToDevice));
        k_ivf_range_count<<<grid, 256>>>(stage.as<long long>(), o, m, doff.as<long long>(), c0, c1, limit, b, e, bits,
                                         cnt.as<long long>(), bad.as<int>());
        CK(cudaGetLastError());
        if (whole) CKS(write(o, m, c0, c1));
    }
    int hbad = 0;
    CK(cudaMemcpy(&hbad, bad.p, 4, cudaMemcpyDeviceToHost));
    if (hbad) return pb_fail(PB_ERR_INVALID, "ivf contains a value outside [0, %lld)", limit);
    if (whole && m_keys > 0)  // the j-th new pair of centroid c after c's file list: file_off[c + 1] + j
        k_ivf_merge_new<<<grid, 256>>>(keys, m_keys, doff.as<long long>(), (uint32_t)limit, out.as<uint32_t>());
    if (!whole) {
        CKS(exclusive_sum(cnt.as<long long>(), out_off.as<long long>(), K + 1, tmp));
        CK(cudaMemcpy(out_len, out_off.as<long long>() + K, 8, cudaMemcpyDeviceToHost));
        CKS(out.ensure(std::max<size_t>((size_t)*out_len * 4, 16)));
        CK(cudaMemcpy(cur.p, out_off.p, (size_t)K * 8, cudaMemcpyDeviceToDevice));
        for (long long o = 0; *out_len > 0 && o < total; o += slab) {
            const long long m = std::min(slab, total - o);
            long long c0, c1;
            lists(o, m, c0, c1);
            if (total > slab) CK(cudaMemcpy(stage.p, ivf + o, (size_t)m * 8, cudaMemcpyHostToDevice));
            CKS(write(o, m, c0, c1));
        }
    }
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    return PB_OK;
}

// The inverted file of an index opened without one, as the part of a directory's ivf.npy that lies in docs [b, e)
pb_status pb_index_upload_ivf_range(pb_index *ix, const int64_t *ivf, const int32_t *lengths, long long total,
                                    long long limit, long long b, long long e) {
    CKS(ivf_from_file(ix, ivf, lengths, total, limit, b, e, nullptr, nullptr, nullptr, 0, ix->ivf, ix->ivf_off,
                      &ix->ivf_len));
    ix->build_ivf = false;
    return PB_OK;
}

// codes + packed residuals of tokens [tok_off, tok_off+n) (one chunk file pair, or everything)
pb_status pb_index_upload_tokens(pb_index *ix, long long tok_off, const int64_t *codes, const uint8_t *residuals,
                                 long long n, int space) {
    if (n == 0) return PB_OK;
    if (tok_off < 0 || tok_off + n > ix->N) return pb_fail(PB_ERR_INVALID, "token range [%lld,+%lld) outside the index", tok_off, n);
    CK(cudaSetDevice(ix->device));
    if (!ix->residuals.owned) {  // PB_OPEN_ADOPT_RESIDUALS: the caller's array is the index
        if (tok_off != 0 || n != ix->N || residuals != ix->residuals.as<uint8_t>())
            return pb_fail(PB_ERR_INVALID, "adopted residuals cover the whole index");
    } else if (ix->host_tier) {
        CKS(ix->host.rows->write((size_t)tok_off * ix->packed, residuals, (size_t)n * ix->packed, space));
    } else
        CK(cudaMemcpy(ix->residuals.as<uint8_t>() + (size_t)tok_off * ix->packed, residuals, (size_t)n * ix->packed,
                      space == PB_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    return upload_narrow(ix->codes, tok_off, codes, n, ix->K, space, "codes");
}

// The offsets of docs of lengths dl starting at token t0 (off[0] = t0, dl.size() + 1 of them); the longest doc is
// folded into *maxlen.  A length outside [0, 2^30] fails.
static pb_status doc_offsets(const std::vector<int64_t> &dl, long long t0, std::vector<long long> &off, int *maxlen) {
    off.assign(dl.size() + 1, t0);
    for (size_t i = 0; i < dl.size(); ++i) {
        if (dl[i] < 0 || dl[i] > (1 << 30)) return pb_fail(PB_ERR_INVALID, "doc_lengths[%zu] = %lld", i, (long long)dl[i]);
        off[i + 1] = off[i] + dl[i];
        *maxlen = std::max<int>(*maxlen, (int)dl[i]);
    }
    return PB_OK;
}

// the longest of the D docs at host offsets off
static int longest_doc(const std::vector<long long> &off, long long D) {
    int m = 0;
    for (long long j = 0; j < D; ++j) m = std::max<int>(m, (int)(off[j + 1] - off[j]));
    return m;
}

// Everything except the per-token arrays (d->codes / d->residuals may be NULL here).
pb_status pb_index_open_begin(const pb_index_desc *d, pb_index **out) {
    if (!d || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    *out = nullptr;
    if (d->nbits <= 0 || 8 % d->nbits != 0)  // codec.rs:161-166
        return pb_fail(PB_ERR_INVALID, "nbits must be a divisor of 8, got %d", d->nbits);
    if (d->dim <= 0 || d->dim % 4 != 0) return pb_fail(PB_ERR_INVALID, "embedding_dim %d must be a positive multiple of 4", d->dim);
    CKS(BuiltDims::check(d->dim));
    if (d->num_centroids <= 0 || d->num_documents < 0 || d->num_embeddings < 0)
        return pb_fail(PB_ERR_INVALID, "bad shapes K=%lld D=%lld N=%lld", (long long)d->num_centroids,
                       (long long)d->num_documents, (long long)d->num_embeddings);
    if (d->num_centroids >= (1ll << 32) - 1 || d->num_documents >= (1ll << 32) - 1)
        return pb_fail(PB_ERR_UNSUPPORTED, "K and D must be below 2^32-1 per shard");
    if (d->doc_id_base < 0 || d->doc_id_base + d->num_documents >= (1ll << 32) - 1)
        return pb_fail(PB_ERR_UNSUPPORTED, "global doc ids must stay below 2^32-1");
    if (!d->centroids || !d->bucket_weights || (!d->doc_lengths && d->num_documents) || (!d->ivf_lengths && d->ivf))
        return pb_fail(PB_ERR_INVALID, "null index array");
    if ((d->flags & PB_OPEN_ADOPT_RESIDUALS) && (d->memory_space != PB_MEM_DEVICE || !d->residuals))
        return pb_fail(PB_ERR_INVALID, "PB_OPEN_ADOPT_RESIDUALS needs device-resident residuals");
    if ((d->flags & PB_OPEN_ADOPT_RESIDUALS) && (d->flags & PB_OPEN_HOST_RESIDUALS))
        return pb_fail(PB_ERR_INVALID, "PB_OPEN_ADOPT_RESIDUALS and PB_OPEN_HOST_RESIDUALS exclude each other");
    if ((d->flags & PB_OPEN_HOST_MUTABLE) && !(d->flags & PB_OPEN_HOST_RESIDUALS))
        return pb_fail(PB_ERR_INVALID, "PB_OPEN_HOST_MUTABLE needs PB_OPEN_HOST_RESIDUALS");
    int seg_shift = 28;
    if (const char *e = getenv("PB_HOST_SEGMENT_BYTES"); e && (d->flags & PB_OPEN_HOST_RESIDUALS)) {
        const long long v = atoll(e);
        if (v < 256 || v > (1ll << 40) || (v & (v - 1)))
            return pb_fail(PB_ERR_INVALID, "PB_HOST_SEGMENT_BYTES=%s is not a power of two in [256, 2^40]", e);
        seg_shift = __builtin_ctzll((unsigned long long)v);
    }
    CKS(check_device(d->device));
    std::unique_ptr<pb_index> ix(new pb_index());
    ix->device = d->device;
    ix->dim = d->dim;
    ix->nbits = d->nbits;
    ix->packed = d->dim * d->nbits / 8;
    ix->K = d->num_centroids;
    ix->D = d->num_documents;
    ix->N = d->num_embeddings;
    ix->doc_id_base = d->doc_id_base;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, d->device));
    ix->sm_count = prop.multiProcessorCount;
    for (const char *name : {"PB_ST_BUDGET_MB", "PB_WS_BUDGET_MB"})
        if (const char *e = getenv(name)) {
            long v = atol(e);
            if (v > 0) ix->st_budget = (size_t)v << 20;
        }
    if (const char *e = getenv("PB_DELETE_WINDOW_TOKENS")) ix->delete_window = std::max(1ll, atoll(e));
    const int sp = d->memory_space;
    // doc offsets (index.rs:1107-1110)
    std::vector<int64_t> dl;
    CKS(fetch_host(dl, d->doc_lengths, (size_t)ix->D, sp));
    std::vector<long long> doff;
    CKS(doc_offsets(dl, 0, doff, &ix->max_doclen));
    if (doff[ix->D] != ix->N)
        return pb_fail(PB_ERR_INVALID, "sum(doc_lengths)=%lld != num_embeddings=%lld", doff[ix->D], ix->N);
    CKS(upload(ix->doc_off, doff.data(), doff.size() * 8, PB_MEM_HOST));
    // ivf offsets (index.rs:1089-1094); without an inverted file it is built from the codes in pb_index_finalize
    ix->build_ivf = d->ivf_lengths == nullptr;
    if (!ix->build_ivf) {
        std::vector<int32_t> il;
        CKS(fetch_host(il, d->ivf_lengths, (size_t)ix->K, sp));
        std::vector<long long> ioff((size_t)ix->K + 1, 0);
        for (long long i = 0; i < ix->K; ++i) {
            if (il[i] < 0) return pb_fail(PB_ERR_INVALID, "ivf_lengths[%lld] < 0", i);
            ioff[i + 1] = ioff[i] + il[i];
        }
        ix->ivf_len = ioff[ix->K];
        if (ix->ivf_len && !d->ivf) return pb_fail(PB_ERR_INVALID, "null ivf");
        CKS(upload(ix->ivf_off, ioff.data(), ioff.size() * 8, PB_MEM_HOST));
    }
    // bucket weights with the packer's bit reversal folded in (codec.rs:168-214, :389-395)
    std::vector<float> w;
    CKS(fetch_host(w, d->bucket_weights, (size_t)1 << ix->nbits, sp));
    std::vector<float> wrev(256, 0.f);
    for (unsigned f = 0; f < (1u << ix->nbits); ++f) wrev[f] = w[bitrev_n(f, ix->nbits)];
    CKS(upload(ix->w_rev, wrev.data(), 256 * sizeof(float), PB_MEM_HOST));
    CKS(upload(ix->centroids, d->centroids, (size_t)ix->K * ix->dim * sizeof(float), sp));
    ix->host_tier = (d->flags & PB_OPEN_HOST_RESIDUALS) != 0;
    ix->host_mutable = (d->flags & PB_OPEN_HOST_MUTABLE) != 0;
    if (d->flags & PB_OPEN_ADOPT_RESIDUALS)
        ix->residuals.adopt(const_cast<uint8_t *>(d->residuals), (size_t)ix->N * ix->packed);
    else if (ix->host_tier) {
        ix->host.rows = std::make_shared<HostRows>();
        ix->host.rows->shift = seg_shift;
        CKS(ix->host.rows->open((size_t)ix->N * ix->packed));
        CK(cudaSetDevice(ix->device));
        CKS(ix->host.sync());
    }
    else CKS(ix->residuals.ensure(std::max<size_t>((size_t)ix->N * ix->packed, 16)));
    CKS(ix->codes.ensure(std::max<size_t>((size_t)ix->N * 4, 16)));
    if (!ix->build_ivf) {
        CKS(ix->ivf.ensure(std::max<size_t>((size_t)ix->ivf_len * 4, 16)));
        CKS(upload_narrow(ix->ivf, 0, d->ivf, ix->ivf_len, std::max<long long>(ix->D, 1), sp, "ivf"));
    }
    *out = ix.release();
    return PB_OK;
}

// The distinct (centroid, doc) pairs of docs [d0, d0 + n) as sorted keys code << 32 | (doc - d0) in `keys` (*m_out of
// them), from the per-doc distinct code lists: k_ivf_pairs, a radix sort, and a unique pass for the raw lists of docs
// longer than PB_UCODE_MAX.  `cap` bounds the pair count (the ucodes entries of those docs).
static pb_status sorted_doc_pairs(pb_index *ix, long long d0, long long n, long long cap, DevBuf &keys, long long *m_out) {
    cap = std::max<long long>(cap, 1);
    DevBuf kb, cnt, tmp;
    CKS(keys.ensure((size_t)cap * 8));
    CKS(kb.ensure((size_t)cap * 8));
    CKS(cnt.ensure(16));
    CK(cudaMemset(cnt.p, 0, 16));
    if (n > 0) {
        k_ivf_pairs<<<ix->sm_count * 8, 256>>>(ix->ucodes.as<uint32_t>(), ix->udoc_off.as<long long>() + d0, n, keys.as<u64>(),
                                               cnt.as<unsigned long long>());
        CK(cudaGetLastError());
    }
    unsigned long long m = 0;
    CK(cudaMemcpy(&m, cnt.p, 8, cudaMemcpyDeviceToHost));
    if (m > (1ull << 31) - 2) return pb_fail(PB_ERR_UNSUPPORTED, "more than 2^31 (centroid, doc) pairs per shard");
    int kbits = 1;
    while ((1ll << kbits) < ix->K) ++kbits;
    size_t tb = 0;
    CK(cub::DeviceRadixSort::SortKeys(nullptr, tb, keys.as<u64>(), kb.as<u64>(), (int)m, 0, 32 + kbits));
    size_t tb2 = 0;
    CK(cub::DeviceSelect::Unique(nullptr, tb2, kb.as<u64>(), keys.as<u64>(), cnt.as<int>() + 2, (int)m));
    CKS(tmp.ensure(std::max(tb, tb2) + 16));
    CK(cub::DeviceRadixSort::SortKeys(tmp.p, tb, keys.as<u64>(), kb.as<u64>(), (int)m, 0, 32 + kbits));
    CK(cub::DeviceSelect::Unique(tmp.p, tb2, kb.as<u64>(), keys.as<u64>(), cnt.as<int>() + 2, (int)m));
    int m2 = 0;
    CK(cudaMemcpy(&m2, cnt.as<int>() + 2, 4, cudaMemcpyDeviceToHost));
    *m_out = m2;
    return PB_OK;
}

// The inverted file of an index opened without one (index.rs:850-873), from the per-doc distinct code lists.
static pb_status build_ivf_on_device(pb_index *ix) {
    CKS(ix->ivf_off.ensure((size_t)(ix->K + 1) * 8));
    DevBuf ka;
    long long m2 = 0;
    CKS(sorted_doc_pairs(ix, 0, ix->D, ix->n_ucodes, ka, &m2));
    ix->ivf_len = m2;
    CKS(ix->ivf.ensure(std::max<size_t>((size_t)m2 * 4, 16)));
    k_ivf_from_keys<<<ix->sm_count * 8, 256>>>(ka.as<u64>(), m2, ix->ivf.as<uint32_t>());
    k_ivf_offsets<<<(unsigned)((ix->K + 256) / 256), 256>>>(ka.as<u64>(), m2, ix->K, ix->ivf_off.as<long long>());
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    return PB_OK;
}

// Operands of the tensor-core kernels that depend on the centroids alone: the scaled hi / lo tiles of the score table
// (k_scores16_tc).
static pb_status build_centroid_operands(pb_index *ix) {
    if ((ix->k1_diag || ix->k1_tc) && ix->cmax > 0.0f && ix->cmax < 3.0e38f) {
        // operands of the tensor-core score table: centroids * 2^cent_exp (max norm in [1, 2)), fp16 hi / lo parts
        ix->cent_exp = -ilogbf(ix->cmax);
        const size_t elems = (size_t)((ix->K + 127) / 128) * 128 * ix->dim;
        CKS(ix->cent_h16t.ensure(elems * 2));
        CKS(ix->cent_l16t.ensure(elems * 2));
        CK(cudaMemset(ix->cent_h16t.p, 0, elems * 2));
        CK(cudaMemset(ix->cent_l16t.p, 0, elems * 2));
        k_rows_to_f16_split_tiles<<<ix->sm_count * 8, 256>>>(ix->centroids.as<float>(), ix->K, ix->dim, ix->cent_exp,
                                                            ix->cent_h16t.as<__half>(), ix->cent_l16t.as<__half>());
        CK(cudaGetLastError());
    }
    return PB_OK;
}

// 1 / |c + w| of n tokens (codes, packed residuals) into inv; min |c + w| and max |w| over them folded into mn[0] / mn[1]
static pb_status launch_min_vnorm(pb_index *ix, const uint32_t *codes, const uint8_t *res, long long n, float *inv,
                                  float *mn) {
    if (n == 0) return PB_OK;
    return TcDims::dispatch(ix->dim, [&](auto dim_c) -> pb_status {
        k_min_vnorm<decltype(dim_c)::value><<<ix->sm_count * 8, 256>>>(ix->centroids.as<float>(), ix->w_rev.as<float>(),
                                                                      ix->nbits, codes, res, n, mn, inv);
        CK(cudaGetLastError());
        return PB_OK;
    });
}
// The filter's token norms of tokens [t0, t.N) of `a` (the handle's arrays, or a rebalance's new ones), at the
// tensor-core widths: 1 / |c + w| into a.tok_inv_norm, and into t.vmin / t.wmax the least |c + w| and the largest |w|
// over those tokens and the seed (0 / 0 over nothing).  An append seeds with the handle's values; open, delete and
// rebalance, which cover every token, with {3e38, 0}.  A handle that had no tokens gets its centroid operands first.
// A host-tier handle's rows go through a device buffer in slabs of 2^22 tokens; the per-token values and the folded
// min / max do not depend on the slabs, so they are bit-identical to a resident open's (the filter's certificate rests
// on them).  mn: 8 bytes of scratch.
static pb_status token_norms(pb_index *ix, DocArrays &a, long long t0, const float seed[2], DocTotals &t, DevBuf &mn) {
    float got[2] = {seed[0], seed[1]};
    if (TcDims::has(ix->dim) && t.N > 0) {
        if (ix->N == 0) CKS(build_centroid_operands(ix));
        const long long n = t.N - t0, slab = ix->host_tier ? 1ll << 22 : std::max(n, 1ll);
        DevBuf st;
        if (ix->host_tier) CKS(st.ensure((size_t)std::min(n, slab) * ix->packed + 16));
        CKS(mn.ensure(16));
        CK(cudaMemcpy(mn.p, seed, 8, cudaMemcpyHostToDevice));
        for (long long o = t0; o < t.N; o += slab) {
            const long long m = std::min(slab, t.N - o);
            const uint8_t *res = st.as<uint8_t>();
            if (ix->host_tier) {
                CKS(ix->host.rows->to_device((size_t)o * ix->packed, st.as<uint8_t>(), (size_t)m * ix->packed, 0));
                CK(cudaStreamSynchronize(0));
            } else
                res = a.residuals.as<uint8_t>() + (size_t)o * ix->packed;
            CKS(launch_min_vnorm(ix, a.codes.as<uint32_t>() + o, res, m, a.tok_inv_norm.as<float>() + o, mn.as<float>()));
        }
        CK(cudaMemcpy(got, mn.p, 8, cudaMemcpyDeviceToHost));
    }
    t.vmin = got[0] < 1e30f ? got[0] : 0.0f;
    t.wmax = got[1];
    return PB_OK;
}

// The distinct-code lists k_approx walks, of docs [d0, d0 + n) of the handle, after the u0 entries of the docs before
// them: a count pass, the offsets on the host into udoc_off [d0, d0 + n] (udoc_off holds d0 + n + 1 entries, absolute
// positions into ucodes), then the lists into ucodes.  ucodes is sized as a first allocation is, or grows keeping its
// first u0 entries.  The new entry count goes to *u1.
static pb_status unique_codes(pb_index *ix, long long d0, long long n, long long u0, long long *u1) {
    std::vector<long long> uoff((size_t)n + 1, u0);
    const int blocks = (int)std::min<long long>(n, (long long)ix->sm_count * 16);
    if (n > 0) {
        DevBuf counts;
        CKS(counts.ensure((size_t)n * 4));
        k_unique_codes<<<blocks, 128>>>(ix->codes.as<uint32_t>(), ix->doc_off.as<long long>() + d0, n, nullptr, nullptr,
                                        counts.as<int>());
        CK(cudaGetLastError());
        std::vector<int> hc((size_t)n);
        CK(cudaMemcpy(hc.data(), counts.p, hc.size() * 4, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < n; ++i) uoff[i + 1] = uoff[i] + hc[i];
    }
    *u1 = uoff[n];
    const size_t bytes = std::max<size_t>((size_t)*u1 * 4, 16);
    CKS(ix->ucodes.p ? ix->ucodes.grow(bytes, (size_t)u0 * 4) : ix->ucodes.ensure(bytes));
    CK(cudaMemcpy(ix->udoc_off.as<long long>() + d0, uoff.data(), uoff.size() * 8, cudaMemcpyHostToDevice));
    if (n > 0) {
        k_unique_codes<<<blocks, 128>>>(ix->codes.as<uint32_t>(), ix->doc_off.as<long long>() + d0, n,
                                        ix->udoc_off.as<long long>() + d0, ix->ucodes.as<uint32_t>(), nullptr);
        CK(cudaGetLastError());
    }
    return PB_OK;
}

// The coalescing a handle starts with: PB_COALESCE (max_queries), PB_COALESCE_WAIT_US, PB_COALESCE_INFLIGHT
static pb_status coalesce_env_defaults(pb_index *ix) {
    if (const char *e = getenv("PB_COALESCE")) {
        pb_coalesce_config c = {atoi(e), 0, 2};
        if (const char *w = getenv("PB_COALESCE_WAIT_US")) c.max_wait_us = std::max(0, atoi(w));
        if (const char *f = getenv("PB_COALESCE_INFLIGHT")) c.max_inflight = std::max(1, atoi(f));
        c.max_queries = std::max(1, c.max_queries);
        CKS(pb_index_set_coalescing(ix, &c));
    }
    return PB_OK;
}

// A deployment's or replica set's handle: no documents of its own; what every member shares, from the first
pb_index *pb_index_new_group(Group *g, const pb_index *first) {
    pb_index *ix = new pb_index();
    ix->group.reset(g);
    pb_index_deployment_rank0(ix, first);
    coalesce_env_defaults(ix);  // cannot fail: the handle joins no group
    return ix;
}
void pb_index_deployment_rank0(pb_index *ix, const pb_index *rank0) {
    ix->device = rank0->device, ix->dim = rank0->dim, ix->nbits = rank0->nbits, ix->packed = rank0->packed;
    ix->K = rank0->K;
}

// The calls a deployment or a replica set refuses: each addresses one rank's handle, one device, or one group
static pb_status refuse_deployment(const pb_index *ix, const char *call) {
    return ix && ix->group ? ix->group->refuse(call) : PB_OK;
}

// Derived arrays that need every token: the per-doc distinct-code lists, the token norms, and the inverted file of an
// index opened without one.
pb_status pb_index_finalize(pb_index *ix) {
    CK(cudaSetDevice(ix->device));
    if ((unsigned long long)ix->K * 1024ull * 4ull >= (1ull << 40)) return pb_fail(PB_ERR_UNSUPPORTED, "K too large");
    {
        DevBuf mx;
        CKS(mx.ensure(16));
        CK(cudaMemset(mx.p, 0, 4));
        k_max_row_norm<<<ix->sm_count * 4, 256>>>(ix->centroids.as<float>(), ix->K, ix->dim, mx.as<float>());
        CK(cudaGetLastError());
        float m2 = 0.f;
        CK(cudaMemcpy(&m2, mx.p, 4, cudaMemcpyDeviceToHost));
        ix->cmax = sqrtf(m2);
        if (const char *e = getenv("PB_FAST_APPROX")) ix->fast_approx = atoi(e) != 0;
        if (const char *e = getenv("PB_FAST_EXACT")) ix->fast_exact = atoi(e) != 0;
        if (const char *e = getenv("PB_FILTER_DIAG")) ix->filter_diag = atoi(e) != 0;
        if (const char *e = getenv("PB_PAIR_EXACT")) ix->pair_exact = atoi(e) != 0;
        if (const char *e = getenv("PB_WS_GRID")) ix->ws_grid = std::max(1, atoi(e));
        if (const char *e = getenv("PB_WS_GRID2")) ix->ws_grid2 = std::max(1, atoi(e));
        if (const char *e = getenv("PB_LANES")) ix->lanes = std::min(8, std::max(1, atoi(e)));
        if (const char *e = getenv("PB_PROBE16")) ix->probe16 = atoi(e) != 0;
        if (const char *e = getenv("PB_K1_TC_DIAG")) ix->k1_diag = atoi(e) != 0;
        if (const char *e = getenv("PB_TABLE_DIAG")) ix->table_diag = atoi(e) != 0;
        if (const char *e = getenv("PB_K1_TC")) ix->k1_tc = atoi(e) != 0;
        if (const char *e = getenv("PB_K1_TC_E")) ix->k1_margin = std::max(1, atoi(e));
        if (const char *e = getenv("PB_APPROX_GRID")) ix->approx_grid = std::max(1, atoi(e));
        if (const char *e = getenv("PB_A5_PRUNE")) ix->a5_prune = atoi(e) != 0;
        if (const char *e = getenv("PB_A5_LIVE")) ix->a5_live = std::max(0ll, atoll(e));
        if (const char *e = getenv("PB_A5_M1")) ix->a5_m1 = std::max(1.0f, (float)atof(e));
        if (const char *e = getenv("PB_A5_WAVES")) ix->a5_waves = std::max(1, atoi(e));
        CKS(coalesce_env_defaults(ix));
    }
    if (TcDims::has(ix->dim) && ix->N > 0) {
        // operands of the tensor-core score table, and the token norms of the filter
        CKS(build_centroid_operands(ix));
        CKS(ix->tok_inv_norm.ensure((size_t)ix->N * 4));
        DevBuf mn;
        const float seed[2] = {3.0e38f, 0.0f};
        CKS(token_norms(ix, *ix, 0, seed, *ix, mn));
    }
    CKS(ix->udoc_off.ensure(std::max<size_t>((size_t)(ix->D + 1) * 8, 16)));
    CKS(unique_codes(ix, 0, ix->D, 0, &ix->n_ucodes));
    CK(cudaDeviceSynchronize());
    if (ix->build_ivf) CKS(build_ivf_on_device(ix));
    return PB_OK;
}

extern "C" pb_status pb_index_export_ivf(pb_index *ix, int64_t *out_ivf, int32_t *out_lengths, int64_t *out_total) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix->group) return ix->group->export_ivf(out_ivf, out_lengths, out_total);
    auto rd = ix->read_lock();
    CK(cudaSetDevice(ix->device));
    if (out_total) *out_total = ix->ivf_len;
    if (!out_ivf && !out_lengths) return PB_OK;
    DevBuf di, dl;
    if (out_ivf) CKS(di.ensure(std::max<size_t>((size_t)ix->ivf_len * 8, 16)));
    if (out_lengths) CKS(dl.ensure(std::max<size_t>((size_t)ix->K * 4, 16)));
    k_ivf_export<<<ix->sm_count * 8, 256>>>(ix->ivf.as<uint32_t>(), ix->ivf_off.as<long long>(), ix->ivf_len, ix->K,
                                           ix->doc_id_base, out_ivf ? di.as<long long>() : nullptr,
                                           out_lengths ? dl.as<int>() : nullptr);
    CK(cudaGetLastError());
    if (out_ivf && ix->ivf_len) CK(cudaMemcpy(out_ivf, di.p, (size_t)ix->ivf_len * 8, cudaMemcpyDeviceToHost));
    if (out_lengths) CK(cudaMemcpy(out_lengths, dl.p, (size_t)ix->K * 4, cudaMemcpyDeviceToHost));
    return PB_OK;
}

extern "C" pb_status pb_index_open(const pb_index_desc *d, pb_index **out) {
    if (!d || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    if (d->num_embeddings > 0 && (!d->codes || !d->residuals)) return pb_fail(PB_ERR_INVALID, "null index array");
    pb_index *ix = nullptr;
    CKS(pb_index_open_begin(d, &ix));
    pb_status s = pb_index_upload_tokens(ix, 0, d->codes, d->residuals, d->num_embeddings, d->memory_space);
    if (s == PB_OK) s = pb_index_finalize(ix);
    if (s != PB_OK) {
        pb_index_close(ix);
        return s;
    }
    *out = ix;
    return PB_OK;
}

extern "C" void pb_index_close(pb_index *ix) {
    if (!ix) return;
    ix->group.reset();  // first: joins its threads, closes its members
    cudaSetDevice(ix->device);
    ix->lane_workers.clear();  // joins the helper threads
    cudaDeviceSynchronize();
    delete ix;
}

// D and N change under pb_index_append; K, dim, nbits and the device are fixed at open
void pb_index_totals(const pb_index *ix, long long *D, long long *N) {
    if (ix->group) return ix->group->totals(D, N);
    auto rd = ix->read_lock();
    *D = ix->D, *N = ix->N;
}
extern "C" int64_t pb_index_num_documents(const pb_index *ix) {
    long long D = 0, N = 0;
    if (ix) pb_index_totals(ix, &D, &N);
    return D;
}
extern "C" int64_t pb_index_num_embeddings(const pb_index *ix) {
    long long D = 0, N = 0;
    if (ix) pb_index_totals(ix, &D, &N);
    return N;
}
extern "C" int64_t pb_index_num_partitions(const pb_index *ix) { return ix ? ix->K : 0; }
extern "C" double pb_index_avg_doclen(const pb_index *ix) {
    long long D = 0, N = 0;
    if (ix) pb_index_totals(ix, &D, &N);
    return D ? (double)N / (double)D : 0.0;
}
extern "C" int32_t pb_index_embedding_dim(const pb_index *ix) { return ix ? ix->dim : 0; }
extern "C" int32_t pb_index_nbits(const pb_index *ix) { return ix ? ix->nbits : 0; }
extern "C" int32_t pb_index_device(const pb_index *ix) {
    if (!ix) return -1;
    int32_t dv = ix->device;  // a group's: its first member's, which a resize may change
    if (ix->group) ix->group->first([&](pb_index *m) { return dv = pb_index_device(m), PB_OK; });
    return dv;
}

extern "C" pb_status pb_index_memory(const pb_index *ix, int64_t *device_bytes, int64_t *host_bytes) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix->group) return ix->group->memory(device_bytes, host_bytes);
    auto rd = ix->read_lock();
    size_t dev = ix->centroids.cap + ix->w_rev.cap + ix->cent_h16t.cap + ix->cent_l16t.cap + ix->rc.rows.cap;
    for (const DevBuf *b : DocArrays::buffers(*ix))
        if (b->owned) dev += b->cap;  // adopted residuals are the caller's allocation
    if (device_bytes) *device_bytes = (int64_t)dev;
    if (host_bytes) *host_bytes = ix->host.rows ? (int64_t)ix->host.rows->bytes : 0;
    return PB_OK;
}

extern "C" pb_status pb_index_shard_layout(const pb_index *ix, int32_t *out_world, int64_t *out_bounds, int32_t *out_devices) {
    if (!ix || !out_world) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix->group) return ix->group->shard_layout(out_world, out_bounds, out_devices);
    auto rd = ix->read_lock();
    *out_world = 1;
    if (out_bounds) out_bounds[0] = ix->doc_id_base, out_bounds[1] = ix->doc_id_base + ix->D;
    if (out_devices) out_devices[0] = ix->device;
    return PB_OK;
}

extern "C" void pb_search_params_default(pb_search_params *p) {  // search.rs:58-69
    if (!p) return;
    p->batch_size = 2000;
    p->n_full_scores = 4096;
    p->top_k = 10;
    p->n_ivf_probe = 8;
    p->centroid_batch_size = 100000;
    p->has_centroid_score_threshold = 1;
    p->centroid_score_threshold = 0.4f;
}

extern "C" void pb_set_fast_approx(pb_index *ix, int32_t enabled) {
    if (!ix) return;
    if (ix->group) return ix->group->each([&](pb_index *m) { pb_set_fast_approx(m, enabled); });
    ix->fast_approx = enabled != 0;  // 0 = single exact pass over every candidate, otherwise two-pass
}
extern "C" void pb_set_scores_tc(pb_index *ix, int32_t enabled) {
    if (ix && ix->group) return ix->group->each([&](pb_index *m) { pb_set_scores_tc(m, enabled); });
    if (ix) ix->k1_tc = enabled != 0;  // effective when the tensor-core operands were built at open (k1_tc_usable)
}
extern "C" void pb_set_lanes(pb_index *ix, int32_t lanes) {
    if (ix && ix->group) return ix->group->each([&](pb_index *m) { pb_set_lanes(m, lanes); });
    if (ix) ix->lanes = std::min(8, std::max(1, (int)lanes));
}
extern "C" pb_status pb_index_set_coalescing(pb_index *ix, const pb_coalesce_config *cfg) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    pbq::Config c;  // off
    if (cfg) {
        if (cfg->max_queries < 1 || cfg->max_wait_us < 0 || cfg->max_inflight < 1)
            return pb_fail(PB_ERR_INVALID, "coalescing: max_queries and max_inflight must be >= 1, max_wait_us >= 0");
        if (cfg->max_queries > 1 && ix->comm.joined())
            return pb_fail(PB_ERR_UNSUPPORTED, "coalescing on a doc-sharded handle: a collective needs the same order on every rank");
        c.max_queries = cfg->max_queries;
        c.max_wait_us = std::min(cfg->max_wait_us, 10000);
        c.max_inflight = cfg->max_inflight;
    }
    auto set = [&](int R) {
        ix->coalesce_cfg = c;
        pb_index_apply_coalescing(ix, R);
    };
    if (Replicas *rs = pb_replicas_of(ix)) pb_rep_sized(rs, set);  // a resize rescales it
    else set(1);
    return PB_OK;
}
// a replica set runs max_inflight merged batches per replica
void pb_index_apply_coalescing(pb_index *ix, int R) {
    pbq::Config c = ix->coalesce_cfg;
    c.max_inflight *= R;
    ix->coalescer.configure(c);
    ix->coalesce_on = c.max_queries > 1;
}
extern "C" pb_status pb_index_coalesce_stats(pb_index *ix, pb_coalesce_stats *out, int32_t reset) {
    if (!ix || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    const pbq::Counters c = ix->coalescer.counters(reset != 0);
    out->n_requests = c.n_requests, out->n_batches = c.n_batches, out->n_bypassed = c.n_bypassed;
    out->n_refused = c.n_refused, out->n_rerun_alone = c.n_rerun_alone, out->max_batch = c.max_batch;
    for (int i = 0; i < 8; ++i) out->batch_hist[i] = c.batch_hist[i];
    out->queue_wait_us = c.queue_wait_us;
    return PB_OK;
}
extern "C" void pb_set_fast_exact(pb_index *ix, int32_t enabled) {
    if (ix && ix->group) return ix->group->each([&](pb_index *m) { pb_set_fast_exact(m, enabled); });
    if (ix) ix->fast_exact = enabled != 0;
}
extern "C" void pb_set_profiling(pb_index *ix, int32_t enabled) {
    if (ix && ix->group) return ix->group->each([&](pb_index *m) { pb_set_profiling(m, enabled); });
    if (ix) ix->profiling = enabled != 0;
}
extern "C" pb_status pb_last_stage_stats(pb_index *, float *out_ms, int32_t *out_launches) {
    for (int i = 0; i < PB_STAGE_COUNT; ++i) {
        if (out_ms) out_ms[i] = g_stats.ms[i];
        if (out_launches) out_launches[i] = g_stats.launches[i];
    }
    return PB_OK;
}
extern "C" pb_status pb_last_call_ms(pb_index *, float *out_ms) {
    if (!out_ms) return pb_fail(PB_ERR_INVALID, "null argument");
    *out_ms = g_stats.call_ms;
    return PB_OK;
}
extern "C" pb_status pb_last_kernel_ms(pb_index *, float *out_ms) {
    if (!out_ms) return pb_fail(PB_ERR_INVALID, "null argument");
    for (int i = 0; i < PB_KERNEL_COUNT; ++i) out_ms[i] = g_stats.kernel_ms[i];
    return PB_OK;
}
extern "C" pb_status pb_last_work_counters(pb_index *, pb_work_counters *out) {
    if (!out) return pb_fail(PB_ERR_INVALID, "null argument");
    *out = g_stats.work;
    return PB_OK;
}
extern "C" pb_status pb_last_staging_stats(pb_index *, int64_t *docs, int64_t *bytes, float *ms) {
    if (docs) *docs = g_stats.staged_docs;
    if (bytes) *bytes = g_stats.staged_bytes;
    if (ms) *ms = g_stats.staging_ms;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// kernel launch helpers shared by the search pipeline and the stage entry points
// ------------------------------------------------------------------------------------------
// a2 on the tensor cores (k_scores_tc.cuh).  err = certified bound of |exact - estimate| in 16-bit code units
// (derivation at the top of that file); E = ceil(err) is the largest difference between an estimate-built code and
// the exact-table code, 2E + 1 the code margin of its consumers.
static float k1_err_codes(int dim) {
    const float chain = (float)dim * 5.9604645e-8f;                 // dim * 2^-24: the pinned fp32 FMA chain
    const float tc = (3.0f * (float)(dim / 16) + 3.0f) * 2.3841858e-7f;  // 2^-22 per MMA accumulation + the dropped split terms
    const float sub = 2.0f * 2.9802322e-8f * sqrtf((float)dim);     // fp16 subnormal spacing of the lo parts
    return (chain + tc + sub) * 32768.0f * 1.0001f;
}
static bool k1_tc_usable(const pb_index *ix) {
    return ix->k1_tc && ix->cent_h16t.p && TcDims::has(ix->dim) && k1_err_codes(ix->dim) < 1.0f;
}

// the 16-bit score table from the split-fp16 wgmma GEMM (k_scores16_tc) into `table`; `flags` gets the per-query
// out-of-range bits the exact kernel would set in qflag; slab_max (or null) the table's 16-row slab maxima
// (8 ceil(K / 128) slabs of k1_slab_rows(B, QS) codes)
static int k1_slab_rows(int B, int QS) { return (int)(((long long)B * QS + 127) / 128) * 128; }
static pb_status launch_k1_table(pb_index *ix, Workspace &ws, int B, int QS, unsigned short *table, int *flags,
                                 unsigned short *slab_max) {
    const int n_groups = (int)(((long long)B * QS + 127) / 128);
    const size_t qelems = (size_t)n_groups * 128 * ix->dim;
    CKS(ws.Qh16t.ensure(qelems * 2));
    CKS(ws.Ql16t.ensure(qelems * 2));
    CKS(ws.qrange_tc.ensure((size_t)B * 8 + 16));
    k_query_split_tiles<<<ix->sm_count, 256, 0, ws.stream>>>(ws.Q.as<float>(), ws.qoff.as<int>(), ws.qexp.as<int>(), B, QS,
                                                             ix->dim, ws.Qh16t.as<__half>(), ws.Ql16t.as<__half>());
    k_query_range_tc<<<(B + 127) / 128, 128, 0, ws.stream>>>(ws.qrange.as<float2>(), ws.qexp.as<int>(), ix->cent_exp, B,
                                                            ws.qrange_tc.as<float2>());
    const int tiles = (int)((ix->K + 127) / 128);
    const size_t sm = (size_t)6 * 128 * ix->dim * 2 + 128;
    return TcDims::dispatch(ix->dim, [&](auto dim_c) -> pb_status {
        auto kern = k_scores16_tc<decltype(dim_c)::value>;
        CKS(set_smem(kern, sm));
        KEV_BEGIN(PB_KERNEL_SCORES);
        kern<<<tiles, 384, sm, ws.stream>>>(ix->cent_h16t.as<__half>(), ix->cent_l16t.as<__half>(), ix->K,
                                            ws.Qh16t.as<__half>(), ws.Ql16t.as<__half>(), n_groups, B, QS,
                                            ws.qoff.as<int>(), ws.qrange_tc.as<float2>(), table, flags, slab_max);
        KEV_END(PB_KERNEL_SCORES);
        CK(cudaGetLastError());
        return PB_OK;
    });
}

// diagnostic twin of the score table on the tensor cores, compared code by code with the exact one
static pb_status launch_k1_diag(pb_index *ix, Workspace &ws, int B, int QS) {
    if (!ix->cent_h16t.p || !TcDims::has(ix->dim)) return PB_OK;
    CKS(ws.ST16b.ensure((size_t)B * ix->K * QS * 2));
    CKS(ws.k1diag.ensure((size_t)(B + 4) * 4));
    CK(cudaMemsetAsync(ws.k1diag.p, 0, (size_t)(B + 4) * 4, ws.stream));
    CKS(launch_k1_table(ix, ws, B, QS, ws.ST16b.as<unsigned short>(), ws.k1diag.as<int>() + 4, nullptr));
    k_diff16<<<dim3(ix->sm_count, B), 256, 0, ws.stream>>>(ws.ST16.as<unsigned short>(), ws.ST16b.as<unsigned short>(),
                                                          ws.qoff.as<int>(), ix->K, QS, ws.k1diag.as<int>());
    CK(cudaGetLastError());
    return PB_OK;
}

// chunk size of the threshold-first probe: 1024 centroids, fewer for small K so that at least 2n chunks exist (tau is
// the n-th largest chunk maximum); *n_chunks < n means the path cannot run
static int probe_chunk_rows(long long K, int n, int *n_chunks) {
    int rows = 1024;
    while (rows > 32 && (K + rows - 1) / rows < 2ll * n) rows >>= 1;
    *n_chunks = (int)((K + rows - 1) / rows);
    return rows;
}

// entries per query token of the threshold-first probe's candidate list
static int probe16_cap(int n) { return n * std::max(2, 128 / n); }

// The threshold-first probe up to its collect kernel: the candidate lists cleared, every chunk's largest code
// (k_chunkmax16 from the table, or k_chunkmax_slabs from the slab maxima the tensor-core table's epilogue kept) and
// each query token's threshold, the n-th largest of them (k_tau16).  *d_fallback is the device flag k_tau16 and the
// kernels after it raise when a query cannot take this path.
static pb_status probe16_thresholds(pb_index *ix, Workspace &ws, int B, int QS, int n, int n_chunks, int chunk_rows,
                                    const int *qn, const unsigned short *slab_max, int **d_fallback) {
    const int cap = probe16_cap(n);
    CKS(ws.cmax16.ensure((size_t)B * n_chunks * QS * 2));
    CKS(ws.tau16.ensure((size_t)B * QS * 4));
    CKS(ws.plist.ensure((size_t)B * QS * cap * 8));
    CKS(ws.pcount.ensure((size_t)B * QS * 4 + 16));
    CK(cudaMemsetAsync(ws.plist.p, 0, (size_t)B * QS * cap * 8, ws.stream));
    CK(cudaMemsetAsync(ws.pcount.p, 0, (size_t)B * QS * 4 + 16, ws.stream));
    int *fb = ws.pcount.as<int>() + (size_t)B * QS;
    if (slab_max)
        k_chunkmax_slabs<<<dim3(n_chunks, (B * QS + 511) / 512), 256, 0, ws.stream>>>(
            slab_max, ix->K, B, QS, k1_slab_rows(B, QS) / 128, n_chunks, chunk_rows, ws.cmax16.as<unsigned short>());
    else
        k_chunkmax16<<<dim3((n_chunks + 3) / 4, B), 128, 0, ws.stream>>>(ws.ST16.as<unsigned short>(), ix->K, QS,
                                                                         n_chunks, chunk_rows, ws.cmax16.as<unsigned short>());
    k_tau16<<<dim3(QS, B), 32, 0, ws.stream>>>(ws.cmax16.as<unsigned short>(), ws.qoff.as<int>(), QS, n, n_chunks,
                                              ws.qflag.as<int>(), ws.tau16.as<uint32_t>(), fb, qn);
    *d_fallback = fb;
    return PB_OK;
}

// the smallest power of two >= x: the shared-memory sort and set sizes of the per-query kernels
static int pow2_at_least(int x) {
    int P = 1;
    while (P < x) P <<= 1;
    return P;
}

// live rows the pruned first approximate pass aims at per query token (k_a5_floor), and the words per query of its
// live-row bitmap (16-byte rows, so that k_a5_bound can bulk-copy one)
static long long a5_live_rows(const pb_index *ix) { return ix->a5_live >= 0 ? ix->a5_live : ix->K / 512; }
static long long a5_live_stride(long long K) { return ((K + 31) / 32 + 3) & ~3ll; }

// a2 + a3 on the tensor-core table.  Nothing is read back here: a flagged query or a probe-list overflow raises
// *d_fallback on the device, the kernels after it stay memory-safe, and the caller redoes the sub-batch on the
// exact path once it sees the flag at the end.
// n: the pass's largest n_ivf_probe; qn / qhas / qthr: each query's own n and threshold, or null (uniform pass).
// live: the pass prunes its first approximate pass; the floors of a5 (k_a5_floor, on a sample of the table) are taken
// before the collect kernel, which then also writes the live-row bitmap from its one stream of the table (ws.a5floor,
// ws.a5live, read by approx_scores).  On a pass that raises *d_fallback the bitmap may be stale or partly written;
// approx_scores still runs on it (memory-safe: the bits only select among a doc's own code rows) and the redo on the
// exact path replaces everything that pass produced.
static pb_status run_k1_tc(pb_index *ix, Workspace &ws, int B, int QS, int nq_max, int n, const int *qn, int has_thr,
                           float thr, const int *qhas, const float *qthr, bool batched, long long slab, bool live,
                           int *L, int *cells_cap_out, const int **d_fallback_out) {
    int n_chunks = 0;
    const int chunk_rows = probe_chunk_rows(ix->K, n, &n_chunks);
    const int cm = 2 * ix->k1_margin + 1;
    CKS(ws.Qi.ensure((size_t)B * QS * ix->dim * 4));
    k_interleave_query_rows<<<dim3(8, B), 256, 0, ws.stream>>>(ws.Q.as<float>(), ws.qoff.as<int>(), QS, ix->dim, ws.Qi.as<float>());
    const int tiles = (int)((ix->K + 127) / 128);
    CKS(ws.smax.ensure((size_t)tiles * 8 * k1_slab_rows(B, QS) * 2));
    CKS(launch_k1_table(ix, ws, B, QS, ws.ST16.as<unsigned short>(), ws.qflag.as<int>(), ws.smax.as<unsigned short>()));
    L[PB_STAGE_CENTROID_SCORES] += 4;
    const int cap = probe16_cap(n);
    const int cells_cap = (int)std::min<long long>((long long)QS * n, ix->K);
    CKS(ws.sel.ensure((size_t)B * QS * n * 8));
    CKS(ws.cells.ensure((size_t)B * cells_cap * 4));
    CKS(ws.ncells.ensure((size_t)B * 4 + 16));
    CKS(ws.ulist.ensure((size_t)B * cells_cap * 4));
    CKS(ws.nulist.ensure((size_t)B * 4 + 16));
    CKS(ws.k1rows.ensure((size_t)B * cells_cap * QS * 4));
    int *d_fallback = nullptr;
    CKS(probe16_thresholds(ix, ws, B, QS, n, n_chunks, chunk_rows, qn, ws.smax.as<unsigned short>(), &d_fallback));
    const long long live_stride = a5_live_stride(ix->K);
    if (live) {
        CKS(ws.a5floor.ensure((size_t)B * QS * 4));
        CKS(ws.a5live.ensure((size_t)B * live_stride * 4));
        k_a5_floor<<<dim3(QS / 8, B), 256, 0, ws.stream>>>(ws.ST16.as<unsigned short>(), ws.qoff.as<int>(), ix->K, QS,
                                                           a5_live_rows(ix), ws.a5floor.as<uint32_t>());
        L[PB_STAGE_PROBE] += 1;
    }
    (live ? k_collect16_tc<true> : k_collect16_tc<false>)<<<dim3((n_chunks + 3) / 4, B), 128, 0, ws.stream>>>(
        ws.ST16.as<unsigned short>(), ws.Q.as<float>(), ws.qoff.as<int>(), ix->centroids.as<float>(), ix->dim, cm, ix->K, QS,
        n_chunks, chunk_rows, ws.tau16.as<uint32_t>(), cap, ws.pcount.as<int>(), ws.plist.as<u64>(), d_fallback,
        live ? ws.a5floor.as<uint32_t>() : nullptr, live ? ws.a5live.as<uint32_t>() : nullptr, live_stride);
    // PB_TABLE_DIAG: the standalone kernels on the same table, compared word by word with the chunk maxima from the
    // slab maxima and with the collect kernel's live bits
    if (ix->table_diag) {
        CKS(ws.tdcmax.ensure((size_t)B * n_chunks * QS * 2));
        CKS(ws.tdiag.ensure(16));
        CK(cudaMemsetAsync(ws.tdiag.p, 0, 16, ws.stream));
        k_chunkmax16<<<dim3((n_chunks + 3) / 4, B), 128, 0, ws.stream>>>(ws.ST16.as<unsigned short>(), ix->K, QS, n_chunks,
                                                                         chunk_rows, ws.tdcmax.as<unsigned short>());
        k_words_diff<<<dim3(4, B), 256, 0, ws.stream>>>(ws.cmax16.as<uint32_t>(), ws.tdcmax.as<uint32_t>(),
                                                        (long long)n_chunks * QS / 2, (long long)n_chunks * QS / 2,
                                                        d_fallback, ws.tdiag.as<unsigned long long>());
        L[PB_STAGE_PROBE] += 2;
        if (live) {
            CKS(ws.tdlive.ensure((size_t)B * live_stride * 4));
            k_a5_live<<<dim3(ix->sm_count * 2, B), 256, 0, ws.stream>>>(ws.ST16.as<unsigned short>(), ix->K, QS,
                                                                         ws.a5floor.as<uint32_t>(), ws.tdlive.as<uint32_t>(),
                                                                         live_stride);
            k_words_diff<<<dim3(4, B), 256, 0, ws.stream>>>(ws.a5live.as<uint32_t>(), ws.tdlive.as<uint32_t>(),
                                                            (ix->K + 31) / 32, live_stride, d_fallback,
                                                            ws.tdiag.as<unsigned long long>());
            L[PB_STAGE_PROBE] += 2;
        }
    }
    k_topn_merge<<<dim3(QS, B), 32, 0, ws.stream>>>(ws.plist.as<u64>(), ws.qoff.as<int>(), QS, n, cap / n, ws.sel.as<u64>(),
                                                  nullptr, 0, qn);
    // the selected centroids, their exact rows, the variant's threshold rule
    const int P = pow2_at_least(std::max(nq_max * n, 1));
    CKS(set_smem(k_cells_unique, (size_t)P * 8));
    k_cells_unique<<<B, 256, (size_t)P * 8, ws.stream>>>(ws.sel.as<u64>(), ws.qoff.as<int>(), QS, n, cells_cap,
                                                         ws.ulist.as<uint32_t>(), ws.nulist.as<int>());
    const size_t smr = (size_t)(PB_TOK_TILE * (ix->dim + 4) + PB_Q_TILE * ix->dim) * sizeof(float);
    PB_DIM_SWITCH(ix->dim, {
        auto kern = k_exact_rows<DIM>;
        CKS(set_smem(kern, smr));
        kern<<<dim3((cells_cap + PB_TOK_TILE - 1) / PB_TOK_TILE, B), 128, smr, ws.stream>>>(
            ws.Qi.as<float>(), ws.qoff.as<int>(), QS, ix->centroids.as<float>(), ws.ulist.as<uint32_t>(), ws.nulist.as<int>(),
            cells_cap, ws.k1rows.as<float>());
    });
    CKS(ws.cellflags.ensure((size_t)B * cells_cap * 4));
    k_cells_thr<<<dim3(8, B), 256, 0, ws.stream>>>(
        ws.sel.as<u64>(), ws.k1rows.as<float>(), ws.ulist.as<uint32_t>(), ws.nulist.as<int>(), ws.qoff.as<int>(), ix->K, QS, n,
        cells_cap, has_thr, thr, batched ? 1 : 0, slab, ws.cellflags.as<int>(), ws.ST16.as<unsigned short>(),
        ws.qrange.as<float2>(), cm, ws.Q.as<float>(), ix->centroids.as<float>(), ix->dim, ws.cmax16.as<unsigned short>(),
        n_chunks, chunk_rows, qn, qhas, qthr);
    k_cells_emit<<<B, 256, 0, ws.stream>>>(ws.ulist.as<uint32_t>(), ws.nulist.as<int>(), ws.cellflags.as<int>(), cells_cap,
                                           ws.cells.as<uint32_t>(), ws.ncells.as<int>());
    CK(cudaGetLastError());
    L[PB_STAGE_PROBE] += 8;
    *cells_cap_out = cells_cap;
    *d_fallback_out = d_fallback;
    return PB_OK;
}

// a2 on the fp32 FMA path: the exact table, with16 also its 16-bit codes
static pb_status launch_centroid_scores(pb_index *ix, Workspace &ws, int B, int QS, int *launches, bool with16 = false) {
    const int tiles = (int)((ix->K + PB_TOK_TILE - 1) / PB_TOK_TILE);
    // enough CTAs to fill the machine twice over; each CTA keeps its centroid tile in smem and walks queries
    int groups = std::max(1, std::min(B, (4 * ix->sm_count + tiles - 1) / tiles));
    // paired fp32 FMA tile: query rows interleaved pairwise, one 8-byte load feeds two dots
    CKS(ws.Qi.ensure((size_t)B * QS * ix->dim * 4));
    k_interleave_query_rows<<<dim3(8, B), 256, 0, ws.stream>>>(ws.Q.as<float>(), ws.qoff.as<int>(), QS, ix->dim,
                                                               ws.Qi.as<float>());
    PB_DIM_SWITCH(ix->dim, {
        auto kern = k_centroid_scores<DIM, true>;
        CKS(set_smem(kern, smem_scores(DIM)));
        KEV_BEGIN(PB_KERNEL_SCORES);
        kern<<<dim3(tiles, groups), 128, smem_scores(DIM), ws.stream>>>(ws.Qi.as<float>(), ws.qoff.as<int>(), B, QS,
                                                                        ix->centroids.as<float>(), ix->K,
                                                                        ws.ST.as<float>(),
                                                                        with16 ? ws.ST16.as<unsigned short>() : nullptr,
                                                                        ws.qrange.as<float2>(), ws.qflag.as<int>());
        KEV_END(PB_KERNEL_SCORES);
    });
    CK(cudaGetLastError());
    if (launches) *launches += 2;
    return PB_OK;
}

struct KeptView {  // the docs the exact stage scores: the cut's output, or the filter's survivors
    uint32_t *kept;
    int *nkept;
    long long *tokp;
    uint32_t *krank;  // global approximate rank (sharded) or nullptr
};

// The token arrays the exact stage reads: the handle's own, or (host tier) a staged copy whose doc_off is indexed by the
// slots the kept lists then hold (k_stage.cuh)
struct TokView {
    const uint32_t *codes;
    const uint8_t *residuals;
    const float *inv_norm;
    const long long *doc_off;
};
static TokView resident_tokens(const pb_index *ix) {
    return {ix->codes.as<uint32_t>(), ix->residuals.as<uint8_t>(), ix->tok_inv_norm.as<float>(), ix->doc_off.as<long long>()};
}

static pb_status launch_exact(pb_index *ix, Workspace &ws, const KeptView &kv, const TokView &tv, int B, int QS, int Mcap,
                              int kept_shared, long long max_tokens, int *launches, const int *only_flagged = nullptr,
                              bool timed = true) {
    // each CTA owns a contiguous range of chunks; aim for 8 waves of 2 CTAs/SM over the whole grid
    long long chunks = (max_tokens + PB_TOK_TILE - 1) / PB_TOK_TILE;
    long long want = std::max<long long>(1, ((long long)ix->sm_count * 16 + B - 1) / B);
    int gx = (int)std::max<long long>(1, std::min<long long>(chunks, want));
    PB_DIM_SWITCH(ix->dim, {
        auto kern = k_exact<DIM, false>;
        CKS(set_smem(kern, smem_exact(DIM, ix->packed)));
        if (timed) KEV_BEGIN(PB_KERNEL_EXACT);
        kern<<<dim3(gx, B), 128, smem_exact(DIM, ix->packed), ws.stream>>>(
            ws.Q.as<float>(), ws.qoff.as<int>(), QS, ix->centroids.as<float>(), ix->w_rev.as<float>(), ix->nbits,
            tv.codes, tv.residuals, tv.doc_off, nullptr,
            kv.kept, kv.nkept, kv.tokp, Mcap, kept_shared, ws.maxkey.as<uint32_t>(), only_flagged);
        if (timed) KEV_END(PB_KERNEL_EXACT);
    });
    CK(cudaGetLastError());
    if (launches) ++*launches;
    return PB_OK;
}

// error of one tensor-core similarity estimate relative to |q| (derivation at the top of k_filter_tc.cuh and in DESIGN.md 4c);
// E = code error of the score table (0 = exact table); 0 = filter unusable
static float filter_eps_unit2(const pb_index *ix, int E) {
    const float u = 1.0f / 2048.0f;
    const float vmin = ix->vmin * 0.9999f, wmax = ix->wmax * 1.0001f;
    if (!(vmin > 0.0f) || !(ix->cmax < 3.0e4f) || !(wmax < 3.0e4f)) return 0.0f;
    const float ds = ((float)E + 1.01f) * 2.0f * ix->cmax * 1.0001f / 65535.0f;
    const float dw = wmax * (2.0f * u + u * u + 3.0517578e-5f);
    // k_maxsim_tc decodes a code with one FFMA whose folded constant (|.| <= 257 R, R = |q| cmax) is rounded once:
    // <= 257 R 2^-24 = 0.503 code units
    const float dfold = 0.53f * 2.0f * ix->cmax * 1.0001f / 65535.0f;
    const float eps = (ds + dw + dfold) / vmin + 8e-6f;
    return eps < 0.05f ? eps : 0.0f;
}

static size_t smem_maxsim_tc(int dim, int packed, int nqt) {
    const int nbits = packed * 8 / dim;
    return (size_t)2 * PB_XTC_STAGE(dim) + (size_t)nqt * dim * 2 + (size_t)256 * (8 / nbits) * 2 * (nbits == 4 ? 4 : 1) +
           4 * 128 * sizeof(MsMeta) + 8 * 8 + (size_t)128 * ACC_LD(nqt) * 4;
}

// the warp-specialised linear estimate over the docs of `in`: pass 1 (pairs == nullptr) leaves per (doc, q) maxima in
// `keys`; pass 2 lists the (token, q) pairs within the certified band of the maxima `keys` holds at src_rank
static pb_status launch_maxsim_tc(pb_index *ix, Workspace &ws, const KeptView &in, const TokView &tv, int B, int QS, int Mcap,
                                  long long max_tokens, int nq_max, uint32_t *keys, const uint32_t *src_rank, float band_unit,
                                  u64 *pairs, int *n_pairs, int pair_cap, int kev) {
    const bool emit = pairs != nullptr;
    // CTAs per SM over the batch: ws_grid for pass 1 (all kept docs), ws_grid2 for pass 2 (the survivors, ~1/10 of the
    // tokens; fewer, longer CTAs measured slower: the pass is latency-bound and wants the parallelism)
    long long chunks = (max_tokens + 127) / 128;
    long long want = std::max<long long>(1, ((long long)ix->sm_count * (emit ? ix->ws_grid2 : ix->ws_grid) + B - 1) / B);
    int gx = (int)std::max<long long>(1, std::min<long long>(chunks, want));
    const int nqt = nq_max <= 32 ? 32 : 64;
    const size_t sm = smem_maxsim_tc(ix->dim, ix->packed, nqt);
    CKS(ws.gbase.ensure((size_t)B * Mcap * 8));
    k_doc_gbase<<<dim3((Mcap + 255) / 256, B), 256, 0, ws.stream>>>(in.kept, in.nkept, in.tokp, tv.doc_off, Mcap,
                                                                    ws.gbase.as<long long>());
    CK(cudaGetLastError());
#define PB_MS_GO(DV, NB, NQ, EM)                                                                                       \
    {                                                                                                                  \
        auto kern = k_maxsim_tc<DV, NB, NQ, EM>;                                                                       \
        CKS(set_smem(kern, sm));                                                                                       \
        if (kev >= 0) KEV_BEGIN(kev);                                                                                  \
        kern<<<dim3(gx, B), 256, sm, ws.stream>>>(ws.Q.as<float>(), ws.qoff.as<int>(), QS, ws.qexp.as<int>(),            \
                                                  ws.ST16.as<unsigned short>(), ix->K, ws.qrange.as<float2>(),         \
                                                  ws.qflag.as<int>(), ix->w_rev.as<float>(),                           \
                                                  tv.codes, tv.residuals,                                              \
                                                  tv.inv_norm, ws.gbase.as<long long>(),                               \
                                                  in.nkept, in.tokp, Mcap, keys, src_rank, ws.qnmax.as<float>(),       \
                                                  band_unit, pairs, n_pairs, pair_cap);                                \
        if (kev >= 0) KEV_END(kev);                                                                                    \
    }
#define PB_MS_LAUNCH(DV, NB)                                                                                           \
    if (emit) {                                                                                                        \
        if (nqt == 32) PB_MS_GO(DV, NB, 32, true) else PB_MS_GO(DV, NB, 64, true)                                      \
    } else {                                                                                                           \
        if (nqt == 32) PB_MS_GO(DV, NB, 32, false) else PB_MS_GO(DV, NB, 64, false)                                    \
    }
    return TcDims::dispatch(ix->dim, [&](auto dim_c) -> pb_status {
        constexpr int DV = decltype(dim_c)::value;
        switch (ix->nbits) {
            case 1:
                // 1-bit rows of DV / 8 bytes: whole 32-bit words unless DV % 32 != 0 (filter_runs keeps those off)
                if constexpr (DV % 32 == 0) {
                    PB_MS_LAUNCH(DV, 1)
                    break;
                } else {
                    return pb_fail(PB_ERR_UNSUPPORTED, "filter: %d-byte 1-bit rows are not whole 32-bit words", DV / 8);
                }
            case 2: PB_MS_LAUNCH(DV, 2) break;
            case 4: PB_MS_LAUNCH(DV, 4) break;
            default: PB_MS_LAUNCH(DV, 8) break;
        }
        CK(cudaGetLastError());
        return PB_OK;
    });
#undef PB_MS_LAUNCH
#undef PB_MS_GO
}

// a7': tensor-core estimate of every kept doc, then the survivors that can still reach the top_k
static pb_status launch_filter(pb_index *ix, Workspace &ws, const KeptView &in, const KeptView &out, const TokView &tv, int B,
                               int QS, int Mcap, int top_k, const int *qtopk, long long max_tokens, float eps_unit,
                               int nq_max, bool keep_keys, int *launches) {
    // keep_keys: the per (doc, q) maxima go to their own buffer and stay there for the pair pass of the exact stage
    uint32_t *keys = keep_keys ? ws.estkey.as<uint32_t>() : ws.maxkey.as<uint32_t>();
    if (keep_keys) CK(cudaMemsetAsync(keys, 0, (size_t)B * Mcap * QS * 4, ws.stream));
    CKS(launch_maxsim_tc(ix, ws, in, tv, B, QS, Mcap, max_tokens, nq_max, keys, nullptr, 0.0f, nullptr, nullptr, 0,
                         PB_KERNEL_FILTER));
    k_tc_finalize<<<dim3((Mcap + 7) / 8, B), 256, 0, ws.stream>>>(keys, ws.qoff.as<int>(), QS, in.nkept, Mcap, in.tokp,
                                                                  ws.est.as<float>(), keep_keys ? 0 : 1);
    CK(cudaGetLastError());
    const int Pm = pow2_at_least(Mcap);
    CKS(set_smem(k_tc_select, (size_t)Pm * 8));
    k_tc_select<<<B, 1024, (size_t)Pm * 8, ws.stream>>>(ws.est.as<float>(), in.kept, in.krank, in.nkept, Mcap, top_k,
                                                        ws.qoff.as<int>(), ws.qnmax.as<float>(), eps_unit,
                                                        tv.doc_off, out.kept, out.krank, out.nkept,
                                                        out.tokp, ws.ktok2.as<long long>(),
                                                        keep_keys ? ws.srcrank.as<uint32_t>() : nullptr, qtopk);
    CK(cudaGetLastError());
    if (launches) *launches += 3 + (keep_keys ? 1 : 0);
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// the search pipeline
// ------------------------------------------------------------------------------------------
struct Fnv64 {  // FNV-1a over the call's arguments
    u64 h = 14695981039346656037ull;
    void add(const void *p, size_t n) {
        for (size_t i = 0; i < n; ++i) h = (h ^ static_cast<const uint8_t *>(p)[i]) * 1099511628211ull;
    }
    template <class T> void put(T v) { add(&v, sizeof v); }
};

struct SearchIO {
    const float *queries;  // host or device
    bool queries_on_device;
    const int64_t *q_off;  // host
    int64_t n_queries;
    // Subsets (host).  Per query: query b's ids are sub_ids[sub_off[b] .. sub_off[b + 1]) when has_sub[b] != 0 (has_sub
    // null: every query has one; sub_off null: none has).  shared_sub: every query has sub_ids[0 .. n_shared).
    const int64_t *sub_ids;
    const int64_t *sub_off;
    const uint8_t *has_sub;
    int64_t n_shared;
    bool shared_sub;
    int64_t *out_ids;  // host or device
    float *out_scores;
    int32_t *out_counts;
    bool out_on_device;
    pb_trace *trace;
    // search parameters: query b's are qp[b * qp_stride] (stride 0: one struct for the call); rows of out_ids /
    // out_scores are out_stride entries apart (the call's largest top_k)
    const pb_search_params *qp;
    int64_t qp_stride;
    int64_t out_stride;
};

static const pb_search_params &query_params(const SearchIO &io, int64_t b) { return io.qp[b * io.qp_stride]; }

// Queries [b0, b1) of a call, as lanes and replica slices search them: the offsets stay absolute into the call's
// queries and subset ids, and the output rows stay io.out_stride apart (a search writes each row's own top_k entries)
static SearchIO slice_io(const SearchIO &io, int64_t b0, int64_t b1) {
    SearchIO s = io;
    s.n_queries = b1 - b0;
    if (io.q_off) s.q_off = io.q_off + b0;
    if (io.sub_off) s.sub_off = io.sub_off + b0;
    if (io.has_sub) s.has_sub = io.has_sub + b0;
    if (io.qp) s.qp = io.qp + b0 * io.qp_stride;
    if (io.out_ids) s.out_ids = io.out_ids + b0 * io.out_stride;
    if (io.out_scores) s.out_scores = io.out_scores + b0 * io.out_stride;
    if (io.out_counts) s.out_counts = io.out_counts + b0;
    return s;
}

// query b's id list [*s, *e) of io.sub_ids, or false when it has no subset
static bool query_subset(const SearchIO &io, int64_t b, int64_t *s, int64_t *e) {
    if (io.shared_sub) {
        *s = 0;
        *e = io.n_shared;
        return true;
    }
    if (!io.sub_off || (io.has_sub && !io.has_sub[b])) return false;
    *s = io.sub_off[b];
    *e = io.sub_off[b + 1];
    return true;
}

// How a query's cells are selected (a3); a pass holds queries of one kind.  TABLE: no eligibility row, the streaming
// probe (the tensor-core table where it applies).  STREAM: the streaming probe over the query's eligible centroids.
// BIG: the row-wise radix select (effective n_ivf_probe beyond the streaming lists).  ALL: every eligible centroid.
// NONE: nothing eligible, an empty result without a pass.
enum ProbeKind : uint8_t { PROBE_TABLE, PROBE_STREAM, PROBE_BIG, PROBE_ALL, PROBE_NONE };

// what a search call decides once, before its first sub-batch
struct SearchPlan {
    int64_t Bt = 0;                           // queries
    int Mcap = 1, top_k_max = 0;              // the largest M and top_k of the call: buffer strides and budget
    bool sharded = false;
    bool empty = false;                       // every result list is empty
    bool prof = false;                        // stage and call times (pb_set_profiling)
    long long Wd = 0, Wk = 0;                 // 32-bit words of a doc / centroid bitmap
    long long Wke = 0;                        // words of an eligibility row (even: rows travel as 64-bit words)
    long long D_total = 0;                    // documents of the deployment (doc-sharded: over every rank)
    // each query's search parameters (DESIGN.md 4l): M = the docs the cut keeps (search.rs:468), M1 = the first round
    // of the pruned a5 pass, the threshold (has / value), the variant (batched: search.rs:337) and its slab width
    std::vector<int> qtopk, qM, qM1, qhas;
    std::vector<float> qthr;
    std::vector<uint8_t> qbatched;
    std::vector<long long> qslab;
    // subsets: one row per distinct id list; the doc bitmap rows, and (dense variant) the eligible-centroid rows
    int rows = 0;
    const uint32_t *d_subset_bits = nullptr;
    const uint32_t *d_elig = nullptr;
    std::vector<int> qrow;          // [Bt] the query's row, -1 = no subset
    std::vector<int> qn;            // [Bt] its effective n_ivf_probe (ALL: its eligible count)
    std::vector<uint8_t> kind;      // [Bt] ProbeKind
    std::vector<int64_t> order;     // the queries in pass order
    std::vector<std::pair<int64_t, int>> passes;  // (first position in `order`, queries)
};

// The checks a query must pass whatever batch it is in.  plan_search and plan_probe apply them to every query of a call
// and pb_search applies them to a request before it joins a merged batch (check_request), so a request refused alone is
// refused before it can fail its neighbours.
static pb_status check_query_args(const pb_search_params &p) {
    if (p.top_k < 0 || p.n_full_scores < 0) return pb_fail(PB_ERR_INVALID, "top_k / n_full_scores must be >= 0");
    if (p.n_ivf_probe < 1) return pb_fail(PB_ERR_INVALID, "n_ivf_probe must be >= 1");
    return PB_OK;
}
// M, the docs the cut keeps
static pb_status query_kept_docs(const pb_search_params &p, int *M) {
    const long long n_dec = std::max<long long>(p.n_full_scores / 4, p.top_k);  // search.rs:468
    const long long Mll = std::min<long long>(p.n_full_scores, n_dec);          // take(nfs).take(n_dec)
    if (Mll > 16384)
        return pb_fail(PB_ERR_UNSUPPORTED, "min(n_full_scores, max(n_full_scores/4, top_k)) = %lld exceeds 16384", Mll);
    *M = (int)Mll;
    return PB_OK;
}
static bool query_batched(const pb_index *ix, const pb_search_params &p) {
    return p.centroid_batch_size > 0 && ix->K > p.centroid_batch_size;  // search.rs:337
}
// effective n_ivf_probe beyond 64: the dense variant switches to a row-wise radix select; the batched variant's
// heap-order threshold rule is tied to the streaming formulation, whose per-lane lists hold up to 192 entries
static pb_status check_batched_probe(const pb_index *ix, const pb_search_params &p) {
    const long long n_probe = std::min<long long>(p.n_ivf_probe, ix->K);
    if (n_probe > 192)
        return pb_fail(PB_ERR_UNSUPPORTED, "n_ivf_probe %d > 192 with the batched variant is not built", (int)n_probe);
    return PB_OK;
}
// the limits of a query of n_tokens tokens whose probe is of `kind` with effective width n
static pb_status check_query_rows(const pb_index *ix, uint8_t kind, int n, int n_tokens) {
    const int QS = query_row_tokens(n_tokens);
    if ((kind == PROBE_TABLE || kind == PROBE_STREAM) && (long long)QS * n > 8192)
        return pb_fail(PB_ERR_UNSUPPORTED, "query tokens x n_ivf_probe = %lld exceeds 8192", (long long)QS * n);
    const size_t per_q = (size_t)ix->K * QS * sizeof(float);
    if (per_q >= ((size_t)1 << 32))
        return pb_fail(PB_ERR_UNSUPPORTED, "num_centroids x query tokens x 4 = %zu bytes per query exceeds 2^32", per_q);
    return PB_OK;
}

// The arguments and what follows from them alone.  Nothing is enqueued here, so a call refused here takes no workspace.
static pb_status plan_search(pb_index *ix, const SearchIO &io, SearchPlan &plan) {
    if (!ix || !io.qp) return pb_fail(PB_ERR_INVALID, "null argument");
    if (io.n_queries < 0) return pb_fail(PB_ERR_INVALID, "n_queries < 0");
    if (io.n_queries > 0 && (!io.queries || !io.q_off)) return pb_fail(PB_ERR_INVALID, "null queries");
    // every query's parameters as pb_search_batch checks its one struct (one struct: also for an empty batch)
    const int64_t n_par = io.qp_stride ? io.n_queries : 1;
    long long top_k_max = 0;
    for (int64_t b = 0; b < n_par; ++b) {
        const pb_search_params &p = query_params(io, b);
        CKS(check_query_args(p));
        top_k_max = std::max<long long>(top_k_max, p.top_k);
    }
    if (top_k_max > 0 && (!io.out_ids || !io.out_scores)) return pb_fail(PB_ERR_INVALID, "null outputs");
    if (!io.out_counts) return pb_fail(PB_ERR_INVALID, "null out_counts");
    CK(cudaSetDevice(ix->device));
    g_stats = Stats();
    plan.Bt = io.n_queries;
    if (plan.Bt == 0) return PB_OK;
    for (int64_t b = 0; b < plan.Bt; ++b)
        if (io.q_off[b + 1] < io.q_off[b]) return pb_fail(PB_ERR_INVALID, "q_tok_offsets not monotone");
    const size_t Bt = (size_t)plan.Bt;
    plan.qtopk.resize(Bt), plan.qM.resize(Bt), plan.qM1.resize(Bt), plan.qhas.resize(Bt), plan.qthr.resize(Bt);
    plan.qbatched.resize(Bt), plan.qslab.resize(Bt);
    bool all_empty = true;
    int M_max = 0;
    for (int64_t b = 0; b < plan.Bt; ++b) {
        const pb_search_params &p = query_params(io, b);
        int M = 0;
        CKS(query_kept_docs(p, &M));
        const bool batched = query_batched(ix, p);
        plan.qtopk[(size_t)b] = (int)p.top_k;
        plan.qM[(size_t)b] = M;
        plan.qM1[(size_t)b] = (int)std::min<double>(ceil((double)ix->a5_m1 * M), (double)INT_MAX);
        plan.qhas[(size_t)b] = p.has_centroid_score_threshold ? 1 : 0;
        plan.qthr[(size_t)b] = p.centroid_score_threshold;
        plan.qbatched[(size_t)b] = batched ? 1 : 0;
        plan.qslab[(size_t)b] = batched ? (long long)p.centroid_batch_size : ix->K;
        all_empty = all_empty && (M == 0 || p.top_k == 0);
        M_max = std::max(M_max, M);
    }
    plan.Mcap = std::max(M_max, 1);
    plan.top_k_max = (int)top_k_max;
    plan.sharded = ix->comm.world > 1;
    // a shard with no documents still takes part in the exchanges
    plan.empty = all_empty || (ix->D == 0 && !plan.sharded);
    plan.prof = ix->profiling;
    return PB_OK;
}

// a query whose parameters leave nothing to return (top_k == 0 or M == 0): count 0, no pass
static bool query_empty(const SearchPlan &plan, int64_t b) { return plan.qtopk[(size_t)b] == 0 || plan.qM[(size_t)b] == 0; }

// a sharded call's refusal that every rank reached from the same exchanged data: the group stays usable
static thread_local bool g_search_agreed = false;

// Doc-sharded: the plan-time exchange of one record per rank (status, D, raw sub-batch bound, fingerprint of the
// subset arguments).  Every rank takes the least bound (equal sub-batches, so the later exchanges agree in size) and
// the deployment's D for the n_ivf_probe scaling; differing subsets refuse the call on every rank.
enum { PX_STATUS, PX_D, PX_QB, PX_PRINT, PX_WORDS };
static pb_status plan_exchange(pb_index *ix, Workspace &ws, pb_status local, u64 print, int *QB, SearchPlan &plan) {
    const int G = ix->comm.world;
    long long mine[PX_WORDS] = {(long long)local, ix->D, *QB, (long long)print};
    std::vector<long long> all((size_t)G * PX_WORDS);
    CKS(ws.xrec.ensure(PX_WORDS * 8));
    CKS(ws.xall.ensure((size_t)G * PX_WORDS * 8));
    CK(cudaMemcpyAsync(ws.xrec.p, mine, PX_WORDS * 8, cudaMemcpyHostToDevice, ws.stream));
    CKS(ix->comm.allgather(ws.stream, ws.xrec.p, ws.xall.p, PX_WORDS));
    CK(cudaMemcpyAsync(all.data(), ws.xall.p, all.size() * 8, cudaMemcpyDeviceToHost, ws.stream));
    CK(cudaStreamSynchronize(ws.stream));
    g_search_agreed = true;  // from here on every rank decides from the same words
    for (int r = 0; r < G; ++r) {
        const pb_status s = (pb_status)all[(size_t)r * PX_WORDS + PX_STATUS];
        if (s == PB_OK) continue;
        if (r == ix->comm.rank) return s;  // g_err holds my own message
        return pb_fail(s, "rank %d of the group failed (status %d)", r, (int)s);
    }
    plan.D_total = 0;
    for (int r = 0; r < G; ++r) {
        const long long *w = all.data() + (size_t)r * PX_WORDS;
        if ((u64)w[PX_PRINT] != print)
            return pb_fail(PB_ERR_INVALID,
                           "the ranks were given different subsets or parameters (rank %d differs from rank %d)", r,
                           ix->comm.rank);
        plan.D_total += w[PX_D];
        *QB = (int)std::min<long long>(*QB, w[PX_QB]);
    }
    g_search_agreed = false;
    return PB_OK;
}

// The subsets, each query's probe kind and width, and the passes.  Subset rows: one doc bitmap per distinct id list,
// and with the dense variant its eligible centroids (search.rs:350-382), counted on the device and read back once.
static pb_status plan_probe(pb_index *ix, Workspace &ws, const SearchIO &io, SearchPlan &plan) {
    const int64_t Bt = plan.Bt;
    plan.Wd = (ix->D + 31) / 32;
    plan.Wk = (ix->K + 31) / 32;
    plan.Wke = (plan.Wk + 1) & ~1ll;
    plan.D_total = ix->D;

    // ---- subset rows: queries with the same id list share one; every empty list is the same row ----
    plan.qrow.assign((size_t)Bt, -1);
    std::vector<long long> span;  // [2 rows] into sub_ids, then relative to `lo`
    std::map<std::pair<int64_t, int64_t>, int> row_of;
    int64_t lo = INT64_MAX, hi = 0;
    for (int64_t b = 0; b < Bt; ++b) {
        int64_t s, e;
        if (!query_subset(io, b, &s, &e)) continue;
        if (s == e) s = e = 0;
        auto it = row_of.emplace(std::make_pair(s, e), (int)(span.size() / 2));
        if (it.second) {
            span.push_back(s);
            span.push_back(e);
            if (s < e) lo = std::min(lo, s), hi = std::max(hi, e);
        }
        plan.qrow[(size_t)b] = it.first->second;
    }
    plan.rows = (int)(span.size() / 2);
    if (lo > hi) lo = hi = 0;
    // eligible-centroid rows: for the dense-variant queries with a subset
    bool elig = false;
    for (int64_t b = 0; b < Bt; ++b) elig = elig || (plan.qrow[(size_t)b] >= 0 && !plan.qbatched[(size_t)b]);

    // ---- the raw sub-batch bound: the score tables (16-bit always, fp32 only on the exact path, the 16-row slab maxima
    // of the 16-bit one on the tensor-core path) and the per-(query,
    // doc) scratch (candidate lists, code sums, approximate scores, cut keys, bitmap: 24.2 bytes per document; the
    // live-row bitmap of the pruned first pass: 1 bit per centroid) share one budget.  A host-tier handle also stages up
    // to Mcap docs of max_doclen rows per query (residuals, codes, 1 / |v|); a call with subsets holds a doc row and
    // (dense variant) an eligibility row per query that has one.
    int nq_max_all = 0;
    for (int64_t b = 0; b < Bt; ++b) nq_max_all = std::max<int>(nq_max_all, (int)(io.q_off[b + 1] - io.q_off[b]));
    const int QS_all = query_row_tokens(nq_max_all);
    const size_t per_q_all = (size_t)ix->K * QS_all * (k1_tc_usable(ix) ? 2 : 6) +
                             (k1_tc_usable(ix) ? (size_t)ix->K * QS_all / 8 : 0) + (size_t)ix->D * 24 + (size_t)ix->D / 8 + (size_t)ix->K / 8 + 4096 +
                             (ix->host_tier ? (size_t)plan.Mcap * std::max(ix->max_doclen, 1) * (ix->packed + 8) : 0) +
                             (plan.rows ? (size_t)plan.Wd * 4 + (elig ? (size_t)plan.Wke * 4 : 0) : 0);
    int QB = (int)std::max<size_t>(1, std::min<size_t>((size_t)Bt, ix->st_budget / std::max(g_budget_div, 1) / per_q_all));
    QB = std::min(QB, 256);

    // ---- the rows on the device: every id of the call in one copy ----
    auto build_rows = [&]() -> pb_status {
        if (!plan.rows) return PB_OK;
        for (size_t i = 0; i < span.size(); i += 2)  // relative to the uploaded ids; empty lists stay [0, 0)
            if (span[i] < span[i + 1]) span[i] -= lo, span[i + 1] -= lo;
        CKS(ws.subset.ensure((size_t)std::max<int64_t>(hi - lo, 2) * 8));
        CKS(ws.subspan.ensure(span.size() * 8));
        if (hi > lo)
            CK(cudaMemcpyAsync(ws.subset.p, io.sub_ids + lo, (size_t)(hi - lo) * 8, cudaMemcpyHostToDevice, ws.stream));
        CK(cudaMemcpyAsync(ws.subspan.p, span.data(), span.size() * 8, cudaMemcpyHostToDevice, ws.stream));
        long long len_max = 0;
        for (int r = 0; r < plan.rows; ++r) len_max = std::max(len_max, span[2 * r + 1] - span[2 * r]);
        const unsigned gx = (unsigned)std::max<long long>(1, std::min<long long>((len_max + 255) / 256,
                                                                                  std::max(1, ix->sm_count * 4 / plan.rows)));
        CKS(ws.subset_bits.ensure(std::max<size_t>((size_t)plan.rows * plan.Wd * 4, 16)));
        CK(cudaMemsetAsync(ws.subset_bits.p, 0, (size_t)plan.rows * plan.Wd * 4, ws.stream));
        k_subset_bits<<<dim3(gx, plan.rows), 256, 0, ws.stream>>>(ws.subset.as<long long>(), ws.subspan.as<long long>(),
                                                                 ix->doc_id_base, ix->D, ws.subset_bits.as<uint32_t>(),
                                                                 plan.Wd);
        plan.d_subset_bits = ws.subset_bits.as<uint32_t>();
        if (elig) {
            CKS(ws.elig.ensure((size_t)plan.rows * plan.Wke * 4));
            CK(cudaMemsetAsync(ws.elig.p, 0, (size_t)plan.rows * plan.Wke * 4, ws.stream));
            // a warp per listed doc; the row in shared memory while it fits (K <= 2^19)
            const size_t sm = (size_t)plan.Wk * 4;
            const bool in_smem = sm <= 64 * 1024;
            if (in_smem) CKS(set_smem(k_eligible_bits, sm));
            const unsigned ge = (unsigned)std::max<long long>(1, std::min<long long>((len_max + 63) / 64,
                                                                                      std::max(1, ix->sm_count * 2 / plan.rows)));
            k_eligible_bits<<<dim3(ge, plan.rows), 256, in_smem ? sm : 0, ws.stream>>>(
                ws.subset.as<long long>(), ws.subspan.as<long long>(), ix->doc_id_base, ix->D, ix->doc_off.as<long long>(),
                ix->codes.as<uint32_t>(), ws.elig.as<uint32_t>(), plan.Wk, plan.Wke, in_smem ? 1 : 0);
            plan.d_elig = ws.elig.as<uint32_t>();
        }
        CK(cudaGetLastError());
        return PB_OK;
    };
    pb_status local = build_rows();
    if (plan.sharded) {
        Fnv64 f;  // the subset arguments as the caller gave them
        f.put(Bt);
        for (int64_t b = 0; b < Bt; ++b) {
            int64_t s = 0, e = 0;
            const uint8_t has = query_subset(io, b, &s, &e) ? 1 : 0;
            f.put(has);
            f.put(e - s);
            if (has && e > s && !io.shared_sub) f.add(io.sub_ids + s, (size_t)(e - s) * 8);
        }
        if (io.shared_sub && io.n_shared > 0) f.add(io.sub_ids, (size_t)io.n_shared * 8);
        for (int64_t b = 0; b < Bt; ++b) {  // the parameters (field by field: the struct has padding)
            const pb_search_params &q = query_params(io, b);
            f.put(q.n_full_scores), f.put(q.top_k), f.put(q.n_ivf_probe), f.put(q.centroid_batch_size);
            f.put(q.has_centroid_score_threshold), f.put(q.centroid_score_threshold);
        }
        CKS(plan_exchange(ix, ws, local, f.h, &QB, plan));
        if (elig) {  // global eligibility: every rank's rows, OR-ed on the device
            const size_t words = (size_t)plan.rows * plan.Wke;
            CKS(ws.gelig.ensure(words * 4 * ix->comm.world));
            CKS(ix->comm.allgather(ws.stream, ws.elig.p, ws.gelig.p, words / 2));
            k_or_ranks<<<ix->sm_count * 4, 256, 0, ws.stream>>>(ws.gelig.as<uint32_t>(), ix->comm.world, (long long)words,
                                                               ws.elig.as<uint32_t>());
            CK(cudaGetLastError());
        }
    } else CKS(local);

    // ---- every query's kind and n: the eligible counts come back in one read ----
    std::vector<unsigned long long> ne((size_t)plan.rows, 0ull);
    if (elig) {
        CKS(ws.eligcnt.ensure((size_t)plan.rows * 8));
        CK(cudaMemsetAsync(ws.eligcnt.p, 0, (size_t)plan.rows * 8, ws.stream));
        const unsigned gp = (unsigned)std::max<long long>(1, std::min<long long>((plan.Wk + 4095) / 4096, 8));
        k_popcount<<<dim3(gp, plan.rows), 256, 0, ws.stream>>>(ws.elig.as<uint32_t>(), plan.Wke,
                                                              ws.eligcnt.as<unsigned long long>());
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(ne.data(), ws.eligcnt.p, (size_t)plan.rows * 8, cudaMemcpyDeviceToHost, ws.stream));
        CK(cudaStreamSynchronize(ws.stream));
    }
    if (plan.sharded) g_search_agreed = true;  // the refusals below follow from exchanged data alone
    for (int64_t b = 0; b < Bt; ++b)
        if (!query_empty(plan, b) && plan.qbatched[(size_t)b]) CKS(check_batched_probe(ix, query_params(io, b)));
    plan.qn.assign((size_t)Bt, 0);
    plan.kind.assign((size_t)Bt, PROBE_TABLE);
    for (int64_t b = 0; b < Bt; ++b) {
        const pb_search_params &p = query_params(io, b);
        const int r = plan.qrow[(size_t)b];
        const int stream_max = plan.qbatched[(size_t)b] ? 192 : 64;
        int n = (int)std::min<long long>(p.n_ivf_probe, ix->K);
        uint8_t k = n > stream_max ? PROBE_BIG : PROBE_TABLE;
        if (query_empty(plan, b)) k = PROBE_NONE, n = 0;
        else if (!plan.qbatched[(size_t)b] && r >= 0) {
            const unsigned long long n_elig = ne[(size_t)r];
            const unsigned long long len = (unsigned long long)(io.shared_sub ? io.n_shared : io.sub_off[b + 1] - io.sub_off[b]);
            // n_ivf_probe scaled by D / |subset| (raw length, duplicates and out-of-range ids counted)
            unsigned long long scaled = len > 0 ? (unsigned long long)p.n_ivf_probe * (unsigned long long)plan.D_total / len
                                                : (unsigned long long)p.n_ivf_probe;
            scaled = std::max<unsigned long long>(scaled, (unsigned long long)p.n_ivf_probe);
            scaled = std::min<unsigned long long>(scaled, n_elig);
            if (n_elig == 0) k = PROBE_NONE, n = 0;  // every per-token pool is empty -> no cells
            else if (scaled >= n_elig) k = PROBE_ALL, n = (int)n_elig;
            else n = (int)scaled, k = n > stream_max ? PROBE_BIG : PROBE_STREAM;
        }
        plan.kind[(size_t)b] = k;
        plan.qn[(size_t)b] = n;
    }
    // the limits of pb_search_batch, query by query
    for (int64_t b = 0; b < Bt; ++b) {
        const uint8_t k = plan.kind[(size_t)b];
        if (k == PROBE_NONE) continue;
        CKS(check_query_rows(ix, k, plan.qn[(size_t)b], (int)(io.q_off[b + 1] - io.q_off[b])));
    }
    g_search_agreed = false;

    // ---- passes: the queries of each pass key in input order, in equal sub-batches of at most QB; a streaming pass
    // also keeps its widest query row x its largest n within 8192.  The key is (probe kind, variant, slab width,
    // whether the query's own n admits the tensor-core table): the batched threshold rule depends on the slab width,
    // and a query whose n rules out the table path must not pull the others of its pass off it ----
    std::vector<uint8_t> tc_ok((size_t)Bt, 0);
    for (int64_t b = 0; b < Bt; ++b) {
        if (plan.kind[(size_t)b] != PROBE_TABLE) continue;
        int n_chunks = 0;
        const int n = plan.qn[(size_t)b];
        probe_chunk_rows(ix->K, n, &n_chunks);
        tc_ok[(size_t)b] = n_chunks >= n && n <= 192;
    }
    const auto same_key = [&](int64_t a, int64_t b) {
        return plan.kind[(size_t)a] == plan.kind[(size_t)b] && plan.qbatched[(size_t)a] == plan.qbatched[(size_t)b] &&
               plan.qslab[(size_t)a] == plan.qslab[(size_t)b] && tc_ok[(size_t)a] == tc_ok[(size_t)b];
    };
    std::vector<uint8_t> placed((size_t)Bt, 0);
    for (uint8_t k = PROBE_TABLE; k < PROBE_NONE; ++k) {
        for (int64_t first = 0; first < Bt; ++first) {
            if (placed[(size_t)first] || plan.kind[(size_t)first] != k) continue;
            std::vector<int64_t> run;
            for (int64_t b = first; b < Bt; ++b)
                if (!placed[(size_t)b] && same_key(first, b)) run.push_back(b), placed[(size_t)b] = 1;
            const int64_t L = (int64_t)run.size();
            const int64_t per = (L + (L + QB - 1) / QB - 1) / ((L + QB - 1) / QB);  // equal sub-batches
            int64_t at = (int64_t)plan.order.size();
            int cur = 0, qs_max = 0, n_max = 0;
            for (int64_t b : run) {
                const int QS = query_row_tokens((int)(io.q_off[b + 1] - io.q_off[b]));
                const int qs2 = std::max(qs_max, QS), n2 = std::max(n_max, plan.qn[(size_t)b]);
                const bool wide = (k == PROBE_TABLE || k == PROBE_STREAM) && (long long)qs2 * n2 > 8192;
                if (cur > 0 && (cur == per || wide)) {
                    plan.passes.emplace_back(at, cur);
                    at += cur;
                    cur = 0;
                    qs_max = n_max = 0;
                }
                qs_max = std::max(qs_max, QS);
                n_max = std::max(n_max, plan.qn[(size_t)b]);
                plan.order.push_back(b);
                ++cur;
            }
            plan.passes.emplace_back(at, cur);
        }
    }
    return PB_OK;
}

// The pinned read-back of one pass (ws.hcounts): the query offsets that go up, then what comes back.  Placed here only.
struct HostCounts {
    int *qoff;                // [B + 1] query token offsets of the sub-batch
    unsigned long long *cnt;  // [B + 4] ws.counters
    long long *surv_tok;      // [B] tokens of the filter's survivors
    int *cells, *cand, *kept, *surv, *recheck, *pairs, *need;  // [B] each
    // [B] each, up in one copy: the queries' subset rows and n_ivf_probe (Pass::rows), then their M, M1, top_k and
    // threshold (Pass::mixed)
    int *qrow, *qn, *qM, *qM1, *qtopk, *qhas;
    float *qthr;
    int *fell;                // the threshold-first probe's fallback flag
};
enum { HC_UP_WORDS = 7 };  // the per-query words from qrow to qthr
static pb_status map_host_counts(HostBuf &hb, int B, HostCounts &h) {
    const size_t at_cnt = ((size_t)(B + 1) * 4 + 15) & ~(size_t)15, at_tok = at_cnt + (size_t)(B + 4) * 8,
                 at_int = at_tok + (size_t)B * 8;
    CKS(hb.ensure(at_int + ((size_t)14 * B + 1) * 4));
    char *base = hb.as<char>();
    h.qoff = reinterpret_cast<int *>(base);
    h.cnt = reinterpret_cast<unsigned long long *>(base + at_cnt);
    h.surv_tok = reinterpret_cast<long long *>(base + at_tok);
    int *c = reinterpret_cast<int *>(base + at_int);
    for (int **f : {&h.cells, &h.cand, &h.kept, &h.surv, &h.recheck, &h.pairs, &h.need, &h.qrow, &h.qn, &h.qM, &h.qM1,
                    &h.qtopk, &h.qhas})
        *f = c, c += B;
    h.qthr = reinterpret_cast<float *>(c), c += B;
    h.fell = c;
    return PB_OK;
}

// One pass of the pipeline over a sub-batch: its inputs, then what one stage hands to a later one
struct Pass {
    const int64_t *q = nullptr;  // [B] the input positions of its queries (ascending within a kind)
    int64_t R = 0;               // the sub-batch's tokens
    int B = 0, nq_max = 0, QS = 0;
    // the probe kind of its queries and their largest n_ivf_probe; rows: the queries' subset rows and n on the device
    // (d_qrow / d_qn), when any query has a row or its own n
    uint8_t kind = PROBE_TABLE;
    int n = 0;
    bool rows = false;
    const int *d_qrow = nullptr, *d_qn = nullptr;
    // the search parameters: the variant and slab width are the pass's (its key); M, M1, top_k and the threshold are
    // its first query's, and with `mixed` (its queries differ in them) each query's on the device (d_qM ...)
    bool batched = false;
    long long slab = 0;
    int M = 0, M1 = 0, top_k = 0, has_thr = 0;
    float thr = 0.0f;
    bool mixed = false;
    bool some_top_k_below_M = false;  // the certified filter has something to drop
    const int *d_qM = nullptr, *d_qM1 = nullptr, *d_qtopk = nullptr, *d_qhas = nullptr;
    const float *d_qthr = nullptr;
    // use_tc: a2 + a3 on the tensor cores.  A flagged query or a probe-list overflow raises a device flag instead of
    // being read back mid-way; the pass then finishes on (memory-safe) garbage and is redone on the exact path.
    bool use_tc = false;
    bool fast = false;  // the two-pass approximate stage on the 16-bit score table
    bool prune = false;  // its first pass bounded from the live table rows (QS <= 64, not on a redo)
    HostCounts hc{};
    // a2 / a3
    int cells_cap = 0;
    const int *d_probe_fallback = nullptr;  // device flag of the threshold-first probe (0 = it did the work)
    bool probe_list_only = false;
    // a5: the candidates that carry an approximate score
    const uint32_t *cand_list = nullptr;
    const int *cand_n = nullptr;
    // a7: whether the certified filter runs (decided before a2, which makes its 16-bit table), its form, and the docs
    // scored exactly
    bool filt = false, pairs = false, diag = false;
    KeptView kv{};
    // a9: the results of the sub-batch on the device
    long long *d_ids = nullptr;
    float *d_sc = nullptr;
    int *d_cn = nullptr;
};

// H2D: the query tokens and offsets of the sub-batch, gathered from their input positions, and their subset rows
static pb_status upload_queries(pb_index *ix, Workspace &ws, const SearchIO &io, const SearchPlan &plan, Pass &pass) {
    const int B = pass.B;
    const size_t bytes = (size_t)pass.R * ix->dim * 4, row = (size_t)ix->dim * 4;
    CKS(ws.Q.ensure(std::max<size_t>(bytes, 16)));
    CKS(ws.qoff.ensure((size_t)(B + 1) * 4));
    CKS(map_host_counts(ws.hcounts, B, pass.hc));
    pass.hc.qoff[0] = 0;
    for (int b = 0; b < B; ++b) pass.hc.qoff[b + 1] = pass.hc.qoff[b] + (int)(io.q_off[pass.q[b] + 1] - io.q_off[pass.q[b]]);
    if (pass.R > 0) {
        if (io.queries_on_device) {  // no subsets: the queries of a pass are consecutive
            const float *src = io.queries + (size_t)io.q_off[pass.q[0]] * ix->dim;
            CK(cudaMemcpyAsync(ws.Q.p, src, bytes, cudaMemcpyDeviceToDevice, ws.stream));
        } else {
            CKS(ws.hq.ensure(bytes));
            for (int b = 0; b < B; ++b)
                memcpy(ws.hq.as<char>() + (size_t)pass.hc.qoff[b] * row, io.queries + (size_t)io.q_off[pass.q[b]] * ix->dim,
                       (size_t)(pass.hc.qoff[b + 1] - pass.hc.qoff[b]) * row);
            CK(cudaMemcpyAsync(ws.Q.p, ws.hq.p, bytes, cudaMemcpyHostToDevice, ws.stream));
        }
    }
    CK(cudaMemcpyAsync(ws.qoff.p, pass.hc.qoff, (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, ws.stream));
    if (pass.rows || pass.mixed) {
        for (int b = 0; b < B; ++b) {
            const size_t g = (size_t)pass.q[b];
            pass.hc.qrow[b] = plan.qrow[g];
            pass.hc.qn[b] = plan.qn[g];
            pass.hc.qM[b] = plan.qM[g];
            pass.hc.qM1[b] = plan.qM1[g];
            pass.hc.qtopk[b] = plan.qtopk[g];
            pass.hc.qhas[b] = plan.qhas[g];
            pass.hc.qthr[b] = plan.qthr[g];
        }
        CKS(ws.qsub.ensure((size_t)B * HC_UP_WORDS * 4));
        CK(cudaMemcpyAsync(ws.qsub.p, pass.hc.qrow, (size_t)B * HC_UP_WORDS * 4, cudaMemcpyHostToDevice, ws.stream));
        const int *up = ws.qsub.as<int>();
        if (pass.rows) pass.d_qrow = up, pass.d_qn = up + B;
        if (pass.mixed) {
            pass.d_qM = up + 2 * B, pass.d_qM1 = up + 3 * B, pass.d_qtopk = up + 4 * B, pass.d_qhas = up + 5 * B;
            pass.d_qthr = ws.qsub.as<float>() + 6 * B;
        }
    }
    return PB_OK;
}

// a2: the centroid score table, fp32 off the tensor cores and 16-bit for a fast pass or the filter; on the tensor cores
// also a3
static pb_status centroid_scores(pb_index *ix, Workspace &ws, Pass &pass) {
    const int B = pass.B, QS = pass.QS;
    int *L = g_stats.launches;
    if (!pass.use_tc) CKS(ws.ST.ensure((size_t)B * ix->K * QS * sizeof(float)));
    const bool with16 = pass.fast || pass.filt;
    if (with16) {
        CKS(ws.ST16.ensure((size_t)B * ix->K * QS * 2));
        CKS(ws.qrange.ensure((size_t)B * 8 + 16));
        CKS(ws.qflag.ensure((size_t)B * 4 + 16));
        CKS(ws.qexp.ensure((size_t)B * 4 + 16));
        CKS(ws.qnmax.ensure((size_t)B * 4 + 16));
        k_query_range<<<B, 256, 0, ws.stream>>>(ws.Q.as<float>(), ws.qoff.as<int>(), ix->dim, ix->cmax,
                                                ws.qrange.as<float2>(), ws.qflag.as<int>(), ws.qexp.as<int>(),
                                                ws.qnmax.as<float>());
        CK(cudaGetLastError());
        L[PB_STAGE_CENTROID_SCORES] += 1;
    }
    if (pass.use_tc)
        return run_k1_tc(ix, ws, B, QS, pass.nq_max, pass.n, pass.d_qn, pass.has_thr, pass.thr, pass.d_qhas, pass.d_qthr,
                         pass.batched, pass.slab, pass.prune, L, &pass.cells_cap, &pass.d_probe_fallback);
    CKS(launch_centroid_scores(ix, ws, B, QS, &L[PB_STAGE_CENTROID_SCORES], with16));
    // PB_K1_TC_DIAG: the tensor-core table next to the exact one, compared code by code
    if (pass.fast && ix->k1_diag && ix->cent_h16t.p) CKS(launch_k1_diag(ix, ws, B, QS));
    return PB_OK;
}

// a3: the cells (centroids) each query probes, on the fp32 table; the tensor-core pass placed them in a2
static pb_status probe(pb_index *ix, Workspace &ws, const SearchPlan &plan, Pass &pass) {
    if (pass.use_tc) return PB_OK;
    const int B = pass.B, QS = pass.QS;
    int *L = g_stats.launches;
    // each query reads its own eligibility row and n (pass.d_qrow / d_qn); lists are sized by the pass's largest n
    const uint32_t *elig = pass.rows ? plan.d_elig : nullptr;
    if (pass.kind == PROBE_ALL) {
        pass.cells_cap = pass.n;  // the largest eligible count of the pass
        CKS(ws.list.ensure((size_t)B * pass.n * 4 + 16));
        CKS(ws.listn.ensure((size_t)B * 4 + 16));
        CKS(ws.cells.ensure((size_t)B * pass.cells_cap * 4));
        CKS(ws.ncells.ensure((size_t)B * 4 + 16));
        k_cells_from_bits<<<B, 1024, 0, ws.stream>>>(plan.d_elig, pass.d_qrow, plan.Wke, ix->K, ws.list.as<uint32_t>(),
                                                     pass.n, ws.listn.as<int>());
        k_cells_filter_list<<<B, 256, 0, ws.stream>>>(ws.list.as<uint32_t>(), pass.n, ws.listn.as<int>(), ws.ST.as<float>(),
                                                      ws.qoff.as<int>(), ix->K, QS, pass.has_thr, pass.thr, pass.cells_cap,
                                                      ws.cells.as<uint32_t>(), ws.ncells.as<int>(), pass.d_qhas,
                                                      pass.d_qthr);
        CK(cudaGetLastError());
        L[PB_STAGE_PROBE] += 2;
        return PB_OK;
    }
    const int n = pass.n;
    pass.cells_cap = (int)std::min<long long>((long long)QS * n, ix->K);
    if (pass.kind == PROBE_BIG) {
        CKS(ws.cellbits.ensure((size_t)B * plan.Wk * 4));
        CKS(ws.cells.ensure((size_t)B * pass.cells_cap * 4));
        CKS(ws.ncells.ensure((size_t)B * 4 + 16));
        k_topn_select_row<<<dim3(QS, B), 256, 0, ws.stream>>>(ws.ST.as<float>(), ws.qoff.as<int>(), ix->K, QS, pass.d_qn,
                                                              elig, pass.d_qrow, plan.Wke, ws.cellbits.as<uint32_t>(),
                                                              plan.Wk);
        k_cells_from_query_bits<<<B, 1024, 0, ws.stream>>>(ws.cellbits.as<uint32_t>(), plan.Wk, ws.ST.as<float>(),
                                                           ws.qoff.as<int>(), ix->K, QS, pass.has_thr, pass.thr,
                                                           pass.cells_cap, ws.cells.as<uint32_t>(), ws.ncells.as<int>(),
                                                           pass.d_qhas, pass.d_qthr);
        CK(cudaGetLastError());
        L[PB_STAGE_PROBE] += 2;
        return PB_OK;
    }
    const int n_chunks = (int)((ix->K + 1023) / 1024);
    CKS(ws.partial.ensure((size_t)B * QS * n_chunks * n * 8));
    CKS(ws.sel.ensure((size_t)B * QS * n * 8));
    CKS(ws.cells.ensure((size_t)B * pass.cells_cap * 4));
    CKS(ws.ncells.ensure((size_t)B * 4 + 16));
    size_t sm1 = (size_t)4 * n * 32 * 8;
    CKS(set_smem(k_topn_partial, sm1));
    // threshold-first selection on the 16-bit table when there is one (k_chunkmax16 / k_collect16);
    // the per-lane list scan of k_topn_partial otherwise, or when the device raises `fallback`
    const int GQ = QS / 8;
    int t_chunks = 0;
    const int t_rows = probe_chunk_rows(ix->K, n, &t_chunks);
    const bool thr_path = pass.fast && pass.kind == PROBE_TABLE && ix->probe16 && GQ <= 32 && t_chunks >= n && n <= 192;
    int *d_fallback = nullptr;
    pass.probe_list_only = !thr_path;
    if (thr_path) {
        const int cap = probe16_cap(n);
        CKS(probe16_thresholds(ix, ws, B, QS, n, t_chunks, t_rows, pass.d_qn, nullptr, &d_fallback));
        pass.d_probe_fallback = d_fallback;
        k_collect16<<<dim3((t_chunks + 3) / 4, B), 128, 0, ws.stream>>>(
            ws.ST16.as<unsigned short>(), ws.ST.as<float>(), ix->K, QS, t_chunks, t_rows, ws.tau16.as<uint32_t>(), cap,
            ws.pcount.as<int>(), ws.plist.as<u64>(), d_fallback);
        k_topn_merge<<<dim3(QS, B), 32, 0, ws.stream>>>(ws.plist.as<u64>(), ws.qoff.as<int>(), QS, n, cap / n,
                                                      ws.sel.as<u64>(), d_fallback, 0, pass.d_qn);
        CK(cudaGetLastError());
        L[PB_STAGE_PROBE] += 4;
    }
    k_topn_partial<<<dim3((n_chunks + 3) / 4, B, (QS + 31) / 32), 128, sm1, ws.stream>>>(
        ws.ST.as<float>(), ws.qoff.as<int>(), ix->K, QS, n, elig, pass.d_qrow, plan.Wke, pass.d_qn, ws.partial.as<u64>(),
        n_chunks, d_fallback, 1);
    k_topn_merge<<<dim3(QS, B), 32, 0, ws.stream>>>(ws.partial.as<u64>(), ws.qoff.as<int>(), QS, n, n_chunks,
                                                  ws.sel.as<u64>(), d_fallback, 1, pass.d_qn);
    const int P = pow2_at_least(std::max(pass.nq_max * n, 1));
    size_t sm2 = (size_t)P * 12;
    CKS(set_smem(k_cells, sm2));
    k_cells<<<B, 256, sm2, ws.stream>>>(ws.sel.as<u64>(), ws.ST.as<float>(), ws.qoff.as<int>(), ix->K, QS, n,
                                        pass.cells_cap, pass.has_thr, pass.thr, pass.batched ? 1 : 0, pass.slab,
                                        ws.cells.as<uint32_t>(), ws.ncells.as<int>(),
                                        thr_path ? ws.cmax16.as<unsigned short>() : nullptr, t_chunks, t_rows,
                                        ws.qrange.as<float2>(), d_fallback, pass.d_qn, pass.d_qhas, pass.d_qthr);
    CK(cudaGetLastError());
    L[PB_STAGE_PROBE] += 3;
    return PB_OK;
}

// a4: the docs of the probed cells (within the subset), compacted per query
static pb_status candidates(pb_index *ix, Workspace &ws, const SearchPlan &plan, const Pass &pass) {
    const int B = pass.B;
    const long long Wd = plan.Wd;
    CKS(ws.bitmap.ensure((size_t)B * Wd * 4));
    CKS(ws.cand.ensure((size_t)B * ix->D * 4));
    CKS(ws.ncand.ensure((size_t)B * 4 + 16));
    k_mark<<<dim3(pass.cells_cap, B), 128, 0, ws.stream>>>(ws.cells.as<uint32_t>(), ws.ncells.as<int>(), pass.cells_cap,
                                                          ix->ivf.as<uint32_t>(), ix->ivf_off.as<long long>(),
                                                          pass.rows ? plan.d_subset_bits : nullptr, pass.d_qrow,
                                                          ws.bitmap.as<uint32_t>(), Wd);
    const int slices = (int)std::max<long long>(1, std::min<long long>(32, (4ll * ix->sm_count + B - 1) / B));
    CKS(ws.slicecnt.ensure((size_t)B * slices * 4));
    k_compact_count<<<dim3(slices, B), 256, 0, ws.stream>>>(ws.bitmap.as<uint32_t>(), Wd, ws.slicecnt.as<int>());
    k_compact_emit<<<dim3(slices, B), 256, 0, ws.stream>>>(ws.bitmap.as<uint32_t>(), Wd, ws.slicecnt.as<int>(),
                                                           ws.cand.as<uint32_t>(), ix->D, ws.ncand.as<int>());
    CK(cudaGetLastError());
    g_stats.launches[PB_STAGE_CANDIDATES] += 3;
    return PB_OK;
}

// a5: the approximate score of every candidate; a fast pass first narrows them to the band around the cut on the
// 16-bit table, and the tensor-core pass re-checks that band with pinned-order dots
static pb_status approx_scores(pb_index *ix, Workspace &ws, const SearchPlan &plan, Pass &pass) {
    const int B = pass.B, QS = pass.QS, Mcap = plan.Mcap;
    int *L = g_stats.launches;
    // [0] candidate codes gathered, [1+b] kept-doc tokens, [B+1] re-check gathers, [B+2] live rows gathered by the
    // pruned first pass, [B+3] docs it scored densely
    CKS(ws.counters.ensure((size_t)(B + 4) * 8));
    CK(cudaMemsetAsync(ws.counters.p, 0, (size_t)(B + 4) * 8, ws.stream));
    CKS(ws.approx.ensure((size_t)B * ix->D * 4));
    CKS(ws.keys.ensure((size_t)B * ix->D * 8));
    if (pass.fast) {
        CKS(ws.lsum.ensure((size_t)B * ix->D * 4));
        CKS(ws.cand2.ensure((size_t)B * ix->D * 4));
        CKS(ws.ncand2.ensure((size_t)B * 4 + 16));
        const dim3 ga(ix->sm_count * ix->approx_grid, B);
        const unsigned short *st16 = ws.ST16.as<unsigned short>();
        const uint32_t *list = ws.cand.as<uint32_t>();
        const int *list_n = ws.ncand.as<int>();
        unsigned long long *cnt = ws.counters.as<unsigned long long>();
        const auto approx16 = QS <= 32 ? k_approx16<4> : k_approx16<8>;
        // band per query token in code units (W = band * nq + 8).  Exact table: +-1 code of rounding per token and side
        // plus the fp32 summation error -> 4.  Estimate table (k_scores_tc.cuh): W = nq (1.004 + 2 err) + nq^2/256 + 4
        // <= nq (ceil(1.004 + 2 err) + 1) + 8 for nq <= 256.
        const int band_per_q =
            pass.use_tc ? (int)ceilf(1.004f + 2.0f * std::max(k1_err_codes(ix->dim), (float)(ix->k1_margin - 1))) + 1 : 4;
        KEV_BEGIN(PB_KERNEL_APPROX16);
        if (pass.prune) {
            // the bound U of every candidate from the live rows, then k_approx16 on the two rounds that can reach the
            // band (k_approx16.cuh); U lives in ws.approx and the round lists in ws.keys until the re-check overwrites them
            const long long live_stride = a5_live_stride(ix->K);
            CKS(ws.a5n1.ensure((size_t)B * 4 + 16));
            CKS(ws.a5n12.ensure((size_t)B * 4 + 16));
            CKS(ws.a5theta.ensure((size_t)B * 4 + 16));
            const int M1 = pass.M1;
            uint32_t *ub = ws.approx.as<uint32_t>(), *rl = ws.keys.as<uint32_t>();
            int *n1 = ws.a5n1.as<int>(), *n12 = ws.a5n12.as<int>();
            if (!pass.use_tc) {  // the tensor-core pass took the floors and the live bits with its probe (run_k1_tc)
                CKS(ws.a5floor.ensure((size_t)B * QS * 4));
                CKS(ws.a5live.ensure((size_t)B * live_stride * 4));
                k_a5_floor<<<dim3(QS / 8, B), 256, 0, ws.stream>>>(st16, ws.qoff.as<int>(), ix->K, QS, a5_live_rows(ix),
                                                                   ws.a5floor.as<uint32_t>());
                k_a5_live<<<dim3(ix->sm_count * 2, B), 256, 0, ws.stream>>>(st16, ix->K, QS, ws.a5floor.as<uint32_t>(),
                                                                             ws.a5live.as<uint32_t>(), live_stride);
                L[PB_STAGE_APPROX] += 2;
            }
            // the bitmap in shared memory up to K = 2^19 (64 KiB, two CTAs per SM), then a5_waves waves of resident
            // CTAs spread over the batch, each a contiguous range of its query's candidates (k_approx16.cuh; the
            // default of 8 waves is measured in DESIGN.md 4b)
            const auto bound = QS <= 32 ? k_a5_bound<4> : k_a5_bound<8>;
            const bool bits_in_smem = live_stride * 4 <= 64 * 1024;
            const size_t smb = a5_bound_smem(live_stride, bits_in_smem);
            CKS(set_smem(bound, smb));
            int resident = 1;
            CKS(resident_ctas(bound, 256, smb, &resident));
            const long long ctas = (long long)resident * ix->sm_count * ix->a5_waves;
            const dim3 gb((unsigned)std::max(1ll, (ctas + B - 1) / B), B);
            bound<<<gb, 256, smb, ws.stream>>>(st16, ws.qoff.as<int>(), ix->K, QS, ix->ucodes.as<uint32_t>(),
                                               ix->udoc_off.as<long long>(), list, ix->D, list_n,
                                               ws.a5floor.as<uint32_t>(), ws.a5live.as<uint32_t>(), live_stride,
                                               bits_in_smem, ub, cnt, cnt + B + 2);
            k_select_u32<<<B, 1024, 0, ws.stream>>>(ub, list_n, M1, 0, ub, list, list_n, ix->D, ws.qoff.as<int>(),
                                                    ws.qflag.as<int>(), rl, n1, ws.a5theta.as<uint32_t>(), nullptr,
                                                    nullptr, nullptr, pass.d_qM1);
            approx16<<<ga, 256, 0, ws.stream>>>(st16, ws.qoff.as<int>(), ix->K, QS, ix->ucodes.as<uint32_t>(),
                                                ix->udoc_off.as<long long>(), rl, ix->D, n1, nullptr,
                                                ws.lsum.as<uint32_t>(), nullptr);
            k_select_u32<<<B, 1024, 0, ws.stream>>>(ws.lsum.as<uint32_t>(), n1, pass.M, band_per_q, ub, list, list_n,
                                                    ix->D, ws.qoff.as<int>(), ws.qflag.as<int>(), rl, n12, nullptr,
                                                    ws.a5theta.as<uint32_t>(), n1, cnt + B + 3, pass.d_qM);
            approx16<<<ga, 256, 0, ws.stream>>>(st16, ws.qoff.as<int>(), ix->K, QS, ix->ucodes.as<uint32_t>(),
                                                ix->udoc_off.as<long long>(), rl, ix->D, n12, n1,
                                                ws.lsum.as<uint32_t>(), nullptr);
            list = rl;
            list_n = n12;
            L[PB_STAGE_APPROX] += 5;
        } else {
            approx16<<<ga, 256, 0, ws.stream>>>(st16, ws.qoff.as<int>(), ix->K, QS, ix->ucodes.as<uint32_t>(),
                                                ix->udoc_off.as<long long>(), list, ix->D, list_n, nullptr,
                                                ws.lsum.as<uint32_t>(), cnt);
            L[PB_STAGE_APPROX] += 1;
        }
        KEV_END(PB_KERNEL_APPROX16);
        k_select_u32<<<B, 1024, 0, ws.stream>>>(ws.lsum.as<uint32_t>(), list_n, pass.M, band_per_q, ws.lsum.as<uint32_t>(),
                                                list, list_n, ix->D, ws.qoff.as<int>(), ws.qflag.as<int>(),
                                                ws.cand2.as<uint32_t>(), ws.ncand2.as<int>(), nullptr, nullptr, nullptr,
                                                nullptr, pass.d_qM);
        CK(cudaGetLastError());
        L[PB_STAGE_APPROX] += 1;
    }
    pass.cand_list = pass.fast ? ws.cand2.as<uint32_t>() : ws.cand.as<uint32_t>();
    pass.cand_n = pass.fast ? ws.ncand2.as<int>() : ws.ncand.as<int>();
    if (pass.use_tc) {  // the exact approximate score of the docs around the cut from pinned-order dots (no dense fp32 S)
        const int rc_cap = 2 * Mcap + 1024, pair_cap = 64 * rc_cap;
        CKS(ws.rcmax.ensure((size_t)B * rc_cap * QS * 4));
        CKS(ws.rcpairs.ensure((size_t)B * pair_cap * 8));
        CKS(ws.rcn.ensure((size_t)B * 4 + 16));
        CK(cudaMemsetAsync(ws.rcn.p, 0, (size_t)B * 4, ws.stream));
        int *d_fb = const_cast<int *>(pass.d_probe_fallback);
        (QS <= 32 ? k_recheck_pairs<4> : k_recheck_pairs<8>)<<<dim3(ix->sm_count * 2, B), 256, 0, ws.stream>>>(
            ws.ST16.as<unsigned short>(), ws.qoff.as<int>(), ix->K, QS, ix->ucodes.as<uint32_t>(), ix->udoc_off.as<long long>(),
            pass.cand_list, ix->D, pass.cand_n, 2 * ix->k1_margin + 1, rc_cap, pair_cap, ws.rcpairs.as<u64>(),
            ws.rcn.as<int>(), d_fb, ws.counters.as<unsigned long long>() + B + 1);
        k_recheck_dots<<<dim3(ix->sm_count * 2, B), 128, 0, ws.stream>>>(ws.rcpairs.as<u64>(), ws.rcn.as<int>(), pair_cap,
                                                                         ws.Q.as<float>(), ws.qoff.as<int>(),
                                                                         ix->centroids.as<float>(), ix->dim, rc_cap, QS,
                                                                         ws.rcmax.as<uint32_t>());
        k_recheck_sum<<<dim3(ix->sm_count, B), 256, 0, ws.stream>>>(ws.rcmax.as<uint32_t>(), ws.qoff.as<int>(), QS,
                                                                    pass.cand_list, ix->D, pass.cand_n, rc_cap,
                                                                    ws.approx.as<float>(), ws.keys.as<u64>(),
                                                                    (uint32_t)ix->doc_id_base);
        L[PB_STAGE_APPROX] += 2;
    } else
        k_approx<<<dim3(ix->sm_count * 8, B), 256, 0, ws.stream>>>(
            ws.ST.as<float>(), ws.qoff.as<int>(), ix->K, QS, ix->ucodes.as<uint32_t>(), ix->udoc_off.as<long long>(),
            pass.cand_list, ix->D, pass.cand_n, ws.approx.as<float>(), ws.keys.as<u64>(),
            pass.fast ? ws.counters.as<unsigned long long>() + B + 1 : ws.counters.as<unsigned long long>(),
            (uint32_t)ix->doc_id_base);
    CK(cudaGetLastError());
    L[PB_STAGE_APPROX] += 1;
    return PB_OK;
}

// a6: the top M by approximate score; doc-sharded, exchange 1 makes it the global cut
static pb_status cut(pb_index *ix, Workspace &ws, const SearchPlan &plan, const Pass &pass) {
    const int B = pass.B, Mcap = plan.Mcap;
    const bool sharded = plan.sharded;
    CKS(ws.kept.ensure((size_t)B * Mcap * 4));
    CKS(ws.nkept.ensure((size_t)B * 4 + 16));
    CKS(ws.tokp.ensure((size_t)B * (Mcap + 1) * 8));
    if (sharded) CKS(ws.lkeys.ensure((size_t)B * Mcap * 8));
    const int Pm = pow2_at_least(Mcap);
    CKS(set_smem(k_cut, (size_t)Pm * 8));
    k_cut<<<B, 1024, (size_t)Pm * 8, ws.stream>>>(ws.keys.as<u64>(), ws.approx.as<float>(), ix->D, pass.cand_n, pass.M,
                                                  Mcap, ix->doc_off.as<long long>(), ws.kept.as<uint32_t>(),
                                                  ws.nkept.as<int>(), ws.tokp.as<long long>(),
                                                  ws.counters.as<long long>() + 1, (uint32_t)ix->doc_id_base,
                                                  sharded ? ws.lkeys.as<u64>() : nullptr, pass.d_qM);
    CK(cudaGetLastError());
    g_stats.launches[PB_STAGE_CUT] += 1;
    if (sharded) {
        // exchange 1: every shard's sorted top-M cut keys (Mcap per query, ~0 past its M) -> global cut -> my members
        // (SURVEY 8e)
        const int G = ix->comm.world;
        CKS(ws.gkeys.ensure((size_t)G * B * Mcap * 8));
        CKS(ws.krank.ensure((size_t)B * Mcap * 4));
        CKS(ix->comm.allgather(ws.stream, ws.lkeys.p, ws.gkeys.p, (size_t)B * Mcap));
        k_merge_cut<<<B, 1024, 0, ws.stream>>>(ws.gkeys.as<u64>(), G, ix->comm.rank, B, pass.M, Mcap, (uint32_t)ix->doc_id_base,
                                               ix->D, ix->doc_off.as<long long>(), ws.kept.as<uint32_t>(),
                                               ws.krank.as<uint32_t>(), ws.nkept.as<int>(),
                                               ws.tokp.as<long long>(), ws.counters.as<long long>() + 1, pass.d_qM);
        CK(cudaGetLastError());
        g_stats.launches[PB_STAGE_CUT] += 2;
    }
    return PB_OK;
}

// k_stage_rows in the form the row length allows, on st: the rows of docs[s] for the slots s of [0, n_slots) (nkept !=
// NULL: slot b Mcap + j only for j < nkept[b]) to s_res / s_codes / s_inv at soff[s] (s_codes == NULL: rows only)
static pb_status launch_stage_rows(pb_index *ix, cudaStream_t st, const uint32_t *docs, const int *nkept, int Mcap,
                                   long long n_slots, const long long *soff, RowCache cache, uint8_t *s_res,
                                   uint32_t *s_codes, float *s_inv) {
    const int pk = ix->packed, grid = ix->sm_count * 8;
    const float *src_inv = s_inv ? ix->tok_inv_norm.as<float>() : nullptr;
    const long long *doff = ix->doc_off.as<long long>();
    const uint32_t *codes = ix->codes.as<uint32_t>();
    if (pk % 16 == 0)
        k_stage_rows<uint4, 4><<<grid, 256, 0, st>>>(docs, nkept, Mcap, n_slots, doff, soff, ix->host.dev(), cache, codes,
                                                     src_inv, pk, s_res, s_codes, s_inv);
    else if (pk % 4 != 0)  // 1-bit rows of dim 48 (6 bytes)
        k_stage_rows<unsigned short, 8><<<grid, 256, 0, st>>>(docs, nkept, Mcap, n_slots, doff, soff, ix->host.dev(), cache,
                                                              codes, src_inv, pk, s_res, s_codes, s_inv);
    else
        k_stage_rows<uint32_t, 8><<<grid, 256, 0, st>>>(docs, nkept, Mcap, n_slots, doff, soff, ix->host.dev(), cache,
                                                        codes, src_inv, pk, s_res, s_codes, s_inv);
    CK(cudaGetLastError());
    return PB_OK;
}

// The handle's row cache as k_stage_rows reads it; count: also the keep counts and the workspace's hit counters
// (search staging only)
static RowCache row_cache_view(const pb_index *ix, Workspace *ws, bool count) {
    if (!ix->cache_off.p) return RowCache{nullptr, FlatRows{nullptr}, nullptr, nullptr};
    return RowCache{ix->cache_off.as<const long long>(), FlatRows{ix->rc.rows.as<uint8_t>()},
                    count ? ix->kept_count.as<uint32_t>() : nullptr,
                    count ? ws->rc_hits.as<unsigned long long>() : nullptr};
}

// The rows of docs[s] for the slots s of [0, n_slots) (nkept != NULL: slot b Mcap + j only for j < nkept[b]) from the
// row cache or the pinned host residuals, and the device codes / 1 / |v|, into the workspace's staging buffers at
// soff[s]; cap_tok bounds the staged tokens.  count: a search's staging, which the row cache counts.  Returns the
// staged arrays as a TokView whose doc_off is soff (indexed by slot).
static pb_status stage_rows(pb_index *ix, Workspace &ws, const uint32_t *docs, const int *nkept, int Mcap, long long n_slots,
                            const long long *soff, long long cap_tok, bool count, TokView &tv) {
    const int pk = ix->packed;
    const bool inv = ix->tok_inv_norm.p != nullptr;
    cap_tok = std::max(cap_tok, 1ll);
    CKS(ws.s_res.ensure((size_t)cap_tok * pk));
    CKS(ws.s_codes.ensure((size_t)cap_tok * 4));
    if (inv) CKS(ws.s_inv.ensure((size_t)cap_tok * 4));
    float *dst_inv = inv ? ws.s_inv.as<float>() : nullptr;
    if (count && ix->cache_off.p) {
        CKS(ws.rc_hits.ensure(16));
        CK(cudaMemsetAsync(ws.rc_hits.p, 0, 16, ws.stream));
    }
    CKS(launch_stage_rows(ix, ws.stream, docs, nkept, Mcap, n_slots, soff, row_cache_view(ix, &ws, count),
                          ws.s_res.as<uint8_t>(), ws.s_codes.as<uint32_t>(), dst_inv));
    tv = {ws.s_codes.as<uint32_t>(), ws.s_res.as<uint8_t>(), dst_inv, soff};
    return PB_OK;
}

// Host tier, after the cut: the sub-batch's kept docs laid out in slot space and staged (k_stage.cuh).  kv then lists
// slots, tv the staged arrays; the cut's own list (ws.kept) stays as it is, and the slots go back to doc ids before
// k_exact_finalize.
static pb_status stage_kept(pb_index *ix, Workspace &ws, const SearchPlan &plan, const Pass &pass, KeptView &kv, TokView &tv) {
    const int B = pass.B, Mcap = plan.Mcap;
    const long long slots = (long long)B * Mcap;
    CKS(ws.soff.ensure((size_t)(slots + 1) * 8));
    CKS(ws.kept_s.ensure((size_t)slots * 4));
    if (plan.prof) CK(cudaEventRecord(ws.sev[0], ws.stream));
    k_stage_layout<<<dim3(std::min((Mcap + 255) / 256, 8), B), 256, 0, ws.stream>>>(
        kv.nkept, kv.tokp, B, Mcap, ws.soff.as<long long>(), ws.kept_s.as<uint32_t>());
    CK(cudaGetLastError());
    CKS(stage_rows(ix, ws, kv.kept, kv.nkept, Mcap, slots, ws.soff.as<long long>(), slots * std::max(ix->max_doclen, 1), true,
                   tv));
    if (plan.prof) CK(cudaEventRecord(ws.sev[1], ws.stream));
    g_stats.launches[PB_STAGE_EXACT] += 2;
    kv.kept = ws.kept_s.as<uint32_t>();
    return PB_OK;
}

// a7 + a8: the exact MaxSim of the kept docs.  Only the top_k need exact scores: the tensor-core filter (a7') first
// drops the docs that provably cannot reach them, and its pass 2 lists the (token, q) pairs k_pair_exact evaluates.
static pb_status exact_scores(pb_index *ix, Workspace &ws, const SearchPlan &plan, Pass &pass) {
    const int B = pass.B, QS = pass.QS, nq_max = pass.nq_max, Mcap = plan.Mcap;
    const bool sharded = plan.sharded;
    const long long max_tokens = (long long)Mcap * std::max(ix->max_doclen, 1);
    int *L = g_stats.launches;
    CKS(ws.maxkey.ensure((size_t)B * Mcap * QS * 4));
    CKS(ws.exact.ensure((size_t)B * Mcap * 4));
    CKS(ws.fkeys.ensure((size_t)B * Mcap * 8));
    KeptView &kv = pass.kv;
    kv = {ws.kept.as<uint32_t>(), ws.nkept.as<int>(), ws.tokp.as<long long>(), sharded ? ws.krank.as<uint32_t>() : nullptr};
    TokView tv = resident_tokens(ix);
    if (ix->host_tier) CKS(stage_kept(ix, ws, plan, pass, kv, tv));
    const float eps_unit = filter_eps_unit2(ix, pass.use_tc ? ix->k1_margin : 0);
    // PB_FILTER_DIAG: the filter runs as usual, then every kept doc is scored exactly (the results of
    // pb_set_fast_exact(0)) and k_filter_diag compares the pass-1 estimate maxima with the exact ones
    pass.diag = pass.filt && ix->filter_diag;
    if (pass.filt) {
        CKS(ws.est.ensure((size_t)B * Mcap * 4));
        CKS(ws.kept2.ensure((size_t)B * Mcap * 4));
        CKS(ws.krank2.ensure((size_t)B * Mcap * 4));
        CKS(ws.nkept2.ensure((size_t)B * 4 + 16));
        CKS(ws.tokp2.ensure((size_t)B * (Mcap + 1) * 8));
        CKS(ws.ktok2.ensure((size_t)B * 8 + 16));
        KeptView kv2{ws.kept2.as<uint32_t>(), ws.nkept2.as<int>(), ws.tokp2.as<long long>(), ws.krank2.as<uint32_t>()};
        // pair form of the exact stage: pass 2 of the estimate over the survivors lists the (token, q) pairs that can
        // hold a per-token maximum, k_pair_exact evaluates them in the pinned order; a query whose list overflows
        // (or that published no estimate) goes through k_exact
        pass.pairs = !pass.diag && ix->pair_exact && Mcap <= 65535 && QS <= 256;
        if (pass.pairs || pass.diag) {
            CKS(ws.estkey.ensure((size_t)B * Mcap * QS * 4));
            CKS(ws.srcrank.ensure((size_t)B * Mcap * 4));
        }
        CKS(launch_filter(ix, ws, kv, kv2, tv, B, QS, Mcap, pass.top_k, pass.d_qtopk, max_tokens, eps_unit, nq_max,
                          pass.pairs || pass.diag, &L[PB_STAGE_EXACT]));
        if (!pass.diag) {
            kv = kv2;
            if (!sharded) kv.krank = nullptr;  // survivors keep their order, so position breaks ties the same way
        }
    }
    if (pass.pairs) {
        const int pair_cap = 16 * Mcap + 4096;  // ~ (top_k + ties) * nq * (1 + a few) pairs per query in practice
        CKS(ws.xpairs.ensure((size_t)B * pair_cap * 8));
        CKS(ws.xnpairs.ensure((size_t)B * 4 + 16));
        CKS(ws.needexact.ensure((size_t)B * 4 + 16));
        CK(cudaMemsetAsync(ws.xnpairs.p, 0, (size_t)B * 4, ws.stream));
        KEV_BEGIN(PB_KERNEL_EXACT);  // pass 2 + pair evaluation + the (normally empty) k_exact of flagged queries
        CKS(launch_maxsim_tc(ix, ws, kv, tv, B, QS, Mcap, max_tokens, nq_max, ws.estkey.as<uint32_t>(),
                             ws.srcrank.as<uint32_t>(), eps_unit, ws.xpairs.as<u64>(), ws.xnpairs.as<int>(), pair_cap, -1));
        k_pair_overflow<<<(B + 255) / 256, 256, 0, ws.stream>>>(ws.xnpairs.as<int>(), pair_cap, ws.qflag.as<int>(), B,
                                                                ws.needexact.as<int>());
        CK(cudaGetLastError());
        const size_t smp = ((size_t)(nq_max + 256) * (ix->dim + 1) + 256) * 4;
        const int pe_ctas = std::max(1, std::min(16, (2 * ix->sm_count + B - 1) / B));  // about one wave over the batch
        CKS(TcDims::dispatch(ix->dim, [&](auto dim_c) -> pb_status {
            auto kern = k_pair_exact<decltype(dim_c)::value>;
            CKS(set_smem(kern, smp));
            kern<<<dim3(pe_ctas, B), 256, smp, ws.stream>>>(ws.xpairs.as<u64>(), ws.xnpairs.as<int>(), pair_cap,
                                                            ws.Q.as<float>(), ws.qoff.as<int>(), QS, ix->centroids.as<float>(),
                                                            ix->w_rev.as<float>(), ix->nbits, tv.codes, tv.residuals, Mcap,
                                                            ws.maxkey.as<uint32_t>());
            return PB_OK;
        }));
        CK(cudaGetLastError());
        L[PB_STAGE_EXACT] += 5;
        CKS(launch_exact(ix, ws, kv, tv, B, QS, Mcap, 0, max_tokens, &L[PB_STAGE_EXACT], ws.needexact.as<int>(), false));
        KEV_END(PB_KERNEL_EXACT);
    } else {
        CKS(launch_exact(ix, ws, kv, tv, B, QS, Mcap, 0, max_tokens, &L[PB_STAGE_EXACT]));
    }
    if (pass.diag) {  // before k_exact_finalize, which clears the exact maxima
        CKS(ws.fdiag.ensure(16));
        CK(cudaMemsetAsync(ws.fdiag.p, 0, 16, ws.stream));
        k_filter_diag<<<dim3(4, B), 256, 0, ws.stream>>>(ws.estkey.as<uint32_t>(), ws.maxkey.as<uint32_t>(), ws.qoff.as<int>(),
                                                         QS, kv.nkept, Mcap, ws.qnmax.as<float>(), ws.qflag.as<int>(), eps_unit,
                                                         ws.fdiag.as<unsigned long long>());
        CK(cudaGetLastError());
        L[PB_STAGE_EXACT] += 1;
    }
    if (ix->host_tier) {  // slots back to doc ids, in the list the scores belong to
        k_unstage_kept<<<dim3((Mcap + 255) / 256, B), 256, 0, ws.stream>>>(kv.kept, kv.nkept, Mcap, ws.kept.as<uint32_t>());
        CK(cudaGetLastError());
        L[PB_STAGE_EXACT] += 1;
    }
    if (sharded) {
        CKS(ws.payload.ensure((size_t)B * Mcap * 8));
        CK(cudaMemsetAsync(ws.fkeys.p, 0xff, (size_t)B * Mcap * 8, ws.stream));  // ~0 = no entry
    }
    k_exact_finalize<<<dim3((Mcap + 7) / 8, B), 256, 0, ws.stream>>>(
        ws.maxkey.as<uint32_t>(), ws.qoff.as<int>(), QS, kv.nkept, Mcap, 0, ws.exact.as<float>(),
        ws.fkeys.as<u64>(), kv.krank, kv.kept, (uint32_t)ix->doc_id_base, sharded ? ws.payload.as<u64>() : nullptr);
    CK(cudaGetLastError());
    L[PB_STAGE_EXACT] += 1;
    return PB_OK;
}

// a9: the top_k by exact score, into the caller's device outputs or the workspace's; doc-sharded, exchange 2 merges
// every shard's
static pb_status select_topk(pb_index *ix, Workspace &ws, const SearchIO &io, const SearchPlan &plan, Pass &pass) {
    // rows of the outputs: the caller's stride on the device, the call's largest top_k in the workspace
    const int B = pass.B, Mcap = plan.Mcap;
    const int ostride = io.out_on_device ? (int)io.out_stride : plan.top_k_max;
    if (io.out_on_device) {  // no subsets: the queries of a pass are consecutive
        pass.d_ids = reinterpret_cast<long long *>(io.out_ids) + (size_t)pass.q[0] * ostride;
        pass.d_sc = io.out_scores + (size_t)pass.q[0] * ostride;
        pass.d_cn = io.out_counts + pass.q[0];
    } else {
        CKS(ws.oids.ensure((size_t)B * ostride * 8));
        CKS(ws.oscores.ensure((size_t)B * ostride * 4));
        CKS(ws.ocounts.ensure((size_t)B * 4 + 16));
        pass.d_ids = ws.oids.as<long long>();
        pass.d_sc = ws.oscores.as<float>();
        pass.d_cn = ws.ocounts.as<int>();
    }
    const int Pm = pow2_at_least(Mcap);
    if (plan.sharded) {
        // exchange 2: (exact key | global approx rank) + (doc id | score) of every shard, merged on every rank
        const int G = ix->comm.world;
        CKS(ws.gfkeys.ensure((size_t)G * B * Mcap * 8));
        CKS(ws.gpayload.ensure((size_t)G * B * Mcap * 8));
        CKS(ix->comm.allgather(ws.stream, ws.fkeys.p, ws.gfkeys.p, (size_t)B * Mcap));
        CKS(ix->comm.allgather(ws.stream, ws.payload.p, ws.gpayload.p, (size_t)B * Mcap));
        CKS(ws.mslot.ensure((size_t)B * Mcap * 4));
        CKS(set_smem(k_merge_topk, (size_t)Pm * 8));
        k_merge_topk<<<B, 1024, (size_t)Pm * 8, ws.stream>>>(ws.gfkeys.as<u64>(), ws.gpayload.as<u64>(), G, B, Mcap,
                                                            pass.top_k, ws.mslot.as<uint32_t>(), pass.d_ids, pass.d_sc,
                                                            pass.d_cn, pass.d_qtopk, ostride);
        CK(cudaGetLastError());
        g_stats.launches[PB_STAGE_TOPK] += 3;
    } else {
        CKS(set_smem(k_topk, (size_t)Pm * 8));
        k_topk<<<B, 1024, (size_t)Pm * 8, ws.stream>>>(ws.fkeys.as<u64>(), ws.exact.as<float>(), pass.kv.kept,
                                                       pass.kv.nkept, Mcap, pass.top_k, ix->doc_id_base, pass.d_ids,
                                                       pass.d_sc, pass.d_cn, pass.d_qtopk, ostride);
        CK(cudaGetLastError());
        g_stats.launches[PB_STAGE_TOPK] += 1;
    }
    return PB_OK;
}

// D2H and the pass's one synchronise.  A tensor-core pass that gave up on the device stops there with *redo: its
// launches stay counted, its stage times are not added.  Otherwise the results go out and the pass is accounted.
static pb_status finish(pb_index *ix, Workspace &ws, const SearchIO &io, const SearchPlan &plan, const Pass &pass,
                        bool *redo) {
    const int B = pass.B, top_k = plan.top_k_max;  // the workspace's row stride (select_topk)
    const HostCounts &hc = pass.hc;
    *hc.fell = 0;
    CK(cudaMemcpyAsync(hc.cells, ws.ncells.p, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
    CK(cudaMemcpyAsync(hc.cand, ws.ncand.p, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
    CK(cudaMemcpyAsync(hc.kept, ws.nkept.p, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
    CK(cudaMemcpyAsync(hc.cnt, ws.counters.p, (size_t)(B + 4) * 8, cudaMemcpyDeviceToHost, ws.stream));
    if (pass.filt) {
        CK(cudaMemcpyAsync(hc.surv_tok, ws.ktok2.p, (size_t)B * 8, cudaMemcpyDeviceToHost, ws.stream));
        CK(cudaMemcpyAsync(hc.surv, ws.nkept2.p, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
    }
    if (pass.fast) CK(cudaMemcpyAsync(hc.recheck, ws.ncand2.p, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
    if (pass.pairs) {
        CK(cudaMemcpyAsync(hc.pairs, ws.xnpairs.p, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
        CK(cudaMemcpyAsync(hc.need, ws.needexact.p, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
    }
    if (pass.d_probe_fallback) CK(cudaMemcpyAsync(hc.fell, pass.d_probe_fallback, 4, cudaMemcpyDeviceToHost, ws.stream));
    if (!io.out_on_device) {
        size_t bytes = (size_t)B * top_k * 12 + (size_t)B * 4;
        CKS(ws.hres.ensure(bytes));
        char *h = ws.hres.as<char>();
        CK(cudaMemcpyAsync(h, pass.d_ids, (size_t)B * top_k * 8, cudaMemcpyDeviceToHost, ws.stream));
        CK(cudaMemcpyAsync(h + (size_t)B * top_k * 8, pass.d_sc, (size_t)B * top_k * 4, cudaMemcpyDeviceToHost, ws.stream));
        CK(cudaMemcpyAsync(h + (size_t)B * top_k * 12, pass.d_cn, (size_t)B * 4, cudaMemcpyDeviceToHost, ws.stream));
    }
    if (plan.prof) CK(cudaEventRecord(ws.ev[9], ws.stream));
    CK(cudaStreamSynchronize(ws.stream));
    if (pass.use_tc && *hc.fell) {  // the tensor-core pass gave up on the device: same sub-batch again on the exact path
        *redo = true;
        return PB_OK;
    }
    if (!io.out_on_device) {  // back to the queries' input positions
        const char *h = ws.hres.as<char>();
        for (int b = 0; b < B; ++b) {
            const int64_t g = pass.q[b];
            const size_t kq = (size_t)plan.qtopk[(size_t)g], os = (size_t)io.out_stride;
            memcpy(io.out_ids + (size_t)g * os, h + (size_t)b * top_k * 8, kq * 8);
            memcpy(io.out_scores + (size_t)g * os, h + (size_t)B * top_k * 8 + (size_t)b * top_k * 4, kq * 4);
            memcpy(io.out_counts + g, h + (size_t)B * top_k * 12 + (size_t)b * 4, 4);
        }
    }
    if (plan.prof) {
        for (int s = 0; s < PB_STAGE_COUNT; ++s) {
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, ws.ev[s], ws.ev[s + 1]));
            g_stats.ms[s] += ms;
        }
        for (int k = 0; k < PB_KERNEL_COUNT; ++k)
            if (g_stats.kernel_seen[k]) {
                float ms = 0.f;
                CK(cudaEventElapsedTime(&ms, ws.kev[2 * k], ws.kev[2 * k + 1]));
                g_stats.kernel_ms[k] += ms;
                g_stats.kernel_seen[k] = false;
            }
    }
    pb_work_counters &w = g_stats.work;
    if (pass.diag) {
        unsigned long long got[2] = {0, 0};
        CK(cudaMemcpy(got, ws.fdiag.p, 16, cudaMemcpyDeviceToHost));
        w.filter_err_ratio_e6 = std::max<long long>(w.filter_err_ratio_e6, (long long)got[0]);
        w.filter_diag_pairs += (long long)got[1];
    }
    if (pass.use_tc && ix->table_diag) {
        unsigned long long got = 0;
        CK(cudaMemcpy(&got, ws.tdiag.p, 8, cudaMemcpyDeviceToHost));
        w.table_diag_mismatch += (long long)got;
    }
    if (pass.fast && ix->k1_diag && ws.k1diag.p) {
        int got[2] = {0, 0};
        CK(cudaMemcpy(got, ws.k1diag.p, 8, cudaMemcpyDeviceToHost));
        w.k1_tc_max_code_diff = std::max<long long>(w.k1_tc_max_code_diff, got[0]);
    }
    w.n_queries += B;
    w.n_query_tokens += pass.R;
    if (pass.use_tc) w.n_k1_tc += 1;
    else if (pass.d_probe_fallback) (*hc.fell ? w.n_probe_list : w.n_probe_threshold) += 1;
    else if (pass.probe_list_only) w.n_probe_list += 1;
    if (pass.fast)
        for (int b = 0; b < B; ++b) w.n_recheck_docs += hc.recheck[b];
    if (pass.pairs)
        for (int b = 0; b < B; ++b) {
            if (hc.need[b]) w.n_pair_fallback_queries += 1;
            else w.n_exact_pairs += hc.pairs[b];
        }
    w.n_candidate_tokens += (long long)hc.cnt[0];
    w.n_a5_live_rows += (long long)hc.cnt[B + 2];
    w.n_a5_dense_docs += (long long)hc.cnt[B + 3];
    for (int b = 0; b < B; ++b) {
        w.n_cells += hc.cells[b];
        w.n_candidates += hc.cand[b];
        if (pass.filt) {
            w.n_filter_docs += hc.kept[b];
            w.n_filter_tokens += (long long)hc.cnt[1 + b];
            w.n_exact_docs += hc.surv[b];
            w.n_exact_tokens += hc.surv_tok[b];
        } else {
            w.n_exact_docs += hc.kept[b];
            w.n_exact_tokens += (long long)hc.cnt[1 + b];
        }
    }
    if (ix->host_tier) {  // every kept doc was staged, filter or not
        for (int b = 0; b < B; ++b) {
            g_stats.staged_docs += hc.kept[b];
            g_stats.staged_bytes += (long long)hc.cnt[1 + b] * ix->packed;
        }
        if (plan.prof) {
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, ws.sev[0], ws.sev[1]));
            g_stats.staging_ms += ms;
        }
        if (ix->cache_off.p) {  // the row cache's staging counters
            unsigned long long hits[2] = {0, 0};
            CK(cudaMemcpyAsync(hits, ws.rc_hits.p, 16, cudaMemcpyDeviceToHost, ws.stream));
            CK(cudaStreamSynchronize(ws.stream));
            long long kept = 0;
            for (int b = 0; b < B; ++b) kept += hc.kept[b];
            ix->rc.staged += kept;
            ix->rc.hit_docs += (long long)hits[0];
            ix->rc.hit_bytes += (long long)hits[1];
        }
    }
    return PB_OK;
}

// the per-stage contents of a pass into the caller's pb_trace (tests only; synchronous copies)
static pb_status dump_trace(pb_index *ix, Workspace &ws, const SearchIO &io, const SearchPlan &plan, const Pass &pass) {
    pb_trace *t = io.trace;
    const HostCounts &hc = pass.hc;
    for (int b = 0; b < pass.B; ++b) {
        const int64_t gb = pass.q[b];
        if (t->n_cells) t->n_cells[gb] = hc.cells[b];
        if (t->n_candidates) t->n_candidates[gb] = hc.cand[b];
        if (t->n_kept) t->n_kept[gb] = hc.kept[b];
        if (t->cells) {
            int n = (int)std::min<int64_t>(hc.cells[b], t->cells_cap);
            std::vector<uint32_t> tmp(n);
            CK(cudaMemcpy(tmp.data(), ws.cells.as<uint32_t>() + (size_t)b * pass.cells_cap, (size_t)n * 4,
                          cudaMemcpyDeviceToHost));
            for (int i = 0; i < n; ++i) t->cells[gb * t->cells_cap + i] = tmp[i];
        }
        if (t->candidates || t->approx) {
            int n = (int)std::min<int64_t>(hc.cand[b], t->cand_cap);
            std::vector<uint32_t> tmp(n);
            CK(cudaMemcpy(tmp.data(), ws.cand.as<uint32_t>() + (size_t)b * ix->D, (size_t)n * 4, cudaMemcpyDeviceToHost));
            if (t->candidates)
                for (int i = 0; i < n; ++i) t->candidates[gb * t->cand_cap + i] = (int64_t)tmp[i] + ix->doc_id_base;
            if (t->approx)
                CK(cudaMemcpy(t->approx + gb * t->cand_cap, ws.approx.as<float>() + (size_t)b * ix->D, (size_t)n * 4,
                              cudaMemcpyDeviceToHost));
        }
        if (t->kept || t->kept_exact) {
            int n = (int)std::min<int64_t>(hc.kept[b], t->kept_cap);
            std::vector<uint32_t> tmp(n);
            CK(cudaMemcpy(tmp.data(), ws.kept.as<uint32_t>() + (size_t)b * plan.Mcap, (size_t)n * 4, cudaMemcpyDeviceToHost));
            if (t->kept)
                for (int i = 0; i < n; ++i) t->kept[gb * t->kept_cap + i] = (int64_t)tmp[i] + ix->doc_id_base;
            if (t->kept_exact)
                CK(cudaMemcpy(t->kept_exact + gb * t->kept_cap, ws.exact.as<float>() + (size_t)b * plan.Mcap, (size_t)n * 4,
                              cudaMemcpyDeviceToHost));
        }
    }
    return PB_OK;
}

// One pass of the pipeline over a sub-batch, stage by stage, with the stage events between them.  *redo: the
// tensor-core pass gave up on the device and nothing of it went out.  `pass` is a copy, so a redo starts clean.
static pb_status run_pass(pb_index *ix, Workspace &ws, const SearchIO &io, const SearchPlan &plan, Pass pass,
                          bool *redo) {
    *redo = false;
    const auto mark = [&](int s) { return plan.prof ? cudaEventRecord(ws.ev[s], ws.stream) : cudaSuccess; };
    CK(mark(0));
    CKS(upload_queries(ix, ws, io, plan, pass));
    CK(mark(1));
    CKS(centroid_scores(ix, ws, pass));
    CK(mark(2));
    CKS(probe(ix, ws, plan, pass));
    CK(mark(3));
    CKS(candidates(ix, ws, plan, pass));
    CK(mark(4));
    CKS(approx_scores(ix, ws, plan, pass));
    CK(mark(5));
    CKS(cut(ix, ws, plan, pass));
    CK(mark(6));
    CKS(exact_scores(ix, ws, plan, pass));
    CK(mark(7));
    CKS(select_topk(ix, ws, io, plan, pass));
    CK(mark(8));
    CKS(finish(ix, ws, io, plan, pass, redo));  // D2H ends at ws.ev[9]
    if (!*redo && io.trace) CKS(dump_trace(ix, ws, io, plan, pass));
    return PB_OK;
}

// a7': whether the certified filter runs on a pass; a2 then makes the pass's 16-bit table, which the estimate reads.
// The certificate depends on the table's code error, so a tensor-core pass redone on the exact path decides again.
// It runs when some query of the pass has top_k < M; a query whose top_k reaches its kept count keeps every kept doc.
static bool filter_runs(const pb_index *ix, const SearchIO &io, const Pass &pass) {
    return ix->fast_exact && !io.trace && ix->tok_inv_norm.p && filter_eps_unit2(ix, pass.use_tc ? ix->k1_margin : 0) > 0.0f &&
           pass.nq_max <= 64 && pass.some_top_k_below_M && ix->packed % 4 == 0;
}

// One search call (or one lane of it): the plan, the workspace, then the sub-batches in order
static pb_status run_search(pb_index *ix, const SearchIO &io) {
    SearchPlan plan;
    CKS(plan_search(ix, io, plan));
    if (plan.Bt == 0) return PB_OK;

    WorkspaceLease lease{ix};
    CKS(lease.acquire());
    Workspace &ws = *lease.ws;

    if (!plan.empty) CKS(plan_probe(ix, ws, io, plan));
    // empty results: the whole call, or the queries with nothing eligible (they get no pass)
    for (int64_t b = 0; b < plan.Bt; ++b) {
        if (!plan.empty && plan.kind[(size_t)b] != PROBE_NONE) continue;
        if (io.out_on_device) CK(cudaMemsetAsync(io.out_counts + b, 0, 4, ws.stream));
        else io.out_counts[b] = 0;
        if (pb_trace *t = io.trace) {
            if (t->n_cells) t->n_cells[b] = 0;
            if (t->n_candidates) t->n_candidates[b] = 0;
            if (t->n_kept) t->n_kept[b] = 0;
        }
    }
    if (plan.empty || plan.passes.empty()) {
        CK(cudaStreamSynchronize(ws.stream));
        lease.done = true;
        return PB_OK;
    }

    if (plan.prof) CK(cudaEventRecord(ws.call_ev[0], ws.stream));
    for (const auto &pp : plan.passes) {
        Pass pass;
        pass.q = plan.order.data() + pp.first;
        pass.B = pp.second;
        for (int b = 0; b < pass.B; ++b) {
            const int64_t g = pass.q[b];
            pass.R += io.q_off[g + 1] - io.q_off[g];
            pass.nq_max = std::max(pass.nq_max, (int)(io.q_off[g + 1] - io.q_off[g]));
            pass.n = std::max(pass.n, plan.qn[(size_t)g]);
            pass.rows = pass.rows || plan.qrow[(size_t)g] >= 0;
        }
        const size_t g0 = (size_t)pass.q[0];
        pass.kind = plan.kind[g0];
        pass.batched = plan.qbatched[g0] != 0;
        pass.slab = plan.qslab[g0];
        pass.M = plan.qM[g0], pass.M1 = plan.qM1[g0], pass.top_k = plan.qtopk[g0], pass.has_thr = plan.qhas[g0];
        pass.thr = plan.qthr[g0];
        for (int b = 0; b < pass.B; ++b) {
            const size_t g = (size_t)pass.q[b];
            pass.rows = pass.rows || plan.qn[g] != pass.n;  // queries of their own n
            pass.mixed = pass.mixed || plan.qM[g] != pass.M || plan.qM1[g] != pass.M1 || plan.qtopk[g] != pass.top_k ||
                         plan.qhas[g] != pass.has_thr ||
                         (pass.has_thr && __builtin_memcmp(&plan.qthr[g], &pass.thr, 4) != 0);
            pass.some_top_k_below_M = pass.some_top_k_below_M || plan.qtopk[g] < plan.qM[g];
        }
        pass.rows = pass.rows || pass.kind != PROBE_TABLE;
        pass.QS = query_row_tokens(pass.nq_max);
        pass.fast = ix->fast_approx && !io.trace;  // trace wants every candidate's exact approx score
        pass.prune = pass.fast && ix->a5_prune && pass.QS <= 64;
        // the score table comes from the tensor cores unless something needs the dense fp32 S (an eligibility filter,
        // the radix-select probe, a trace) or the shape is outside the kernel's (DESIGN.md "a2")
        int n_chunks_k = 0;
        probe_chunk_rows(ix->K, pass.n, &n_chunks_k);
        pass.use_tc = k1_tc_usable(ix) && pass.fast && ix->probe16 && !ix->k1_diag && pass.kind == PROBE_TABLE &&
                      pass.QS / 8 <= 32 && n_chunks_k >= pass.n && pass.n <= 192;
        pass.filt = filter_runs(ix, io, pass);
        bool redo = false;
        CKS(run_pass(ix, ws, io, plan, pass, &redo));
        if (redo) {
            g_stats.work.n_k1_tc_redo += 1;
            pass.use_tc = false;
            pass.prune = false;
            pass.filt = filter_runs(ix, io, pass);
            CKS(run_pass(ix, ws, io, plan, pass, &redo));
        }
    }
    if (plan.prof) {
        CK(cudaEventRecord(ws.call_ev[1], ws.stream));
        CK(cudaEventSynchronize(ws.call_ev[1]));
        CK(cudaEventElapsedTime(&g_stats.call_ms, ws.call_ev[0], ws.call_ev[1]));
    }
    lease.done = true;
    return PB_OK;
}

static void merge_stats(Stats &a, const Stats &b) {
    for (int i = 0; i < PB_STAGE_COUNT; ++i) {
        a.ms[i] += b.ms[i];
        a.launches[i] += b.launches[i];
    }
    for (int i = 0; i < PB_KERNEL_COUNT; ++i) a.kernel_ms[i] += b.kernel_ms[i];
    a.staged_docs += b.staged_docs;
    a.staged_bytes += b.staged_bytes;
    a.staging_ms += b.staging_ms;
    const int64_t *src = reinterpret_cast<const int64_t *>(&b.work);
    int64_t *dst = reinterpret_cast<int64_t *>(&a.work);
    const size_t kdiff = offsetof(pb_work_counters, k1_tc_max_code_diff) / 8;
    const size_t kratio = offsetof(pb_work_counters, filter_err_ratio_e6) / 8;
    for (size_t i = 0; i < sizeof(pb_work_counters) / 8; ++i)
        dst[i] = (i == kdiff || i == kratio) ? std::max(dst[i], src[i]) : dst[i] + src[i];
}

// the stats of a call cut into the slices s[0 .. n) (lanes, replica slices): merged, with the longest slice's call time
static Stats merge_slices(const Stats *s, size_t n) {
    Stats total = s[0];
    for (size_t i = 1; i < n; ++i) {
        merge_stats(total, s[i]);
        total.call_ms = std::max(total.call_ms, s[i].call_ms);
    }
    return total;
}

// events of the calling thread around a laned call (the lanes' own call events live on different streams)
struct LaneClock {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[2] = {};
    int device = -1;
};
static thread_local LaneClock g_lane_clock;

static pb_status search_impl(pb_index *ix, const SearchIO &io) {
    // the lanes' helper threads run under this caller's lock (they must not take it themselves: a waiting append
    // would block them while this thread waits for them)
    std::shared_lock<std::shared_mutex> rd;
    if (ix) rd = ix->read_lock();
    g_search_agreed = false;
    // Lanes: the queries of a batch are independent, so the batch is cut into `lanes` slices searched concurrently, each
    // through the whole pipeline on its own workspace and stream (helper threads do the launching).  Not with a trace
    // (per-stage dumps), not doc-sharded (the exchanges are collective calls in batch order), not for small batches.
    int lanes = 1;
    if (ix && io.qp && ix->lanes > 1 && !io.trace && ix->comm.world == 1 && io.n_queries >= 16)
        lanes = (int)std::min<int64_t>(ix->lanes, io.n_queries / 8);
    std::unique_lock<std::mutex> lane_lock;
    if (lanes > 1) {
        lane_lock = std::unique_lock<std::mutex>(ix->lane_mu, std::try_to_lock);
        if (!lane_lock.owns_lock()) lanes = 1;  // another host thread is using the helpers: it already provides the overlap
    }
    if (lanes <= 1) {
        const pb_status st = run_search(ix, io);
        // the peers must not wait for a rank that gave up; a refusal every rank reached together leaves the group usable
        if (st != PB_OK && ix && !g_search_agreed) ix->comm.fail();
        return st;
    }
    while ((int)ix->lane_workers.size() < lanes - 1)
        ix->lane_workers.emplace_back(new RankWorker((int)ix->lane_workers.size() + 1));
    const bool prof = ix->profiling;
    LaneClock &clk = g_lane_clock;
    if (prof) {
        CK(cudaSetDevice(ix->device));
        if (clk.device != ix->device) {
            CK(cudaStreamCreateWithFlags(&clk.stream, cudaStreamNonBlocking));
            CK(cudaEventCreate(&clk.ev[0]));
            CK(cudaEventCreate(&clk.ev[1]));
            clk.device = ix->device;
        }
        CK(cudaEventRecord(clk.ev[0], clk.stream));
    }
    std::vector<Stats> stats(lanes);
    std::vector<pb_status> sts;
    std::vector<std::string> errs;
    const int64_t Bt = io.n_queries;
    run_slots(lanes, [&](int l) {
        g_budget_div = lanes;
        const pb_status st = run_search(ix, slice_io(io, Bt * l / lanes, Bt * (l + 1) / lanes));
        g_budget_div = 1;
        stats[l] = g_stats;
        return st;
    }, ix->lane_workers.data(), sts, errs);
    Stats total = merge_slices(stats.data(), lanes);
    if (prof) {
        CK(cudaEventRecord(clk.ev[1], clk.stream));
        CK(cudaEventSynchronize(clk.ev[1]));
        CK(cudaEventElapsedTime(&total.call_ms, clk.ev[0], clk.ev[1]));
    }
    g_stats = total;
    for (int l = 0; l < lanes; ++l)
        if (sts[l] != PB_OK) {
            g_err = errs[l];
            return sts[l];
        }
    return PB_OK;
}

// One batch search on any handle; each batch entry point builds its SearchIO and calls this.  `traced` names the call
// in a deployment's refusal of a trace.
// - A replica set (replicas.cpp) cuts the call into contiguous slices, each searched as slice_io on one of the
//   least-loaded replicas.  A call that the host checks of a plain handle refuse (null or non-monotone offsets, a
//   query's parameters) is not cut: it runs whole on one replica, so it is refused there, once, with the plain handle's
//   status, message and outputs.  A cut call that a slice still refuses on the device runs again whole on one
//   replica, for the plain handle's status and message.  A trace follows one call through the pipeline: never cut.
// - A deployment runs the call on every rank, rank 0 into the caller's outputs.
// - A plain handle searches it.
static pb_status search_io(pb_index *ix, const SearchIO &io, const char *traced) {
    if (Replicas *rs = pb_replicas_of(ix)) {
        auto whole = [&] {
            return ix->group->one(io.n_queries, [&](pb_index *m) { return search_io(m, io, traced); });
        };
        bool cut = !io.trace && io.n_queries > 1 && io.queries && io.q_off && io.qp;
        for (int64_t b = 0; cut && b < io.n_queries; ++b) {
            int M = 0;
            const pb_search_params &p = query_params(io, b);
            cut = io.q_off[b + 1] >= io.q_off[b] && (!io.sub_off || io.sub_off[b + 1] >= io.sub_off[b]) &&
                  check_query_args(p) == PB_OK && query_kept_docs(p, &M) == PB_OK;
        }
        if (!cut) return whole();
        std::vector<Stats> stats(PB_MAX_MEMBERS);  // a slice per replica: R may change until pb_rep_search holds the set
        size_t slices = 0;
        const pb_status st = pb_rep_search(rs, io.n_queries, [&](pb_index *m, int64_t b0, int64_t b1, int k) {
            const pb_status r = search_io(m, slice_io(io, b0, b1), traced);
            stats[k] = g_stats;
            if (b1 == io.n_queries) slices = k + 1;  // the last slice ends the call
            return r;
        });
        if (st != PB_OK) return whole();
        g_stats = merge_slices(stats.data(), slices);
        return PB_OK;
    }
    if (Deployment *d = ix && ix->group ? ix->group->as_deployment() : nullptr) {
        if (io.trace) CKS(refuse_deployment(ix, traced));
        return pb_dep_search(d, io.n_queries, io.out_stride, io.out_ids, io.out_scores, io.out_counts,
                             [&](pb_index *m, int64_t *ids, float *sc, int32_t *cn) {
                                 SearchIO rank = io;
                                 rank.out_ids = ids, rank.out_scores = sc, rank.out_counts = cn;
                                 return search_io(m, rank, traced);
                             });
    }
    // before search_impl: a refusal there leaves a deployment's group broken
    if (io.shared_sub && io.n_shared < 0) return pb_fail(PB_ERR_INVALID, "n_subset < 0");
    return search_impl(ix, io);
}

extern "C" pb_status pb_search_batch_traced(pb_index *ix, const float *queries, const int64_t *q_tok_offsets,
                                            int64_t n_queries, const pb_search_params *params, const int64_t *subset,
                                            int64_t n_subset, int64_t *out_ids, float *out_scores, int32_t *out_counts,
                                            pb_trace *trace) {
    SearchIO io{queries, false, q_tok_offsets, n_queries, subset, nullptr, nullptr, subset ? n_subset : 0,
                subset != nullptr, out_ids, out_scores, out_counts, false, trace,
                params, 0, params ? params->top_k : 0};
    return search_io(ix, io, "pb_search_batch_traced with a trace");
}

// pb_search_batch_subsets and pb_search_batch_params: params[b * params_stride] are query b's parameters
static pb_status search_subsets(pb_index *ix, const float *queries, const int64_t *q_tok_offsets, int64_t n_queries,
                                const pb_search_params *params, int64_t params_stride, const int64_t *subset_offsets,
                                const int64_t *subset_ids, const uint8_t *has_subset, int64_t *out_ids,
                                float *out_scores, int32_t *out_counts, pb_trace *trace) {
    // the subset arguments, checked whole before any slice is taken
    if (n_queries < 0) return pb_fail(PB_ERR_INVALID, "n_queries < 0");
    if (subset_offsets) {
        if (subset_offsets[0] != 0) return pb_fail(PB_ERR_INVALID, "subset_offsets[0] must be 0");
        for (int64_t b = 0; b < n_queries; ++b)
            if (subset_offsets[b + 1] < subset_offsets[b]) return pb_fail(PB_ERR_INVALID, "subset_offsets not monotone");
        if (n_queries > 0 && subset_offsets[n_queries] > 0 && !subset_ids)
            return pb_fail(PB_ERR_INVALID, "null subset_ids");
    }
    int64_t out_stride = 0;  // the call's largest top_k (negative ones are refused in plan_search)
    if (params)
        for (int64_t b = 0; b < (params_stride ? n_queries : 1); ++b)
            out_stride = std::max<int64_t>(out_stride, params[b * params_stride].top_k);
    SearchIO io{queries, false, q_tok_offsets, n_queries, subset_ids, subset_offsets, has_subset, 0, false,
                out_ids, out_scores, out_counts, false, trace, params, params_stride, out_stride};
    return search_io(ix, io, "a search with a trace");
}

extern "C" pb_status pb_search_batch_subsets(pb_index *ix, const float *queries, const int64_t *q_tok_offsets,
                                             int64_t n_queries, const pb_search_params *params,
                                             const int64_t *subset_offsets, const int64_t *subset_ids,
                                             const uint8_t *has_subset, int64_t *out_ids, float *out_scores,
                                             int32_t *out_counts, pb_trace *trace) {
    return search_subsets(ix, queries, q_tok_offsets, n_queries, params, 0, subset_offsets, subset_ids, has_subset,
                          out_ids, out_scores, out_counts, trace);
}

extern "C" pb_status pb_search_batch_params(pb_index *ix, const float *queries, const int64_t *q_tok_offsets,
                                            int64_t n_queries, const pb_search_params *params,
                                            const int64_t *subset_offsets, const int64_t *subset_ids,
                                            const uint8_t *has_subset, int64_t *out_ids, float *out_scores,
                                            int32_t *out_counts, pb_trace *trace) {
    if (!params) return pb_fail(PB_ERR_INVALID, "null params");
    return search_subsets(ix, queries, q_tok_offsets, n_queries, params, 1, subset_offsets, subset_ids, has_subset,
                          out_ids, out_scores, out_counts, trace);
}

// ---- pb_search: one query per call, merged with the other callers' when coalescing is on (DESIGN.md 4m) ----
struct SearchRequest : pbq::Request {
    const float *query;
    int64_t n_tokens;
    const pb_search_params *params;
    const int64_t *subset;  // null = None
    int64_t n_subset;
    int64_t *out_ids;
    float *out_scores;
    int32_t *out_count;
    Stats stats;  // of the call the request was answered by; installed in the caller's thread-local slot
};

// a request as a batch of one, straight into its own outputs
static pb_status search_alone(pb_index *ix, const SearchRequest &r) {
    const int64_t q_off[2] = {0, r.n_tokens}, sub_off[2] = {0, r.subset ? r.n_subset : 0};
    const uint8_t has = r.subset ? 1 : 0;
    return pb_search_batch_params(ix, r.query, q_off, 1, r.params, r.subset ? sub_off : nullptr, r.subset, &has,
                                  r.out_ids, r.out_scores, r.out_count, nullptr);
}

// What pb_search_batch_params of the request alone would refuse, as far as the host can tell, on a handle of D
// documents with ix's K (the caller holds ix's read lock: K decides the variant).  Not covered: a dense-variant query
// with a subset, whose effective n_ivf_probe follows from its eligible centroids, counted on the device; such a request
// can still fail its merged call, which then re-runs its members alone.
static pb_status check_request(const pb_index *ix, long long D, const SearchRequest &r) {
    if (!r.params) return pb_fail(PB_ERR_INVALID, "null params");
    if (r.subset && r.n_subset < 0) return pb_fail(PB_ERR_INVALID, "subset_offsets not monotone");
    if (!r.query) return pb_fail(PB_ERR_INVALID, "null queries");
    const pb_search_params &p = *r.params;
    CKS(check_query_args(p));
    if (p.top_k > 0 && (!r.out_ids || !r.out_scores)) return pb_fail(PB_ERR_INVALID, "null outputs");
    if (!r.out_count) return pb_fail(PB_ERR_INVALID, "null out_counts");
    if (r.n_tokens < 0) return pb_fail(PB_ERR_INVALID, "q_tok_offsets not monotone");
    int M = 0;
    CKS(query_kept_docs(p, &M));
    if (M == 0 || p.top_k == 0 || D == 0) return PB_OK;  // an empty result, no pass
    const bool batched = query_batched(ix, p);
    if (batched) CKS(check_batched_probe(ix, p));
    const int n = (int)std::min<long long>(p.n_ivf_probe, ix->K);
    const uint8_t kind = (!batched && r.subset) ? PROBE_ALL : n > (batched ? 192 : 64) ? PROBE_BIG : PROBE_TABLE;
    return check_query_rows(ix, kind, n, (int)r.n_tokens);
}

int CoalescedRun::operator()(pbq::Request *const *reqs, size_t n, std::string &err) const {
    if (pb_replicas_of(ix)) {  // a replica set: the merged batch goes whole to the least-loaded replica
        int r = 0;
        ix->group->one((int64_t)n, [&](pb_index *m) { return (pb_status)(r = CoalescedRun{m}(reqs, n, err)); });
        return r;
    }
    pb_status st;
    if (n == 1) st = search_alone(ix, *static_cast<SearchRequest *>(reqs[0]));
    else {
        std::unique_ptr<GatherBuf> gb;
        {
            std::lock_guard<std::mutex> g(ix->mu);
            if (!ix->gather_pool.empty()) {
                gb = std::move(ix->gather_pool.back());
                ix->gather_pool.pop_back();
            }
        }
        if (!gb) gb.reset(new GatherBuf());
        GatherBuf &g = *gb;
        g.queries.clear(), g.q_off.assign(1, 0), g.sub_off.assign(1, 0), g.sub_ids.clear(), g.params.clear(), g.has_sub.clear();
        int64_t top_k = 0;
        bool any_subset = false;
        for (size_t i = 0; i < n; ++i) {
            const SearchRequest &r = *static_cast<SearchRequest *>(reqs[i]);
            g.queries.insert(g.queries.end(), r.query, r.query + (size_t)r.n_tokens * ix->dim);
            g.q_off.push_back(g.q_off.back() + r.n_tokens);
            if (r.subset) g.sub_ids.insert(g.sub_ids.end(), r.subset, r.subset + r.n_subset);
            g.sub_off.push_back((int64_t)g.sub_ids.size());
            g.has_sub.push_back(r.subset ? 1 : 0);
            any_subset = any_subset || r.subset;
            g.params.push_back(*r.params);
            top_k = std::max(top_k, r.params->top_k);
        }
        g.ids.resize(n * (size_t)top_k), g.scores.resize(n * (size_t)top_k), g.counts.resize(n);
        if (g.queries.empty()) g.queries.push_back(0.f);  // every query has no tokens: the pointer must not be null
        st = pb_search_batch_params(ix, g.queries.data(), g.q_off.data(), (int64_t)n, g.params.data(),
                                    any_subset ? g.sub_off.data() : nullptr, g.sub_ids.data(), g.has_sub.data(),
                                    g.ids.data(), g.scores.data(), g.counts.data(), nullptr);
        if (st == PB_OK)
            for (size_t i = 0; i < n; ++i) {
                const SearchRequest &r = *static_cast<SearchRequest *>(reqs[i]);
                const size_t c = (size_t)g.counts[i];
                *r.out_count = g.counts[i];
                if (c) {
                    memcpy(r.out_ids, g.ids.data() + i * (size_t)top_k, c * 8);
                    memcpy(r.out_scores, g.scores.data() + i * (size_t)top_k, c * 4);
                }
            }
        std::lock_guard<std::mutex> lk(ix->mu);
        ix->gather_pool.push_back(std::move(gb));
    }
    if (st != PB_OK) err = g_err;
    for (size_t i = 0; i < n; ++i) static_cast<SearchRequest *>(reqs[i])->stats = g_stats;
    return (int)st;
}

extern "C" pb_status pb_search(pb_index *ix, const float *query, int64_t n_query_tokens, const pb_search_params *params,
                               const int64_t *subset, int64_t n_subset, int64_t *out_ids, float *out_scores,
                               int32_t *out_count) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    SearchRequest r;
    r.query = query, r.n_tokens = n_query_tokens, r.params = params, r.subset = subset, r.n_subset = n_subset;
    r.out_ids = out_ids, r.out_scores = out_scores, r.out_count = out_count;
    // a doc-sharded search is a collective, issued in the same order on every rank: never queued
    if (!ix->coalesce_on || ix->comm.joined()) {
        ix->coalescer.count_bypassed();
        return search_alone(ix, r);
    }
    pb_status st;
    if (ix->group) {  // as one handle of the whole index: every rank's K, the deployment's D (rank 0 may be empty)
        const long long D = pb_index_num_documents(ix);
        auto check = [&](pb_index *h) {
            auto rd = h->read_lock();
            return check_request(h, D, r);
        };
        // a deployment's rank 0; a replica set's replica 0, or its rank 0
        st = ix->group->first([&](pb_index *m) { return m->group ? m->group->first(check) : check(m); });
    } else {
        auto rd = ix->read_lock();
        st = check_request(ix, ix->D, r);
    }
    if (st != PB_OK) {
        ix->coalescer.count_refused();
        return st;
    }
    ix->coalescer.submit(r);
    g_stats = r.stats;
    if (r.status != 0) g_err = r.error;
    return (pb_status)r.status;
}

extern "C" pb_status pb_search_batch(pb_index *ix, const float *queries, const int64_t *q_tok_offsets, int64_t n_queries,
                                     const pb_search_params *params, const int64_t *subset, int64_t n_subset,
                                     int64_t *out_ids, float *out_scores, int32_t *out_counts) {
    return pb_search_batch_traced(ix, queries, q_tok_offsets, n_queries, params, subset, n_subset, out_ids, out_scores,
                                  out_counts, nullptr);
}

extern "C" pb_status pb_search_batch_device(pb_index *ix, const float *d_queries, const int64_t *q_tok_offsets_host,
                                            int64_t n_queries, const pb_search_params *params, int64_t *d_out_ids,
                                            float *d_out_scores, int32_t *d_out_counts) {
    CKS(refuse_deployment(ix, "pb_search_batch_device"));  // its pointers belong to one device
    SearchIO io{d_queries, true, q_tok_offsets_host, n_queries, nullptr, nullptr, nullptr, 0, false,
                d_out_ids, d_out_scores, d_out_counts, true, nullptr, params, 0, params ? params->top_k : 0};
    return search_impl(ix, io);
}

// ------------------------------------------------------------------------------------------
// stage entry points
// ------------------------------------------------------------------------------------------
extern "C" pb_status pb_centroid_scores(pb_index *ix, const float *query_tokens, int64_t n, float *out) {
    if (ix && ix->group)  // the centroids are replicated: a deployment's rank 0, a replica
        return ix->group->one(0, [&](pb_index *m) { return pb_centroid_scores(m, query_tokens, n, out); });
    if (!ix || (!query_tokens && n) || (!out && n)) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n == 0) return PB_OK;
    auto rd = ix->read_lock();
    CK(cudaSetDevice(ix->device));
    WorkspaceLease lease{ix};
    CKS(lease.acquire());
    Workspace &ws = *lease.ws;
    // one pseudo-query per block of <= 64 tokens keeps the per-query transposed layout small
    const int blk = 64;
    DevBuf S;
    CKS(S.ensure((size_t)blk * ix->K * 4));
    for (int64_t r0 = 0; r0 < n; r0 += blk) {
        int nq = (int)std::min<int64_t>(blk, n - r0);
        int QS = std::max(8, (nq + 7) & ~7);
        CKS(ws.Q.ensure((size_t)nq * ix->dim * 4));
        CKS(ws.qoff.ensure(8));
        int qoff[2] = {0, nq};
        CK(cudaMemcpyAsync(ws.Q.p, query_tokens + (size_t)r0 * ix->dim, (size_t)nq * ix->dim * 4, cudaMemcpyHostToDevice, ws.stream));
        CK(cudaMemcpyAsync(ws.qoff.p, qoff, 8, cudaMemcpyHostToDevice, ws.stream));
        CKS(ws.ST.ensure((size_t)ix->K * QS * 4));
        CKS(launch_centroid_scores(ix, ws, 1, QS, nullptr));
        k_transpose_scores<<<(unsigned)((ix->K + 255) / 256), 256, 0, ws.stream>>>(ws.ST.as<float>(), ix->K, QS, nq, S.as<float>());
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(out + (size_t)r0 * ix->K, S.p, (size_t)nq * ix->K * 4, cudaMemcpyDeviceToHost, ws.stream));
        CK(cudaStreamSynchronize(ws.stream));
    }
    lease.done = true;
    return PB_OK;
}

extern "C" pb_status pb_decompress_documents(pb_index *ix, const int64_t *doc_ids, int64_t n_docs, float *out_embeddings,
                                             int64_t *out_lengths) {
    if (ix && ix->group) return ix->group->decompress(doc_ids, n_docs, out_embeddings, out_lengths);
    if (!ix || (!doc_ids && n_docs) || !out_lengths) return pb_fail(PB_ERR_INVALID, "null argument");
    auto rd = ix->read_lock();
    CK(cudaSetDevice(ix->device));
    if (n_docs == 0) return PB_OK;
    std::vector<long long> doff((size_t)ix->D + 1);
    CK(cudaMemcpy(doff.data(), ix->doc_off.p, doff.size() * 8, cudaMemcpyDeviceToHost));
    std::vector<uint32_t> docs;
    std::vector<long long> prefix(1, 0);
    for (int64_t i = 0; i < n_docs; ++i) {
        int64_t d = doc_ids[i] - ix->doc_id_base;
        if (d < 0 || d >= ix->D) {  // index.rs:1202-1204: unknown id -> length 0
            out_lengths[i] = 0;
            continue;
        }
        out_lengths[i] = doff[d + 1] - doff[d];
        docs.push_back((uint32_t)d);
        prefix.push_back(prefix.back() + out_lengths[i]);
    }
    if (!out_embeddings || docs.empty() || prefix.back() == 0) return PB_OK;
    const long long total = prefix.back();
    DevBuf ddocs, dpre, dout, ident;
    CKS(upload(ddocs, docs.data(), docs.size() * 4, PB_MEM_HOST));
    CKS(upload(dpre, prefix.data(), prefix.size() * 8, PB_MEM_HOST));
    const long long chunk_tok = 1ll << 22;  // bound the staging buffer (2 GiB at dim 128)
    CKS(dout.ensure((size_t)std::min(total, chunk_tok + ix->max_doclen) * ix->dim * 4));
    // host tier: each range's docs are staged first (slot j = its j-th doc, at the range-local prefix), then decompressed
    // from the staged rows with the identity as doc list
    WorkspaceLease lease{ix};
    if (ix->host_tier) {
        CKS(lease.acquire());
        CKS(ident.ensure(docs.size() * 4 + 16));
        k_fill_identity<<<64, 256, 0, lease.ws->stream>>>(ident.as<uint32_t>(), (long long)docs.size(), 0u);
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(lease.ws->stream));
    }
    // process doc ranges whose token count fits the staging buffer
    size_t i0 = 0;
    while (i0 < docs.size()) {
        size_t i1 = i0;
        while (i1 < docs.size() && prefix[i1] - prefix[i0] < chunk_tok) ++i1;  // <= chunk_tok + max_doclen tokens
        const int nd = (int)(i1 - i0);
        const long long ntok = prefix[i1] - prefix[i0];
        std::vector<long long> local(nd + 1);
        for (int j = 0; j <= nd; ++j) local[j] = prefix[i0 + j] - prefix[i0];
        CK(cudaMemcpy(dpre.p, local.data(), local.size() * 8, cudaMemcpyHostToDevice));
        int blocks = (int)std::max<long long>(1, std::min<long long>((ntok + 7) / 8, (long long)ix->sm_count * 8));
        TokView tv = resident_tokens(ix);
        const uint32_t *list = ddocs.as<uint32_t>() + i0;
        if (ix->host_tier) {
            CKS(stage_rows(ix, *lease.ws, list, nullptr, nd, nd, dpre.as<long long>(), ntok, false, tv));
            CK(cudaStreamSynchronize(lease.ws->stream));
            list = ident.as<uint32_t>();
        }
        PB_DIM_SWITCH(ix->dim, {
            k_decompress<DIM><<<blocks, 256>>>(ix->centroids.as<float>(), ix->w_rev.as<float>(), ix->nbits,
                                               tv.codes, tv.residuals, tv.doc_off, list, dpre.as<long long>(),
                                               nd, dout.as<float>());
        });
        CK(cudaGetLastError());
        CK(cudaMemcpy(out_embeddings + (size_t)prefix[i0] * ix->dim, dout.p, (size_t)ntok * ix->dim * 4, cudaMemcpyDeviceToHost));
        i0 = i1;
    }
    lease.done = true;
    return PB_OK;
}

extern "C" pb_status pb_maxsim_scores(int32_t device, const float *query, int32_t nq, int32_t dim, const float *doc_tokens,
                                      const int64_t *doc_tok_offsets, int64_t n_docs, float *out_scores) {
    if ((!query && nq) || (!doc_tok_offsets) || (!out_scores && n_docs)) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(BuiltDims::check(dim));
    if (nq < 0 || n_docs < 0) return pb_fail(PB_ERR_INVALID, "negative size");
    CKS(check_device(device));
    if (n_docs == 0) return PB_OK;
    if (n_docs > (1 << 30)) return pb_fail(PB_ERR_UNSUPPORTED, "too many documents in one call");
    const long long total = doc_tok_offsets[n_docs] - doc_tok_offsets[0];
    const int QS = std::max(8, (nq + 7) & ~7);
    const int Mcap = (int)n_docs;
    DevBuf dQ, dqoff, dtok, dkept, dnk, dtp, dmax, dex;
    dmax.zero_on_grow = true;
    int qoff[2] = {0, nq};
    std::vector<long long> tp(n_docs + 1);
    for (int64_t i = 0; i <= n_docs; ++i) tp[i] = doc_tok_offsets[i] - doc_tok_offsets[0];
    CKS(upload(dQ, query, (size_t)nq * dim * 4, PB_MEM_HOST));
    CKS(upload(dqoff, qoff, 8, PB_MEM_HOST));
    CKS(upload(dtok, doc_tokens + (size_t)doc_tok_offsets[0] * dim, (size_t)total * dim * 4, PB_MEM_HOST));
    CKS(upload(dtp, tp.data(), tp.size() * 8, PB_MEM_HOST));
    CKS(upload(dnk, &Mcap, 4, PB_MEM_HOST));
    CKS(dkept.ensure((size_t)Mcap * 4));
    CKS(dmax.ensure((size_t)Mcap * QS * 4));
    CKS(dex.ensure((size_t)Mcap * 4));
    long long chunks = (total + PB_TOK_TILE - 1) / PB_TOK_TILE;
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    int gx = (int)std::max<long long>(1, std::min<long long>(chunks, (long long)sms * 16));
    PB_DIM_SWITCH(dim, {
        auto kern = k_exact<DIM, true>;
        CKS(set_smem(kern, smem_exact(DIM, 0)));
        kern<<<dim3(gx, 1), 128, smem_exact(DIM, 0)>>>(dQ.as<float>(), dqoff.as<int>(), QS, nullptr, nullptr, 8, nullptr,
                                                       nullptr, nullptr, dtok.as<float>(), dkept.as<uint32_t>(), dnk.as<int>(),
                                                       dtp.as<long long>(), Mcap, 0, dmax.as<uint32_t>(), nullptr);
    });
    CK(cudaGetLastError());
    k_exact_finalize<<<dim3((Mcap + 7) / 8, 1), 256>>>(dmax.as<uint32_t>(), dqoff.as<int>(), QS, dnk.as<int>(), Mcap, 0,
                                                      dex.as<float>(), nullptr, nullptr, nullptr, 0u, nullptr);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out_scores, dex.p, (size_t)Mcap * 4, cudaMemcpyDeviceToHost));
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// pool_document_embeddings (next-plaid-onnx lib.rs:1632, DESIGN §4p)
// ------------------------------------------------------------------------------------------
// pool_embeddings_hierarchical's length rule (lib.rs:1636-1641, :2257-2266) with protected_tokens = 1
extern "C" int64_t pb_pooled_doc_length(int64_t n_tokens, int64_t pool_factor) {
    if (n_tokens < 0 || pool_factor < 0) return -1;
    if (pool_factor <= 1 || n_tokens <= 2) return n_tokens;
    const int64_t t = n_tokens - 1, k = std::max<int64_t>(t / pool_factor, 1);
    return k >= t ? n_tokens : 1 + k;
}

static thread_local float g_pool_ms[3];
extern "C" pb_status pb_last_pool_ms(float *out_ms) {
    if (!out_ms) return pb_fail(PB_ERR_INVALID, "null argument");
    memcpy(out_ms, g_pool_ms, sizeof g_pool_ms);
    return PB_OK;
}

// d^2 workspace of one wave of documents (a document that needs more runs alone)
static constexpr size_t POOL_WAVE_BYTES = size_t(1) << 30;

extern "C" pb_status pb_pool_embeddings(int32_t device, const float *embeddings, const int64_t *doc_lengths,
                                        int64_t n_docs, int32_t dim, int64_t pool_factor, int32_t memory_space,
                                        float *out_embeddings, int64_t *out_doc_lengths) {
    if (n_docs < 0 || pool_factor < 0) return pb_fail(PB_ERR_INVALID, "negative n_docs or pool_factor");
    if (n_docs > INT_MAX) return pb_fail(PB_ERR_UNSUPPORTED, "more than %d documents in one call", INT_MAX);
    if (n_docs && (!doc_lengths || !out_doc_lengths)) return pb_fail(PB_ERR_INVALID, "null argument");
    if (memory_space != PB_MEM_HOST && memory_space != PB_MEM_DEVICE)
        return pb_fail(PB_ERR_INVALID, "memory_space %d is neither PB_MEM_HOST nor PB_MEM_DEVICE", memory_space);
    CKS(BuiltDims::check(dim));
    std::vector<PoolDoc> docs(n_docs);
    long long total = 0, total_out = 0;
    for (int64_t i = 0; i < n_docs; ++i) {
        const int64_t n = doc_lengths[i];
        if (n < 0) return pb_fail(PB_ERR_INVALID, "doc_lengths[%lld] = %lld is negative", (long long)i, (long long)n);
        const int64_t o = pb_pooled_doc_length(n, pool_factor);
        const int k = o < n ? (int)(o - 1) : 0;
        if (n > INT_MAX || (k && n - 1 > PB_POOL_MAX_T))
            return pb_fail(PB_ERR_UNSUPPORTED, "document %lld has %lld tokens; pooling clusters at most %d", (long long)i,
                           (long long)n, PB_POOL_MAX_T);
        docs[i] = PoolDoc{total, total_out, 0, 0, (int)n, k};
        total += n;
        total_out += o;
    }
    if ((total && !embeddings) || (total_out && !out_embeddings)) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(check_device(device));
    memset(g_pool_ms, 0, sizeof g_pool_ms);
    // waves: consecutive documents whose d^2 matrices fit POOL_WAVE_BYTES; per wave the pooled documents and the
    // (doc, I, J) tiles of k_pool_dist
    struct Wave {
        int d0, d1;
        size_t p0, p1, i0, i1;
        int max_t, max_means_smem;
    };
    std::vector<Wave> waves;
    std::vector<int> pooled;
    std::vector<int4> items;
    size_t ws_max = 0, par_max = 0;
    for (int64_t i = 0; i < n_docs;) {
        Wave w{(int)i, (int)i, pooled.size(), 0, items.size(), 0, 0, 0};
        size_t ws = 0, par = 0;
        for (; i < n_docs; ++i) {
            PoolDoc &d = docs[i];
            const size_t t = d.n - 1, need = d.k ? t * t : 0;
            if (w.d1 > w.d0 && (ws + need) * sizeof(double) > POOL_WAVE_BYTES) break;
            if (d.k) {
                d.ws_off = (long long)ws;
                d.par_off = (long long)par;
                ws += need;
                par += t;
                pooled.push_back((int)i);
                const int nb = (int)((t + PB_POOL_TILE - 1) / PB_POOL_TILE);
                for (int I = 0; I < nb; ++I)
                    for (int J = I; J < nb; ++J) items.push_back(make_int4((int)i, I, J, 0));
                w.max_t = std::max(w.max_t, (int)t);
                w.max_means_smem = std::max(w.max_means_smem, (int)(4 * t + 2 * d.k) * 4);
            }
            w.d1 = (int)i + 1;
        }
        w.p1 = pooled.size();
        w.i1 = items.size();
        ws_max = std::max(ws_max, ws);
        par_max = std::max(par_max, par);
        waves.push_back(w);
    }

    OwnedStream st;
    CK(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
    DevBuf din, dout, ddocs, dpooled, ditems, dws, dpar, derr;
    const size_t in_bytes = (size_t)total * dim * 4, out_bytes = (size_t)total_out * dim * 4;
    const float *x = embeddings;
    float *y = out_embeddings;
    if (memory_space == PB_MEM_HOST) {
        CKS(din.ensure(std::max<size_t>(in_bytes, 16)));
        CKS(dout.ensure(std::max<size_t>(out_bytes, 16)));
        if (in_bytes) CK(cudaMemcpyAsync(din.p, embeddings, in_bytes, cudaMemcpyHostToDevice, st.s));
        x = din.as<float>();
        y = dout.as<float>();
    }
    CKS(derr.ensure(16));
    CK(cudaMemsetAsync(derr.p, 0, 4, st.s));
    int sms = 0, err = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    if (total) {
        const long long nv = total * dim;
        k_pool_finite<<<(int)std::min<long long>((nv + 255) / 256, (long long)sms * 8), 256, 0, st.s>>>(x, nv, derr.as<int>());
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(&err, derr.p, 4, cudaMemcpyDeviceToHost, st.s));
    CK(cudaStreamSynchronize(st.s));
    if (err & 1) return pb_fail(PB_ERR_INVALID, "the embeddings hold a value that is not finite");

    CKS(ddocs.ensure(std::max<size_t>(docs.size() * sizeof(PoolDoc), 16)));
    CKS(dpooled.ensure(std::max<size_t>(pooled.size() * 4, 16)));
    CKS(ditems.ensure(std::max<size_t>(items.size() * sizeof(int4), 16)));
    CKS(dws.ensure(std::max<size_t>(ws_max * sizeof(double), 16)));
    CKS(dpar.ensure(std::max<size_t>(par_max * 4, 16)));
    if (n_docs) CK(cudaMemcpyAsync(ddocs.p, docs.data(), docs.size() * sizeof(PoolDoc), cudaMemcpyHostToDevice, st.s));
    if (!pooled.empty()) CK(cudaMemcpyAsync(dpooled.p, pooled.data(), pooled.size() * 4, cudaMemcpyHostToDevice, st.s));
    if (!items.empty())
        CK(cudaMemcpyAsync(ditems.p, items.data(), items.size() * sizeof(int4), cudaMemcpyHostToDevice, st.s));
    struct Events {
        cudaEvent_t e[4] = {};
        ~Events() {
            for (cudaEvent_t v : e)
                if (v) cudaEventDestroy(v);
        }
    } ev;
    for (cudaEvent_t &v : ev.e) CK(cudaEventCreate(&v));
    for (const Wave &w : waves) {
        const int np = (int)(w.p1 - w.p0), ni = (int)(w.i1 - w.i0);
        CK(cudaEventRecord(ev.e[0], st.s));
        if (ni) {
            PB_DIM_SWITCH(dim, {
                k_pool_dist<DIM><<<ni, 256, 0, st.s>>>(x, ddocs.as<PoolDoc>(), ditems.as<int4>() + w.i0, dws.as<double>());
            });
            CK(cudaGetLastError());
        }
        CK(cudaEventRecord(ev.e[1], st.s));
        if (np) {
            const size_t smem = (size_t)w.max_t * 24;
            CKS(set_smem(k_pool_chain, smem));
            k_pool_chain<<<np, 32, smem, st.s>>>(ddocs.as<PoolDoc>(), dpooled.as<int>() + w.p0, dws.as<double>(),
                                                 dpar.as<int>(), derr.as<int>());
            CK(cudaGetLastError());
        }
        CK(cudaEventRecord(ev.e[2], st.s));
        PB_DIM_SWITCH(dim, {
            auto kern = k_pool_means<DIM>;
            CKS(set_smem(kern, w.max_means_smem));
            kern<<<w.d1 - w.d0, 256, w.max_means_smem, st.s>>>(x, ddocs.as<PoolDoc>(), w.d0, dpar.as<int>(), y,
                                                              derr.as<int>());
        });
        CK(cudaGetLastError());
        CK(cudaEventRecord(ev.e[3], st.s));
        CK(cudaEventSynchronize(ev.e[3]));
        for (int p = 0; p < 3; ++p) {
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, ev.e[p], ev.e[p + 1]));
            g_pool_ms[p] += ms;
        }
    }
    CK(cudaMemcpyAsync(&err, derr.p, 4, cudaMemcpyDeviceToHost, st.s));
    CK(cudaStreamSynchronize(st.s));
    if (err & 2)
        return pb_fail(PB_ERR_UNSUPPORTED, "a nearest-neighbour chain revisited a cluster (the reference does not terminate)");
    if (err) return pb_fail(PB_ERR_CUDA, "pooling cut did not give the expected number of clusters (error bits %d)", err);
    if (memory_space == PB_MEM_HOST && out_bytes) {
        CK(cudaMemcpyAsync(out_embeddings, dout.p, out_bytes, cudaMemcpyDeviceToHost, st.s));
        CK(cudaStreamSynchronize(st.s));
    }
    for (int64_t i = 0; i < n_docs; ++i) out_doc_lengths[i] = pb_pooled_doc_length(doc_lengths[i], pool_factor);
    return PB_OK;
}

extern "C" pb_status pb_exhaustive_scores(pb_index *ix, const float *queries, const int64_t *q_off, int64_t n_queries,
                                          float *out_scores) {
    if (ix && ix->group) return ix->group->exhaustive(queries, q_off, n_queries, out_scores);
    if (!ix || (!queries && n_queries) || !q_off || (!out_scores && n_queries)) return pb_fail(PB_ERR_INVALID, "null argument");
    auto rd = ix->read_lock();
    CK(cudaSetDevice(ix->device));
    if (n_queries == 0 || ix->D == 0) return PB_OK;
    WorkspaceLease lease{ix};
    CKS(lease.acquire());
    Workspace &ws = *lease.ws;
    std::vector<long long> doff((size_t)ix->D + 1);
    CK(cudaMemcpy(doff.data(), ix->doc_off.p, doff.size() * 8, cudaMemcpyDeviceToHost));
    const int QBmax = 32;
    const int Mblk = 1 << 16;
    for (int64_t b0 = 0; b0 < n_queries; b0 += QBmax) {
        const int B = (int)std::min<int64_t>(QBmax, n_queries - b0);
        const int64_t r0 = q_off[b0], R = q_off[b0 + B] - r0;
        std::vector<int> qoff(B + 1);
        int nq_max = 0;
        for (int b = 0; b <= B; ++b) qoff[b] = (int)(q_off[b0 + b] - r0);
        for (int b = 0; b < B; ++b) nq_max = std::max(nq_max, qoff[b + 1] - qoff[b]);
        const int QS = std::max(8, (nq_max + 7) & ~7);
        CKS(ws.Q.ensure(std::max<size_t>((size_t)R * ix->dim * 4, 16)));
        CKS(ws.qoff.ensure((size_t)(B + 1) * 4));
        if (R) CK(cudaMemcpyAsync(ws.Q.p, queries + (size_t)r0 * ix->dim, (size_t)R * ix->dim * 4, cudaMemcpyHostToDevice, ws.stream));
        CK(cudaMemcpyAsync(ws.qoff.p, qoff.data(), (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, ws.stream));
        CK(cudaStreamSynchronize(ws.stream));
        CKS(ws.kept.ensure((size_t)Mblk * 4));
        CKS(ws.nkept.ensure(16));
        CKS(ws.tokp.ensure((size_t)(Mblk + 1) * 8));
        CKS(ws.maxkey.ensure((size_t)B * Mblk * QS * 4));
        CKS(ws.exact.ensure((size_t)B * Mblk * 4));
        // maxkey layout changes with QS/Mcap: rows are reset by finalize, but only those < n_kept
        for (long long d0 = 0, nd = 0; d0 < ix->D; d0 += nd) {
            nd = std::min<long long>(Mblk, ix->D - d0);
            // host tier: a window of at most 2^22 tokens (or one doc) is one H2D copy into the staging buffer, scored with
            // window-local ids and offsets (the window's token prefix is its doc_off)
            if (ix->host_tier) {
                const long long win = std::max(1ll << 22, (long long)ix->max_doclen);
                nd = std::upper_bound(doff.begin() + d0 + 1, doff.begin() + d0 + nd + 1, doff[d0] + win) - doff.begin() - 1 - d0;
            }
            const long long ntok = doff[d0 + nd] - doff[d0];
            k_fill_identity<<<64, 256, 0, ws.stream>>>(ws.kept.as<uint32_t>(), nd, ix->host_tier ? 0u : (uint32_t)d0);
            k_range_prefix<<<64, 256, 0, ws.stream>>>(ix->doc_off.as<long long>(), d0, (int)nd, ws.tokp.as<long long>());
            const int nd32 = (int)nd;
            CK(cudaMemcpyAsync(ws.nkept.p, &nd32, 4, cudaMemcpyHostToDevice, ws.stream));
            const KeptView kv{ws.kept.as<uint32_t>(), ws.nkept.as<int>(), ws.tokp.as<long long>(), nullptr};
            TokView tv = resident_tokens(ix);
            if (ix->host_tier) {
                CKS(ws.s_res.ensure((size_t)std::max(ntok, 1ll) * ix->packed));
                CKS(ix->host.rows->to_device((size_t)doff[d0] * ix->packed, ws.s_res.as<uint8_t>(), (size_t)ntok * ix->packed,
                                             ws.stream));
                tv = {ix->codes.as<uint32_t>() + doff[d0], ws.s_res.as<uint8_t>(), nullptr, ws.tokp.as<long long>()};
            }
            CKS(launch_exact(ix, ws, kv, tv, B, QS, Mblk, 1, ntok, nullptr));
            k_exact_finalize<<<dim3((Mblk + 7) / 8, B), 256, 0, ws.stream>>>(ws.maxkey.as<uint32_t>(), ws.qoff.as<int>(), QS,
                                                                           ws.nkept.as<int>(), Mblk, 1, ws.exact.as<float>(),
                                                                           nullptr, nullptr, nullptr, 0u, nullptr);
            CK(cudaGetLastError());
            for (int b = 0; b < B; ++b)
                CK(cudaMemcpyAsync(out_scores + (size_t)(b0 + b) * ix->D + d0, ws.exact.as<float>() + (size_t)b * Mblk,
                                   (size_t)nd * 4, cudaMemcpyDeviceToHost, ws.stream));
            CK(cudaStreamSynchronize(ws.stream));
        }
    }
    lease.done = true;
    return PB_OK;
}


// ------------------------------------------------------------------------------------------
// doc-sharded deployment: one process per GPU, NCCL all-gathers of the per-shard top lists.
// The host passes the 128-byte NCCL unique id between ranks however it likes (torch.distributed,
// MPI, a file); nothing else crosses the C-ABI.
// ------------------------------------------------------------------------------------------
extern "C" pb_status pb_comm_unique_id(uint8_t *out128) {
    if (!out128) return pb_fail(PB_ERR_INVALID, "null argument");
    if (!g_nccl.load()) return pb_fail(PB_ERR_COMM, "libnccl.so.2 not found (%s)", dlerror());
    ncclUniqueId id;
    CKN(g_nccl.GetUniqueId(&id));
    memcpy(out128, id.internal, 128);
    return PB_OK;
}

extern "C" pb_status pb_index_comm_init(pb_index *ix, const uint8_t *id128, int32_t rank, int32_t world) {
    if (!ix || !id128) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_deployment(ix, "pb_index_comm_init"));
    CKS(ix->comm.init_nccl(id128, rank, world, ix->device));
    // a sharded search is a collective: arrival order is not a rank-agreed order
    if (ix->comm.joined()) pb_index_set_coalescing(ix, nullptr);
    return PB_OK;
}

// In-process alternative to NCCL: one handle per shard, one host thread per handle (any devices, peer copies)
extern "C" pb_status pb_shard_group_create(int32_t world, pb_shard_group **out) {
    if (!out || world < 1 || world > 64) return pb_fail(PB_ERR_INVALID, "shard group: world must be in [1, 64]");
    pb_shard_group *g = new pb_shard_group();
    g->world = world;
    g->table.assign((size_t)world, nullptr);
    g->dev.assign((size_t)world, 0);
    *out = g;
    return PB_OK;
}
extern "C" void pb_shard_group_destroy(pb_shard_group *g) { delete g; }
extern "C" pb_status pb_index_group_join(pb_index *ix, pb_shard_group *g, int32_t rank) {
    if (!ix || !g) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_deployment(ix, "pb_index_group_join"));
    CKS(ix->comm.join(g, rank, ix->device));
    pb_index_set_coalescing(ix, nullptr);  // as pb_index_comm_init
    return PB_OK;
}
pb_status pb_index_group_move(pb_index *ix, pb_shard_group *g, int rank) {
    ix->comm.leave();
    return pb_index_group_join(ix, g, rank);
}

// ------------------------------------------------------------------------------------------
// index-build path (SURVEY 8 a12, secondary): ResidualCodec on the device
// ------------------------------------------------------------------------------------------
struct pb_codec {
    int device = 0, dim = 0, nbits = 0, sm_count = 132;
    long long K = 0;
    DevBuf centroids, cutoffs, cent_bf16, cent_norm;
    bool has_cutoffs = false;
    bool use_tc = false;   // tensor-core certified filter in front of the exact assignment
    float cmax = 0.f;
    int c_finite = 1;
    long long last_tokens = 0, last_fallback = 0;
};

static size_t smem_assign_tc(int dim) {
    return (size_t)2 * PB_TC_M * dim * 2 + (size_t)PB_TC_STAGES * PB_TC_N * dim * 2 + (2 * PB_TC_STAGES + 5) * 8 + 16;
}

static size_t smem_assign(int dim) { return (size_t)((dim <= 128 ? 2 : 1) * PB_TOK_TILE + 64) * (dim + 4) * sizeof(float); }

static pb_status launch_assign(int dim, int sm_count, const float *dX, long long n, const float *dC, long long K,
                               const float *bias, long long *codes64, uint32_t *codes32, cudaStream_t st) {
    if (n == 0) return PB_OK;
    (void)sm_count;
    const unsigned blocks = (unsigned)((n + 63) / 64);
    PB_DIM_SWITCH(dim, {
        auto kern = k_assign<DIM>;
        CKS(set_smem(kern, smem_assign(DIM)));
        kern<<<blocks, 256, smem_assign(DIM), st>>>(dX, n, dC, K, bias, codes64, codes32);
    });
    CK(cudaGetLastError());
    return PB_OK;
}

extern "C" pb_status pb_codec_open(int32_t device, const float *centroids, int64_t K, int32_t dim, int32_t nbits,
                                   const float *bucket_cutoffs, pb_codec **out) {
    if (!centroids || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    *out = nullptr;
    if (nbits <= 0 || 8 % nbits != 0) return pb_fail(PB_ERR_INVALID, "nbits must be a divisor of 8, got %d", nbits);
    if (K <= 0 || K >= (1ll << 32) - 1) return pb_fail(PB_ERR_INVALID, "bad num_centroids %lld", (long long)K);
    CKS(BuiltDims::check(dim));
    CKS(check_device(device));
    std::unique_ptr<pb_codec> c(new pb_codec());
    c->device = device;
    c->dim = dim;
    c->nbits = nbits;
    c->K = K;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    CKS(upload(c->centroids, centroids, (size_t)K * dim * 4, PB_MEM_HOST));
    if (bucket_cutoffs) {
        CKS(upload(c->cutoffs, bucket_cutoffs, (size_t)((1 << nbits) - 1) * 4, PB_MEM_HOST));
        c->has_cutoffs = true;
    }
    // tensor-core filter: fp16 copy of the centroids (tile order), their largest norm, finiteness
    c->use_tc = TcDims::has(dim) && K >= 256 && !getenv("PB_ASSIGN_EXACT") &&
                smem_assign_tc(dim) <= 227 * 1024;
    if (c->use_tc) {
        const size_t kpad = (size_t)((K + 127) / 128) * 128;  // tile order, zero padded
        CKS(c->cent_bf16.ensure(kpad * dim * 2));
        CK(cudaMemset(c->cent_bf16.p, 0, kpad * dim * 2));
        CKS(c->cent_norm.ensure((size_t)K * 4));
        k_rows_to_bf16<<<c->sm_count * 8, 256>>>(c->centroids.as<float>(), K, dim, c->cent_bf16.as<__nv_bfloat16>(),
                                                 c->cent_norm.as<float>());
        CK(cudaGetLastError());
        std::vector<float> nr((size_t)K);
        CK(cudaMemcpy(nr.data(), c->cent_norm.p, (size_t)K * 4, cudaMemcpyDeviceToHost));
        float mx = 0.f;
        for (float v : nr) {
            if (!(v < 1e18f)) c->c_finite = 0;
            else mx = std::max(mx, v);
        }
        c->cmax = mx;
    }
    *out = c.release();
    return PB_OK;
}

extern "C" pb_status pb_codec_last_assign_stats(pb_codec *c, int64_t *n_tokens, int64_t *n_exact_fallback, int32_t *used_tensor_cores) {
    if (!c) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_tokens) *n_tokens = c->last_tokens;
    if (n_exact_fallback) *n_exact_fallback = c->last_fallback;
    if (used_tensor_cores) *used_tensor_cores = c->use_tc ? 1 : 0;
    return PB_OK;
}

// nearest-centroid codes of m device-resident rows: tensor-core shortlist + certified exact re-score,
// exact kernel for whatever cannot be certified
static pb_status assign_codes(pb_codec *c, const float *dX, long long m, long long *dcodes) {
    if (!c->use_tc) {
        c->last_fallback += m;
        return launch_assign(c->dim, c->sm_count, dX, m, c->centroids.as<float>(), c->K, nullptr, dcodes, nullptr, 0);
    }
    DevBuf xb, xn, ts, ti, nfb, fl;
    const size_t mpad = (size_t)((m + 255) / 256) * 256;  // two 128-token tiles per CTA, zero padded
    CKS(xb.ensure(mpad * c->dim * 2));
    CK(cudaMemset(xb.p, 0, mpad * c->dim * 2));
    CKS(xn.ensure((size_t)m * 4));
    CKS(ts.ensure((size_t)m * 16));
    CKS(ti.ensure((size_t)m * 16));
    CKS(nfb.ensure(16));
    CKS(fl.ensure((size_t)m * 8));
    CK(cudaMemset(nfb.p, 0, 4));
    k_rows_to_bf16<<<c->sm_count * 8, 256>>>(dX, m, c->dim, xb.as<__nv_bfloat16>(), xn.as<float>());
    const unsigned blocks = (unsigned)((m + 2 * PB_TC_M - 1) / (2 * PB_TC_M));
    const size_t sm = smem_assign_tc(c->dim);
    CKS(TcDims::dispatch(c->dim, [&](auto dim_c) -> pb_status {
        auto kern = k_assign_tc<decltype(dim_c)::value, false>;
        CKS(set_smem(kern, sm));
        kern<<<blocks, 288, sm>>>(xb.as<__nv_bfloat16>(), m, c->cent_bf16.as<__nv_bfloat16>(), c->K, ts.as<float>(),
                                  ti.as<uint32_t>(), nullptr);
        return PB_OK;
    }));
    CK(cudaGetLastError());
    k_assign_certify<<<c->sm_count * 8, 256>>>(dX, m, c->dim, c->centroids.as<float>(), xn.as<float>(), c->cmax, c->c_finite,
                                               ts.as<float>(), ti.as<uint32_t>(), dcodes, nfb.as<int>(), fl.as<long long>());
    CK(cudaGetLastError());
    int nf = 0;
    CK(cudaMemcpy(&nf, nfb.p, 4, cudaMemcpyDeviceToHost));
    c->last_fallback += nf;
    if (nf > 0) {
        DevBuf gx, gc;
        CKS(gx.ensure((size_t)nf * c->dim * 4));
        CKS(gc.ensure((size_t)nf * 8));
        k_gather_rows_i64<<<c->sm_count * 8, 256>>>(dX, fl.as<long long>(), nf, c->dim, gx.as<float>());
        CKS(launch_assign(c->dim, c->sm_count, gx.as<float>(), nf, c->centroids.as<float>(), c->K, nullptr, gc.as<long long>(),
                          nullptr, 0));
        k_scatter_codes<<<(nf + 255) / 256, 256>>>(gc.as<long long>(), fl.as<long long>(), nf, dcodes);
        CK(cudaGetLastError());
    }
    return PB_OK;
}

extern "C" void pb_codec_close(pb_codec *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    delete c;
}

// encode_index_chunk on m device-resident rows: codes (i64) and, when asked, the packed residuals and / or the f32 residuals
static pb_status codec_encode_device(pb_codec *c, const float *dX, long long m, long long *dcodes, uint8_t *dpacked,
                                     float *dres) {
    CKS(assign_codes(c, dX, m, dcodes));
    if (dpacked || dres) {
        PB_DIM_SWITCH(c->dim, {
            k_quantize_pack<DIM><<<c->sm_count * 8, 256>>>(dX, m, c->centroids.as<float>(), dcodes, c->cutoffs.as<float>(),
                                                            c->nbits, dpacked, dres);
        });
        CK(cudaGetLastError());
    }
    return PB_OK;
}

// embeddings are processed in slabs so the staging buffers stay bounded
static pb_status codec_run(pb_codec *c, const float *emb, int64_t n, int64_t *out_codes, uint8_t *out_packed,
                           float *out_residuals) {
    if (!c || (!emb && n) || n < 0) return pb_fail(PB_ERR_INVALID, "null argument");
    if ((out_packed) && !c->has_cutoffs) return pb_fail(PB_ERR_INVALID, "bucket_cutoffs required for quantization");  // codec.rs:359-362
    CK(cudaSetDevice(c->device));
    if (n == 0) return PB_OK;
    const long long slab = 1ll << 20;
    const int packed = c->dim * c->nbits / 8;
    c->last_tokens = n;
    c->last_fallback = 0;
    DevBuf dX, dcodes, dpk, dres;
    CKS(dX.ensure((size_t)std::min<long long>(n, slab) * c->dim * 4));
    CKS(dcodes.ensure((size_t)std::min<long long>(n, slab) * 8));
    if (out_packed) CKS(dpk.ensure((size_t)std::min<long long>(n, slab) * packed));
    if (out_residuals) CKS(dres.ensure((size_t)std::min<long long>(n, slab) * c->dim * 4));
    for (long long o = 0; o < n; o += slab) {
        const long long m = std::min(slab, n - o);
        CK(cudaMemcpy(dX.p, emb + (size_t)o * c->dim, (size_t)m * c->dim * 4, cudaMemcpyHostToDevice));
        CKS(codec_encode_device(c, dX.as<float>(), m, dcodes.as<long long>(), out_packed ? dpk.as<uint8_t>() : nullptr,
                                out_residuals ? dres.as<float>() : nullptr));
        if (out_codes) CK(cudaMemcpy(out_codes + o, dcodes.p, (size_t)m * 8, cudaMemcpyDeviceToHost));
        if (out_packed) CK(cudaMemcpy(out_packed + (size_t)o * packed, dpk.p, (size_t)m * packed, cudaMemcpyDeviceToHost));
        if (out_residuals) CK(cudaMemcpy(out_residuals + (size_t)o * c->dim, dres.p, (size_t)m * c->dim * 4, cudaMemcpyDeviceToHost));
    }
    return PB_OK;
}

extern "C" pb_status pb_codec_compress_into_codes(pb_codec *c, const float *embeddings, int64_t n, int64_t *out_codes) {
    if (!out_codes && n) return pb_fail(PB_ERR_INVALID, "null argument");
    return codec_run(c, embeddings, n, out_codes, nullptr, nullptr);
}

extern "C" pb_status pb_codec_encode_chunk(pb_codec *c, const float *embeddings, int64_t n, int64_t *out_codes,
                                           uint8_t *out_residuals_packed) {
    if ((!out_codes || !out_residuals_packed) && n) return pb_fail(PB_ERR_INVALID, "null argument");
    return codec_run(c, embeddings, n, out_codes, out_residuals_packed, nullptr);
}

extern "C" pb_status pb_codec_compress_and_residuals(pb_codec *c, const float *embeddings, int64_t n, int64_t *out_codes,
                                                     float *out_residuals) {
    if ((!out_codes || !out_residuals) && n) return pb_fail(PB_ERR_INVALID, "null argument");
    // residuals only need the subtraction: run the pack kernel without a packed output
    bool had = c && c->has_cutoffs;
    if (c && !had) {  // the kernel reads ncut cutoffs only when packing; give it a valid (unused) pointer
        float zero[255] = {0};
        CKS(upload(c->cutoffs, zero, sizeof zero, PB_MEM_HOST));
    }
    return codec_run(c, embeddings, n, out_codes, nullptr, out_residuals);
}

// prepare_codec_artifacts' arithmetic (index.rs:228-287) for held-out embeddings the caller selected: residuals of
// the nearest centroid, cluster_threshold = quantile 0.75 of their L2 norms, avg_residual = per-dimension mean of
// |residual|, bucket cutoffs / weights = quantiles of the flattened residuals at i/2^b and (i+1/2)/2^b
// (utils.rs:125-149: sort, position q (n-1) in f64, lo (1-w) + hi w with w cast to f32).  The codec keeps the cutoffs.
static float quantile_pick(const std::vector<float> &sorted_at, const std::vector<long long> &pos, long long n, double q) {
    // sorted_at[i] = sorted[pos[i]]; pos holds floor/ceil positions of every requested quantile in order
    const double idx = q * (double)(n - 1);
    const long long lo = (long long)floor(idx), hi = (long long)ceil(idx);
    float vlo = 0.f, vhi = 0.f;
    for (size_t i = 0; i < pos.size(); ++i) {
        if (pos[i] == lo) vlo = sorted_at[i];
        if (pos[i] == hi) vhi = sorted_at[i];
    }
    if (lo == hi) return vlo;
    const float w = (float)(idx - (double)lo);
    return vlo * (1.0f - w) + vhi * w;
}

static pb_status device_quantiles(DevBuf &vals, long long n, const std::vector<double> &qs, std::vector<float> &out) {
    out.assign(qs.size(), 0.0f);
    if (n == 0) return PB_OK;
    DevBuf sorted, tmp;
    CKS(sorted.ensure((size_t)n * 4));
    size_t tb = 0;
    CK(cub::DeviceRadixSort::SortKeys(nullptr, tb, vals.as<float>(), sorted.as<float>(), (int)n));
    CKS(tmp.ensure(tb + 16));
    CK(cub::DeviceRadixSort::SortKeys(tmp.p, tb, vals.as<float>(), sorted.as<float>(), (int)n));
    std::vector<long long> pos;
    for (double q : qs) {
        const double idx = q * (double)(n - 1);
        pos.push_back((long long)floor(idx));
        pos.push_back((long long)ceil(idx));
    }
    std::vector<float> at(pos.size());
    for (size_t i = 0; i < pos.size(); ++i)
        CK(cudaMemcpy(&at[i], sorted.as<float>() + pos[i], 4, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < qs.size(); ++i) out[i] = quantile_pick(at, pos, n, qs[i]);
    return PB_OK;
}

extern "C" pb_status pb_codec_train(pb_codec *c, const float *heldout, int64_t n, float *out_cutoffs, float *out_weights,
                                    float *out_avg_residual, float *out_cluster_threshold) {
    if (!c || (!heldout && n) || n < 0 || !out_cutoffs || !out_weights) return pb_fail(PB_ERR_INVALID, "null argument");
    if ((long long)n * c->dim >= (1ll << 31)) return pb_fail(PB_ERR_UNSUPPORTED, "held-out sample too large");
    CK(cudaSetDevice(c->device));
    const int nopt = 1 << c->nbits;
    DevBuf dX, dcodes, dres, dnorm, davg;
    CKS(dX.ensure(std::max<size_t>((size_t)n * c->dim * 4, 16)));
    CKS(dcodes.ensure(std::max<size_t>((size_t)n * 8, 16)));
    CKS(dres.ensure(std::max<size_t>((size_t)n * c->dim * 4, 16)));
    CKS(dnorm.ensure(std::max<size_t>((size_t)n * 4, 16)));
    CKS(davg.ensure((size_t)c->dim * 4));
    if (n > 0) {
        CK(cudaMemcpy(dX.p, heldout, (size_t)n * c->dim * 4, cudaMemcpyHostToDevice));
        CKS(assign_codes(c, dX.as<float>(), n, dcodes.as<long long>()));
        if (!c->has_cutoffs) {  // the residual kernel takes a cutoff pointer it does not read without a packed output
            float zero[255] = {0};
            CKS(upload(c->cutoffs, zero, sizeof zero, PB_MEM_HOST));
        }
        PB_DIM_SWITCH(c->dim, {
            k_quantize_pack<DIM><<<c->sm_count * 8, 256>>>(dX.as<float>(), n, c->centroids.as<float>(), dcodes.as<long long>(),
                                                            c->cutoffs.as<float>(), c->nbits, nullptr, dres.as<float>());
        });
        k_residual_stats<<<c->sm_count * 4, 256>>>(dres.as<float>(), n, c->dim, dnorm.as<float>());
        k_column_abs_mean<<<(c->dim + 31) / 32, 32>>>(dres.as<float>(), n, c->dim, davg.as<float>());
        CK(cudaGetLastError());
    }
    std::vector<double> q75{0.75}, qc, qw;
    for (int i = 1; i < nopt; ++i) qc.push_back((double)i / (double)nopt);
    for (int i = 0; i < nopt; ++i) qw.push_back(((double)i + 0.5) / (double)nopt);
    std::vector<float> r75, rc, rw;
    CKS(device_quantiles(dnorm, n, q75, r75));
    CKS(device_quantiles(dres, (long long)n * c->dim, qc, rc));
    CKS(device_quantiles(dres, (long long)n * c->dim, qw, rw));
    for (int i = 0; i < nopt - 1; ++i) out_cutoffs[i] = rc[i];
    for (int i = 0; i < nopt; ++i) out_weights[i] = rw[i];
    if (out_cluster_threshold) *out_cluster_threshold = n ? r75[0] : 0.0f;
    if (out_avg_residual) {
        if (n) CK(cudaMemcpy(out_avg_residual, davg.p, (size_t)c->dim * 4, cudaMemcpyDeviceToHost));
        else memset(out_avg_residual, 0, (size_t)c->dim * 4);
    }
    float cut[255] = {0};
    for (int i = 0; i < nopt - 1; ++i) cut[i] = rc[i];
    CKS(upload(c->cutoffs, cut, sizeof cut, PB_MEM_HOST));
    c->has_cutoffs = true;
    return PB_OK;
}

// compute_kmeans' sizing rules (kmeans.rs:273-312) and prepare_codec_artifacts' (index.rs:195-212), as the host
// side needs them to pick its samples
extern "C" int64_t pb_kmeans_num_sample_docs(int64_t num_documents) {  // min(floor(1 + 16 sqrt(120 D)), D)
    const double v = 1.0 + 16.0 * sqrt(120.0 * (double)num_documents);
    return std::min<int64_t>((int64_t)v, num_documents);
}
extern "C" int64_t pb_kmeans_num_partitions(int64_t num_documents, double avg_sample_doclen, int64_t num_sample_tokens) {
    const double est = avg_sample_doclen * (double)num_documents;  // K = 2^floor(log2(16 sqrt(avg_doclen * D)))
    const double k = pow(2.0, floor(log2(16.0 * sqrt(est))));
    return std::max<int64_t>(1, std::min<int64_t>((int64_t)k, num_sample_tokens));
}
extern "C" int64_t pb_codec_num_sample_docs(int64_t num_documents) {  // clamp(floor(16 sqrt(120 D)), 1, D)
    const int64_t v = (int64_t)(16.0 * sqrt(120.0 * (double)num_documents));
    return std::max<int64_t>(1, std::min<int64_t>(v, num_documents));
}
extern "C" int64_t pb_codec_heldout_tokens(int64_t num_embeddings) {  // min(0.05 N, 50 000)
    return (int64_t)std::min(0.05 * (double)num_embeddings, 50000.0);
}

// k-means assignment step.  TcDims with K >= 256: the fp16 wgmma GEMM of the encode path with the
// -|c|^2/2 bias added in its epilogue, best shortlist entry taken as is; otherwise the exact fp32 kernel.
struct KmeansAssign {
    DevBuf xb, cb, bias, ts, ti, scratch;
    bool tc = false;
    long long n = 0, K = 0;
    int dim = 0, sms = 0;
    pb_status init(const float *dX, long long n_, int dim_, long long K_, int sms_, cudaStream_t st) {
        n = n_; K = K_; dim = dim_; sms = sms_;
        tc = TcDims::has(dim) && K >= 256 && n > 0 && !getenv("PB_KMEANS_EXACT");
        if (!tc) return PB_OK;
        const size_t npad = (size_t)((n + 255) / 256) * 256, kpad = (size_t)((K + 127) / 128) * 128;
        CKS(xb.ensure(npad * dim * 2));
        CKS(cb.ensure(kpad * dim * 2));
        CKS(bias.ensure(kpad * 4));
        CKS(ts.ensure((size_t)n * 16));
        CKS(ti.ensure((size_t)n * 16));
        CKS(scratch.ensure(std::max<size_t>((size_t)std::max(n, K) * 4, 16)));
        CK(cudaMemsetAsync(xb.p, 0, npad * dim * 2, st));
        k_rows_to_bf16<<<sms * 8, 256, 0, st>>>(dX, n, dim, xb.as<__nv_bfloat16>(), scratch.as<float>());
        CK(cudaGetLastError());
        return PB_OK;
    }
    pb_status run(const float *dX, const float *dC, float *dbias_exact, uint32_t *codes, cudaStream_t st) {
        if (!tc) {
            k_half_sqnorm<<<sms * 4, 256, 0, st>>>(dC, K, dim, dbias_exact);
            return launch_assign(dim, sms, dX, n, dC, K, dbias_exact, nullptr, codes, st);
        }
        const size_t kpad = (size_t)((K + 127) / 128) * 128;
        CK(cudaMemsetAsync(cb.p, 0, kpad * dim * 2, st));
        k_rows_to_bf16<<<sms * 8, 256, 0, st>>>(dC, K, dim, cb.as<__nv_bfloat16>(), scratch.as<float>());
        k_half_sqnorm_padded<<<sms * 4, 256, 0, st>>>(dC, K, (long long)kpad, dim, bias.as<float>());
        const unsigned blocks = (unsigned)((n + 2 * PB_TC_M - 1) / (2 * PB_TC_M));
        const size_t sm = (size_t)2 * PB_TC_M * dim * 2 + (size_t)PB_TC_STAGES * PB_TC_N * dim * 2 + (2 * PB_TC_STAGES + 5) * 8 + 16;
        CKS(TcDims::dispatch(dim, [&](auto dim_c) -> pb_status {
            auto kern = k_assign_tc<decltype(dim_c)::value, true>;
            CKS(set_smem(kern, sm));
            kern<<<blocks, 288, sm, st>>>(xb.as<__nv_bfloat16>(), n, cb.as<__nv_bfloat16>(), K, ts.as<float>(),
                                          ti.as<uint32_t>(), bias.as<float>());
            return PB_OK;
        }));
        k_take_top1<<<sms * 4, 256, 0, st>>>(ti.as<uint32_t>(), n, codes);
        CK(cudaGetLastError());
        return PB_OK;
    }
};

// Lloyd iterations from the K centroids in dC over the n points dX (k-means assignment, coordinate sums and counts,
// new centroids), then L2 normalisation (kmeans.rs:415-419).  With `comm`, the points are this rank's share and one
// all-reduce per iteration sums every rank's [K][dim] sums and [K] counts, so every rank moves the same centroids.
static pb_status lloyd(ShardComm *comm, DevBuf *stage, cudaStream_t st, const float *dX, long long n, int dim, long long K,
                       int niters, int sms, float *dC) {
    DevBuf dbias, dcodes, dacc;
    CKS(dbias.ensure((size_t)K * 4));
    CKS(dcodes.ensure((size_t)std::max<long long>(n, 1) * 4));
    CKS(dacc.ensure((size_t)K * (dim + 1) * 4));  // [K][dim] sums followed by [K] counts: one all-reduce
    float *sums = dacc.as<float>(), *counts = dacc.as<float>() + (size_t)K * dim;
    KmeansAssign ka;
    CKS(ka.init(dX, n, dim, K, sms, st));
    for (int it = 0; it < niters; ++it) {
        CKS(ka.run(dX, dC, dbias.as<float>(), dcodes.as<uint32_t>(), st));
        CK(cudaMemsetAsync(dacc.p, 0, (size_t)K * (dim + 1) * 4, st));
        if (n > 0) k_accumulate<<<sms * 8, 256, 0, st>>>(dX, n, dim, dcodes.as<uint32_t>(), sums, counts);
        CK(cudaGetLastError());
        if (comm) CKS(comm->allreduce_sum(st, dacc.as<float>(), (size_t)K * (dim + 1), *stage));
        k_update_centroids<<<sms * 4, 256, 0, st>>>(dC, K, dim, sums, counts);
        CK(cudaGetLastError());
    }
    k_normalize_rows<<<sms * 4, 256, 0, st>>>(dC, K, dim);
    CK(cudaGetLastError());
    return PB_OK;
}

// the first K entries of a partial Fisher-Yates shuffle of 0..n-1 with a 64-bit LCG from state s: the sample points
// pb_kmeans_fit starts from
static std::vector<long long> lcg_seeds(long long n, long long K, uint64_t s) {
    std::vector<long long> perm((size_t)n);
    for (long long i = 0; i < n; ++i) perm[i] = i;
    for (long long i = 0; i < K; ++i) {
        s = s * 6364136223846793005ull + 1442695040888963407ull;
        long long j = i + (long long)((s >> 11) % (uint64_t)(n - i));
        std::swap(perm[i], perm[j]);
    }
    perm.resize((size_t)K);
    return perm;
}

extern "C" pb_status pb_kmeans_fit(int32_t device, const float *samples, int64_t n, int32_t dim, int64_t K, int32_t niters,
                                   uint64_t seed, float *out_centroids) {
    if (!samples || !out_centroids) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n <= 0 || K <= 0 || K > n) return pb_fail(PB_ERR_INVALID, "need 0 < K <= n (K=%lld, n=%lld)", (long long)K, (long long)n);
    CKS(BuiltDims::check(dim));
    CKS(check_device(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    const int sms = prop.multiProcessorCount;
    DevBuf dX, dC, didx;
    CKS(upload(dX, samples, (size_t)n * dim * 4, PB_MEM_HOST));
    CKS(dC.ensure((size_t)K * dim * 4));
    // initial centroids: K distinct sample points
    const std::vector<long long> perm = lcg_seeds(n, K, seed * 6364136223846793005ull + 1442695040888963407ull);
    CKS(upload(didx, perm.data(), (size_t)K * 8, PB_MEM_HOST));
    k_gather_rows<<<sms * 4, 256>>>(dX.as<float>(), didx.as<long long>(), K, dim, dC.as<float>());
    CK(cudaGetLastError());
    CKS(lloyd(nullptr, nullptr, 0, dX.as<float>(), n, dim, K, niters, sms, dC.as<float>()));
    CK(cudaMemcpy(out_centroids, dC.p, (size_t)K * dim * 4, cudaMemcpyDeviceToHost));
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// Data-parallel k-means (SURVEY 8e "Build path"): every rank holds a shard of the sample points, the centroids are
// replicated, and one all-reduce per iteration sums the per-rank [K][dim] coordinate sums and [K] counts (135 MB at
// K = 2^18, dim 128) -- over NCCL when the communicator came from pb_build_comm_init, or through the in-process shard
// group (peer copies + a rank-ordered sum, identical on every rank) when it came from pb_build_comm_group.
// ------------------------------------------------------------------------------------------
struct pb_build_comm {
    OwnedStream stream;
    DevBuf stage;  // every rank's buffer, gathered by the in-process all-reduce
    ShardComm comm;  // declared last, so destroyed first: an NCCL communicator goes before the stream it ran on
};

extern "C" pb_status pb_build_comm_init(const uint8_t *id128, int32_t rank, int32_t world, int32_t device, pb_build_comm **out) {
    if (!id128 || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(check_device(device));
    std::unique_ptr<pb_build_comm> c(new pb_build_comm());
    CK(cudaStreamCreateWithFlags(&c->stream.s, cudaStreamNonBlocking));
    CKS(c->comm.init_nccl(id128, rank, world, device));
    *out = c.release();
    return PB_OK;
}
extern "C" pb_status pb_build_comm_group(pb_shard_group *g, int32_t rank, int32_t device, pb_build_comm **out) {
    if (!g || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(check_device(device));
    std::unique_ptr<pb_build_comm> c(new pb_build_comm());
    CK(cudaStreamCreateWithFlags(&c->stream.s, cudaStreamNonBlocking));
    CKS(c->comm.join(g, rank, device));
    *out = c.release();
    return PB_OK;
}
extern "C" void pb_build_comm_destroy(pb_build_comm *c) {
    if (!c) return;
    cudaSetDevice(c->comm.device);
    delete c;
}

extern "C" pb_status pb_kmeans_fit_dp(pb_build_comm *c, const float *samples, int64_t n_local, int32_t dim, int64_t K,
                                      int32_t niters, uint64_t seed, float *out_centroids) {
    if (!c || (!samples && n_local) || !out_centroids) return pb_fail(PB_ERR_INVALID, "null argument");
    if (n_local < 0 || K <= 0) return pb_fail(PB_ERR_INVALID, "bad sizes");
    CKS(BuiltDims::check(dim));
    CK(cudaSetDevice(c->comm.device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, c->comm.device));
    const int sms = prop.multiProcessorCount;
    const long long n = n_local;
    // rank r seeds centroids [k0, k1) with distinct points of its shard; one all-reduce of the zero-padded table
    // gives every rank the same start
    const long long k0 = K * c->comm.rank / c->comm.world, k1 = K * (c->comm.rank + 1) / c->comm.world, kmine = k1 - k0;
    if (kmine > n) return pb_fail(PB_ERR_INVALID, "rank %d holds %lld points but seeds %lld centroids", c->comm.rank, n, kmine);
    DevBuf dX, dC, didx;
    CKS(upload(dX, samples, (size_t)std::max<long long>(n, 1) * dim * 4, PB_MEM_HOST));
    CKS(dC.ensure((size_t)K * dim * 4));
    const std::vector<long long> perm = lcg_seeds(
        n, kmine, (seed + 0x9e3779b97f4a7c15ull * (uint64_t)(c->comm.rank + 1)) * 6364136223846793005ull + 1442695040888963407ull);
    CK(cudaMemsetAsync(dC.p, 0, (size_t)K * dim * 4, c->stream.s));
    if (kmine > 0) {
        CKS(upload(didx, perm.data(), (size_t)kmine * 8, PB_MEM_HOST));
        k_gather_rows<<<sms * 4, 256, 0, c->stream.s>>>(dX.as<float>(), didx.as<long long>(), kmine, dim, dC.as<float>() + (size_t)k0 * dim);
        CK(cudaGetLastError());
    }
    CKS(c->comm.allreduce_sum(c->stream.s, dC.as<float>(), (size_t)K * dim, c->stage));
    CKS(lloyd(&c->comm, &c->stage, c->stream.s, dX.as<float>(), n, dim, K, niters, sms, dC.as<float>()));
    CK(cudaMemcpyAsync(out_centroids, dC.p, (size_t)K * dim * 4, cudaMemcpyDeviceToHost, c->stream.s));
    CK(cudaStreamSynchronize(c->stream.s));
    return PB_OK;
}

// find_outliers (update.rs:490-608) on the codec's centroids
extern "C" pb_status pb_codec_find_outliers(pb_codec *c, const float *embeddings, int64_t n, float threshold_sq,
                                            int64_t *out_indices, int64_t *out_count) {
    if (!c || (!embeddings && n) || !out_count || (!out_indices && n)) return pb_fail(PB_ERR_INVALID, "null argument");
    *out_count = 0;
    if (n <= 0) return n == 0 ? PB_OK : pb_fail(PB_ERR_INVALID, "negative size");
    CK(cudaSetDevice(c->device));
    DevBuf cn, dX, xn, md, fl;
    CKS(cn.ensure((size_t)c->K * 4));
    k_squared_norms_ref<<<c->sm_count * 4, 256>>>(c->centroids.as<float>(), c->K, c->dim, cn.as<float>());
    const long long slab = 1ll << 20;
    CKS(dX.ensure((size_t)std::min<long long>(n, slab) * c->dim * 4));
    CKS(xn.ensure((size_t)std::min<long long>(n, slab) * 4));
    CKS(md.ensure((size_t)std::min<long long>(n, slab) * 4));
    CKS(fl.ensure((size_t)std::min<long long>(n, slab)));
    std::vector<uint8_t> hf((size_t)std::min<long long>(n, slab));
    int64_t cnt = 0;
    for (long long o = 0; o < n; o += slab) {
        const long long m = std::min(slab, n - o);
        CK(cudaMemcpy(dX.p, embeddings + (size_t)o * c->dim, (size_t)m * c->dim * 4, cudaMemcpyHostToDevice));
        k_squared_norms_ref<<<c->sm_count * 4, 256>>>(dX.as<float>(), m, c->dim, xn.as<float>());
        const unsigned blocks = (unsigned)((m + 63) / 64);
        PB_DIM_SWITCH(c->dim, {
            auto kern = k_min_dist<DIM>;
            CKS(set_smem(kern, smem_assign(DIM)));
            kern<<<blocks, 256, smem_assign(DIM)>>>(dX.as<float>(), m, xn.as<float>(), c->centroids.as<float>(), c->K,
                                                    cn.as<float>(), md.as<float>());
        });
        k_outlier_decide<<<c->sm_count * 8, 256>>>(dX.as<float>(), m, c->dim, c->centroids.as<float>(), c->K, md.as<float>(),
                                                   threshold_sq, fl.as<uint8_t>());
        CK(cudaGetLastError());
        CK(cudaMemcpy(hf.data(), fl.p, (size_t)m, cudaMemcpyDeviceToHost));
        for (long long i = 0; i < m; ++i)
            if (hf[i]) out_indices[cnt++] = o + i;
    }
    *out_count = cnt;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// incremental append: MmapIndex::update_append (index.rs:1675) + reload on a live handle
// ------------------------------------------------------------------------------------------
// the u32 inverted file ivf [L] at off [K + 1] on the host in the directory's dtypes: ivf.npy <i8, ivf_lengths.npy <i4
// (widened on the device one slab of at most 2^26 entries at a time, so the i64 copy is never whole on the device)
static pb_status ivf_to_host(pb_index *ix, const DevBuf &ivf, const DevBuf &off, long long L, std::vector<int64_t> &hivf,
                             std::vector<int32_t> &hlen) {
    hivf.assign((size_t)std::max(L, 1ll), 0);
    hlen.assign((size_t)ix->K, 0);
    const long long slab = 1ll << 26;
    DevBuf di, dln;
    CKS(di.ensure(std::max<size_t>((size_t)std::min(L, slab) * 8, 16)));
    CKS(dln.ensure((size_t)ix->K * 4));
    for (long long o = 0; o < std::max(L, 1ll); o += slab) {  // the first launch also writes the lengths
        const long long m = std::min(slab, L - o);
        k_ivf_export<<<ix->sm_count * 8, 256>>>(ivf.as<uint32_t>() + o, off.as<long long>(), m, ix->K, 0,
                                               di.as<long long>(), o == 0 ? dln.as<int>() : nullptr);
        CK(cudaGetLastError());
        if (m > 0) CK(cudaMemcpy(hivf.data() + o, di.p, (size_t)m * 8, cudaMemcpyDeviceToHost));
    }
    CK(cudaMemcpy(hlen.data(), dln.p, (size_t)ix->K * 4, cudaMemcpyDeviceToHost));
    return PB_OK;
}

pb_status pb_index_patch_ivf(pb_index *ix, const int64_t *file_ivf, const int32_t *file_lengths, long long total, long long D,
                             const uint32_t *bits, const long long *word_pre, const uint64_t *keys, long long m,
                             std::vector<int64_t> &ivf, std::vector<int32_t> &lengths) {
    DevBuf out, off;
    long long L = 0;
    CKS(ivf_from_file(ix, file_ivf, file_lengths, total, D, 0, D, bits, word_pre,
                      reinterpret_cast<const u64 *>(keys), m, out, off, &L));
    return ivf_to_host(ix, out, off, L, ivf, lengths);
}

// What an append computes before anything becomes visible: the new tokens in the tails of the per-token arrays, the
// new docs' offsets and distinct codes, the merged inverted file in the spare half of the ping-pong, and the totals the
// commit publishes.  keys holds the new docs' sorted (centroid << 32 | doc in the batch) pairs.
struct AppendPrep {
    long long D0 = 0, n = 0, ntok = 0, m = 0;
    DocTotals t;
    std::vector<int64_t> dl, hcodes;  // doc lengths; the i64 codes for a directory (keep_codes)
    DevBuf keys;
};

// Capacity for D1 docs of N1 tokens in the per-token and per-doc arrays, keeping their contents
static pb_status grow_docs(pb_index *ix, long long D1, long long N1, bool geometric) {
    const size_t pk = (size_t)ix->packed;
    CKS(ix->codes.grow((size_t)N1 * 4, (size_t)ix->N * 4, geometric));
    if (!ix->host_tier) CKS(ix->residuals.grow((size_t)N1 * pk, (size_t)ix->N * pk, geometric));
    if (TcDims::has(ix->dim)) CKS(ix->tok_inv_norm.grow((size_t)N1 * 4, (size_t)ix->N * 4, geometric));
    CKS(ix->doc_off.grow((size_t)(D1 + 1) * 8, (size_t)(ix->D + 1) * 8, geometric));
    CKS(ix->udoc_off.grow((size_t)(D1 + 1) * 8, (size_t)(ix->D + 1) * 8, geometric));
    if (ix->cache_off.p) {
        CKS(ix->cache_off.grow((size_t)D1 * 8, (size_t)ix->D * 8, geometric));
        CKS(ix->kept_count.grow((size_t)D1 * 4, (size_t)ix->D * 4, geometric));
    }
    return PB_OK;
}

// Makes a prepared mutation visible: its totals, with either the inverted file an append or a delete merged into the
// spare halves, or (rebalance) a whole set of arrays built out of place, swapped in; the old ones leave with `fresh`
static void publish(pb_index *ix, const DocTotals &t, DocArrays *fresh = nullptr) {
    if (fresh) {
        const auto mine = DocArrays::buffers(*ix), theirs = DocArrays::buffers(*fresh);
        for (size_t i = 0; i < mine.size(); ++i) mine[i]->swap(*theirs[i]);
    } else {
        ix->ivf.swap(ix->ivf_spare);
        ix->ivf_off.swap(ix->ivf_off_spare);
    }
    static_cast<DocTotals &>(*ix) = t;
    ++ix->doc_gen;
}

// Every check, allocation and device write of an append that stays invisible until publish.  The caller holds
// the handle's writer lock.  A host-tier handle's new rows go to its store's tail, past the rows a search reads;
// write_rows = false: another replica sharing the store has written them.
static pb_status append_prepare(pb_index *ix, pb_codec *codec, const float *embeddings, const int64_t *codes,
                                const uint8_t *residuals, const int64_t *doc_lengths, int64_t n_docs, int32_t space,
                                bool keep_codes, int64_t *out_first, AppendPrep &p, bool write_rows = true) {
    CK(cudaSetDevice(ix->device));
    CK(cudaDeviceSynchronize());  // work earlier readers left queued (pb_search_batch_device) reads the arrays
    if (codec) {  // same K, dim, nbits and bit-identical centroids as the index; cutoffs required (codec.rs:359-362)
        if (codec->K != ix->K || codec->dim != ix->dim || codec->nbits != ix->nbits || codec->device != ix->device)
            return pb_fail(PB_ERR_INVALID, "codec (K=%lld dim=%d nbits=%d device %d) does not match the index (K=%lld dim=%d nbits=%d device %d)",
                           codec->K, codec->dim, codec->nbits, codec->device, ix->K, ix->dim, ix->nbits, ix->device);
        if (!codec->has_cutoffs) return pb_fail(PB_ERR_INVALID, "bucket_cutoffs required for quantization");
        DevBuf flag;
        CKS(flag.ensure(16));
        CK(cudaMemset(flag.p, 0, 4));
        k_words_differ<<<ix->sm_count * 8, 256>>>(codec->centroids.as<uint32_t>(), ix->centroids.as<uint32_t>(),
                                                  ix->K * (long long)ix->dim, flag.as<int>());
        CK(cudaGetLastError());
        int differ = 0;
        CK(cudaMemcpy(&differ, flag.p, 4, cudaMemcpyDeviceToHost));
        if (differ) return pb_fail(PB_ERR_INVALID, "the codec's centroids differ from the index's");
    }
    const long long D0 = ix->D, N0 = ix->N, n = n_docs;
    if (out_first) *out_first = ix->doc_id_base + D0;
    p.D0 = D0;
    DocTotals &t = p.t;
    t.max_doclen = ix->max_doclen;
    CKS(fetch_host(p.dl, doc_lengths, (size_t)n, space));
    std::vector<long long> doff;  // doc_off[D0 ..]
    CKS(doc_offsets(p.dl, N0, doff, &t.max_doclen));
    if (n == 0) return PB_OK;
    const long long ntok = doff[n] - N0;
    // the limits of pb_index_open_begin for the new totals
    if (D0 + n >= (1ll << 32) - 1 || ix->doc_id_base + D0 + n >= (1ll << 32) - 1)
        return pb_fail(PB_ERR_UNSUPPORTED, "D and global doc ids must stay below 2^32-1");
    if (ntok > 0 && ((codec && !embeddings) || (!codec && (!codes || !residuals)))) return pb_fail(PB_ERR_INVALID, "null argument");
    p.ntok = ntok;
    t.N = N0 + ntok;
    t.D = D0 + n;
    const size_t pk = (size_t)ix->packed;

    // capacity: grown arrays keep their contents; nothing below is visible until the commit
    if (ix->host_tier) CKS(write_rows ? ix->host.grow((size_t)t.N * pk) : ix->host.sync());
    CKS(grow_docs(ix, t.D, t.N, true));

    // 1. tokens into the tails of codes / residuals: encoded on the device, or narrowed and range-checked
    std::vector<int64_t> &hcodes = p.hcodes;  // i64 codes for the chunk files
    if (codec) {
        codec->last_tokens = ntok;
        codec->last_fallback = 0;
        const long long slab = 1ll << 20;
        DevBuf dX, dcodes, dres;  // dres: a host-tier slab's rows on their way to the store
        CKS(dcodes.ensure((size_t)std::max(std::min(ntok, slab), 1ll) * 8));
        if (space == PB_MEM_HOST) CKS(dX.ensure((size_t)std::max(std::min(ntok, slab), 1ll) * ix->dim * 4));
        if (ix->host_tier) CKS(dres.ensure((size_t)std::max(std::min(ntok, slab), 1ll) * pk));
        if (keep_codes) hcodes.resize((size_t)ntok);
        for (long long o = 0; o < ntok; o += slab) {
            const long long m = std::min(slab, ntok - o);
            const float *x = embeddings + (size_t)o * ix->dim;
            if (space == PB_MEM_HOST) {
                CK(cudaMemcpy(dX.p, x, (size_t)m * ix->dim * 4, cudaMemcpyHostToDevice));
                x = dX.as<float>();
            }
            uint8_t *res = ix->host_tier ? dres.as<uint8_t>() : ix->residuals.as<uint8_t>() + (size_t)(N0 + o) * pk;
            CKS(codec_encode_device(codec, x, m, dcodes.as<long long>(), res, nullptr));
            if (ix->host_tier) CKS(ix->host.rows->write((size_t)(N0 + o) * pk, res, (size_t)m * pk, PB_MEM_DEVICE));
            CKS(upload_narrow(ix->codes, N0 + o, reinterpret_cast<const int64_t *>(dcodes.p), m, ix->K, PB_MEM_DEVICE, "codes"));
            if (keep_codes) CK(cudaMemcpy(hcodes.data() + o, dcodes.p, (size_t)m * 8, cudaMemcpyDeviceToHost));
        }
    } else if (ntok > 0) {
        if (!ix->host_tier)
            CK(cudaMemcpy(ix->residuals.as<uint8_t>() + (size_t)N0 * pk, residuals, (size_t)ntok * pk,
                          space == PB_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
        else if (write_rows)
            CKS(ix->host.rows->write((size_t)N0 * pk, residuals, (size_t)ntok * pk, space));
        CKS(upload_narrow(ix->codes, N0, codes, ntok, ix->K, space, "codes"));
    }

    // 2. doc offsets; with a row cache the new docs are not cached and have not been kept
    CK(cudaMemcpy(ix->doc_off.as<long long>() + D0 + 1, doff.data() + 1, (size_t)n * 8, cudaMemcpyHostToDevice));
    if (ix->cache_off.p) {
        CK(cudaMemset(ix->cache_off.as<long long>() + D0, 0xff, (size_t)n * 8));
        CK(cudaMemset(ix->kept_count.as<uint32_t>() + D0, 0, (size_t)n * 4));
    }

    // 3. distinct code lists of the new docs, after the old ones
    CKS(unique_codes(ix, D0, n, ix->n_ucodes, &t.n_ucodes));

    // 4. 1 / |c + w| of the new tokens; min / max seeded with the index's, which is what an open over all tokens finds
    DevBuf mn;
    const float seed[2] = {N0 > 0 ? ix->vmin : 3.0e38f, N0 > 0 ? ix->wmax : 0.0f};
    CKS(token_norms(ix, *ix, N0, seed, t, mn));

    // 5. inverted file: the new docs' sorted distinct (centroid, doc) pairs merged behind each centroid's old list
    DevBuf add_before;
    long long m = 0;
    CKS(sorted_doc_pairs(ix, D0, n, t.n_ucodes - ix->n_ucodes, p.keys, &m));
    t.ivf_len = ix->ivf_len + m;
    if (t.ivf_len > (1ll << 31) - 2) return pb_fail(PB_ERR_UNSUPPORTED, "more than 2^31 (centroid, doc) pairs per shard");
    CKS(add_before.ensure((size_t)(ix->K + 1) * 8));
    CKS(ix->ivf_spare.grow(std::max<size_t>((size_t)t.ivf_len * 4, 16), 0));
    CKS(ix->ivf_off_spare.ensure((size_t)(ix->K + 1) * 8));
    k_ivf_offsets<<<(unsigned)((ix->K + 256) / 256), 256>>>(p.keys.as<u64>(), m, ix->K, add_before.as<long long>());
    k_ivf_merge_old<<<ix->sm_count * 8, 256>>>(ix->ivf.as<uint32_t>(), ix->ivf_off.as<long long>(), add_before.as<long long>(),
                                               ix->K, ix->ivf_spare.as<uint32_t>(), ix->ivf_off_spare.as<long long>());
    if (m > 0)
        k_ivf_merge_new<<<ix->sm_count * 8, 256>>>(p.keys.as<u64>(), m, ix->ivf_off.as<long long>(), (uint32_t)D0,
                                                   ix->ivf_spare.as<uint32_t>());
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    p.n = n;
    p.m = m;
    return PB_OK;
}

// the packed rows of tokens [t0, t0 + n) into host memory, from the device array or the host tier's store
static pb_status rows_to_host(const pb_index *ix, long long t0, long long n, uint8_t *dst) {
    const size_t pk = (size_t)ix->packed;
    if (n == 0) return PB_OK;
    if (ix->host_tier) return ix->host.rows->read((size_t)t0 * pk, dst, (size_t)n * pk);
    CK(cudaMemcpy(dst, ix->residuals.as<uint8_t>() + (size_t)t0 * pk, (size_t)n * pk, cudaMemcpyDeviceToHost));
    return PB_OK;
}

// update_index's file changes for the prepared documents, on a directory of old_D documents whose new inverted file
// is (hivf [L], hlen [K])
static pb_status append_dir(pb_index *ix, const AppendPrep &p, const char *index_dir, long long old_D, int64_t batch_size,
                            const std::vector<int64_t> &hivf, long long L, const std::vector<int32_t> &hlen) {
    const size_t pk = (size_t)ix->packed;
    std::vector<uint8_t> hres((size_t)p.ntok * pk);
    CKS(rows_to_host(ix, p.t.N - p.ntok, p.ntok, hres.data()));
    return pb_dir_append(index_dir, old_D, ix->K, ix->dim, ix->nbits, batch_size, p.hcodes.data(), hres.data(), p.dl.data(),
                         p.n, hivf.data(), L, hlen.data());
}

// Mutations need residual rows the library owns and may grow: not the caller's array (PB_OPEN_ADOPT_RESIDUALS), not
// pinned host memory opened without PB_OPEN_HOST_MUTABLE
static pb_status refuse_fixed_residuals(const pb_index *ix) {
    if (!ix->residuals.owned)
        return pb_fail(PB_ERR_UNSUPPORTED, "the handle uses the caller's residual array (PB_OPEN_ADOPT_RESIDUALS)");
    if (ix->host_tier && !ix->host_mutable)
        return pb_fail(PB_ERR_UNSUPPORTED, "the handle keeps its residuals in host memory (PB_OPEN_HOST_RESIDUALS)");
    return PB_OK;
}

static pb_status append_impl(pb_index *ix, pb_codec *codec, const float *embeddings, const int64_t *codes,
                             const uint8_t *residuals, const int64_t *doc_lengths, int64_t n_docs, int32_t space,
                             const char *index_dir, int64_t batch_size, int64_t *out_first) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    return pb_members_append({ix}, codec, embeddings, codes, residuals, doc_lengths, n_docs, space, index_dir, batch_size,
                             out_first);
}

extern "C" pb_status pb_index_append(pb_index *ix, pb_codec *codec, const float *embeddings, const int64_t *doc_lengths,
                                     int64_t n_docs, int32_t memory_space, const char *index_dir, int64_t batch_size,
                                     int64_t *out_first_doc_id) {
    if (!codec) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix && ix->group)
        return ix->group->append(codec, embeddings, nullptr, nullptr, doc_lengths, n_docs, memory_space, index_dir,
                                 batch_size, out_first_doc_id);
    return append_impl(ix, codec, embeddings, nullptr, nullptr, doc_lengths, n_docs, memory_space, index_dir, batch_size,
                       out_first_doc_id);
}

extern "C" pb_status pb_index_append_encoded(pb_index *ix, const int64_t *codes, const uint8_t *residuals,
                                             const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space,
                                             int64_t *out_first_doc_id) {
    if (ix && ix->group)
        return ix->group->append(nullptr, nullptr, codes, residuals, doc_lengths, n_docs, memory_space, nullptr, 0,
                                 out_first_doc_id);
    return append_impl(ix, nullptr, nullptr, codes, residuals, doc_lengths, n_docs, memory_space, nullptr, 0, out_first_doc_id);
}

extern "C" pb_status pb_index_reserve(pb_index *ix, int64_t num_documents, int64_t num_embeddings) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix->group) return ix->group->reserve(num_documents, num_embeddings);
    std::lock_guard<std::mutex> gate(ix->gate);
    std::unique_lock<std::shared_mutex> wr(ix->rw);
    if (ix->comm.joined()) return pb_fail(PB_ERR_UNSUPPORTED, "appends to a doc-sharded handle are not supported");
    CKS(refuse_fixed_residuals(ix));
    if (num_documents >= (1ll << 32) - 1 || num_embeddings < 0) return pb_fail(PB_ERR_INVALID, "bad reserve sizes");
    CK(cudaSetDevice(ix->device));
    CK(cudaDeviceSynchronize());
    const long long D1 = std::max<long long>(num_documents, ix->D), N1 = std::max<long long>(num_embeddings, ix->N);
    const long long dd = D1 - ix->D, dn = N1 - ix->N;
    // a new doc adds at most its length rounded up to 8 distinct-code entries, and at most that many (centroid, doc) pairs
    const long long U1 = ix->n_ucodes + dn + 7 * dd, L1 = ix->ivf_len + dn;
    if (ix->host_tier) CKS(ix->host.grow((size_t)N1 * ix->packed));
    CKS(grow_docs(ix, D1, N1, false));
    CKS(ix->ucodes.grow((size_t)U1 * 4, (size_t)ix->n_ucodes * 4, false));
    CKS(ix->ivf.grow((size_t)L1 * 4, (size_t)ix->ivf_len * 4, false));
    CKS(ix->ivf_spare.grow((size_t)L1 * 4, 0, false));
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// incremental delete: MmapIndex::delete_with_options (index.rs:1805) -> delete_from_index (delete.rs:43) + reload on a
// live handle
// ------------------------------------------------------------------------------------------
struct Events {
    cudaEvent_t e[5] = {};
    ~Events() {
        for (cudaEvent_t x : e)
            if (x) cudaEventDestroy(x);
    }
};

// The deleted set among docs [base, base + D): one bit per doc in bits [ceil(D / 32)], its per-word prefix counts in
// word_pre [ceil(D / 32) + 1], and the number of docs it holds
static pb_status del_bitmap(pb_index *ix, const int64_t *doc_ids, long long n_ids, long long base, long long D, DevBuf &bits,
                            DevBuf &wpre, long long *n_del) {
    const long long nw = (D + 31) / 32;
    const int grid = ix->sm_count * 8;
    DevBuf wcnt, tmp;
    CKS(bits.ensure(std::max<size_t>((size_t)nw * 4, 16)));
    CK(cudaMemset(bits.p, 0, (size_t)nw * 4));
    if (n_ids > 0 && D > 0) {
        const long long slab = 1ll << 20;
        DevBuf dids;
        CKS(dids.ensure((size_t)std::min<long long>(n_ids, slab) * 8));
        for (long long o = 0; o < n_ids; o += slab) {
            const long long m = std::min(slab, n_ids - o);
            CK(cudaMemcpy(dids.p, doc_ids + o, (size_t)m * 8, cudaMemcpyHostToDevice));
            k_del_mark<<<grid, 256>>>(dids.as<long long>(), m, base, D, bits.as<uint32_t>());
            CK(cudaGetLastError());
        }
    }
    CKS(wcnt.ensure((size_t)(nw + 1) * 8));
    CKS(wpre.ensure((size_t)(nw + 1) * 8));
    k_del_popc<<<grid, 256>>>(bits.as<uint32_t>(), nw, wcnt.as<long long>());
    CK(cudaGetLastError());
    CKS(exclusive_sum(wcnt.as<long long>(), wpre.as<long long>(), nw + 1, tmp));
    CK(cudaMemcpy(n_del, wpre.as<long long>() + nw, 8, cudaMemcpyDeviceToHost));
    return PB_OK;
}

// What a delete computes before its first in-place write: the deleted set, the survivors and their new offsets, the
// filtered inverted file in the spare half, the compaction windows with their staging buffers, and the new totals
struct DeletePrep {
    long long D0 = 0, n_del = 0;
    DocTotals t;
    DevBuf bits, wpre, kept, new_doff, new_uoff, st_codes, st_res, st_u, mn;
    DevBuf cache_off, kept_count;  // with a row cache: the survivors' map and counts under their new ids
    long long dead_docs = 0, dead_tok = 0;  // the cached docs among the deleted ones, and their tokens
    std::vector<long long> hoff, hu;
    std::vector<uint32_t> hbits;
    std::vector<std::pair<long long, long long>> wins;
    Events ev;
};

// Every check and allocation of a delete and everything it computes out of place; nothing visible changes.  n_del = 0:
// nothing to do.  The caller holds the handle's writer lock.
static pb_status delete_prepare(pb_index *ix, const int64_t *doc_ids, int64_t n_ids, DeletePrep &p) {
    CK(cudaSetDevice(ix->device));
    CK(cudaDeviceSynchronize());  // work earlier readers left queued (pb_search_batch_device) reads the arrays
    const long long D0 = ix->D, K = ix->K, nw = (D0 + 31) / 32;
    const int grid = ix->sm_count * 8;
    p.D0 = D0;
    if (ix->profiling)
        for (cudaEvent_t &x : p.ev.e) CK(cudaEventCreate(&x));

    // 1. the deleted set: one bit per doc, its per-word prefix counts, and the number of docs deleted
    CKS(del_bitmap(ix, doc_ids, n_ids, ix->doc_id_base, D0, p.bits, p.wpre, &p.n_del));
    if (p.n_del == 0) return PB_OK;
    const long long D1 = D0 - p.n_del;

    // 2. the survivors kept[j] and their new doc_off / udoc_off, into scratch: the old ones are read until the commit
    DevBuf tlen, ulen, tmp;
    CKS(p.kept.ensure((size_t)std::max(D1, 1ll) * 8));
    CKS(tlen.ensure((size_t)(D1 + 1) * 8));
    CKS(ulen.ensure((size_t)(D1 + 1) * 8));
    CKS(p.new_doff.ensure((size_t)(D1 + 1) * 8));
    CKS(p.new_uoff.ensure((size_t)(D1 + 1) * 8));
    CK(cudaMemset(tlen.as<long long>() + D1, 0, 8));
    CK(cudaMemset(ulen.as<long long>() + D1, 0, 8));
    k_del_kept<<<grid, 256>>>(p.bits.as<uint32_t>(), p.wpre.as<long long>(), D0, ix->doc_off.as<long long>(),
                              ix->udoc_off.as<long long>(), p.kept.as<long long>(), tlen.as<long long>(), ulen.as<long long>());
    CK(cudaGetLastError());
    CKS(exclusive_sum(tlen.as<long long>(), p.new_doff.as<long long>(), D1 + 1, tmp));
    CKS(exclusive_sum(ulen.as<long long>(), p.new_uoff.as<long long>(), D1 + 1, tmp));
    std::vector<long long> &hoff = p.hoff, &hu = p.hu;
    hoff.resize((size_t)D1 + 1);
    hu.resize((size_t)D1 + 1);
    CK(cudaMemcpy(hoff.data(), p.new_doff.p, hoff.size() * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hu.data(), p.new_uoff.p, hu.size() * 8, cudaMemcpyDeviceToHost));
    p.t.D = D1;
    p.t.N = hoff[D1];
    p.t.n_ucodes = hu[D1];
    p.t.max_doclen = longest_doc(hoff, D1);
    if (ix->cache_off.p) {  // the row cache: survivors keep their entries, deleted cached docs' rows become dead
        DevBuf dead;
        CKS(p.cache_off.ensure((size_t)std::max(D1, 1ll) * 8));
        CKS(p.kept_count.ensure((size_t)std::max(D1, 1ll) * 4));
        CKS(dead.ensure(16));
        CK(cudaMemset(dead.p, 0, 16));
        k_cache_compact<<<grid, 256>>>(ix->cache_off.as<long long>(), ix->kept_count.as<uint32_t>(), p.kept.as<long long>(),
                                       D1, p.cache_off.as<long long>(), p.kept_count.as<uint32_t>());
        k_cache_dead<<<grid, 256>>>(ix->cache_off.as<long long>(), p.bits.as<uint32_t>(), ix->doc_off.as<long long>(), D0,
                                    dead.as<unsigned long long>());
        CK(cudaGetLastError());
        long long got[2] = {0, 0};
        CK(cudaMemcpy(got, dead.p, 16, cudaMemcpyDeviceToHost));
        p.dead_docs = got[0], p.dead_tok = got[1];
    }

    // 3. the inverted file without the deleted ids, renumbered, into the spare half
    if (ix->profiling) CK(cudaEventRecord(p.ev.e[0]));
    DevBuf icnt;
    CKS(icnt.ensure((size_t)(K + 1) * 8));
    CKS(ix->ivf_off_spare.ensure((size_t)(K + 1) * 8));
    k_ivf_delete_count<<<grid, 256>>>(ix->ivf.as<uint32_t>(), ix->ivf_off.as<long long>(), K, p.bits.as<uint32_t>(),
                                      icnt.as<long long>());
    CK(cudaGetLastError());
    CKS(exclusive_sum(icnt.as<long long>(), ix->ivf_off_spare.as<long long>(), K + 1, tmp));
    CK(cudaMemcpy(&p.t.ivf_len, ix->ivf_off_spare.as<long long>() + K, 8, cudaMemcpyDeviceToHost));
    CKS(ix->ivf_spare.grow(std::max<size_t>((size_t)p.t.ivf_len * 4, 16), 0));
    k_ivf_delete_write<<<grid, 256>>>(ix->ivf.as<uint32_t>(), ix->ivf_off.as<long long>(), K, p.bits.as<uint32_t>(),
                                      p.wpre.as<long long>(), ix->ivf_off_spare.as<long long>(), ix->ivf_spare.as<uint32_t>());
    CK(cudaGetLastError());
    if (ix->profiling) CK(cudaEventRecord(p.ev.e[1]));

    // 4. compaction windows over the survivors that move: those from the first deleted doc on (survivors before it keep
    // their rows; a delete of the newest docs moves nothing).  Each window is a run of survivors whose rows fit
    // delete_window tokens (a longer doc is a window of its own).
    p.hbits.resize((size_t)nw);
    CK(cudaMemcpy(p.hbits.data(), p.bits.p, (size_t)nw * 4, cudaMemcpyDeviceToHost));
    long long first = 0;
    while (p.hbits[(size_t)(first >> 5)] == 0) first += 32;
    first += __builtin_ctz(p.hbits[(size_t)(first >> 5)]);
    long long max_tok = 0, max_u = 0;
    for (long long j0 = first, j1; j0 < D1; j0 = j1) {
        for (j1 = j0 + 1; j1 < D1 && hoff[j1 + 1] - hoff[j0] <= ix->delete_window; ++j1) {}
        p.wins.emplace_back(j0, j1);
        max_tok = std::max(max_tok, hoff[j1] - hoff[j0]);
        max_u = std::max(max_u, hu[j1] - hu[j0]);
    }
    const size_t pk = (size_t)ix->packed;
    if (!p.wins.empty()) {
        CKS(p.st_codes.ensure(std::max<size_t>((size_t)max_tok * 4, 16)));
        CKS(p.st_res.ensure(std::max<size_t>((size_t)max_tok * pk, 16)));
        CKS(p.st_u.ensure(std::max<size_t>((size_t)max_u * 4, 16)));
    }
    CKS(p.mn.ensure(16));
    CK(cudaDeviceSynchronize());
    return PB_OK;
}

// The in-place part of a prepared delete, in two steps (delete_move, then delete_finish): only a CUDA runtime error
// can fail them.  delete_move compacts the arrays; a host-tier handle's survivors are gathered over the mapping into
// the device staging and copied back to the store at their new offsets, one copy per segment piece.  write_rows =
// false: another replica sharing the store moves them, before this handle's delete_finish reads them.
static pb_status delete_move(pb_index *ix, DeletePrep &p, bool write_rows) {
    if (p.n_del == 0) return PB_OK;
    const bool prof = ix->profiling && p.ev.e[0];
    const int grid = ix->sm_count * 8;
    const std::vector<long long> &hoff = p.hoff, &hu = p.hu;
    const size_t pk = (size_t)ix->packed;
    // 5. compaction
    if (prof) CK(cudaEventRecord(p.ev.e[2]));
    for (const auto &w : p.wins) {
        const long long j0 = w.first, j1 = w.second;
        const unsigned blocks = (unsigned)std::min<long long>((j1 - j0 + 7) / 8, grid);
        const long long *kp = p.kept.as<long long>();
        k_compact_gather<uint32_t><<<blocks, 256>>>(FlatRows{ix->codes.as<uint8_t>()}, ix->doc_off.as<long long>(), kp,
                                                    p.new_doff.as<long long>(), j0, j1, 4, p.st_codes.as<uint8_t>());
        auto gather_rows = [&](auto src) {
            if (pk % 16 == 0)
                k_compact_gather<uint4><<<blocks, 256>>>(src, ix->doc_off.as<long long>(), kp, p.new_doff.as<long long>(), j0,
                                                         j1, (int)pk, p.st_res.as<uint8_t>());
            else if (pk % 4 != 0)  // 1-bit rows of dim 48 (6 bytes)
                k_compact_gather<unsigned short><<<blocks, 256>>>(src, ix->doc_off.as<long long>(), kp,
                                                                  p.new_doff.as<long long>(), j0, j1, (int)pk,
                                                                  p.st_res.as<uint8_t>());
            else
                k_compact_gather<uint32_t><<<blocks, 256>>>(src, ix->doc_off.as<long long>(), kp, p.new_doff.as<long long>(),
                                                            j0, j1, (int)pk, p.st_res.as<uint8_t>());
        };
        if (!ix->host_tier) gather_rows(FlatRows{ix->residuals.as<uint8_t>()});
        else if (write_rows) gather_rows(ix->host.dev());
        // distinct-code blocks start at multiples of 8 codes (32 bytes)
        k_compact_gather<uint4><<<blocks, 256>>>(FlatRows{ix->ucodes.as<uint8_t>()}, ix->udoc_off.as<long long>(), kp,
                                                 p.new_uoff.as<long long>(), j0, j1, 4, p.st_u.as<uint8_t>());
        CK(cudaGetLastError());
        const long long nt = hoff[j1] - hoff[j0], nu = hu[j1] - hu[j0];
        CK(cudaMemcpy(ix->codes.as<uint8_t>() + (size_t)hoff[j0] * 4, p.st_codes.p, (size_t)nt * 4, cudaMemcpyDeviceToDevice));
        if (!ix->host_tier)
            CK(cudaMemcpy(ix->residuals.as<uint8_t>() + (size_t)hoff[j0] * pk, p.st_res.p, (size_t)nt * pk, cudaMemcpyDeviceToDevice));
        else if (write_rows)
            CKS(ix->host.rows->write((size_t)hoff[j0] * pk, p.st_res.as<uint8_t>(), (size_t)nt * pk, PB_MEM_DEVICE));
        CK(cudaMemcpy(ix->ucodes.as<uint8_t>() + (size_t)hu[j0] * 4, p.st_u.p, (size_t)nu * 4, cudaMemcpyDeviceToDevice));
    }
    CK(cudaMemcpy(ix->doc_off.p, p.new_doff.p, (size_t)(p.t.D + 1) * 8, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(ix->udoc_off.p, p.new_uoff.p, (size_t)(p.t.D + 1) * 8, cudaMemcpyDeviceToDevice));
    if (ix->cache_off.p) {
        ix->cache_off.swap(p.cache_off);
        ix->kept_count.swap(p.kept_count);
        const long long b = p.dead_tok * ix->packed;
        ix->rc.docs -= p.dead_docs, ix->rc.bytes -= b, ix->rc.dead += b;
    }
    if (prof) CK(cudaEventRecord(p.ev.e[3]));
    return PB_OK;
}

static pb_status delete_finish(pb_index *ix, DeletePrep &p) {
    if (p.n_del == 0) return PB_OK;
    const bool prof = ix->profiling && p.ev.e[0];
    // 6. 1 / |c + w| of the survivors in their new order, and vmin / wmax over them as an open computes them: the old
    // constants would still bound the error, but the work counters would differ from a fresh open
    const float seed[2] = {3.0e38f, 0.0f};
    CKS(token_norms(ix, *ix, 0, seed, p.t, p.mn));
    if (prof) CK(cudaEventRecord(p.ev.e[4]));
    CK(cudaDeviceSynchronize());

    // 7. commit
    publish(ix, p.t);
    if (prof) {
        CK(cudaEventElapsedTime(&ix->delete_ms[0], p.ev.e[2], p.ev.e[3]));
        CK(cudaEventElapsedTime(&ix->delete_ms[1], p.ev.e[0], p.ev.e[1]));
        CK(cudaEventElapsedTime(&ix->delete_ms[2], p.ev.e[3], p.ev.e[4]));
    }
    return PB_OK;
}

static pb_status delete_commit(pb_index *ix, DeletePrep &p, bool write_rows = true) {
    CKS(delete_move(ix, p, write_rows));
    return delete_finish(ix, p);
}

extern "C" pb_status pb_index_delete(pb_index *ix, const int64_t *doc_ids, int64_t n_ids, const char *index_dir,
                                     int64_t *out_deleted) {
    if (!ix || (!doc_ids && n_ids) || n_ids < 0) return pb_fail(PB_ERR_INVALID, "null argument");
    if (out_deleted) *out_deleted = 0;
    if (ix->group) return ix->group->del(doc_ids, n_ids, index_dir, out_deleted);
    return pb_members_delete({ix}, doc_ids, n_ids, index_dir, out_deleted);
}

// ------------------------------------------------------------------------------------------
// device row cache of a host-tier handle (DESIGN.md 4s): the rows of a chosen set of docs, in spare device memory, which
// search staging copies device to device instead of over PCIe
// ------------------------------------------------------------------------------------------
static pb_status refuse_row_cache(const pb_index *ix) {
    if (!ix->residuals.owned)
        return pb_fail(PB_ERR_UNSUPPORTED, "the handle uses the caller's residual array (PB_OPEN_ADOPT_RESIDUALS)");
    if (!ix->host_tier)
        return pb_fail(PB_ERR_UNSUPPORTED, "a row cache serves host-tier handles (PB_OPEN_HOST_RESIDUALS) only");
    return PB_OK;
}

// The cache emptied: no rows, every map entry -1.  The caller holds the writer lock.
static pb_status row_cache_clear(pb_index *ix) {
    CK(cudaDeviceSynchronize());  // pb_search_batch_device may have left staging work that reads the rows
    DevBuf().swap(ix->rc.rows);
    CK(cudaMemset(ix->cache_off.p, 0xff, (size_t)ix->D * 8));
    ix->rc.docs = ix->rc.bytes = ix->rc.dead = 0;
    return PB_OK;
}

extern "C" pb_status pb_index_set_row_cache(pb_index *ix, int64_t max_bytes) {
    if (max_bytes < 0) return pb_fail(PB_ERR_INVALID, "row cache budget %lld < 0", (long long)max_bytes);
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix->group) return ix->group->in_turn(true, [&](pb_index *m) { return pb_index_set_row_cache(m, max_bytes); });
    CKS(refuse_row_cache(ix));
    std::lock_guard<std::mutex> f(ix->rc.fill_mu);
    DevBuf off, cnt;  // the old arrays leave with these, after the locks
    std::lock_guard<std::mutex> gate(ix->gate);
    std::unique_lock<std::shared_mutex> wr(ix->rw);
    CK(cudaSetDevice(ix->device));
    if (max_bytes == 0) {
        if (ix->cache_off.p) CKS(row_cache_clear(ix));
        ix->cache_off.swap(off);
        ix->kept_count.swap(cnt);
        ix->rc.budget = 0;
        return PB_OK;
    }
    if (!ix->cache_off.p) {  // every allocation before the first change
        CKS(off.ensure((size_t)std::max(ix->D, 1ll) * 8));
        CKS(cnt.ensure((size_t)std::max(ix->D, 1ll) * 4));
        CK(cudaMemset(off.p, 0xff, (size_t)ix->D * 8));
        CK(cudaMemset(cnt.p, 0, (size_t)ix->D * 4));
        ix->cache_off.swap(off);
        ix->kept_count.swap(cnt);
    }
    ix->rc.budget = (size_t)max_bytes;
    if ((size_t)(ix->rc.bytes + ix->rc.dead) > ix->rc.budget) CKS(row_cache_clear(ix));
    return PB_OK;
}

// The docs a fill caches, in the order it takes them: by counts (doc_ids == NULL) the docs kept at least once, most
// kept first and ties by id, else the caller's ids in its order, those outside [0, D) and repeats ignored; each taken
// when its rows still fit the budget, skipped otherwise.  off: their token offsets in the new cache, and the total.
static void row_cache_pick(const std::vector<long long> &doff, const std::vector<uint32_t> *count, const int64_t *doc_ids,
                           int64_t n_ids, long long base, long long pk, size_t budget, std::vector<uint32_t> &pick,
                           std::vector<long long> &off) {
    const long long D = (long long)doff.size() - 1;
    std::vector<uint32_t> order;
    if (count) {
        for (long long d = 0; d < D; ++d)
            if ((*count)[d]) order.push_back((uint32_t)d);
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return (*count)[a] > (*count)[b]; });
    } else {
        std::vector<uint8_t> seen((size_t)D, 0);
        for (int64_t i = 0; i < n_ids; ++i) {
            const long long d = doc_ids[i] - base;
            if (d < 0 || d >= D || seen[d]) continue;
            seen[d] = 1;
            order.push_back((uint32_t)d);
        }
    }
    off.assign(1, 0);
    for (uint32_t d : order) {
        const long long len = doff[d + 1] - doff[d];
        if ((size_t)((off.back() + len) * pk) > budget) continue;
        pick.push_back(d);
        off.push_back(off.back() + len);
    }
}

// A plain handle's fill: the new map and rows built out of place under the reader lock, so that searches go on with
// the old cache and mutations wait; then swapped under the writer lock.  A mutation that ran between the two (the
// reader lock cannot become the writer lock in place) makes the fill start again on the new documents.
static pb_status row_cache_fill(pb_index *ix, const int64_t *doc_ids, int64_t n_ids, int64_t *out_ids, int64_t out_cap,
                                int64_t *out_n) {
    CKS(refuse_row_cache(ix));
    std::lock_guard<std::mutex> f(ix->rc.fill_mu);
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
        std::vector<uint32_t> pick;
        std::vector<long long> off;
        DevBuf map, rows, dpick, doff;  // the new cache; after the swap the old one, freed after the locks
        unsigned long long gen = 0;
        {
            auto rd = ix->read_lock();
            if (!ix->rc.budget) return pb_fail(PB_ERR_INVALID, "the handle has no row cache budget (pb_index_set_row_cache)");
            CK(cudaSetDevice(ix->device));
            gen = ix->doc_gen;
            const long long D = ix->D;
            std::vector<long long> hoff((size_t)D + 1);
            CK(cudaMemcpy(hoff.data(), ix->doc_off.p, hoff.size() * 8, cudaMemcpyDeviceToHost));
            std::vector<uint32_t> count;
            if (!doc_ids) {
                count.resize((size_t)D);
                CK(cudaMemcpy(count.data(), ix->kept_count.p, (size_t)D * 4, cudaMemcpyDeviceToHost));
            }
            row_cache_pick(hoff, doc_ids ? nullptr : &count, doc_ids, n_ids, ix->doc_id_base, ix->packed, ix->rc.budget,
                           pick, off);
            std::vector<long long> hmap((size_t)D, -1);
            for (size_t i = 0; i < pick.size(); ++i) hmap[pick[i]] = off[i];
            CKS(map.ensure((size_t)std::max(D, 1ll) * 8));
            if (D) CK(cudaMemcpy(map.p, hmap.data(), (size_t)D * 8, cudaMemcpyHostToDevice));
            const long long tok = off.back();
            if (tok > 0) {  // the chosen docs' rows: already cached ones device to device, the others over PCIe
                CKS(rows.grow((size_t)tok * ix->packed, 0, false));
                CKS(upload(dpick, pick.data(), pick.size() * 4, PB_MEM_HOST));
                CKS(upload(doff, off.data(), off.size() * 8, PB_MEM_HOST));
                CKS(launch_stage_rows(ix, 0, dpick.as<uint32_t>(), nullptr, 0, (long long)pick.size(), doff.as<long long>(),
                                      row_cache_view(ix, nullptr, false), rows.as<uint8_t>(), nullptr, nullptr));
                CK(cudaStreamSynchronize(0));
            }
        }
        std::lock_guard<std::mutex> gate(ix->gate);
        std::unique_lock<std::shared_mutex> wr(ix->rw);
        if (ix->doc_gen != gen) continue;
        CK(cudaSetDevice(ix->device));
        CK(cudaDeviceSynchronize());  // pb_search_batch_device may have left staging work that reads the old cache
        ix->cache_off.swap(map);
        ix->rc.rows.swap(rows);
        if (!doc_ids) CK(cudaMemset(ix->kept_count.p, 0, (size_t)ix->D * 4));
        ix->rc.docs = (long long)pick.size();
        ix->rc.bytes = off.back() * ix->packed;
        ix->rc.dead = 0;
        ix->rc.fill_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        *out_n = (int64_t)pick.size();
        for (size_t i = 0; out_ids && i < pick.size() && (int64_t)i < out_cap; ++i)
            out_ids[i] = (int64_t)pick[i] + ix->doc_id_base;
        return PB_OK;
    }
}

extern "C" pb_status pb_index_fill_row_cache(pb_index *ix, const int64_t *doc_ids, int64_t n_ids, int64_t *out_ids,
                                             int64_t out_cap, int64_t *out_n) {
    if (!ix || !out_n || (!doc_ids && n_ids > 0) || (doc_ids && n_ids < 0) || (out_ids && out_cap < 0))
        return pb_fail(PB_ERR_INVALID, "null argument");
    *out_n = 0;
    if (!ix->group) return row_cache_fill(ix, doc_ids, n_ids, out_ids, out_cap, out_n);
    // ranks or replicas in order, each writing its ids after the previous ones'
    auto one = [&](pb_index *m) {
        const int64_t at = std::min(*out_n, out_cap);
        int64_t n = 0;
        const pb_status s = pb_index_fill_row_cache(m, doc_ids, n_ids, out_ids ? out_ids + at : nullptr, out_cap - at, &n);
        *out_n += n;
        return s;
    };
    return ix->group->in_turn(true, one);
}

extern "C" pb_status pb_index_row_cache_stats(pb_index *ix, pb_row_cache_stats *out, int32_t reset) {
    if (!ix || !out) return pb_fail(PB_ERR_INVALID, "null argument");
    *out = pb_row_cache_stats{};
    if (ix->group) {  // sums over the ranks or replicas
        auto one = [&](pb_index *m) {
            pb_row_cache_stats s{};
            CKS(pb_index_row_cache_stats(m, &s, reset));
            out->budget_bytes += s.budget_bytes, out->cached_docs += s.cached_docs, out->cached_bytes += s.cached_bytes;
            out->dead_bytes += s.dead_bytes, out->staged_docs += s.staged_docs, out->hit_docs += s.hit_docs;
            out->hit_bytes += s.hit_bytes, out->last_fill_ms += s.last_fill_ms;
            return PB_OK;
        };
        return ix->group->in_turn(false, one);
    }
    auto rd = ix->read_lock();
    RowCacheState &c = ix->rc;
    out->budget_bytes = (int64_t)c.budget, out->cached_docs = c.docs, out->cached_bytes = c.bytes;
    out->dead_bytes = c.dead, out->last_fill_ms = c.fill_ms;
    out->staged_docs = reset ? c.staged.exchange(0) : c.staged.load();
    out->hit_docs = reset ? c.hit_docs.exchange(0) : c.hit_docs.load();
    out->hit_bytes = reset ? c.hit_bytes.exchange(0) : c.hit_bytes.load();
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// replicas (DESIGN §4q): a handle copied onto another device, and appends and deletes applied to several plain handles
// of the same documents as one
// ------------------------------------------------------------------------------------------
// dst: a copy of src's whole allocation (on the current device, which is dst_dev), issued on st
static pb_status clone_buf(DevBuf &dst, const DevBuf &src, int dst_dev, int src_dev, cudaStream_t st) {
    if (!src.p) return PB_OK;
    cudaError_t e = cudaMalloc(&dst.p, src.cap);
    if (e != cudaSuccess) {
        cudaGetLastError();
        dst.p = nullptr;
        return pb_fail(PB_ERR_NOMEM, "cudaMalloc(%zu bytes) failed: %s", src.cap, cudaGetErrorString(e));
    }
    dst.cap = src.cap, dst.owned = true, dst.zero_on_grow = src.zero_on_grow;
    CK(cudaMemcpyPeerAsync(dst.p, dst_dev, src.p, src_dev, src.cap, st));
    return PB_OK;
}

pb_status pb_index_clone(const pb_index *src, int device, pb_index **out) {
    *out = nullptr;
    auto rd = src->read_lock();
    CKS(check_device(device));
    std::unique_ptr<pb_index> ix(new pb_index());
    static_cast<DocTotals &>(*ix) = static_cast<const DocTotals &>(*src);
    ix->device = device;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    ix->sm_count = prop.multiProcessorCount;  // the grids sized from it follow the copy's device
    ix->dim = src->dim, ix->nbits = src->nbits, ix->packed = src->packed, ix->K = src->K, ix->doc_id_base = src->doc_id_base;
    ix->host_tier = src->host_tier, ix->build_ivf = src->build_ivf, ix->cmax = src->cmax, ix->cent_exp = src->cent_exp;
    static_cast<Switches &>(*ix) = static_cast<const Switches &>(*src);
    ix->host_mutable = src->host_mutable;
    if (src->host_tier) {  // the store is shared; the table is the copy's device's own
        ix->host.rows = src->host.rows;
        CK(cudaSetDevice(device));
        CKS(ix->host.sync());
    }
    OwnedStream st;
    CK(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
    const auto mine = DocArrays::buffers(*ix);
    const auto theirs = DocArrays::buffers(*src);
    for (size_t i = 0; i < mine.size(); ++i) CKS(clone_buf(*mine[i], *theirs[i], device, src->device, st.s));
    CKS(clone_buf(ix->centroids, src->centroids, device, src->device, st.s));
    CKS(clone_buf(ix->w_rev, src->w_rev, device, src->device, st.s));
    CKS(clone_buf(ix->cent_h16t, src->cent_h16t, device, src->device, st.s));
    CKS(clone_buf(ix->cent_l16t, src->cent_l16t, device, src->device, st.s));
    // a row cache: its map and counts are per-doc arrays (above), its rows and what they hold follow
    CKS(clone_buf(ix->rc.rows, src->rc.rows, device, src->device, st.s));
    ix->rc.budget = src->rc.budget, ix->rc.docs = src->rc.docs, ix->rc.bytes = src->rc.bytes, ix->rc.dead = src->rc.dead;
    CK(cudaStreamSynchronize(st.s));
    CKS(coalesce_env_defaults(ix.get()));
    *out = ix.release();
    return PB_OK;
}

pb_status pb_index_clone_empty(const pb_index *src, int device, long long doc_id_base, pb_index **out) {
    *out = nullptr;
    auto rd = src->read_lock();
    if (!src->residuals.owned || src->host_tier)
        return pb_fail(PB_ERR_UNSUPPORTED, "an empty rank beside one that uses the caller's residual array or host memory "
                                           "(PB_OPEN_ADOPT_RESIDUALS / PB_OPEN_HOST_RESIDUALS)");
    CKS(check_device(device));
    std::unique_ptr<pb_index> ix(new pb_index());
    ix->device = device;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    ix->sm_count = prop.multiProcessorCount;
    ix->dim = src->dim, ix->nbits = src->nbits, ix->packed = src->packed, ix->K = src->K, ix->doc_id_base = doc_id_base;
    ix->cmax = src->cmax;
    static_cast<Switches &>(*ix) = static_cast<const Switches &>(*src);
    // the per-doc arrays of no documents, allocated as an open of an empty range allocates them
    const long long zero = 0;
    CKS(upload(ix->doc_off, &zero, 8, PB_MEM_HOST));
    CKS(upload(ix->udoc_off, &zero, 8, PB_MEM_HOST));
    CKS(ix->ivf_off.ensure((size_t)(ix->K + 1) * 8));
    for (DevBuf *b : {&ix->codes, &ix->residuals, &ix->ucodes, &ix->ivf}) CKS(b->ensure(16));
    OwnedStream st;
    CK(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
    CK(cudaMemsetAsync(ix->ivf_off.p, 0, (size_t)(ix->K + 1) * 8, st.s));
    CKS(clone_buf(ix->centroids, src->centroids, device, src->device, st.s));
    CKS(clone_buf(ix->w_rev, src->w_rev, device, src->device, st.s));
    CK(cudaStreamSynchronize(st.s));
    CKS(coalesce_env_defaults(ix.get()));
    *out = ix.release();
    return PB_OK;
}

// The encoded rows of tokens [t0, t0 + n) of a handle, on the host: codes widened to i64 and packed residual rows
static pb_status tail_rows(const pb_index *ix, long long t0, long long n, std::vector<int64_t> &codes,
                           std::vector<uint8_t> &res) {
    const size_t pk = (size_t)ix->packed;
    std::vector<uint32_t> c32((size_t)n);
    res.resize((size_t)n * pk);
    if (n) {
        CK(cudaSetDevice(ix->device));
        CK(cudaMemcpy(c32.data(), ix->codes.as<uint32_t>() + t0, (size_t)n * 4, cudaMemcpyDeviceToHost));
        CKS(rows_to_host(ix, t0, n, res.data()));
    }
    codes.assign(c32.begin(), c32.end());
    return PB_OK;
}

Replicas *pb_replicas_of(const pb_index *ix) { return ix && ix->group ? ix->group->as_replicas() : nullptr; }
void pb_index_copy_switches(pb_index *dst, pb_index *src) {
    if (!dst->group) {
        static_cast<Switches &>(*dst) = static_cast<const Switches &>(*src);
        return;
    }
    int32_t world = 0;
    pb_index_shard_layout(dst, &world, nullptr, nullptr);
    for (int r = 0; r < world; ++r) pb_index_copy_switches(pb_rank_of(dst, r), pb_rank_of(src, r));
}
pb_index *pb_rank_of(pb_index *ix, int r) { return ix->group && ix->group->as_deployment() ? ix->group->member(r) : ix; }
bool pb_host_rows_shared(pb_index *ix) { return pb_rank_of(ix, 0)->host_mutable; }
pb_status pb_sync_devices(pb_index *ix) {
    pb_status st = PB_OK;
    auto sync = [&](pb_index *r) {
        if (st == PB_OK && (cudaSetDevice(r->device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess))
            st = pb_fail(PB_ERR_CUDA, "synchronizing device %d failed", r->device);
    };
    if (ix->group) ix->group->each(sync);
    else sync(ix);
    return st;
}

// Every member's writer lock, in member order
struct MembersLock {
    std::vector<std::unique_lock<std::mutex>> gates;
    std::vector<std::unique_lock<std::shared_mutex>> rws;
    explicit MembersLock(const std::vector<pb_index *> &ms) {
        for (pb_index *m : ms) {
            gates.emplace_back(m->gate);
            rws.emplace_back(m->rw);
        }
    }
};

pb_status pb_members_append(const std::vector<pb_index *> &ms, pb_codec *codec, const float *embeddings,
                            const int64_t *codes, const uint8_t *residuals, const int64_t *doc_lengths, int64_t n_docs,
                            int32_t space, const char *index_dir, int64_t batch_size, int64_t *out_first) {
    pb_index *ix = ms[0];
    // append_impl's checks, in its order
    if ((!doc_lengths && n_docs) || n_docs < 0) return pb_fail(PB_ERR_INVALID, "null argument");
    if (space != PB_MEM_HOST && space != PB_MEM_DEVICE) return pb_fail(PB_ERR_INVALID, "bad memory_space %d", space);
    MembersLock lock(ms);
    if (ix->comm.joined()) return pb_fail(PB_ERR_UNSUPPORTED, "appends to a doc-sharded handle are not supported");
    CKS(refuse_fixed_residuals(ix));
    if (index_dir && ix->doc_id_base != 0) return pb_fail(PB_ERR_UNSUPPORTED, "an index directory holds doc ids from 0");
    if (index_dir && batch_size <= 0) return pb_fail(PB_ERR_INVALID, "batch_size must be positive");
    std::vector<std::unique_ptr<AppendPrep>> p;
    for (size_t g = 0; g < ms.size(); ++g) p.emplace_back(new AppendPrep());
    // 1. prepare: member 0 as one handle would (with a codec, the only encode); the others from its encoded rows
    pb_status st = append_prepare(ix, codec, embeddings, codes, residuals, doc_lengths, n_docs, space,
                                  index_dir != nullptr, out_first, *p[0]);
    // host tier: member 0 wrote the rows to the store the members share, and may have moved its segments
    for (size_t g = 1; g < ms.size() && ix->host_tier; ++g) {
        CK(cudaSetDevice(ms[g]->device));
        const pb_status s = ms[g]->host.sync();
        if (st == PB_OK) st = s;
    }
    CKS(st);
    if (p[0]->n == 0) return PB_OK;
    if (ms.size() > 1) {
        const AppendPrep &a = *p[0];
        std::vector<int64_t> hc;
        std::vector<uint8_t> hr;
        CKS(tail_rows(ix, a.t.N - a.ntok, a.ntok, hc, hr));
        for (size_t g = 1; g < ms.size(); ++g)
            CKS(append_prepare(ms[g], nullptr, nullptr, hc.data(), hr.data(), a.dl.data(), n_docs, PB_MEM_HOST, false,
                               nullptr, *p[g], false));
    }
    // 2. the directory, once, before any commit: a failure leaves every member as it was
    if (index_dir) {
        std::vector<int64_t> hivf;
        std::vector<int32_t> hlen;
        CK(cudaSetDevice(ix->device));
        CKS(ivf_to_host(ix, ix->ivf_spare, ix->ivf_off_spare, p[0]->t.ivf_len, hivf, hlen));
        CKS(append_dir(ix, *p[0], index_dir, p[0]->D0, batch_size, hivf, p[0]->t.ivf_len, hlen));
    }
    // 3. commit everywhere
    for (size_t g = 0; g < ms.size(); ++g) publish(ms[g], p[g]->t);
    return PB_OK;
}

pb_status pb_members_delete(const std::vector<pb_index *> &ms, const int64_t *doc_ids, int64_t n_ids, const char *index_dir,
                            int64_t *out_deleted) {
    pb_index *ix = ms[0];
    if (out_deleted) *out_deleted = 0;
    MembersLock lock(ms);
    // pb_index_delete's checks, in its order
    if (ix->comm.joined()) return pb_fail(PB_ERR_UNSUPPORTED, "deletes from a doc-sharded handle are not supported");
    CKS(refuse_fixed_residuals(ix));
    if (index_dir && ix->doc_id_base != 0) return pb_fail(PB_ERR_UNSUPPORTED, "an index directory holds doc ids from 0");
    std::vector<std::unique_ptr<DeletePrep>> p;
    for (size_t g = 0; g < ms.size(); ++g) {
        p.emplace_back(new DeletePrep());
        CKS(delete_prepare(ms[g], doc_ids, n_ids, *p[g]));
        if (p[0]->n_del == 0) return PB_OK;
    }
    if (index_dir) {
        std::vector<int64_t> hivf;
        std::vector<int32_t> hlen;
        CK(cudaSetDevice(ix->device));
        CKS(ivf_to_host(ix, ix->ivf_spare, ix->ivf_off_spare, p[0]->t.ivf_len, hivf, hlen));
        CKS(pb_dir_delete(index_dir, p[0]->D0, ix->K, ix->dim, ix->nbits, p[0]->hbits.data(), hivf.data(), p[0]->t.ivf_len,
                          hlen.data()));
    }
    // from here only a CUDA runtime error can fail a member, and that leaves the set to be reloaded.  Host tier: member
    // 0 moves the rows of the store the members share, and every member's norm pass reads them after it
    for (size_t g = 0; g < ms.size(); ++g) {
        CK(cudaSetDevice(ms[g]->device));
        CKS(delete_commit(ms[g], *p[g], g == 0));
    }
    if (out_deleted) *out_deleted = p[0]->n_del;
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// appends and deletes on a doc-sharded deployment (DESIGN §4h).  Every rank prepares locally, then one all-gather of a
// fixed record lets all ranks reach the same verdict from the same data: commit everywhere or nowhere.  Rank world - 1
// writes the directory from ivf.npy on disk; a second exchange carries its status.  After the vote only a CUDA runtime
// error can fail a rank.
// ------------------------------------------------------------------------------------------
// The first exchange of a sharded collective (update or rebalance) carries one record per rank: this head, then the
// operation's own word (the local deletion count of an update, the adopt flag of a rebalance), then an FNV-1a
// fingerprint of the arguments
enum { LR_STATUS, LR_RANK, LR_WORLD, LR_BASE, LR_D, LR_N, LR_K, LR_DIM, LR_NBITS, LR_OWN, LR_PRINT, LR_WORDS };
enum { SH_OP_DELETE = 1, SH_OP_APPEND = 2, SH_OP_APPEND_ENCODED = 3 };

// every rank's `words` 64-bit words, in rank order; a communicator outside any group is a group of one
static pb_status gather_words(ShardComm &comm, const long long *mine, int words, std::vector<long long> &all,
                              bool unbounded = false) {
    all.assign(mine, mine + words);
    if (!comm.joined()) return PB_OK;
    all.resize((size_t)words * comm.world);
    OwnedStream st;
    DevBuf send, recv;
    CK(cudaSetDevice(comm.device));
    CK(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
    CKS(send.ensure((size_t)words * 8));
    CKS(recv.ensure((size_t)words * 8 * comm.world));
    CK(cudaMemcpy(send.p, mine, (size_t)words * 8, cudaMemcpyHostToDevice));
    CKS(comm.allgather(st.s, send.p, recv.p, (size_t)words, unbounded));
    CK(cudaStreamSynchronize(st.s));
    CK(cudaMemcpy(all.data(), recv.p, all.size() * 8, cudaMemcpyDeviceToHost));
    return PB_OK;
}
static pb_status gather_words(pb_index *ix, const long long *mine, int words, std::vector<long long> &all,
                              bool unbounded = false) {
    return gather_words(ix->comm, mine, words, all, unbounded);
}

// the status of the lowest failing rank, or PB_OK; the failing rank keeps its own message, the others name it
static pb_status first_failure(const ShardComm &comm, const std::vector<long long> &all, int words, const char *what) {
    for (int r = 0; r < comm.world; ++r) {
        const pb_status s = (pb_status)all[(size_t)r * words];
        if (s == PB_OK) continue;
        if (r == comm.rank) {
            const std::string own = g_err;
            return pb_fail(s, "rank %d: %s", r, own.c_str());
        }
        return pb_fail(s, "rank %d of the group failed (status %d)%s", r, (int)s, what);
    }
    return PB_OK;
}
static pb_status first_failure(pb_index *ix, const std::vector<long long> &all, int words, const char *what) {
    return first_failure(ix->comm, all, words, what);
}

// Exchange A of a sharded collective and the verdict every rank reaches from the same records.  The caller has set
// the status, its own word and the fingerprint of `rec`; the head is filled in here.  The lowest failing rank's
// status, a rank whose layout differs from rank 0's, documents that do not tile [0, D) and a fingerprint that differs
// from rank 0's (a call with other `args`) fail every rank.  Gives every rank's record (all), the ranks' first
// documents (base [W + 1], base[W] = D_total) and first tokens (tok [W + 1]).
static pb_status layout_vote(pb_index *ix, long long *rec, const char *args, std::vector<long long> &all,
                             std::vector<long long> &base, std::vector<long long> &tok) {
    const int W = ix->comm.world;
    rec[LR_RANK] = ix->comm.rank;
    rec[LR_WORLD] = W;
    rec[LR_BASE] = ix->doc_id_base;
    rec[LR_D] = ix->D;
    rec[LR_N] = ix->N;
    rec[LR_K] = ix->K;
    rec[LR_DIM] = ix->dim;
    rec[LR_NBITS] = ix->nbits;
    CKS(gather_words(ix, rec, LR_WORDS, all));
    CKS(first_failure(ix, all, LR_WORDS, "; nothing changed"));
    auto at = [&](int r, int w) { return all[(size_t)r * LR_WORDS + w]; };
    base.assign((size_t)W + 1, 0);
    tok.assign((size_t)W + 1, 0);
    for (int r = 0; r < W; ++r) {
        if (at(r, LR_RANK) != r || at(r, LR_WORLD) != W || at(r, LR_K) != at(0, LR_K) || at(r, LR_DIM) != at(0, LR_DIM) ||
            at(r, LR_NBITS) != at(0, LR_NBITS))
            return pb_fail(PB_ERR_INVALID, "rank %d's layout (rank %lld of %lld, K=%lld dim=%lld nbits=%lld) differs from rank 0's",
                           r, at(r, LR_RANK), at(r, LR_WORLD), at(r, LR_K), at(r, LR_DIM), at(r, LR_NBITS));
        if (at(r, LR_BASE) != base[r])
            return pb_fail(PB_ERR_INVALID, "the ranks' documents do not tile [0, D): rank %d starts at %lld, not %lld", r,
                           at(r, LR_BASE), base[r]);
        if (at(r, LR_PRINT) != at(0, LR_PRINT))
            return pb_fail(PB_ERR_INVALID, "rank %d was called with other %s than rank 0", r, args);
        base[r + 1] = base[r] + at(r, LR_D);
        tok[r + 1] = tok[r] + at(r, LR_N);
    }
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// The replicas of a set of deployments (S > 1, replicas.cpp, DESIGN §4q) vote on a mutation together, so that it
// commits on every replica or on none: every rank of every replica takes the same rounds, and a rank that returns
// early counts, for every later round, with the status it returned.  A round fails with the lowest failing replica's
// status.  With a codec, replica 0's last rank also hands the rows it encoded to the other replicas, which wait for them
// before they prepare: the append encodes once.
// ------------------------------------------------------------------------------------------
struct RepVote {
    int ranks = 0;
    bool with_dir = false, share_rows = false;
    std::mutex mu;
    std::condition_variable cv;
    struct Entry {
        int round, replica;
        pb_status st;
        std::string msg;
        bool left;
    };
    std::vector<Entry> entries;
    bool rows_ready = false;
    pb_status rows_st = PB_OK;
    std::string rows_msg;
    std::vector<int64_t> dl, codes;
    std::vector<uint8_t> res;
    // round k's votes: the ranks that voted in it and the ranks that left before or at it
    int count(int k) const {
        int c = 0;
        for (const Entry &e : entries) c += e.left ? e.round <= k : e.round == k;
        return c;
    }
    const Entry *failure(int k) const {
        const Entry *f = nullptr;
        for (const Entry &e : entries)
            if (e.st != PB_OK && (e.left ? e.round <= k : e.round == k) && (!f || e.replica < f->replica)) f = &e;
        return f;
    }
};

RepVote *pb_rep_vote_new(int ranks, bool with_dir, bool share_rows) {
    RepVote *v = new RepVote();
    v->ranks = ranks, v->with_dir = with_dir, v->share_rows = share_rows;
    return v;
}
void pb_rep_vote_free(RepVote *v) { delete v; }
void pb_index_set_rep_vote(pb_index *member, RepVote *v, int replica) {
    auto set = [&](pb_index *r) { r->rep_vote = v, r->rep_index = replica; };
    if (member->group) member->group->each(set);
    else set(member);
}

// One rank's turns in its replica set's vote (nothing without one)
struct RepTurn {
    RepVote *v;
    int replica, round = 0;
    explicit RepTurn(const pb_index *ix) : v(ix->rep_vote), replica(ix->rep_index) {}
    bool with_dir() const { return v && v->with_dir; }
    // waits for every rank; the round's verdict (a failing rank keeps its own message)
    pb_status vote(pb_status mine) {
        if (!v) return mine;
        const std::string msg = mine == PB_OK ? std::string() : g_err;
        std::unique_lock<std::mutex> lk(v->mu);
        const int k = round++;
        v->entries.push_back({k, replica, mine, msg, false});
        v->cv.notify_all();
        v->cv.wait(lk, [&] { return v->count(k) >= v->ranks; });
        const RepVote::Entry *f = v->failure(k);
        if (!f) return PB_OK;
        if (mine != PB_OK) return mine;
        return pb_fail(f->st, "replica %d failed (%s); nothing changed", f->replica, f->msg.c_str());
    }
    // the rank returns with status st: it counts so for the rounds it did not take
    void leave(pb_status st) {
        if (!v) return;
        std::lock_guard<std::mutex> lk(v->mu);
        v->entries.push_back({round, replica, st, st == PB_OK ? std::string() : g_err, true});
        if (v->share_rows && replica == 0 && !v->rows_ready && st != PB_OK)  // replica 0 failed before it could share
            v->rows_ready = true, v->rows_st = st, v->rows_msg = g_err;
        v->cv.notify_all();
    }
    // replica 0's last rank: the rows its prepare encoded (or why it failed), for the other replicas
    void share(pb_status st, pb_index *ix, const AppendPrep &ap) {
        std::vector<int64_t> codes;
        std::vector<uint8_t> res;
        if (st == PB_OK && ap.n > 0) st = tail_rows(ix, ap.t.N - ap.ntok, ap.ntok, codes, res);
        std::lock_guard<std::mutex> lk(v->mu);
        v->rows_st = st, v->rows_msg = st == PB_OK ? std::string() : g_err;
        v->dl = ap.dl, v->codes = std::move(codes), v->res = std::move(res);
        v->rows_ready = true;
        v->cv.notify_all();
    }
    // another replica's rank: replica 0's encoded rows, once they are there
    pb_status rows(const std::vector<int64_t> *&dl, const std::vector<int64_t> *&codes, const std::vector<uint8_t> *&res) {
        std::unique_lock<std::mutex> lk(v->mu);
        v->cv.wait(lk, [&] { return v->rows_ready; });
        if (v->rows_st != PB_OK) return pb_fail(v->rows_st, "replica 0 failed (%s); nothing changed", v->rows_msg.c_str());
        dl = &v->dl, codes = &v->codes, res = &v->res;
        return PB_OK;
    }
};

static pb_status sharded_update_body(pb_index *ix, RepTurn &turn, int op, pb_codec *codec, const float *embeddings,
                                     const int64_t *codes, const uint8_t *residuals, const int64_t *doc_lengths,
                                     const int64_t *doc_ids, int64_t n, int32_t space, const char *index_dir,
                                     int64_t batch_size, int64_t *out);

static pb_status sharded_update(pb_index *ix, int op, pb_codec *codec, const float *embeddings, const int64_t *codes,
                                const uint8_t *residuals, const int64_t *doc_lengths, const int64_t *doc_ids, int64_t n,
                                int32_t space, const char *index_dir, int64_t batch_size, int64_t *out) {
    if (out) *out = 0;
    std::lock_guard<std::mutex> gate(ix->gate);
    std::unique_lock<std::shared_mutex> wr(ix->rw);
    RepTurn turn(ix);
    const pb_status s = sharded_update_body(ix, turn, op, codec, embeddings, codes, residuals, doc_lengths, doc_ids, n,
                                            space, index_dir, batch_size, out);
    turn.leave(s);
    return s;
}

static pb_status sharded_update_body(pb_index *ix, RepTurn &turn, int op, pb_codec *codec, const float *embeddings,
                                     const int64_t *codes, const uint8_t *residuals, const int64_t *doc_lengths,
                                     const int64_t *doc_ids, int64_t n, int32_t space, const char *index_dir,
                                     int64_t batch_size, int64_t *out) {
    const bool last = ix->comm.rank == ix->comm.world - 1;
    DeletePrep dp;
    AppendPrep ap;
    long long rec[LR_WORDS] = {};
    // a replica other than 0 of an append with a codec: every rank waits for replica 0's encoded rows, so that the
    // group's exchange below does not time out while replica 0 encodes; the last rank appends them
    const bool takes_rows = turn.v && turn.v->share_rows && turn.replica > 0;
    // host tier: rank r of every replica shares replica 0's rank r's row store, which only replica 0 writes
    const bool write_rows = !(ix->host_tier && turn.v && turn.replica > 0);
    pb_status rows_st = PB_OK;
    if (takes_rows) {
        const std::vector<int64_t> *dl = nullptr, *cd = nullptr;
        const std::vector<uint8_t> *rs = nullptr;
        rows_st = turn.rows(dl, cd, rs);
        if (rows_st == PB_OK) codes = cd->data(), residuals = rs->data(), doc_lengths = dl->data(), space = PB_MEM_HOST;
        // replica 0's prepare may have moved the store's segments, whether it then failed or not
        if (ix->host_tier) {
            pb_status s = cudaSetDevice(ix->device) == cudaSuccess ? ix->host.sync()
                                                                    : pb_fail(PB_ERR_CUDA, "cudaSetDevice failed");
            if (rows_st == PB_OK) rows_st = s;
        }
    }
    // 1. local checks, the fingerprint of the arguments, and the prepare: no early return, or the peers would wait
    auto local = [&]() -> pb_status {
        CKS(rows_st);
        if (n < 0 || (n && !(op == SH_OP_DELETE ? doc_ids : doc_lengths))) return pb_fail(PB_ERR_INVALID, "null argument");
        if (op != SH_OP_DELETE && space != PB_MEM_HOST && space != PB_MEM_DEVICE)
            return pb_fail(PB_ERR_INVALID, "bad memory_space %d", space);
        CKS(refuse_fixed_residuals(ix));
        if (index_dir && op == SH_OP_APPEND && batch_size <= 0) return pb_fail(PB_ERR_INVALID, "batch_size must be positive");
        if (op == SH_OP_APPEND && last && !codec && !takes_rows) return pb_fail(PB_ERR_INVALID, "null argument");
        std::vector<int64_t> args;
        if (op == SH_OP_DELETE) args.assign(doc_ids, doc_ids + n);
        else CKS(fetch_host(args, doc_lengths, (size_t)n, space));
        Fnv64 f;
        f.put(op);
        f.put((long long)n);
        f.add(args.data(), args.size() * 8);
        f.put(index_dir != nullptr);
        if (index_dir) f.add(index_dir, strlen(index_dir) + 1);
        f.put((long long)(op == SH_OP_APPEND ? batch_size : 0));
        rec[LR_PRINT] = (long long)f.h;
        if (op == SH_OP_DELETE) {
            CKS(delete_prepare(ix, doc_ids, n, dp));
            rec[LR_OWN] = dp.n_del;
        } else if (last) {
            CKS(append_prepare(ix, takes_rows ? nullptr : codec, embeddings, codes, residuals, doc_lengths, n, space,
                               index_dir != nullptr, nullptr, ap, write_rows));
        }
        return PB_OK;
    };
    rec[LR_STATUS] = local();
    if (turn.v && turn.v->share_rows && turn.replica == 0 && last) turn.share((pb_status)rec[LR_STATUS], ix, ap);

    // 2. exchange A and the verdict every rank reaches from the same records
    std::vector<long long> all, base, tok;
    CKS(layout_vote(ix, rec, "arguments", all, base, tok));
    const long long D_total = base[ix->comm.world];
    long long n_del = 0, del_before = 0;
    for (int r = 0; r < ix->comm.world; ++r) {
        if (r < ix->comm.rank) del_before += all[(size_t)r * LR_WORDS + LR_OWN];
        n_del += all[(size_t)r * LR_WORDS + LR_OWN];
    }
    if (op == SH_OP_DELETE && n_del == 0) return PB_OK;  // nothing changes, on any rank or on disk
    if (op != SH_OP_DELETE && out) *out = D_total;
    if (op != SH_OP_DELETE && n == 0) return PB_OK;

    // the replicas of a set: every replica prepared, or none writes the directory
    CKS(turn.vote(PB_OK));

    // 3. the directory, written by the last rank from ivf.npy as it is on disk; exchange B carries its status
    if (index_dir) {
        long long wrec = PB_OK;
        if (last) {
            auto total = [](const std::vector<int32_t> &len) {
                long long t = 0;
                for (int32_t x : len) t += x;
                return t;
            };
            auto write = [&]() -> pb_status {
                CKS(pb_dir_check_documents(index_dir, ix->nbits, D_total));
                std::vector<int64_t> hivf;
                std::vector<int32_t> hlen;
                if (op == SH_OP_DELETE) {
                    DevBuf gbits, gwpre;
                    long long g = 0;
                    CKS(del_bitmap(ix, doc_ids, n, 0, D_total, gbits, gwpre, &g));
                    CKS(pb_dir_patch_ivf(ix, index_dir, D_total, gbits.as<uint32_t>(), gwpre.as<long long>(), nullptr, 0, hivf, hlen));
                    std::vector<uint32_t> hbits((size_t)(D_total + 31) / 32);
                    CK(cudaMemcpy(hbits.data(), gbits.p, hbits.size() * 4, cudaMemcpyDeviceToHost));
                    return pb_dir_delete(index_dir, D_total, ix->K, ix->dim, ix->nbits, hbits.data(), hivf.data(),
                                         total(hlen), hlen.data());
                }
                CKS(pb_dir_patch_ivf(ix, index_dir, D_total, nullptr, nullptr, ap.keys.as<uint64_t>(), ap.m, hivf, hlen));
                return append_dir(ix, ap, index_dir, D_total, batch_size, hivf, total(hlen), hlen);
            };
            wrec = write();
        }
        // the peers wait for the writer however long the write takes: a timeout here would leave the directory
        // changed and every handle unchanged
        std::vector<long long> wall;
        CKS(gather_words(ix, &wrec, 1, wall, true));
        CKS(first_failure(ix, wall, 1, " writing the index directory; no rank changed"));
    }

    if (turn.with_dir()) CKS(turn.vote(PB_OK));  // replica 0 wrote the directory

    // 4. commit everywhere: from here only a CUDA runtime error can fail a rank, and that leaves the group inconsistent
    if (op == SH_OP_DELETE) {
        CKS(delete_move(ix, dp, write_rows));
        // host tier: every replica's norm pass reads the rows replica 0 has just moved
        if (ix->host_tier && turn.v) CKS(turn.vote(PB_OK));
        CKS(delete_finish(ix, dp));
        ix->doc_id_base -= del_before;
        if (out) *out = n_del;
    } else if (last) {
        publish(ix, ap.t);
    }
    return PB_OK;
}

extern "C" pb_status pb_index_delete_sharded(pb_index *ix, const int64_t *doc_ids, int64_t n_ids, const char *index_dir,
                                             int64_t *out_deleted) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_deployment(ix, "pb_index_delete_sharded (call pb_index_delete)"));
    return sharded_update(ix, SH_OP_DELETE, nullptr, nullptr, nullptr, nullptr, nullptr, doc_ids, n_ids, PB_MEM_HOST,
                          index_dir, 0, out_deleted);
}

extern "C" pb_status pb_index_append_sharded(pb_index *ix, pb_codec *codec, const float *embeddings,
                                             const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space,
                                             const char *index_dir, int64_t batch_size, int64_t *out_first_doc_id) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_deployment(ix, "pb_index_append_sharded (call pb_index_append)"));
    return sharded_update(ix, SH_OP_APPEND, codec, embeddings, nullptr, nullptr, doc_lengths, nullptr, n_docs, memory_space,
                          index_dir, batch_size, out_first_doc_id);
}

extern "C" pb_status pb_index_append_encoded_sharded(pb_index *ix, const int64_t *codes, const uint8_t *residuals,
                                                     const int64_t *doc_lengths, int64_t n_docs, int32_t memory_space,
                                                     int64_t *out_first_doc_id) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_deployment(ix, "pb_index_append_encoded_sharded (call pb_index_append_encoded)"));
    return sharded_update(ix, SH_OP_APPEND_ENCODED, nullptr, nullptr, codes, residuals, doc_lengths, nullptr, n_docs,
                          memory_space, nullptr, 0, out_first_doc_id);
}

// ------------------------------------------------------------------------------------------
// rebalance of a doc-sharded deployment (DESIGN §4i): the ranks take new document ranges over the same global ids.
// Exchange A checks the layout as §4h does; balanced bounds come from one offer per boundary and rank; every rank
// derives the same plan from the old bounds a and the new ones b: the piece s -> r is docs [max(a_s, b_r),
// min(a_s+1, b_r+1)).  A rank whose range changes builds its new arrays out of place: its pieces' rows arrive at their
// final offsets, then the scans, the merge of the inverted file and the norm pass run over them.  The old arrays stay
// until the last vote, so a failure anywhere leaves every rank as it was.
// ------------------------------------------------------------------------------------------
enum { SZ_TOK, SZ_UCODES, SZ_IVF, SZ_WORDS };  // per piece in the size exchange
// what moves with a piece of documents, in the order both ends issue it
enum { XF_CODES, XF_RES, XF_UCODES, XF_TLEN, XF_ULEN, XF_IVF_OFF, XF_IVF, XF_ITEMS };

struct RebalancePrep {
    std::vector<long long> hoff, huoff;  // the rank's doc_off / udoc_off as they are
    // sender: its pieces' bounds q [W + 1] in local ids, per-doc lengths, the inverted file split by destination with
    // its offsets [W][K + 1], and where each piece's entries start in it (hsplit [W + 1])
    DevBuf q, tlen, ulen, split, split_off;
    std::vector<long long> hsplit;
    // receiver: the new arrays with their totals, and the per-doc lengths and inverted-file segments of its pieces as
    // they arrive
    DocArrays nx;
    DevBuf rlen, rulen, seg, seg_off, meta, mn;
};

static pb_status rebalance_body(pb_index *ix, RepTurn &turn, const int64_t *bounds, const uint8_t *shares,
                                int64_t *out_bounds);

extern "C" pb_status pb_index_rebalance_sharded(pb_index *ix, const int64_t *bounds, int64_t *out_bounds) {
    if (!ix) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix->group) return ix->group->rebalance(bounds, out_bounds);
    return pb_index_rebalance_shares(ix, bounds, nullptr, out_bounds);
}

// The calls that change a deployment's number of ranks (DESIGN §4t) address a deployment of pb_index_load_devices only;
// those that change a replica set's number of replicas (§4u), a replica set of pb_index_load_replicas only
static pb_status refuse_resize(const pb_index *ix, const char *call, bool replicas = false) {
    if (ix->group) {
        const bool mine = replicas ? ix->group->as_replicas() != nullptr : ix->group->as_deployment() != nullptr;
        return mine ? PB_OK : ix->group->refuse(call);
    }
    return pb_fail(PB_ERR_UNSUPPORTED, "%s needs %s (this handle is %s)", call,
                   replicas ? "a replica set of pb_index_load_replicas" : "a multi-device handle of pb_index_load_devices",
                   ix->comm.joined() ? "a rank of a doc-sharded group" : "a single index");
}

extern "C" pb_status pb_index_add_devices(pb_index *ix, const int32_t *devices, int32_t n_devices, const int64_t *bounds,
                                          int64_t *out_bounds) {
    if (!ix || !devices) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_resize(ix, "pb_index_add_devices"));
    return pb_dep_add_devices(ix->group->as_deployment(), devices, n_devices, bounds, out_bounds);
}

extern "C" pb_status pb_index_remove_ranks(pb_index *ix, const int32_t *ranks, int32_t n_ranks, const int64_t *bounds,
                                           int64_t *out_bounds) {
    if (!ix || !ranks) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_resize(ix, "pb_index_remove_ranks"));
    return pb_dep_remove_ranks(ix->group->as_deployment(), ix, ranks, n_ranks, bounds, out_bounds);
}

extern "C" pb_status pb_index_add_replicas(pb_index *ix, const int32_t *devices, int32_t n_devices) {
    if (!ix || !devices) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_resize(ix, "pb_index_add_replicas", true));
    return pb_rep_add(ix->group->as_replicas(), ix, devices, n_devices);
}

extern "C" pb_status pb_index_remove_replicas(pb_index *ix, const int32_t *replicas, int32_t n_replicas) {
    if (!ix || !replicas) return pb_fail(PB_ERR_INVALID, "null argument");
    CKS(refuse_resize(ix, "pb_index_remove_replicas", true));
    return pb_rep_remove(ix->group->as_replicas(), ix, replicas, n_replicas);
}

pb_status pb_index_rebalance_shares(pb_index *ix, const int64_t *bounds, const uint8_t *shares, int64_t *out_bounds) {
    std::lock_guard<std::mutex> gate(ix->gate);
    std::unique_lock<std::shared_mutex> wr(ix->rw);
    RepTurn turn(ix);
    const pb_status s = rebalance_body(ix, turn, bounds, shares, out_bounds);
    turn.leave(s);
    return s;
}

static pb_status rebalance_body(pb_index *ix, RepTurn &turn, const int64_t *bounds, const uint8_t *shares,
                                int64_t *out_bounds) {
    const int W = ix->comm.world, me = ix->comm.rank;
    const long long K = ix->K;
    const size_t pk = (size_t)ix->packed;
    const int grid = ix->sm_count * 8;
    RebalancePrep p;
    long long rec[LR_WORDS] = {};
    // 1. local checks, the fingerprint of the bounds and the host copies of the offsets: no early return, or the peers
    // would wait
    auto local = [&]() -> pb_status {
        Fnv64 f;
        f.put(bounds != nullptr);
        if (bounds) f.add(bounds, (size_t)(W + 1) * 8);
        f.put(shares != nullptr);
        if (shares) f.add(shares, (size_t)W);
        rec[LR_PRINT] = (long long)f.h;
        if (!ix->comm.has_p2p())
            return pb_fail(PB_ERR_COMM, "the NCCL library lacks ncclSend / ncclRecv / ncclGroupStart / ncclGroupEnd");
        CK(cudaSetDevice(ix->device));
        CK(cudaDeviceSynchronize());  // work earlier readers left queued (pb_search_batch_device) reads the arrays
        p.hoff.resize((size_t)ix->D + 1);
        p.huoff.resize((size_t)ix->D + 1);
        CK(cudaMemcpy(p.hoff.data(), ix->doc_off.p, p.hoff.size() * 8, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(p.huoff.data(), ix->udoc_off.p, p.huoff.size() * 8, cudaMemcpyDeviceToHost));
        return PB_OK;
    };
    rec[LR_STATUS] = local();
    rec[LR_OWN] = !ix->residuals.owned || ix->host_tier;  // a residual array that cannot move

    // 2. exchange A and the verdict every rank reaches from the same records
    std::vector<long long> all, a, tok;  // records, old bounds, global token offsets
    CKS(layout_vote(ix, rec, "bounds", all, a, tok));
    for (int r = 0; r < W; ++r)
        if (all[(size_t)r * LR_WORDS + LR_OWN])
            return pb_fail(PB_ERR_UNSUPPORTED,
                           "rank %d uses the caller's residual array or host memory (PB_OPEN_ADOPT_RESIDUALS / "
                           "PB_OPEN_HOST_RESIDUALS)", r);
    const long long D_total = a[W], N_total = tok[W];

    // 3. the new bounds: the caller's, or the token-balanced split c[j] = min { d : off[d] S >= N j } of the global doc
    // offsets over the S ranks that take a share (every rank, unless `shares` leaves some out).  For that each rank
    // offers the least d of its closed range [a_me, a_me+1] that qualifies (global off[d] = tok[me] + its own
    // doc_off), or D_total; the least offer wins.  The j-th sharing rank takes [c[j], c[j+1]), and a rank without a
    // share the empty range where the next sharing rank starts.
    std::vector<long long> b((size_t)W + 1, 0);
    if (bounds) {
        b.assign(bounds, bounds + W + 1);
        bool ok = b[0] == 0 && b[W] == D_total;
        for (int r = 0; r < W; ++r) ok = ok && b[r] <= b[r + 1];
        if (!ok) return pb_fail(PB_ERR_INVALID, "bounds must be non-decreasing from 0 to D_total = %lld", D_total);
    } else {
        int S = 0;
        for (int r = 0; r < W; ++r) S += !shares || shares[r];
        if (S == 0) return pb_fail(PB_ERR_INVALID, "no rank takes a share of the documents");
        std::vector<long long> offer((size_t)S + 1, D_total), offers, c((size_t)S + 1, D_total);
        for (int j = 1; j < S; ++j) {
            long long lo = 0, hi = ix->D + 1;  // the first local i with (tok[me] + doc_off[i]) S >= N j, or D + 1
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if ((tok[me] + p.hoff[mid]) * S >= N_total * j) hi = mid; else lo = mid + 1;
            }
            if (lo <= ix->D) offer[j] = a[me] + lo;
        }
        CKS(gather_words(ix, offer.data(), S + 1, offers));
        c[0] = 0;
        for (int j = 1; j < S; ++j)
            for (int s = 0; s < W; ++s) c[j] = std::min(c[j], offers[(size_t)s * (S + 1) + j]);
        for (int r = 0, j = 0; r < W; ++r) {
            b[r] = c[j];
            j += !shares || shares[r];
        }
        b[W] = D_total;
    }
    if (b == a) {  // nothing moves
        if (out_bounds) std::copy(b.begin(), b.end(), out_bounds);
        return PB_OK;
    }

    // 4. the plan, and the sender's side of the prepare: per-doc lengths and the inverted file split by destination
    auto piece = [&](int s, int r, long long &lo, long long &hi) {
        lo = std::max(a[s], b[r]);
        hi = std::min(a[s + 1], b[r + 1]);
        return lo < hi;
    };
    const bool changes = a[me] != b[me] || a[me + 1] != b[me + 1];
    const int SW = 1 + SZ_WORDS * W;  // status, then per destination its piece's tokens, distinct codes, ivf entries
    std::vector<long long> srec((size_t)SW, 0);
    auto prepare = [&]() -> pb_status {
        if (!changes) return PB_OK;
        const long long Dm = ix->D, n = (long long)W * (K + 1);
        std::vector<long long> q((size_t)W + 1);
        for (int r = 0; r <= W; ++r) q[r] = std::min(std::max(b[r] - a[me], 0ll), Dm);
        CKS(upload(p.q, q.data(), q.size() * 8, PB_MEM_HOST));
        CKS(p.tlen.ensure(std::max<size_t>((size_t)Dm * 8, 16)));
        CKS(p.ulen.ensure(std::max<size_t>((size_t)Dm * 8, 16)));
        if (Dm > 0)
            k_doc_lengths<<<grid, 256>>>(ix->doc_off.as<long long>(), ix->udoc_off.as<long long>(), Dm,
                                         p.tlen.as<long long>(), p.ulen.as<long long>());
        DevBuf cnt, tmp;
        CKS(cnt.ensure((size_t)n * 8));
        CKS(p.split_off.ensure((size_t)n * 8));
        CK(cudaMemset(cnt.p, 0, (size_t)n * 8));
        k_ivf_split_count<<<grid, 256>>>(ix->ivf.as<uint32_t>(), ix->ivf_off.as<long long>(), K, p.q.as<long long>(), W,
                                         cnt.as<long long>());
        CK(cudaGetLastError());
        CKS(exclusive_sum(cnt.as<long long>(), p.split_off.as<long long>(), n, tmp));
        p.hsplit.assign((size_t)W + 1, 0);
        for (int r = 0; r < W; ++r)
            CK(cudaMemcpy(&p.hsplit[r], p.split_off.as<long long>() + (size_t)r * (K + 1), 8, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(&p.hsplit[W], p.split_off.as<long long>() + n - 1, 8, cudaMemcpyDeviceToHost));  // cnt[n - 1] = 0
        CKS(p.split.ensure(std::max<size_t>((size_t)p.hsplit[W] * 4, 16)));
        CK(cudaMemcpy(cnt.p, p.split_off.p, (size_t)n * 8, cudaMemcpyDeviceToDevice));  // the write pass's cursors
        k_ivf_split_write<<<grid, 256>>>(ix->ivf.as<uint32_t>(), ix->ivf_off.as<long long>(), K, p.q.as<long long>(), W,
                                         cnt.as<long long>(), p.split.as<uint32_t>());
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        for (int r = 0; r < W; ++r) {
            long long lo, hi;
            if (!piece(me, r, lo, hi)) continue;
            lo -= a[me];
            hi -= a[me];
            srec[1 + SZ_WORDS * r + SZ_TOK] = p.hoff[hi] - p.hoff[lo];
            srec[1 + SZ_WORDS * r + SZ_UCODES] = p.huoff[hi] - p.huoff[lo];
            srec[1 + SZ_WORDS * r + SZ_IVF] = p.hsplit[r + 1] - p.hsplit[r];
        }
        return PB_OK;
    };
    srec[0] = prepare();
    std::vector<long long> sizes;
    CKS(gather_words(ix, srec.data(), SW, sizes));
    CKS(first_failure(ix, sizes, SW, "; nothing changed"));
    auto sz = [&](int s, int r, int k) { return sizes[(size_t)s * SW + 1 + SZ_WORDS * r + k]; };

    // the receiver's side: where each source's piece lands, and the new arrays, sized to their contents (the last rank
    // keeps the spare capacity it had, so appends provisioned by pb_index_reserve still need no growth copy)
    std::vector<long long> tpos((size_t)W + 1, 0), upos((size_t)W + 1, 0), ipos((size_t)W + 1, 0);
    for (int s = 0; s < W; ++s) {
        tpos[s + 1] = tpos[s] + sz(s, me, SZ_TOK);
        upos[s + 1] = upos[s] + sz(s, me, SZ_UCODES);
        ipos[s + 1] = ipos[s] + sz(s, me, SZ_IVF);
    }
    DocArrays &nx = p.nx;
    auto allocate = [&]() -> pb_status {
        if (!changes) return PB_OK;
        nx.D = b[me + 1] - b[me];
        nx.N = tpos[W];
        nx.n_ucodes = upos[W];
        nx.ivf_len = ipos[W];
        if (nx.ivf_len > (1ll << 31) - 2) return pb_fail(PB_ERR_UNSUPPORTED, "more than 2^31 (centroid, doc) pairs per shard");
        const bool last = me == W - 1;
        auto alloc = [&](DevBuf &nb, const DevBuf &old, long long old_bytes, long long bytes) {
            const size_t spare = last && (long long)old.cap > old_bytes ? old.cap - (size_t)old_bytes : 0;
            return nb.grow(std::max<size_t>((size_t)bytes + spare, 16), 0, false);
        };
        const long long D0 = ix->D, N0 = ix->N, D1 = nx.D;
        CKS(alloc(nx.codes, ix->codes, N0 * 4, nx.N * 4));
        CKS(alloc(nx.residuals, ix->residuals, N0 * (long long)pk, nx.N * (long long)pk));
        CKS(alloc(nx.ucodes, ix->ucodes, ix->n_ucodes * 4, nx.n_ucodes * 4));
        CKS(alloc(nx.doc_off, ix->doc_off, (D0 + 1) * 8, (D1 + 1) * 8));
        CKS(alloc(nx.udoc_off, ix->udoc_off, (D0 + 1) * 8, (D1 + 1) * 8));
        CKS(alloc(nx.ivf, ix->ivf, ix->ivf_len * 4, nx.ivf_len * 4));
        if (last && ix->ivf_spare.cap) CKS(alloc(nx.ivf_spare, ix->ivf_spare, ix->ivf_len * 4, nx.ivf_len * 4));
        if (TcDims::has(ix->dim) && nx.N > 0) CKS(alloc(nx.tok_inv_norm, ix->tok_inv_norm, N0 * 4, nx.N * 4));
        CKS(nx.ivf_off.grow((size_t)(K + 1) * 8, 0, false));
        // the spare offsets hold K + 1 entries whatever the documents: a rank that had them keeps their capacity
        if (ix->ivf_off_spare.cap) CKS(nx.ivf_off_spare.grow(ix->ivf_off_spare.cap, 0, false));
        CKS(p.rlen.ensure((size_t)(D1 + 1) * 8));
        CKS(p.rulen.ensure((size_t)(D1 + 1) * 8));
        CKS(p.seg.ensure(std::max<size_t>((size_t)nx.ivf_len * 4, 16)));
        CKS(p.seg_off.ensure((size_t)W * (K + 1) * 8));
        CK(cudaMemset(p.seg_off.p, 0, (size_t)W * (K + 1) * 8));  // a source without a piece has empty lists
        CKS(p.mn.ensure(16));
        std::vector<long long> meta((size_t)2 * W, 0);  // [segbase W][idoff W]
        for (int s = 0; s < W; ++s) {
            long long lo, hi;
            meta[s] = ipos[s];
            if (piece(s, me, lo, hi)) meta[W + s] = lo - b[me];
        }
        CKS(upload(p.meta, meta.data(), meta.size() * 8, PB_MEM_HOST));
        return PB_OK;
    };
    long long vote = allocate();
    std::vector<long long> votes;
    CKS(gather_words(ix, &vote, 1, votes));
    CKS(first_failure(ix, votes, 1, " allocating its new arrays; nothing changed"));

    // 5. the transfer: rows of codes, residuals, distinct codes and per-doc lengths as contiguous ranges, and the
    // inverted-file pieces, from the senders' arrays into the receivers' new arrays at their final offsets
    std::vector<const void *> sp((size_t)W * XF_ITEMS, nullptr);  // what I send, [destination][item]
    std::vector<size_t> sbytes((size_t)W * XF_ITEMS, 0);
    std::vector<void *> rp((size_t)W * XF_ITEMS, nullptr);  // where I receive, [source][item]
    std::vector<size_t> rbytes((size_t)W * XF_ITEMS, 0);
    if (changes) {
        for (int r = 0; r < W; ++r) {
            long long lo, hi;
            if (!piece(me, r, lo, hi)) continue;
            lo -= a[me];
            hi -= a[me];
            const void **s = &sp[(size_t)r * XF_ITEMS];
            size_t *n = &sbytes[(size_t)r * XF_ITEMS];
            s[XF_CODES] = ix->codes.as<uint8_t>() + (size_t)p.hoff[lo] * 4;
            n[XF_CODES] = (size_t)sz(me, r, SZ_TOK) * 4;
            s[XF_RES] = ix->residuals.as<uint8_t>() + (size_t)p.hoff[lo] * pk;
            n[XF_RES] = (size_t)sz(me, r, SZ_TOK) * pk;
            s[XF_UCODES] = ix->ucodes.as<uint8_t>() + (size_t)p.huoff[lo] * 4;
            n[XF_UCODES] = (size_t)sz(me, r, SZ_UCODES) * 4;
            s[XF_TLEN] = p.tlen.as<long long>() + lo;
            s[XF_ULEN] = p.ulen.as<long long>() + lo;
            n[XF_TLEN] = n[XF_ULEN] = (size_t)(hi - lo) * 8;
            s[XF_IVF_OFF] = p.split_off.as<long long>() + (size_t)r * (K + 1);
            n[XF_IVF_OFF] = (size_t)(K + 1) * 8;
            s[XF_IVF] = p.split.as<uint32_t>() + p.hsplit[r];
            n[XF_IVF] = (size_t)sz(me, r, SZ_IVF) * 4;
        }
        for (int s = 0; s < W; ++s) {
            long long lo, hi;
            if (!piece(s, me, lo, hi)) continue;
            void **d = &rp[(size_t)s * XF_ITEMS];
            size_t *n = &rbytes[(size_t)s * XF_ITEMS];
            d[XF_CODES] = nx.codes.as<uint8_t>() + (size_t)tpos[s] * 4;
            n[XF_CODES] = (size_t)sz(s, me, SZ_TOK) * 4;
            d[XF_RES] = nx.residuals.as<uint8_t>() + (size_t)tpos[s] * pk;
            n[XF_RES] = (size_t)sz(s, me, SZ_TOK) * pk;
            d[XF_UCODES] = nx.ucodes.as<uint8_t>() + (size_t)upos[s] * 4;
            n[XF_UCODES] = (size_t)sz(s, me, SZ_UCODES) * 4;
            d[XF_TLEN] = p.rlen.as<long long>() + (lo - b[me]);
            d[XF_ULEN] = p.rulen.as<long long>() + (lo - b[me]);
            n[XF_TLEN] = n[XF_ULEN] = (size_t)(hi - lo) * 8;
            d[XF_IVF_OFF] = p.seg_off.as<long long>() + (size_t)s * (K + 1);
            n[XF_IVF_OFF] = (size_t)(K + 1) * 8;
            d[XF_IVF] = p.seg.as<uint32_t>() + ipos[s];
            n[XF_IVF] = (size_t)sz(s, me, SZ_IVF) * 4;
        }
    }
    auto transfer = [&]() -> pb_status {
        OwnedStream st;
        const cudaError_t ce = cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking);
        if (ce != cudaSuccess) {
            ix->comm.fail();  // the peers must not wait for me at the barriers of the exchange
            return pb_fail(PB_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(ce));
        }
        return ix->comm.exchange(st.s, XF_ITEMS, sp.data(), sbytes.data(), rp.data(), rbytes.data());
    };
    // the receiver's new doc_off / udoc_off (scans of the arrived lengths), inverted file and norms
    auto build = [&]() -> pb_status {
        const long long D1 = nx.D;
        DevBuf tmp, len;
        CK(cudaMemset(p.rlen.as<long long>() + D1, 0, 8));
        CK(cudaMemset(p.rulen.as<long long>() + D1, 0, 8));
        CKS(exclusive_sum(p.rlen.as<long long>(), nx.doc_off.as<long long>(), D1 + 1, tmp));
        CKS(exclusive_sum(p.rulen.as<long long>(), nx.udoc_off.as<long long>(), D1 + 1, tmp));
        std::vector<long long> hoff((size_t)D1 + 1);
        long long u1 = 0, l1 = 0;
        CK(cudaMemcpy(hoff.data(), nx.doc_off.p, hoff.size() * 8, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(&u1, nx.udoc_off.as<long long>() + D1, 8, cudaMemcpyDeviceToHost));
        nx.max_doclen = longest_doc(hoff, D1);
        CKS(len.ensure((size_t)(K + 1) * 8));
        k_ivf_rebalance_count<<<(unsigned)((K + 256) / 256), 256>>>(p.seg_off.as<long long>(), W, K, len.as<long long>());
        CK(cudaGetLastError());
        CKS(exclusive_sum(len.as<long long>(), nx.ivf_off.as<long long>(), K + 1, tmp));
        CK(cudaMemcpy(&l1, nx.ivf_off.as<long long>() + K, 8, cudaMemcpyDeviceToHost));
        if (hoff[D1] != nx.N || u1 != nx.n_ucodes || l1 != nx.ivf_len)
            return pb_fail(PB_ERR_CUDA, "the received pieces (%lld tokens, %lld codes, %lld ivf entries) differ from the "
                           "plan (%lld, %lld, %lld)", hoff[D1], u1, l1, nx.N, nx.n_ucodes, nx.ivf_len);
        if (nx.ivf_len > 0)
            k_ivf_rebalance_merge<<<grid, 256>>>(p.seg.as<uint32_t>(), p.seg_off.as<long long>(), p.meta.as<long long>(),
                                                 p.meta.as<long long>() + W, W, K, nx.ivf_off.as<long long>(),
                                                 nx.ivf.as<uint32_t>());
        CK(cudaGetLastError());
        // 1 / |c + w| of the new tokens and vmin / wmax over them, as an open computes them
        const float seed[2] = {3.0e38f, 0.0f};
        CKS(token_norms(ix, nx, 0, seed, nx, p.mn));
        CK(cudaDeviceSynchronize());
        return PB_OK;
    };
    long long fin = transfer();
    if (fin == PB_OK && changes) fin = build();

    // 6. the last vote covers the transfer and the build; then every rank swaps in its new arrays, which cannot fail
    CKS(gather_words(ix, &fin, 1, votes, true));
    CKS(first_failure(ix, votes, 1, " moving the documents; nothing changed"));
    CKS(turn.vote(PB_OK));  // the replicas of a set: every replica moved its documents, or none commits
    if (changes) {
        publish(ix, nx, &nx);
        ix->doc_id_base = b[me];
    }
    if (out_bounds) std::copy(b.begin(), b.end(), out_bounds);
    return PB_OK;  // the old arrays are freed with p
}

extern "C" pb_status pb_last_delete_ms(pb_index *ix, float *out_ms) {
    if (!ix || !out_ms) return pb_fail(PB_ERR_INVALID, "null argument");
    if (ix->group) return ix->group->last_delete_ms(out_ms);
    auto rd = ix->read_lock();
    memcpy(out_ms, ix->delete_ms, sizeof ix->delete_ms);
    return PB_OK;
}

// ------------------------------------------------------------------------------------------
// Collective index build (DESIGN §4n): pb_create_index_sharded, with pb_create_index as its one-rank case.  Every rank
// computes the same sample plan over global doc ids; it uploads only its own rows (k-means fit points and seeds, and
// held-out rows for the trainer, rank 0), encodes its documents straight into its shard, writes the chunks that start
// in its range (the head of a chunk that crosses into a later rank comes over the communicator) and its pieces of
// ivf.npy.  A vote ends every phase that can fail on one rank alone.
// ------------------------------------------------------------------------------------------
enum { CV_STATUS, CV_RANK, CV_WORLD, CV_D, CV_N, CV_DIM, CV_NBITS, CV_NITERS, CV_MPP, CV_PARTS, CV_BATCH, CV_SEED, CV_K,
       CV_CENT, CV_DIR, CV_TOKEN, CV_WORDS };
enum { CP_PLAN, CP_KMEANS, CP_CODEC, CP_ENCODE, CP_SHARD, CP_CHUNKS, CP_IVF, CP_COUNT };
static thread_local float g_create_ms[CP_COUNT];

// one word per rank: the lowest failing rank's status on every rank.  Waits for late peers (a phase may keep one rank
// busy much longer than the others)
static pb_status create_vote(ShardComm &comm, pb_status local, const char *what) {
    const long long v = local;
    std::vector<long long> all;
    CKS(gather_words(comm, &v, 1, all, true));
    return first_failure(comm, all, 1, what);
}

// rows `tok` (this rank's token ids) of its embeddings [N][dim] (host or device) into out, in that order
static pb_status gather_rows(const float *emb, int space, int dim, const std::vector<long long> &tok, DevBuf &out, int sms,
                             cudaStream_t st) {
    CKS(out.ensure(std::max<size_t>(tok.size() * dim * 4, 16)));
    if (tok.empty()) return PB_OK;
    if (space == PB_MEM_HOST) {
        std::vector<float> h(tok.size() * dim);
        for (size_t i = 0; i < tok.size(); ++i) memcpy(h.data() + i * dim, emb + (size_t)tok[i] * dim, (size_t)dim * 4);
        CK(cudaMemcpy(out.p, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
        return PB_OK;
    }
    DevBuf idx;
    CKS(upload(idx, tok.data(), tok.size() * 8, PB_MEM_HOST));
    k_gather_rows_i64<<<sms * 8, 256, 0, st>>>(emb, idx.as<long long>(), (long long)tok.size(), dim, out.as<float>());
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    return PB_OK;
}

struct IndexCloser {
    void operator()(pb_index *ix) const { pb_index_close(ix); }
};

static pb_status create_collective(pb_build_comm *c, const float *emb, const int64_t *doc_lengths, int64_t n_docs, int dim,
                                   int space, const float *centroids_in, int64_t num_centroids, const pb_create_params *params,
                                   const char *index_dir, pb_index **out_shard, int64_t *out_first) {
    using clock = std::chrono::steady_clock;
    for (float &v : g_create_ms) v = 0.0f;
    auto t_lap = clock::now();
    auto lap = [&](int phase) {
        const auto now = clock::now();
        g_create_ms[phase] += std::chrono::duration<float, std::milli>(now - t_lap).count();
        t_lap = now;
    };
    ShardComm &comm = c->comm;
    const int R = comm.rank, W = comm.world;
    cudaStream_t st = c->stream.s;
    CK(cudaSetDevice(comm.device));

    // ---- 1. the vote on the arguments, and the directory check ----
    long long rec[CV_WORDS] = {};
    long long n_tok = 0;
    bool token = false;
    auto local = [&]() -> pb_status {
        if (!params || !index_dir || n_docs < 0 || (n_docs && !doc_lengths)) return pb_fail(PB_ERR_INVALID, "null or negative argument");
        if (space != PB_MEM_HOST && space != PB_MEM_DEVICE) return pb_fail(PB_ERR_INVALID, "bad memory_space %d", space);
        const pb_create_params &p = *params;
        if (p.nbits <= 0 || 8 % p.nbits != 0) return pb_fail(PB_ERR_INVALID, "nbits must be a divisor of 8, got %d", p.nbits);
        if (p.batch_size <= 0 || p.kmeans_niters < 0 || p.max_points_per_centroid <= 0)
            return pb_fail(PB_ERR_INVALID, "bad create parameters");
        if (centroids_in && (num_centroids <= 0 || num_centroids >= (1ll << 32) - 1))
            return pb_fail(PB_ERR_INVALID, "bad num_centroids %lld", (long long)num_centroids);
        for (long long i = 0; i < n_docs; ++i) {
            if (doc_lengths[i] < 0 || doc_lengths[i] > (1 << 30))
                return pb_fail(PB_ERR_INVALID, "doc_lengths[%lld] = %lld", i, (long long)doc_lengths[i]);
            n_tok += doc_lengths[i];
        }
        if (n_tok && !emb) return pb_fail(PB_ERR_INVALID, "null argument");
        if (W > 1 && !comm.has_p2p()) return pb_fail(PB_ERR_COMM, "libnccl.so.2 lacks ncclSend / ncclRecv");
        CKS(BuiltDims::check(dim));
        const long long words[] = {dim, p.nbits, p.kmeans_niters, p.max_points_per_centroid, (long long)p.num_partitions,
                                   (long long)p.batch_size, (long long)p.seed, centroids_in ? (long long)num_centroids : 0};
        memcpy(rec + CV_DIM, words, sizeof words);
        Fnv64 fc, fd;
        if (centroids_in) fc.add(centroids_in, (size_t)num_centroids * dim * 4);
        fd.add(index_dir, strlen(index_dir) + 1);
        rec[CV_CENT] = (long long)fc.h;
        rec[CV_DIR] = (long long)fd.h;
        if (R == 0) {
            Fnv64 ft;
            ft.put(clock::now().time_since_epoch().count());
            ft.put((uintptr_t)c);
            rec[CV_TOKEN] = (long long)(ft.h >> 1);
            token = true;
            CKS(pb_dir_token_put(index_dir, rec[CV_TOKEN]));
        }
        return PB_OK;
    };
    rec[CV_STATUS] = local();
    rec[CV_RANK] = R;
    rec[CV_WORLD] = W;
    rec[CV_D] = n_docs;
    rec[CV_N] = n_tok;
    std::vector<long long> all;
    pb_status s = gather_words(comm, rec, CV_WORDS, all, true);
    if (!s) s = first_failure(comm, all, CV_WORDS, "; nothing was written");
    auto at = [&](int r, int w) { return all[(size_t)r * CV_WORDS + w]; };
    std::vector<long long> base((size_t)W + 1, 0), tokb((size_t)W + 1, 0);
    for (int r = 0; r < W && !s; ++r) {
        bool same = at(r, CV_RANK) == r && at(r, CV_WORLD) == W;
        for (int w = CV_DIM; w <= CV_DIR; ++w) same = same && at(r, w) == at(0, w);
        if (!same) s = pb_fail(PB_ERR_INVALID, "rank %d was called with other arguments than rank 0", r);
        base[r + 1] = base[r] + at(r, CV_D);
        tokb[r + 1] = tokb[r] + at(r, CV_N);
    }
    const long long D = base[W], N = tokb[W];
    if (!s && D <= 0) s = pb_fail(PB_ERR_INVALID, "no documents");
    if (!s && N <= 0) s = pb_fail(PB_ERR_INVALID, "no embeddings");
    if (!s && D >= (1ll << 32) - 1) s = pb_fail(PB_ERR_UNSUPPORTED, "global doc ids must stay below 2^32-1");
    if (!s) s = create_vote(comm, R ? pb_dir_token_check(index_dir, at(0, CV_TOKEN)) : PB_OK,
                            " finding the index directory; nothing was written");
    if (token) pb_dir_token_drop(index_dir);
    if (s) return s;
    const pb_create_params &cfg = *params;
    const std::string dir = std::string(index_dir) + "/";
    const int packed = dim * cfg.nbits / 8, nopt = 1 << cfg.nbits;
    const long long T0 = tokb[R];
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, comm.device));
    const int sms = prop.multiProcessorCount;

    // every document's length: O(D) host words, as pb_create_index's own plan
    long long maxD = 0;
    for (int r = 0; r < W; ++r) maxD = std::max(maxD, at(r, CV_D));
    std::vector<long long> mine((size_t)maxD, 0), gl;
    for (long long i = 0; i < n_docs; ++i) mine[i] = doc_lengths[i];
    CKS(gather_words(comm, mine.data(), (int)maxD, gl, true));
    std::vector<int64_t> lens((size_t)D);
    std::vector<long long> off((size_t)D + 1, 0);
    for (int r = 0; r < W; ++r)
        for (long long i = 0; i < at(r, CV_D); ++i) lens[base[r] + i] = gl[(size_t)r * maxD + i];
    for (long long d = 0; d < D; ++d) off[d + 1] = off[d] + lens[d];
    std::vector<long long>().swap(gl);
    auto owner_tok = [&](long long t) { return (int)(std::upper_bound(tokb.begin(), tokb.end(), t) - tokb.begin()) - 1; };
    auto owner_doc = [&](long long d) { return (int)(std::upper_bound(base.begin(), base.end(), d) - base.begin()) - 1; };
    lap(CP_PLAN);

    // ---- 2. centroids (kmeans.rs:273-419): this rank's fit points in global fit order, its seeds, one Lloyd loop ----
    long long K = num_centroids;
    std::vector<float> cent;
    if (centroids_in) {
        cent.assign(centroids_in, centroids_in + (size_t)K * dim);
    } else {
        const long long n_sdocs = pb_kmeans_num_sample_docs(D);
        const std::vector<long long> sdocs = shuffled_prefix(D, n_sdocs, cfg.seed);
        std::vector<long long> srow((size_t)n_sdocs + 1, 0);  // first sample row of each sampled doc
        for (long long j = 0; j < n_sdocs; ++j) srow[j + 1] = srow[j] + lens[sdocs[j]];
        const long long n_stok = srow[n_sdocs];
        if (n_stok <= 0) return pb_fail(PB_ERR_INVALID, "the k-means sample holds no embeddings");
        K = cfg.num_partitions > 0 ? std::min<long long>(cfg.num_partitions, n_stok)
                                   : pb_kmeans_num_partitions(D, (double)n_stok / (double)n_sdocs, n_stok);
        long long n_fit = n_stok;
        std::vector<long long> pick;  // at most max_points_per_centroid points per centroid
        if (n_stok > K * (long long)cfg.max_points_per_centroid) {
            n_fit = K * (long long)cfg.max_points_per_centroid;
            pick = shuffled_prefix(n_stok, n_fit, cfg.seed ^ 0x5bd1e995u);
        }
        std::vector<long long> my_fit, my_tok;  // my fit points: their fit indices (ascending) and my token ids
        for (long long i = 0; i < n_fit; ++i) {
            const long long r = pick.empty() ? i : pick[i];
            const long long j = (long long)(std::upper_bound(srow.begin(), srow.end(), r) - srow.begin()) - 1;
            const long long t = off[sdocs[j]] + (r - srow[j]);
            if (owner_tok(t) == R) {
                my_fit.push_back(i);
                my_tok.push_back(t - T0);
            }
        }
        const std::vector<long long> seeds = lcg_seeds(n_fit, K, cfg.seed * 6364136223846793005ull + 1442695040888963407ull);
        std::vector<long long> sidx((size_t)K, -1);  // my fit point of each seed I own
        for (long long k = 0; k < K; ++k) {
            auto it = std::lower_bound(my_fit.begin(), my_fit.end(), seeds[k]);
            if (it != my_fit.end() && *it == seeds[k]) sidx[k] = it - my_fit.begin();
        }
        DevBuf dX, dC, didx;
        auto prep = [&]() -> pb_status {
            CKS(gather_rows(emb, space, dim, my_tok, dX, sms, st));
            CKS(dC.ensure((size_t)K * dim * 4));
            CKS(upload(didx, sidx.data(), (size_t)K * 8, PB_MEM_HOST));
            k_seed_rows<<<sms * 4, 256, 0, st>>>(dX.as<float>(), didx.as<long long>(), K, dim, dC.as<float>());
            CK(cudaGetLastError());
            return PB_OK;
        };
        CKS(create_vote(comm, prep(), " gathering its k-means points; nothing was written"));
        CKS(comm.allreduce_sum(st, dC.as<float>(), (size_t)K * dim, c->stage));
        CKS(lloyd(comm.joined() ? &comm : nullptr, &c->stage, st, dX.as<float>(), (long long)my_tok.size(), dim, K,
                  cfg.kmeans_niters, sms, dC.as<float>()));
        cent.resize((size_t)K * dim);
        CK(cudaMemcpyAsync(cent.data(), dC.p, cent.size() * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    lap(CP_KMEANS);

    // ---- 3. codec training on rank 0, on pb_create_index's held-out rows in its order (index.rs:195-287) ----
    const long long n_cdocs = pb_codec_num_sample_docs(D);
    const std::vector<long long> cdocs = shuffled_prefix(D, n_cdocs, cfg.seed + 1);
    const long long want = pb_codec_heldout_tokens(N);
    std::vector<std::pair<long long, long long>> held;  // (first global token, rows), from the end of the sample list
    std::vector<long long> my_held, held_rows((size_t)W, 0);
    long long got = 0;
    for (long long i = (long long)cdocs.size() - 1; i >= 0 && got < want; --i) {
        const long long d = cdocs[(size_t)i], take = std::min<long long>(want - got, lens[d]);
        got += take;
        if (!take) continue;
        held.emplace_back(off[d], take);
        const int r = owner_doc(d);
        held_rows[r] += take;
        if (r == R)
            for (long long t = 0; t < take; ++t) my_held.push_back(off[d] - T0 + t);
    }
    std::vector<float> cutoffs((size_t)std::max(nopt - 1, 1)), weights((size_t)nopt), avg_res((size_t)dim);
    float threshold = 0.0f;
    {
        DevBuf hs, hr;
        std::vector<size_t> first((size_t)W + 1, 0);
        for (int r = 0; r < W; ++r) first[r + 1] = first[r] + (size_t)held_rows[r] * dim * 4;
        auto gather = [&]() -> pb_status {
            CKS(gather_rows(emb, space, dim, my_held, hs, sms, st));
            if (R == 0) CKS(hr.ensure(std::max<size_t>(first[W], 16)));
            return PB_OK;
        };
        CKS(create_vote(comm, gather(), " gathering its held-out rows; nothing was written"));
        std::vector<float> rows(R == 0 ? (size_t)got * dim : 0);
        if (comm.joined()) {
            std::vector<const void *> sp((size_t)W, nullptr);
            std::vector<void *> rp((size_t)W, nullptr);
            std::vector<size_t> sb((size_t)W, 0), rb((size_t)W, 0);
            sp[0] = hs.p;
            sb[0] = first[R + 1] - first[R];
            for (int r = 0; r < W && R == 0; ++r) {
                rp[r] = hr.as<char>() + first[r];
                rb[r] = first[r + 1] - first[r];
            }
            CKS(comm.exchange(st, 1, sp.data(), sb.data(), rp.data(), rb.data()));
            if (R == 0 && got) CK(cudaMemcpy(rows.data(), hr.p, first[W], cudaMemcpyDeviceToHost));
        } else if (got) {
            CK(cudaMemcpy(rows.data(), hs.p, first[W], cudaMemcpyDeviceToHost));
        }
        // the trainer reassembles the sample order from the ranks' pieces, trains, and shares the codec's numbers
        const int nf = (nopt - 1) + nopt + dim + 1, words = 1 + (nf + 1) / 2;
        std::vector<long long> mine_w((size_t)words, 0), allw;
        if (R == 0) {
            auto train = [&]() -> pb_status {
                std::vector<float> heldout((size_t)got * dim);
                std::vector<size_t> cur(first.begin(), first.end() - 1);
                size_t w = 0;
                for (const auto &pc : held) {
                    const int r = owner_tok(pc.first);
                    const size_t b = (size_t)pc.second * dim * 4;
                    memcpy(reinterpret_cast<char *>(heldout.data()) + w, reinterpret_cast<char *>(rows.data()) + cur[r], b);
                    cur[r] += b;
                    w += b;
                }
                pb_codec *tc = nullptr;
                CKS(pb_codec_open(comm.device, cent.data(), K, dim, cfg.nbits, nullptr, &tc));
                pb_status ts = pb_codec_train(tc, heldout.data(), got, cutoffs.data(), weights.data(), avg_res.data(), &threshold);
                pb_codec_close(tc);
                return ts;
            };
            mine_w[0] = train();
            float *f = reinterpret_cast<float *>(mine_w.data() + 1);
            memcpy(f, cutoffs.data(), (size_t)(nopt - 1) * 4);
            memcpy(f + nopt - 1, weights.data(), (size_t)nopt * 4);
            memcpy(f + 2 * nopt - 1, avg_res.data(), (size_t)dim * 4);
            f[nf - 1] = threshold;
        }
        CKS(gather_words(comm, mine_w.data(), words, allw, true));
        CKS(first_failure(comm, allw, words, " training the codec; nothing was written"));
        const float *f = reinterpret_cast<const float *>(allw.data() + 1);  // rank 0's record
        memcpy(cutoffs.data(), f, (size_t)(nopt - 1) * 4);
        memcpy(weights.data(), f + nopt - 1, (size_t)nopt * 4);
        memcpy(avg_res.data(), f + 2 * nopt - 1, (size_t)dim * 4);
        threshold = f[nf - 1];
    }
    lap(CP_CODEC);

    // ---- 4. encode this rank's documents straight into its shard, slab by slab ----
    std::unique_ptr<pb_index, IndexCloser> ix;
    pb_codec *enc = nullptr;
    auto encode = [&]() -> pb_status {
        CKS(pb_codec_open(comm.device, cent.data(), K, dim, cfg.nbits, cutoffs.data(), &enc));
        pb_index_desc d;
        memset(&d, 0, sizeof d);
        d.dim = dim;
        d.nbits = cfg.nbits;
        d.num_centroids = K;
        d.num_documents = n_docs;
        d.num_embeddings = n_tok;
        d.centroids = cent.data();
        d.bucket_weights = weights.data();
        d.doc_lengths = doc_lengths;
        d.device = comm.device;
        d.memory_space = PB_MEM_HOST;
        d.doc_id_base = base[R];
        pb_index *h = nullptr;
        CKS(pb_index_open_begin(&d, &h));
        ix.reset(h);
        const long long slab = 1ll << 20;
        DevBuf dX, dcodes, dpk;
        if (space == PB_MEM_HOST) CKS(dX.ensure((size_t)std::min(n_tok, slab) * dim * 4 + 16));
        CKS(dcodes.ensure((size_t)std::min(n_tok, slab) * 8 + 16));
        CKS(dpk.ensure((size_t)std::min(n_tok, slab) * packed + 16));
        for (long long o = 0; o < n_tok; o += slab) {
            const long long m = std::min(slab, n_tok - o);
            const float *x = emb + (size_t)o * dim;
            if (space == PB_MEM_HOST) {
                CK(cudaMemcpy(dX.p, x, (size_t)m * dim * 4, cudaMemcpyHostToDevice));
                x = dX.as<float>();
            }
            CKS(codec_encode_device(enc, x, m, dcodes.as<long long>(), dpk.as<uint8_t>(), nullptr));
            CKS(pb_index_upload_tokens(ix.get(), o, dcodes.as<int64_t>(), dpk.as<uint8_t>(), m, PB_MEM_DEVICE));
        }
        lap(CP_ENCODE);
        CKS(pb_index_finalize(ix.get()));
        lap(CP_SHARD);
        return PB_OK;
    };
    s = encode();
    if (enc) pb_codec_close(enc);
    CKS(create_vote(comm, s, " encoding its documents; nothing was written"));

    // ---- 5. chunk files: chunk i is written by the rank holding its first document; the head of a rank's range that
    // lies in a chunk begun on an earlier rank goes to that chunk's writer ----
    const long long bs = cfg.batch_size, n_chunks = (D + bs - 1) / bs;
    std::vector<int> head_to((size_t)W, -1);  // writer of each rank's head, or -1
    std::vector<long long> head_end((size_t)W, 0);
    bool any_head = false;
    for (int r = 0; r < W; ++r) {
        if (base[r] == base[r + 1] || base[r] % bs == 0) continue;
        const long long c0 = base[r] / bs * bs;
        head_to[r] = owner_doc(c0);
        head_end[r] = std::min(c0 + bs, base[r + 1]);
        any_head = true;
    }
    DevBuf rc, rr;  // the heads this rank receives, in rank order
    std::vector<long long> recv_tok((size_t)W + 1, 0);
    for (int r = 0; r < W; ++r)
        recv_tok[r + 1] = recv_tok[r] + (head_to[r] == R && r != R ? off[head_end[r]] - off[base[r]] : 0);
    if (any_head) {
        CKS(rc.ensure((size_t)recv_tok[W] * 4 + 16));
        CKS(rr.ensure((size_t)recv_tok[W] * packed + 16));
        std::vector<const void *> sp((size_t)W * 2, nullptr);
        std::vector<void *> rp((size_t)W * 2, nullptr);
        std::vector<size_t> sb((size_t)W * 2, 0), rb((size_t)W * 2, 0);
        if (head_to[R] >= 0) {
            const long long n = off[head_end[R]] - off[base[R]];
            sp[(size_t)head_to[R] * 2] = ix->codes.p;
            sp[(size_t)head_to[R] * 2 + 1] = ix->residuals.p;
            sb[(size_t)head_to[R] * 2] = (size_t)n * 4;
            sb[(size_t)head_to[R] * 2 + 1] = (size_t)n * packed;
        }
        for (int r = 0; r < W; ++r) {
            const long long n = recv_tok[r + 1] - recv_tok[r];
            rp[(size_t)r * 2] = rc.as<uint32_t>() + recv_tok[r];
            rp[(size_t)r * 2 + 1] = rr.as<uint8_t>() + (size_t)recv_tok[r] * packed;
            rb[(size_t)r * 2] = (size_t)n * 4;
            rb[(size_t)r * 2 + 1] = (size_t)n * packed;
        }
        CKS(comm.exchange(st, 2, sp.data(), sb.data(), rp.data(), rb.data()));
    }
    auto write_chunks = [&]() -> pb_status {
        for (long long ch = (base[R] + bs - 1) / bs; n_docs && ch * bs < base[R + 1]; ++ch) {
            const long long d0 = ch * bs, d1 = std::min(D, d0 + bs), dm = std::min(d1, base[R + 1]);
            const long long t0 = off[d0], n_own = off[dm] - t0, n = off[d1] - t0;
            const long long n_in = dm < d1 ? recv_tok[W] : 0;  // only the last chunk crosses into later ranks
            std::vector<uint32_t> c32((size_t)n);
            std::vector<int64_t> codes((size_t)n);
            std::vector<uint8_t> res((size_t)n * packed);
            if (n_own) {
                CK(cudaMemcpy(c32.data(), ix->codes.as<uint32_t>() + (t0 - T0), (size_t)n_own * 4, cudaMemcpyDeviceToHost));
                CK(cudaMemcpy(res.data(), ix->residuals.as<uint8_t>() + (size_t)(t0 - T0) * packed, (size_t)n_own * packed,
                              cudaMemcpyDeviceToHost));
            }
            if (n_in) {
                CK(cudaMemcpy(c32.data() + n_own, rc.p, (size_t)n_in * 4, cudaMemcpyDeviceToHost));
                CK(cudaMemcpy(res.data() + (size_t)n_own * packed, rr.p, (size_t)n_in * packed, cudaMemcpyDeviceToHost));
            }
            if (n_own + n_in != n) return pb_fail(PB_ERR_INVALID, "chunk %lld: %lld of %lld rows", ch, n_own + n_in, n);
            for (long long i = 0; i < n; ++i) codes[i] = c32[i];
            CKS(pb_write_chunk(dir, ch, codes.data(), res.data(), n, packed, lens.data() + d0, d1 - d0, t0));
        }
        return PB_OK;
    };
    CKS(create_vote(comm, write_chunks(), " writing its chunk files"));
    lap(CP_CHUNKS);

    // ---- 6. ivf.npy: list k is the ranks' lists of k in rank order (each ascending, so the whole list is); rank 0
    // creates the file at its final size and every rank writes its pieces at their offsets.  Then the codec's files,
    // and metadata.json last ----
    int64_t my_total = 0;
    std::vector<int64_t> my_ivf;
    std::vector<int32_t> my_len((size_t)K);
    CKS(create_vote(comm, [&]() -> pb_status {
        CKS(pb_index_export_ivf(ix.get(), nullptr, nullptr, &my_total));
        my_ivf.resize((size_t)std::max<int64_t>(my_total, 1));
        return pb_index_export_ivf(ix.get(), my_ivf.data(), my_len.data(), &my_total);
    }(), " exporting its inverted file"));
    const int lw = (int)((K + 1) / 2);
    std::vector<long long> lw_mine((size_t)lw, 0), lw_all;
    memcpy(lw_mine.data(), my_len.data(), (size_t)K * 4);
    CKS(gather_words(comm, lw_mine.data(), lw, lw_all, true));
    auto len_of = [&](int r, long long k) { return (long long)reinterpret_cast<const int32_t *>(lw_all.data() + (size_t)r * lw)[k]; };
    std::vector<int32_t> tot((size_t)K, 0);
    std::vector<NpyPiece> pieces;
    long long ivf_total = 0, src = 0;
    for (long long k = 0; k < K; ++k) {
        long long before = 0;
        for (int r = 0; r < W; ++r) {
            if (r < R) before += len_of(r, k);
            tot[k] += (int32_t)len_of(r, k);
        }
        if (my_len[k])
            pieces.push_back({(size_t)(ivf_total + before) * 8, (size_t)my_len[k] * 8, reinterpret_cast<const char *>(my_ivf.data() + src)});
        src += my_len[k];
        ivf_total += tot[k];
    }
    CKS(create_vote(comm, R ? PB_OK : [&]() -> pb_status {
        CKS(npy_create(dir + "ivf.npy", "<i8", {ivf_total}, (size_t)ivf_total * 8));
        CKS(write_npy(dir + "ivf_lengths.npy", "<i4", {K}, tot.data(), (size_t)K * 4));
        return pb_write_codec_files(dir, K, dim, cfg.nbits, cent.data(), cutoffs.data(), weights.data(), avg_res.data(),
                                    threshold, n_chunks);
    }(), " writing the index files"));
    CKS(create_vote(comm, npy_put(dir + "ivf.npy", "<i8", {ivf_total}, pieces), " writing its part of ivf.npy"));
    CKS(create_vote(comm, R ? PB_OK : pb_write_create_meta(dir, n_chunks, cfg.nbits, K, N, D, dim), " writing metadata.json"));
    lap(CP_IVF);
    if (out_first) *out_first = base[R];
    if (out_shard) *out_shard = ix.release();
    return PB_OK;
}

extern "C" pb_status pb_create_index_sharded(pb_build_comm *c, const float *embeddings, const int64_t *doc_lengths,
                                             int64_t n_docs, int32_t dim, int32_t memory_space, const float *centroids,
                                             int64_t num_centroids, const pb_create_params *params, const char *index_dir,
                                             pb_index **out_shard, int64_t *out_first_doc_id) {
    if (out_shard) *out_shard = nullptr;
    if (out_first_doc_id) *out_first_doc_id = 0;
    if (!c) return pb_fail(PB_ERR_INVALID, "null argument");
    return create_collective(c, embeddings, doc_lengths, n_docs, dim, memory_space, centroids, num_centroids, params,
                             index_dir, out_shard, out_first_doc_id);
}

pb_status pb_create_local(const float *embeddings, const int64_t *doc_lengths, int64_t n_docs, int32_t dim,
                          const pb_create_params *params, const char *index_dir, pb_index **out_index) {
    CKS(check_device(params->device));
    pb_build_comm c;
    c.comm.device = params->device;
    CK(cudaSetDevice(params->device));
    CK(cudaStreamCreateWithFlags(&c.stream.s, cudaStreamNonBlocking));
    return create_collective(&c, embeddings, doc_lengths, n_docs, dim, PB_MEM_HOST, nullptr, 0, params, index_dir, out_index,
                             nullptr);
}

extern "C" pb_status pb_last_create_ms(float *out_ms) {
    if (!out_ms) return pb_fail(PB_ERR_INVALID, "null argument");
    memcpy(out_ms, g_create_ms, sizeof g_create_ms);
    return PB_OK;
}
