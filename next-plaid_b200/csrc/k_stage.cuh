// k_stage.cuh -- the exact stage of a handle whose packed residuals live in pinned, mapped host memory
// (PB_OPEN_HOST_RESIDUALS, DESIGN.md 4j).  After the cut the kept docs of a sub-batch are gathered into a device staging
// buffer in "slot space", and every token-addressing kernel of the stage then runs unchanged on the staged arrays.
//
// Slot s = b * Mcap + j stands for kept doc j of query b.  Query b's docs are staged back to back from
//   base_b = sum over b' < b of tokp[b'][nkept[b']]   (the tokens the queries before it keep)
// and doc j at base_b + tokp[b][j].  soff[s] is that offset; a slot past nkept[b] takes base_{b+1}, so that
// soff[s + 1] - soff[s] is the length of every slot, and soff[B * Mcap] is the total.  kept_s[s] = s, so that the
// kernels' doc_off[kept[j]] reads soff[s].
// A handle with a device row cache (DESIGN.md 4s) stages its cached docs from there, device to device.
#pragma once
#include "common.cuh"

__global__ void __launch_bounds__(256) k_stage_layout(const int *__restrict__ nkept, const long long *__restrict__ tokp, int B,
                                                      int Mcap, long long *__restrict__ soff, uint32_t *__restrict__ kept_s) {
    __shared__ long long warp_sum[8];
    const int b = blockIdx.y;
    long long acc = 0;
    for (int i = threadIdx.x; i < b; i += blockDim.x) acc += tokp[(size_t)i * (Mcap + 1) + nkept[i]];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
    __syncthreads();
    long long base = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) base += warp_sum[w];
    const int nk = nkept[b];
    const long long *tp = tokp + (size_t)b * (Mcap + 1);
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < Mcap; j += gridDim.x * blockDim.x) {
        const size_t s = (size_t)b * Mcap + j;
        soff[s] = base + tp[min(j, nk)];
        kept_s[s] = (uint32_t)s;
    }
    if (b == B - 1 && blockIdx.x == 0 && threadIdx.x == 0) soff[(size_t)B * Mcap] = base + tp[nk];
}

// The device row cache of a host-tier handle (DESIGN.md 4s) as k_stage_rows reads it: doc d's rows start at token off[d]
// of `rows` (off[d] < 0: not cached; off == NULL: no cache).  Cached rows start at token offsets, so a load unit sits at
// the same alignment as in the store.  count (search staging only) gains 1 per staged slot of its doc; hits[0] / hits[1]
// gain the slots staged from the cache and their bytes (NULL: not counted).
struct RowCache {
    const long long *off;
    FlatRows rows;
    uint32_t *count;
    unsigned long long *hits;
};

// Words [0, nv) of V from src at byte b0 into dst, U loads in flight per lane before the stores
template <class V, int U, class Src> PB_DEV void stage_copy(Src src, long long b0, long long nv, V *dst, int lane) {
    long long i = lane;
    for (; i + 32 * (U - 1) < nv; i += 32 * U) {
        V r[U];
#pragma unroll
        for (int u = 0; u < U; ++u) r[u] = *src.template at<V>(b0 + (i + 32 * u) * (long long)sizeof(V));
#pragma unroll
        for (int u = 0; u < U; ++u) dst[i + 32 * u] = r[u];
    }
    for (; i < nv; i += 32) dst[i] = *src.template at<V>(b0 + i * (long long)sizeof(V));
}

// One warp per slot: the rows [doc_off[d], doc_off[d + 1]) of doc d = kept[s] go to staged rows [soff[s], ..).  The
// packed residuals come from the row cache when it holds d (device to device), else from the mapped host segments,
// in V-sized words (16 bytes when the row length allows), each located through the segment table, since this kernel's
// PCIe read rate sets the speed of the tier; codes and 1 / |v| (inv_norm may be NULL) come from their device arrays
// (s_codes == NULL: residuals only, as the cache's fill stages them).  nkept == NULL: every slot of [0, n_slots) holds
// a doc.  No launch bounds: with __launch_bounds__(256) ptxas spills the uint4 form at 40 registers; without, it
// spills nothing.
template <class V, int U>
__global__ void k_stage_rows(const uint32_t *__restrict__ kept, const int *__restrict__ nkept, int Mcap, long long n_slots,
                             const long long *__restrict__ doc_off, const long long *__restrict__ soff,
                             SegRows host_res, RowCache cache, const uint32_t *__restrict__ codes,
                             const float *__restrict__ inv_norm, int packed, uint8_t *__restrict__ s_res,
                             uint32_t *__restrict__ s_codes, float *__restrict__ s_inv) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    unsigned long long hit_docs = 0, hit_bytes = 0;
    for (long long s = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < n_slots; s += nw) {
        if (nkept) {  // slot ids fit 32 bits (B * Mcap <= 2^22)
            const unsigned b = (unsigned)s / (unsigned)Mcap;
            if ((int)((unsigned)s - b * (unsigned)Mcap) >= nkept[b]) continue;
        }
        const uint32_t d = kept[s];
        const long long g0 = doc_off[d], len = doc_off[d + 1] - g0, t0 = soff[s];
        const long long c0 = cache.off ? cache.off[d] : -1;  // one address per warp: the branch below is uniform
        if (s_codes)
            for (long long t = lane; t < len; t += 32) {
                s_codes[t0 + t] = codes[g0 + t];
                if (inv_norm) s_inv[t0 + t] = inv_norm[g0 + t];
            }
        const long long nv = len * packed / (long long)sizeof(V);
        V *dst = reinterpret_cast<V *>(s_res + (size_t)t0 * packed);
        if (c0 >= 0) {
            stage_copy<V, U>(cache.rows, c0 * packed, nv, dst, lane);
            hit_docs += 1;
            hit_bytes += (unsigned long long)(len * packed);
        } else {
            stage_copy<V, U>(host_res, g0 * packed, nv, dst, lane);
        }
        if (cache.count && lane == 0) atomicAdd(cache.count + d, 1u);
    }
    if (cache.hits && lane == 0 && hit_docs) {
        atomicAdd(cache.hits, hit_docs);
        atomicAdd(cache.hits + 1, hit_bytes);
    }
}

// The row cache's map and keep counts of a delete's survivors under their new ids (kept[j] = old id of survivor j)
__global__ void k_cache_compact(const long long *__restrict__ off, const uint32_t *__restrict__ count,
                                const long long *__restrict__ kept, long long D1, long long *__restrict__ new_off,
                                uint32_t *__restrict__ new_count) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < D1; j += (long long)gridDim.x * blockDim.x) {
        new_off[j] = off[kept[j]];
        new_count[j] = count[kept[j]];
    }
}

// The cached docs among a delete's deleted set (bit d of `bits`): dead[0] += 1 and dead[1] += its tokens per such doc
__global__ void k_cache_dead(const long long *__restrict__ off, const uint32_t *__restrict__ bits,
                             const long long *__restrict__ doc_off, long long D0, unsigned long long *__restrict__ dead) {
    for (long long d = (long long)blockIdx.x * blockDim.x + threadIdx.x; d < D0; d += (long long)gridDim.x * blockDim.x)
        if (((bits[d >> 5] >> (d & 31)) & 1u) && off[d] >= 0) {
            atomicAdd(dead, 1ull);
            atomicAdd(dead + 1, (unsigned long long)(doc_off[d + 1] - doc_off[d]));
        }
}

// Slot ids back to doc ids, in place: kept[b][j] = kept_flat[kept[b][j]] for j < nkept[b] (before k_exact_finalize,
// which writes the ids)
__global__ void k_unstage_kept(uint32_t *__restrict__ kept, const int *__restrict__ nkept, int Mcap,
                               const uint32_t *__restrict__ kept_flat) {
    const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < nkept[b]) {
        const size_t s = (size_t)b * Mcap + j;
        kept[s] = kept_flat[kept[s]];
    }
}
