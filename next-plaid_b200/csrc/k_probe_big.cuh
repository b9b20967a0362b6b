// k_probe_big.cuh -- a3 for large effective n_ivf_probe.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ------------------------------------------------------------------------------------------
// a3 for large effective n_ivf_probe (dense variant; the subset rule scales n_ivf_probe by
// D / |subset|, search.rs:370-382, far beyond the 64 the streaming lists hold).  One CTA per query
// token: MSB radix select of the n-th best selection key among the eligible centroids, then every
// centroid at or above it is marked in the query's cell bitmap.  grid = (QS, B), 256 threads.  Each query reads its own
// n and eligibility row, so queries of different subsets share a launch.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_topn_select_row(const float *__restrict__ ST, const int *__restrict__ q_off, long long K, int QS,
                  const int *__restrict__ qn, const uint32_t *__restrict__ elig_rows, const int *__restrict__ qrow,
                  long long Wke, uint32_t *__restrict__ cellbits, long long Wk) {
    __shared__ int hist[256];
    __shared__ u64 prefix_s, mask_s;
    __shared__ long long remaining_s;
    const int q = blockIdx.x, b = blockIdx.y;
    const int nq = q_off[b + 1] - q_off[b];
    if (q >= nq) return;
    // the query's own n and eligibility row (per-query subsets), or none
    const long long n = qn[b];
    const uint32_t *eligible = (elig_rows && qrow[b] >= 0) ? elig_rows + (size_t)qrow[b] * Wke : nullptr;
    const float *col = ST + (size_t)b * K * QS + q;
    uint32_t *bits = cellbits + (size_t)b * Wk;
    if (threadIdx.x == 0) {
        prefix_s = 0ull;
        mask_s = 0ull;
        remaining_s = n;
    }
    __syncthreads();
    bool all = false;
    for (int pass = 7; pass >= 0; --pass) {
        const int shift = pass * 8;
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        const u64 prefix = prefix_s, mask = mask_s;
        for (long long c = threadIdx.x; c < K; c += blockDim.x) {
            if (eligible && !((eligible[c >> 5] >> (c & 31)) & 1u)) continue;
            const u64 key = ~(((u64)score_key_asc(col[(size_t)c * QS]) << 32) | (uint32_t)(~(uint32_t)c));  // ascending = best first
            if ((key & mask) == prefix) atomicAdd(&hist[(int)((key >> shift) & 255ull)], 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long rem = remaining_s, cum = 0;
            int d = 0;
            for (; d < 256; ++d) {
                if (cum + hist[d] >= rem) break;
                cum += hist[d];
            }
            if (d == 256) {  // fewer than n eligible centroids: take them all
                d = 255;
                remaining_s = -1;
            } else remaining_s = rem - cum;
            prefix_s = prefix | ((u64)d << shift);
            mask_s = mask | (255ull << shift);
        }
        __syncthreads();
        if (remaining_s < 0) {
            all = true;
            break;
        }
    }
    const u64 pivot = prefix_s;  // inverted key of the n-th best centroid
    for (long long c = threadIdx.x; c < K; c += blockDim.x) {
        if (eligible && !((eligible[c >> 5] >> (c & 31)) & 1u)) continue;
        const u64 key = ~(((u64)score_key_asc(col[(size_t)c * QS]) << 32) | (uint32_t)(~(uint32_t)c));
        if (all || key <= pivot) atomicOr(&bits[c >> 5], 1u << (c & 31));
    }
}

// per query: the marked centroids that pass the dense threshold rule (search.rs:417-425), ascending;
// clears the bitmap for the next call.  grid = B, 1024 threads.
__global__ void __launch_bounds__(1024)
k_cells_from_query_bits(uint32_t *__restrict__ cellbits, long long Wk, const float *__restrict__ ST,
                        const int *__restrict__ q_off, long long K, int QS, int has_thr, float thr, int cells_cap,
                        uint32_t *__restrict__ cells, int *__restrict__ n_cells, const int *__restrict__ qhas,
                        const float *__restrict__ qthr) {
    __shared__ int scan_tmp[33];
    const int b = blockIdx.x;
    const int nq = q_off[b + 1] - q_off[b];
    if (qhas) has_thr = qhas[b], thr = qthr[b];  // the query's own threshold (DESIGN.md 4l)
    uint32_t *bits = cellbits + (size_t)b * Wk;
    const float *STb = ST + (size_t)b * K * QS;
    const long long per = (Wk + blockDim.x - 1) / blockDim.x;
    const long long w0 = min(Wk, (long long)threadIdx.x * per), w1 = min(Wk, w0 + per);
    // drop the centroids under the threshold, count the survivors
    int cnt = 0;
    for (long long i = w0; i < w1; ++i) {
        uint32_t x = bits[i], keep = 0;
        while (x) {
            const int bit = __ffs(x) - 1;
            x &= x - 1;
            bool ok = nq > 0;
            if (ok && has_thr) {
                const float *row = STb + (size_t)(i * 32 + bit) * QS;
                uint32_t best = 0u;
                for (int q = 0; q < nq; ++q) best = max(best, score_key_asc(row[q]));
                const float mval = best ? key_to_score(best) : row[nq - 1];
                ok = mval >= thr;
            }
            if (ok) keep |= 1u << bit;
        }
        bits[i] = keep;
        cnt += __popc(keep);
    }
    int total;
    int pos = block_exclusive_scan(cnt, scan_tmp, &total);
    for (long long i = w0; i < w1; ++i) {
        uint32_t x = bits[i];
        if (x) bits[i] = 0u;
        while (x) {
            const int bit = __ffs(x) - 1;
            x &= x - 1;
            if (pos < cells_cap) cells[(size_t)b * cells_cap + pos] = (uint32_t)(i * 32 + bit);
            ++pos;
        }
    }
    if (threadIdx.x == 0) n_cells[b] = min(total, cells_cap);
}
