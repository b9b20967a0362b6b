// k_subset_shard.cuh -- subset pre-filter helpers and the doc-sharded merges.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// Subsets are per query.  A call's ids are uploaded once; subset row r lists ids[span[2r] .. span[2r + 1]) and every
// query with that list reads row r (a query without a subset reads none).
// k_subset_bits: row r's doc bitmap.  Ids outside [base, base+D) set nothing: `candidates.retain` can never match
// them.  grid = (x, rows)
__global__ void k_subset_bits(const long long *__restrict__ ids, const long long *__restrict__ span, long long base,
                              long long D, uint32_t *__restrict__ bits, long long Wd) {
    const long long s = span[2 * blockIdx.y], e = span[2 * blockIdx.y + 1];
    uint32_t *row = bits + (size_t)blockIdx.y * Wd;
    for (long long i = s + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (long long)gridDim.x * blockDim.x) {
        const long long d = ids[i] - base;
        if (d >= 0 && d < D) atomicOr(&row[d >> 5], 1u << (d & 31));
    }
}

// k_eligible_bits: row r's eligible centroids (search.rs:350-364), every code of every listed in-range doc; a warp per
// listed id, so the cost is the subset's tokens.  With `smem` the CTA ORs into a shared copy of the row (Wk words) and
// flushes its non-zero words once.  grid = (x, rows), 256 threads
__global__ void __launch_bounds__(256)
k_eligible_bits(const long long *__restrict__ ids, const long long *__restrict__ span, long long base, long long D,
                const long long *__restrict__ doc_off, const uint32_t *__restrict__ codes, uint32_t *__restrict__ elig,
                long long Wk, long long Wke, int smem) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t *sh = reinterpret_cast<uint32_t *>(smem_raw);
    uint32_t *row = elig + (size_t)blockIdx.y * Wke;
    uint32_t *dst = smem ? sh : row;
    if (smem) {
        for (long long i = threadIdx.x; i < Wk; i += blockDim.x) sh[i] = 0u;
        __syncthreads();
    }
    const long long s = span[2 * blockIdx.y], e = span[2 * blockIdx.y + 1];
    const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    for (long long i = s + (long long)blockIdx.x * wpb + (threadIdx.x >> 5); i < e; i += (long long)gridDim.x * wpb) {
        const long long d = ids[i] - base;
        if (d < 0 || d >= D) continue;  // warp-uniform
        for (long long t = doc_off[d] + lane; t < doc_off[d + 1]; t += 32) {
            const uint32_t c = codes[t];
            atomicOr(&dst[c >> 5], 1u << (c & 31));
        }
    }
    if (smem) {
        __syncthreads();
        for (long long i = threadIdx.x; i < Wk; i += blockDim.x)
            if (sh[i]) atomicOr(&row[i], sh[i]);
    }
}

// doc-sharded: the OR of every rank's eligibility rows (`words` 32-bit words per rank) into `out`
__global__ void k_or_ranks(const uint32_t *__restrict__ gathered, int G, long long words, uint32_t *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (long long)gridDim.x * blockDim.x) {
        uint32_t v = 0u;
        for (int g = 0; g < G; ++g) v |= gathered[(size_t)g * words + i];
        out[i] = v;
    }
}

// out[r] += the set bits of row r.  grid = (x, rows)
__global__ void k_popcount(const uint32_t *__restrict__ bits, long long W, unsigned long long *__restrict__ out) {
    const uint32_t *row = bits + (size_t)blockIdx.y * W;
    unsigned long long c = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < W; i += (long long)gridDim.x * blockDim.x)
        c += __popc(row[i]);
    for (int m = 16; m >= 1; m >>= 1) c += __shfl_xor_sync(PB_FULL, c, m);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out + blockIdx.y, c);
}

// "all eligible centroids" as the selected set (n_probe_eff >= |eligible|, search.rs:379): query b's row, ascending,
// into list[b][lcap].  grid = B, 1024 threads
__global__ void k_cells_from_bits(const uint32_t *__restrict__ elig, const int *__restrict__ qrow, long long Wke,
                                  long long K, uint32_t *__restrict__ list, int lcap, int *__restrict__ count) {
    __shared__ int scan_tmp[33];
    const int b = blockIdx.x;
    const uint32_t *row = elig + (size_t)qrow[b] * Wke;
    uint32_t *out = list + (size_t)b * lcap;
    const long long W = (K + 31) / 32;
    const long long per = (W + blockDim.x - 1) / blockDim.x;
    const long long w0 = min(W, (long long)threadIdx.x * per), w1 = min(W, w0 + per);
    int cnt = 0;
    for (long long i = w0; i < w1; ++i) cnt += __popc(row[i]);
    int total;
    int pos = block_exclusive_scan(cnt, scan_tmp, &total);
    for (long long i = w0; i < w1; ++i) {
        uint32_t x = row[i];
        while (x) {
            int bit = __ffs(x) - 1;
            x &= x - 1;
            if (pos < lcap) out[pos] = (uint32_t)(i * 32 + bit);
            ++pos;
        }
    }
    if (threadIdx.x == 0) count[b] = min(total, lcap);
}

// threshold filter over each query's centroid list (dense variant only; subset path).  grid = B, 256 threads
__global__ void __launch_bounds__(256)
k_cells_filter_list(const uint32_t *__restrict__ list, int lcap, const int *__restrict__ list_n,
                    const float *__restrict__ ST, const int *__restrict__ q_off, long long K, int QS, int has_thr,
                    float thr, int cells_cap, uint32_t *__restrict__ cells, int *__restrict__ n_cells,
                    const int *__restrict__ qhas, const float *__restrict__ qthr) {
    __shared__ int scan_tmp[33];
    const int b = blockIdx.x;
    const int nq = q_off[b + 1] - q_off[b];
    const int n = list_n[b];
    if (qhas) has_thr = qhas[b], thr = qthr[b];  // the query's own threshold (DESIGN.md 4l)
    const uint32_t *lst = list + (size_t)b * lcap;
    const float *STb = ST + (size_t)b * K * QS;
    int outn = 0;
    for (int base = 0; base < n; base += blockDim.x) {
        int i = base + threadIdx.x;
        int f = 0;
        uint32_t c = 0;
        if (i < n && nq > 0) {
            c = lst[i];
            f = 1;
            if (has_thr) {
                const float *row = STb + (size_t)c * QS;
                uint32_t best = 0u;
                for (int q = 0; q < nq; ++q) best = max(best, score_key_asc(row[q]));
                float mval = best ? key_to_score(best) : row[nq - 1];
                f = (mval >= thr);
            }
        }
        int tot;
        int pos = block_exclusive_scan(f, scan_tmp, &tot);
        if (f && outn + pos < cells_cap) cells[(size_t)b * cells_cap + outn + pos] = c;
        outn += tot;
    }
    if (threadIdx.x == 0) n_cells[b] = min(outn, cells_cap);
}


// ------------------------------------------------------------------------------------------
// doc-sharded search (SURVEY 8e).  The reference cuts to n_full_scores/4 GLOBALLY on the approximate
// score (search.rs:460-469), so shards exchange their sorted top-M cut keys, every shard derives the
// global cut and exact-scores only its own members, then the exact triples are exchanged and merged
// with the stable-sort rule of search.rs:496.  Both kernels: grid = B, 1024 threads.
// ------------------------------------------------------------------------------------------
// k_merge_cut: every shard's list is sorted (best first) and keys are unique (global doc id in the low word), so the
// global rank of my j-th entry is j + the number of smaller keys in every other shard's list (one binary search
// each); it is in the global cut iff that rank < M.  No sort, no shared memory: any number of shards.  Lists are Mcap
// keys per query (~0 past the shard's own); qM: each query's own M (or null: M).
__global__ void __launch_bounds__(1024)
k_merge_cut(const u64 *__restrict__ gkeys, int G, int my_rank, int B, int M, int Mcap, uint32_t doc_id_base, long long D,
            const long long *__restrict__ doc_off, uint32_t *__restrict__ kept, uint32_t *__restrict__ krank,
            int *__restrict__ n_kept, long long *__restrict__ tok_prefix, long long *__restrict__ kept_tokens,
            const int *__restrict__ qM) {
    __shared__ int scan_tmp[33];
    const int b = blockIdx.x;
    if (qM) M = qM[b];
    const u64 *mine = gkeys + ((size_t)my_rank * B + b) * Mcap;
    long long run = 0;
    int outn = 0;
    for (int base = 0; base < M; base += blockDim.x) {
        const int j = base + threadIdx.x;
        int f = 0, len = 0;
        uint32_t d = 0, grank = 0;
        if (j < M && mine[j] != ~0ull) {
            const u64 key = mine[j];
            int r = j;
            for (int g = 0; g < G && r < M; ++g) {
                if (g == my_rank) continue;
                const u64 *lst = gkeys + ((size_t)g * B + b) * Mcap;
                int lo = 0, hi = M;  // first position with lst[pos] >= key (~0 padding sorts last)
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (lst[mid] < key) lo = mid + 1; else hi = mid;
                }
                r += lo;
            }
            const long long gd = (long long)(uint32_t)key - (long long)doc_id_base;
            if (r < M && gd >= 0 && gd < D) {
                f = 1;
                d = (uint32_t)gd;
                grank = (uint32_t)r;
                len = (int)(doc_off[d + 1] - doc_off[d]);
            }
        }
        int tot, ttot;
        const int pos = block_exclusive_scan(f, scan_tmp, &tot);
        const int tpos = block_exclusive_scan(len, scan_tmp, &ttot);
        if (f) {
            kept[(size_t)b * Mcap + outn + pos] = d;
            krank[(size_t)b * Mcap + outn + pos] = grank;
            tok_prefix[(size_t)b * (Mcap + 1) + outn + pos] = run + tpos;
        }
        outn += tot;
        run += ttot;
    }
    if (threadIdx.x == 0) {
        tok_prefix[(size_t)b * (Mcap + 1) + outn] = run;
        n_kept[b] = outn;
        kept_tokens[b] = run;
    }
}

// k_merge_topk: the global cut has at most M members and every global approximate rank belongs to exactly one shard,
// so the real entries of all shards fit M slots indexed by rank: sort those (smem = pow2(M) keys), payloads stay in
// global memory.  `slot` is scratch [B][M] (source position of every rank).  Lists are M = Mcap entries per query;
// qtopk: each query's own top_k (or null: top_k); rows of the outputs are `ostride` apart.
__global__ void __launch_bounds__(1024)
k_merge_topk(const u64 *__restrict__ gfkeys, const u64 *__restrict__ gpayload, int G, int B, int M, int top_k,
             uint32_t *__restrict__ slot, long long *__restrict__ out_ids, float *__restrict__ out_scores,
             int *__restrict__ out_counts, const int *__restrict__ qtopk, int ostride) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int b = blockIdx.x;
    if (qtopk) top_k = qtopk[b];
    const int P = next_pow2(max(M, 1));
    u64 *sk = reinterpret_cast<u64 *>(smem_raw);  // [P], indexed by global approximate rank before the sort
    uint32_t *sl = slot + (size_t)b * M;
    __shared__ int n_real;
    if (threadIdx.x == 0) n_real = 0;
    for (int i = threadIdx.x; i < P; i += blockDim.x) sk[i] = ~0ull;
    __syncthreads();
    int mine = 0;
    for (int i = threadIdx.x; i < G * M; i += blockDim.x) {
        const int g = i / M, j = i - g * M;
        const size_t src = ((size_t)g * B + b) * M + j;
        const u64 v = gfkeys[src];
        if (v != ~0ull) {
            const uint32_t r = (uint32_t)v;  // global approximate rank < M
            sk[r] = v;
            sl[r] = (uint32_t)i;
            ++mine;
        }
    }
    if (mine) atomicAdd(&n_real, mine);
    __syncthreads();
    bitonic_sort_u64(sk, P);
    const int cnt = min(top_k, n_real);
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const uint32_t src = sl[(uint32_t)sk[i]];
        const int g = (int)(src / (uint32_t)M), j = (int)(src - (uint32_t)g * (uint32_t)M);
        const u64 pv = gpayload[((size_t)g * B + b) * M + j];
        out_ids[(size_t)b * ostride + i] = (long long)(pv >> 32);
        out_scores[(size_t)b * ostride + i] = __uint_as_float((uint32_t)pv);
    }
    if (threadIdx.x == 0) out_counts[b] = cnt;
}
