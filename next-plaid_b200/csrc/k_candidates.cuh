// k_candidates.cuh -- a4 candidates, a5 single-pass approximate score, a6 cut.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ------------------------------------------------------------------------------------------
// a4: candidates = sorted unique union of the posting lists of the surviving cells.
// k_mark: grid = (cells_cap, B): set one bit per (query, doc) of the query's subset row, if it has one.  k_compact_count / k_compact_emit turn the bitmap
// into an ascending doc-id list (and clear it for the next call).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_mark(const uint32_t *__restrict__ cells, const int *__restrict__ n_cells, int cells_cap,
       const uint32_t *__restrict__ ivf, const long long *__restrict__ ivf_off,
       const uint32_t *__restrict__ subset_bits, const int *__restrict__ qrow, uint32_t *__restrict__ bitmap,
       long long W) {
    const int b = blockIdx.y;
    if ((int)blockIdx.x >= n_cells[b]) return;
    const uint32_t c = cells[(size_t)b * cells_cap + blockIdx.x];
    uint32_t *bm = bitmap + (size_t)b * W;
    // the query's subset row (k_subset_bits), or none
    const uint32_t *sb = (subset_bits && qrow[b] >= 0) ? subset_bits + (size_t)qrow[b] * W : nullptr;
    for (long long i = ivf_off[c] + threadIdx.x; i < ivf_off[c + 1]; i += blockDim.x) {
        uint32_t d = ivf[i];
        if (sb && !((sb[d >> 5] >> (d & 31)) & 1u)) continue;
        atomicOr(&bm[d >> 5], 1u << (d & 31));
    }
}

// k_compact_count / k_compact_emit: grid = (slices, B), 256 threads.  A query's bitmap is cut into `slices` equal word
// ranges; pass 1 counts the bits of every slice, pass 2 places its slice after the slices before it (ascending doc
// ids overall), clears the words for the next call and -- the last slice -- publishes the total.
__global__ void __launch_bounds__(256)
k_compact_count(const uint32_t *__restrict__ bitmap, long long W, int *__restrict__ slice_counts) {
    __shared__ int red[8];
    const int b = blockIdx.y, S = gridDim.x;
    const long long per = (W + S - 1) / S, w0 = min(W, (long long)blockIdx.x * per), w1 = min(W, w0 + per);
    const uint32_t *bm = bitmap + (size_t)b * W;
    int cnt = 0;
    for (long long i = w0 + threadIdx.x; i < w1; i += blockDim.x) cnt += __popc(bm[i]);
    cnt = __reduce_add_sync(PB_FULL, cnt);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int i = 0; i < 8; ++i) t += red[i];
        slice_counts[(size_t)b * S + blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(256)
k_compact_emit(uint32_t *__restrict__ bitmap, long long W, const int *__restrict__ slice_counts, uint32_t *__restrict__ cand,
               long long cand_cap, int *__restrict__ n_cand) {
    __shared__ int scan_tmp[33];
    const int b = blockIdx.y, S = gridDim.x;
    const long long per = (W + S - 1) / S, w0 = min(W, (long long)blockIdx.x * per), w1 = min(W, w0 + per);
    uint32_t *bm = bitmap + (size_t)b * W;
    int base = 0;
    for (int i = 0; i < (int)blockIdx.x; ++i) base += slice_counts[(size_t)b * S + i];
    // each thread owns a contiguous run of the slice's words, so positions ascend with the doc id
    const long long tper = (w1 - w0 + blockDim.x - 1) / blockDim.x;
    const long long t0 = min(w1, w0 + (long long)threadIdx.x * tper), t1 = min(w1, t0 + tper);
    int cnt = 0;
    for (long long i = t0; i < t1; ++i) cnt += __popc(bm[i]);
    int total;
    int pos = base + block_exclusive_scan(cnt, scan_tmp, &total);
    uint32_t *out = cand + (size_t)b * cand_cap;
    for (long long i = t0; i < t1; ++i) {
        uint32_t x = bm[i];
        if (x) bm[i] = 0u;
        while (x) {
            const int bit = __ffs(x) - 1;
            x &= x - 1;
            out[pos++] = (uint32_t)(i * 32 + bit);
        }
    }
    if (blockIdx.x == S - 1 && threadIdx.x == 0) n_cand[b] = base + total;
}

// ------------------------------------------------------------------------------------------
// a5: approximate score, one warp per candidate doc, lane = query token.
// grid = (blocks, B), 256 threads.  Emits the cut key (~score_key << 32 | doc): ascending key order
// == (approx desc in the score order, doc id asc) == the stable sort of search.rs:460.
// ------------------------------------------------------------------------------------------
// Max over a doc's distinct codes of one column of the score table, 16 row gathers in flight per
// lane (the stage is bound by L2 request latency, not bytes: keep the queue full) with the next 16
// codes prefetched.  Lists are padded to a multiple of 8 and 32-byte aligned.
struct GatherF32 {
    typedef float T;
    static PB_DEV T init() { return -INFINITY; }
    static PB_DEV T ld(const char *p) { return *reinterpret_cast<const float *>(p); }
    // `if (v > m) m = v` of search.rs:313-315 == fmaxf here: m never becomes NaN, a NaN v is ignored
    // by both, and -0/+0 cannot change the q-ordered sum taken afterwards
    static PB_DEV T mx(T a, T b) { return fmaxf(a, b); }
};
struct GatherU16 {
    typedef uint32_t T;
    static PB_DEV T init() { return 0u; }
    static PB_DEV T ld(const char *p) { return *reinterpret_cast<const unsigned short *>(p); }
    static PB_DEV T mx(T a, T b) { return max(a, b); }
};

template <class G>
PB_DEV typename G::T gather_max(const char *__restrict__ col, unsigned rowb, const uint32_t *__restrict__ ucodes,
                                long long t0, long long t1) {
    typedef typename G::T T;
    T m = G::init();
    long long t = t0;
    uint4 c0, c1, c2, c3;
    if (t + 16 <= t1) {
        c0 = *reinterpret_cast<const uint4 *>(ucodes + t);
        c1 = *reinterpret_cast<const uint4 *>(ucodes + t + 4);
        c2 = *reinterpret_cast<const uint4 *>(ucodes + t + 8);
        c3 = *reinterpret_cast<const uint4 *>(ucodes + t + 12);
    }
    while (t + 16 <= t1) {
        uint4 n0 = c0, n1 = c1, n2 = c2, n3 = c3;
        if (t + 32 <= t1) {
            n0 = *reinterpret_cast<const uint4 *>(ucodes + t + 16);
            n1 = *reinterpret_cast<const uint4 *>(ucodes + t + 20);
            n2 = *reinterpret_cast<const uint4 *>(ucodes + t + 24);
            n3 = *reinterpret_cast<const uint4 *>(ucodes + t + 28);
        }
        const T v0 = G::ld(col + (size_t)c0.x * rowb), v1 = G::ld(col + (size_t)c0.y * rowb);
        const T v2 = G::ld(col + (size_t)c0.z * rowb), v3 = G::ld(col + (size_t)c0.w * rowb);
        const T v4 = G::ld(col + (size_t)c1.x * rowb), v5 = G::ld(col + (size_t)c1.y * rowb);
        const T v6 = G::ld(col + (size_t)c1.z * rowb), v7 = G::ld(col + (size_t)c1.w * rowb);
        const T v8 = G::ld(col + (size_t)c2.x * rowb), v9 = G::ld(col + (size_t)c2.y * rowb);
        const T va = G::ld(col + (size_t)c2.z * rowb), vb = G::ld(col + (size_t)c2.w * rowb);
        const T vc = G::ld(col + (size_t)c3.x * rowb), vd = G::ld(col + (size_t)c3.y * rowb);
        const T ve = G::ld(col + (size_t)c3.z * rowb), vf = G::ld(col + (size_t)c3.w * rowb);
        const T a = G::mx(G::mx(G::mx(v0, v1), G::mx(v2, v3)), G::mx(G::mx(v4, v5), G::mx(v6, v7)));
        const T b = G::mx(G::mx(G::mx(v8, v9), G::mx(va, vb)), G::mx(G::mx(vc, vd), G::mx(ve, vf)));
        m = G::mx(m, G::mx(a, b));
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        t += 16;
    }
    if (t < t1) {  // one block of 8 left
        const uint4 ca = *reinterpret_cast<const uint4 *>(ucodes + t);
        const uint4 cb = *reinterpret_cast<const uint4 *>(ucodes + t + 4);
        const T v0 = G::ld(col + (size_t)ca.x * rowb), v1 = G::ld(col + (size_t)ca.y * rowb);
        const T v2 = G::ld(col + (size_t)ca.z * rowb), v3 = G::ld(col + (size_t)ca.w * rowb);
        const T v4 = G::ld(col + (size_t)cb.x * rowb), v5 = G::ld(col + (size_t)cb.y * rowb);
        const T v6 = G::ld(col + (size_t)cb.z * rowb), v7 = G::ld(col + (size_t)cb.w * rowb);
        m = G::mx(m, G::mx(G::mx(G::mx(v0, v1), G::mx(v2, v3)), G::mx(G::mx(v4, v5), G::mx(v6, v7))));
    }
    return m;
}

__global__ void __launch_bounds__(256)
k_approx(const float *__restrict__ ST, const int *__restrict__ q_off, long long K, int QS,
         const uint32_t *__restrict__ ucodes, const long long *__restrict__ udoc_off,
         const uint32_t *__restrict__ cand, long long cand_cap, const int *__restrict__ n_cand,
         float *__restrict__ approx, u64 *__restrict__ keys, unsigned long long *__restrict__ tok_counter,
         uint32_t doc_id_base) {
    // ucodes: per doc its DISTINCT centroid codes (max over tokens == max over distinct codes),
    // padded to a multiple of 8 by repeating the last code, 32-byte aligned: uniform 128-bit
    // loads feed the row gathers (gather_max).
    const int b = blockIdx.y;
    const int nq = q_off[b + 1] - q_off[b];
    const int n = n_cand[b];
    const int lane = threadIdx.x & 31;
    const int warps_per_grid = gridDim.x * (blockDim.x >> 5);
    const float *STb = ST + (size_t)b * K * QS;
    const unsigned rowb = (unsigned)QS * 4u;  // K * QS * 4 < 2^32 is checked on the host
    unsigned long long my_tokens = 0;
    int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    uint32_t d = 0;
    long long t0 = 0, t1 = 0;
    if (i < n) {
        d = cand[(size_t)b * cand_cap + i];
        t0 = udoc_off[d];
        t1 = udoc_off[d + 1];
    }
    for (; i < n; i += warps_per_grid) {
        // next doc's metadata is fetched under this doc's gathers
        const int i2 = i + warps_per_grid;
        uint32_t dn = 0;
        long long t0n = 0, t1n = 0;
        if (i2 < n) {
            dn = cand[(size_t)b * cand_cap + i2];
            t0n = udoc_off[dn];
            t1n = udoc_off[dn + 1];
        }
        my_tokens += (unsigned long long)(t1 - t0);
        float score = 0.0f;
        for (int qc = 0; qc < nq; qc += 32) {
            const int q = qc + lane;
            const char *col = reinterpret_cast<const char *>(STb + (q < nq ? q : 0));
            const float m = gather_max<GatherF32>(col, rowb, ucodes, t0, t1);
            // score += m for q ascending, skipping rows whose max stayed -inf (search.rs:318-320)
            const int lim = min(32, nq - qc);
            for (int qq = 0; qq < lim; ++qq) {
                float mv = __shfl_sync(PB_FULL, m, qq);
                if (mv > -INFINITY) score = __fadd_rn(score, mv);
            }
        }
        if (lane == 0) {
            approx[(size_t)b * cand_cap + i] = score;
            // tie-break on the GLOBAL doc id so shards merge into the unsharded order
            keys[(size_t)b * cand_cap + i] = ((u64)(~score_key_asc(score)) << 32) | (d + doc_id_base);
        }
        d = dn;
        t0 = t0n;
        t1 = t1n;
    }
    if (lane == 0 && my_tokens) atomicAdd(tok_counter, my_tokens);  // work counter for bench.py
}

// index-open transform behind k_approx: per doc the sorted distinct codes.  One CTA (128 threads)
// per doc, bitonic sort in shared memory; docs longer than PB_UCODE_MAX keep their raw code list
// (duplicates are harmless for a max).  pass 0 counts (padded to 8), pass 1 writes.
#define PB_UCODE_MAX 4096
__global__ void __launch_bounds__(128)
k_unique_codes(const uint32_t *__restrict__ codes, const long long *__restrict__ doc_off, long long D,
               const long long *__restrict__ udoc_off, uint32_t *__restrict__ ucodes, int *__restrict__ counts) {
    __shared__ u64 sk[PB_UCODE_MAX];
    __shared__ int scan_tmp[33];
    for (long long d = blockIdx.x; d < D; d += gridDim.x) {
        const long long t0 = doc_off[d];
        const int len = (int)(doc_off[d + 1] - t0);
        __syncthreads();
        if (len > PB_UCODE_MAX) {  // raw copy
            const int padded = (len + 7) & ~7;
            if (!ucodes) {
                if (threadIdx.x == 0) counts[d] = padded;
            } else {
                uint32_t *out = ucodes + udoc_off[d];
                for (int i = threadIdx.x; i < padded; i += blockDim.x) out[i] = codes[t0 + min(i, len - 1)];
            }
            continue;
        }
        const int P = next_pow2(max(len, 1));
        for (int i = threadIdx.x; i < P; i += blockDim.x) sk[i] = i < len ? (u64)codes[t0 + i] : ~0ull;
        __syncthreads();
        bitonic_sort_u64(sk, P);
        int nu = 0;
        for (int base = 0; base < P; base += blockDim.x) {
            const int i = base + threadIdx.x;
            const int f = (i < len && (i == 0 || sk[i - 1] != sk[i])) ? 1 : 0;
            int tot;
            const int pos = block_exclusive_scan(f, scan_tmp, &tot);
            if (f && ucodes) ucodes[udoc_off[d] + nu + pos] = (uint32_t)sk[i];
            nu += tot;
        }
        const int padded = (nu + 7) & ~7;
        if (!ucodes) {
            if (threadIdx.x == 0) counts[d] = padded;
        } else if (threadIdx.x < padded - nu) {
            ucodes[udoc_off[d] + nu + threadIdx.x] = (uint32_t)sk[len - 1];  // repeat the largest code
        }
    }
}

// ------------------------------------------------------------------------------------------
// a6: per query, the M smallest cut keys in ascending order (M = min(n_full_scores, n_decompress)),
// via MSB radix select + bitonic sort; also the token prefix sums the exact stage walks.
// grid = B, 1024 threads, dynamic smem = Mpow2*8 bytes.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
k_cut(const u64 *__restrict__ keys, const float *__restrict__ approx_in, long long cand_cap,
      const int *__restrict__ n_cand, int M, int Mcap, const long long *__restrict__ doc_off,
      uint32_t *__restrict__ kept, int *__restrict__ n_kept, long long *__restrict__ tok_prefix,
      long long *__restrict__ kept_tokens, uint32_t doc_id_base, u64 *__restrict__ out_keys) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64 *sk = reinterpret_cast<u64 *>(smem_raw);
    __shared__ int hist[256];
    __shared__ int scan_tmp[33];
    __shared__ u64 prefix_s, mask_s;
    __shared__ int remaining_s, fill_s;
    const int b = blockIdx.x;
    const int n = n_cand[b];
    const int Mq = min(M, n);
    const u64 *kb = keys + (size_t)b * cand_cap;
    const int P = next_pow2(max(Mq, 1));
    if (n <= M) {
        for (int i = threadIdx.x; i < P; i += blockDim.x) sk[i] = i < n ? kb[i] : ~0ull;
        __syncthreads();
    } else {
        if (threadIdx.x == 0) {
            prefix_s = 0ull;
            mask_s = 0ull;
            remaining_s = Mq;
        }
        for (int pass = 7; pass >= 0; --pass) {
            const int shift = pass * 8;
            for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
            __syncthreads();
            const u64 prefix = prefix_s, mask = mask_s;
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                u64 k = kb[i];
                if ((k & mask) == prefix) atomicAdd(&hist[(int)((k >> shift) & 255ull)], 1);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                int rem = remaining_s, cum = 0, d = 0;
                for (; d < 256; ++d) {
                    if (cum + hist[d] >= rem) break;
                    cum += hist[d];
                }
                remaining_s = rem - cum;
                prefix_s = prefix | ((u64)d << shift);
                mask_s = mask | (255ull << shift);
            }
            __syncthreads();
        }
        const u64 pivot = prefix_s;  // the Mq-th smallest key (keys are unique: doc id in the low word)
        if (threadIdx.x == 0) fill_s = 0;
        for (int i = threadIdx.x; i < P; i += blockDim.x) sk[i] = ~0ull;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            u64 k = kb[i];
            if (k <= pivot) sk[atomicAdd(&fill_s, 1)] = k;
        }
        __syncthreads();
    }
    bitonic_sort_u64(sk, P);
    if (out_keys) {  // doc-sharded mode: the shard's sorted top-M goes to the all-gather; kept docs come from k_merge_cut
        for (int i = threadIdx.x; i < M; i += blockDim.x) out_keys[(size_t)b * M + i] = i < Mq ? sk[i] : ~0ull;
        return;
    }
    // outputs + token prefix sums
    long long run = 0;
    for (int base = 0; base < Mq; base += blockDim.x) {
        int i = base + threadIdx.x;
        int len = 0;
        uint32_t d = 0;
        if (i < Mq) {
            d = (uint32_t)sk[i] - doc_id_base;
            len = (int)(doc_off[d + 1] - doc_off[d]);
            kept[(size_t)b * Mcap + i] = d;
        }
        int tot;
        int pos = block_exclusive_scan(len, scan_tmp, &tot);
        if (i < Mq) tok_prefix[(size_t)b * (Mcap + 1) + i] = run + pos;
        run += tot;
    }
    if (threadIdx.x == 0) {
        tok_prefix[(size_t)b * (Mcap + 1) + Mq] = run;
        n_kept[b] = Mq;
        kept_tokens[b] = run;
    }
    (void)approx_in;
}

