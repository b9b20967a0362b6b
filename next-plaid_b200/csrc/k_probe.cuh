// k_probe.cuh -- a3 probe selection: list scan, threshold-first on the 16-bit table, merge, cells.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ------------------------------------------------------------------------------------------
// a3: per-token top-n.  Selection key = (score_key << 32) | ~c : larger is better, exact score
// ties go to the lower centroid index (the oracle's pinned rule; the reference leaves it to
// select_nth_unstable / heap order).
// k_topn_partial: grid = (ceil(K/4096), B, ceil(QS/32)); 128 threads; each warp streams 1024
// centroid rows, lane = query token, per-lane list of the n best keys in shared memory.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_topn_partial(const float *__restrict__ ST, const int *__restrict__ q_off, long long K, int QS, int n_max,
               const uint32_t *__restrict__ elig_rows, const int *__restrict__ qrow, long long Wke,
               const int *__restrict__ qn, u64 *__restrict__ partial, int n_chunks,
               const int *__restrict__ gate, int gate_want) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    if (gate && (*gate != 0) != (gate_want != 0)) return;  // the threshold path (k_collect16) did the work
    u64 *lists = reinterpret_cast<u64 *>(smem_raw);  // [4 warps][n_max][32 lanes]
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.y, q = blockIdx.z * 32 + lane;
    const int nq = q_off[b + 1] - q_off[b];
    // the query's own n and eligibility row (per-query subsets), lists laid out for the pass's n_max
    const int n = qn ? qn[b] : n_max;
    const uint32_t *eligible = (elig_rows && qrow[b] >= 0) ? elig_rows + (size_t)qrow[b] * Wke : nullptr;
    u64 *mine = lists + (size_t)w * n_max * 32 + lane;
    const int wchunk = blockIdx.x * 4 + w;  // 1024-centroid chunk index
    long long c_begin = (long long)wchunk * 1024, c_end = min(K, c_begin + 1024);
    int cnt = 0, minslot = 0;
    u64 minkey = ~0ull;
    float thr_f = -INFINITY;  // score of the list's worst entry once it is full
    const bool active = q < nq;
    const float *row = ST + ((size_t)b * K) * QS + q;
    for (long long cb = c_begin; cb < c_end; cb += 8) {
        float vals[8];
#pragma unroll
        for (int e = 0; e < 8; ++e)  // 8 independent loads in flight before the (serial) list update
            vals[e] = (active && cb + e < c_end) ? row[(size_t)(cb + e) * QS] : 0.0f;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const long long c = cb + e;
            if (c >= c_end) break;
            if (eligible && !((eligible[c >> 5] >> (c & 31)) & 1u)) continue;  // warp-uniform
            if (!active) continue;
            // fast reject on the raw float once the list is full: a value below the list's worst score
            // (or a NaN, which can only lose to entries scanned earlier) cannot enter
            if (cnt == n && !(vals[e] >= thr_f)) continue;
            u64 key = ((u64)score_key_asc(vals[e]) << 32) | (uint32_t)(~(uint32_t)c);
            if (cnt < n) {
                mine[(size_t)cnt * 32] = key;
                if (key < minkey) {
                    minkey = key;
                    minslot = cnt;
                }
                ++cnt;
            } else if (key > minkey) {
                mine[(size_t)minslot * 32] = key;
                minkey = ~0ull;
                for (int s2 = 0; s2 < n; ++s2) {
                    u64 k2 = mine[(size_t)s2 * 32];
                    if (k2 < minkey) {
                        minkey = k2;
                        minslot = s2;
                    }
                }
            }
            if (cnt == n) {
                const uint32_t hi = (uint32_t)(minkey >> 32);
                thr_f = hi ? key_to_score(hi) : -INFINITY;
            }
        }
    }
    if (q < QS && wchunk < n_chunks) {
        u64 *out = partial + (((size_t)b * QS + q) * n_chunks + wchunk) * n_max;
        for (int s = 0; s < n_max; ++s) out[s] = (active && s < cnt) ? mine[(size_t)s * 32] : 0ull;
    }
}

// ------------------------------------------------------------------------------------------
// a3 on the 16-bit table: threshold first, select second.
// The 16-bit code of a score is a monotone image of it, so with tau = the n-th largest of the per-chunk maxima
// of a token's codes (n entries with code >= tau exist) every entry with code < tau is beaten by n others and
// cannot be in the token's top n.  k_chunkmax16 and k_collect16 stream the 16-bit table (half the bytes of S,
// no per-lane lists, no divergence in the common case); the few entries with code >= tau get their exact key
// from S and k_topn_merge ranks them as before.  More than `cap` such entries (massive ties), a flagged
// query (non-finite scores, no valid table) or an eligibility filter fall back to k_topn_partial: *fallback
// is set on the device and gates the two paths.
// ST16 rows are QS codes; a lane owns one 16-byte group (8 query tokens) of a row, GQ = QS/8 lanes per row.
// grid = (ceil(n_chunks/4), B), 128 threads, one warp per chunk of `chunk_rows` centroids (1024, fewer for small K so
// that at least n chunks exist).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_chunkmax16(const unsigned short *__restrict__ ST16, long long K, int QS, int n_chunks, int chunk_rows,
             unsigned short *__restrict__ cmax) {
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
    const int chunk = blockIdx.x * 4 + w;
    if (chunk >= n_chunks) return;
    // GQ lanes cover one row; L = the largest multiple of GQ that fits a warp, so a lane keeps its 8 query
    // tokens for the whole scan (GQ a power of two: L = 32; nq = 48: GQ = 6, L = 30, two lanes idle)
    const int GQ = QS >> 3, L = (32 / GQ) * GQ;
    const long long c0 = (long long)chunk * chunk_rows;
    const int rows = (int)min((long long)chunk_rows, K - c0);
    const uint4 *base = reinterpret_cast<const uint4 *>(ST16 + ((size_t)b * K + c0) * QS);
    const int total = rows * GQ;
    uint4 acc = make_uint4(0, 0, 0, 0);
    if (lane < L) {
        int idx = lane;
        for (; idx + 7 * L < total; idx += 8 * L) {
            uint4 v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = __ldg(base + idx + L * e);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                acc.x = __vmaxu2(acc.x, v[e].x);
                acc.y = __vmaxu2(acc.y, v[e].y);
                acc.z = __vmaxu2(acc.z, v[e].z);
                acc.w = __vmaxu2(acc.w, v[e].w);
            }
        }
        for (; idx < total; idx += L) {
            const uint4 v = __ldg(base + idx);
            acc.x = __vmaxu2(acc.x, v.x);
            acc.y = __vmaxu2(acc.y, v.y);
            acc.z = __vmaxu2(acc.z, v.z);
            acc.w = __vmaxu2(acc.w, v.w);
        }
    }
    for (int off = GQ; off < L; off <<= 1) {  // lanes g, g + GQ, g + 2 GQ, ... hold the same query tokens
        const uint32_t ox = __shfl_down_sync(PB_FULL, acc.x, off), oy = __shfl_down_sync(PB_FULL, acc.y, off);
        const uint32_t oz = __shfl_down_sync(PB_FULL, acc.z, off), ow = __shfl_down_sync(PB_FULL, acc.w, off);
        if (lane + off < L) {
            acc.x = __vmaxu2(acc.x, ox);
            acc.y = __vmaxu2(acc.y, oy);
            acc.z = __vmaxu2(acc.z, oz);
            acc.w = __vmaxu2(acc.w, ow);
        }
    }
    if (lane < GQ) *reinterpret_cast<uint4 *>(cmax + ((size_t)b * n_chunks + chunk) * QS + 8 * lane) = acc;
}

// tau[b][q] = the largest t with at least n chunk maxima >= t; 65536 for padding rows.  grid = (QS, B), 32 threads.
__global__ void k_tau16(const unsigned short *__restrict__ cmax, const int *__restrict__ q_off, int QS, int n, int n_chunks,
                        const int *__restrict__ qflag, uint32_t *__restrict__ tau, int *__restrict__ fallback) {
    const int q = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
    const int nq = q_off[b + 1] - q_off[b];
    if (q == 0 && lane == 0 && qflag[b]) atomicOr(fallback, 1);
    if (q >= nq) {
        if (lane == 0) tau[(size_t)b * QS + q] = 65536u;
        return;
    }
    const unsigned short *col = cmax + (size_t)b * n_chunks * QS + q;
    uint32_t lo = 0u, hi = 65536u;  // count(lo) >= n holds (n_chunks >= n), count(hi) = 0
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        int cnt = 0;
        for (int i = lane; i < n_chunks; i += 32) cnt += (col[(size_t)i * QS] >= mid) ? 1 : 0;
        for (int m = 16; m >= 1; m >>= 1) cnt += __shfl_xor_sync(PB_FULL, cnt, m);
        if (cnt >= n) lo = mid; else hi = mid;
    }
    if (lane == 0) tau[(size_t)b * QS + q] = lo;
}

__global__ void __launch_bounds__(128)
k_collect16(const unsigned short *__restrict__ ST16, const float *__restrict__ ST, long long K, int QS, int n_chunks,
            int chunk_rows, const uint32_t *__restrict__ tau, int cap, int *__restrict__ counts, u64 *__restrict__ list,
            int *__restrict__ fallback) {
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
    const int chunk = blockIdx.x * 4 + w;
    if (chunk >= n_chunks || *fallback) return;
    const int GQ = QS >> 3, L = (32 / GQ) * GQ, g = lane % GQ;  // lane -> query-token group as in k_chunkmax16
    if (lane >= L) return;
    const long long c0 = (long long)chunk * chunk_rows;
    const int rows = (int)min((long long)chunk_rows, K - c0);
    const uint4 *base = reinterpret_cast<const uint4 *>(ST16 + ((size_t)b * K + c0) * QS);
    const int total = rows * GQ;
    // this lane's 8 thresholds as packed halfwords; padding rows (tau = 65536) never match
    uint32_t t2[4], live[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const uint32_t a = tau[(size_t)b * QS + 8 * g + 2 * e], c = tau[(size_t)b * QS + 8 * g + 2 * e + 1];
        t2[e] = min(a, 65535u) | (min(c, 65535u) << 16);
        live[e] = (a < 65536u ? 0xffffu : 0u) | (c < 65536u ? 0xffff0000u : 0u);
    }
    for (int i0 = lane; i0 < total; i0 += 8 * L) {
        uint4 v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = (i0 + L * e < total) ? __ldg(base + i0 + L * e) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const uint32_t hx = __vcmpgeu2(v[e].x, t2[0]) & live[0], hy = __vcmpgeu2(v[e].y, t2[1]) & live[1];
            const uint32_t hz = __vcmpgeu2(v[e].z, t2[2]) & live[2], hw = __vcmpgeu2(v[e].w, t2[3]) & live[3];
            if ((hx | hy | hz | hw) == 0u || i0 + L * e >= total) continue;  // the common case
            const long long c = c0 + (i0 + L * e) / GQ;
            const uint32_t hits[4] = {hx, hy, hz, hw};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (!((hits[j >> 1] >> (16 * (j & 1))) & 1u)) continue;
                const int q = 8 * g + j;
                const int slot = atomicAdd(&counts[(size_t)b * QS + q], 1);
                if (slot < cap)
                    list[((size_t)b * QS + q) * cap + slot] =
                        ((u64)score_key_asc(ST[((size_t)b * K + c) * QS + q]) << 32) | (uint32_t)(~(uint32_t)c);
                else atomicOr(fallback, 1);
            }
        }
    }
}

// k_topn_merge: one warp per (b, q): n rounds of "largest key strictly below the previous winner".
// grid = (QS, B), 32 threads.  sel[b][q][n] gets the winning keys in rank order (0 = none).  qn: each query's own n
// (rows keep the stride n, the rest zero), or null.
__global__ void k_topn_merge(const u64 *__restrict__ partial, const int *__restrict__ q_off, int QS,
                             int n, int n_chunks, u64 *__restrict__ sel, const int *__restrict__ gate, int gate_want,
                             const int *__restrict__ qn) {
    if (gate && (*gate != 0) != (gate_want != 0)) return;
    const int q = blockIdx.x, b = blockIdx.y, lane = threadIdx.x;
    const int nq = q_off[b + 1] - q_off[b];
    u64 *out = sel + ((size_t)b * QS + q) * n;
    if (q >= nq) {
        for (int s = lane; s < n; s += 32) out[s] = 0ull;
        return;
    }
    const u64 *in = partial + ((size_t)b * QS + q) * n_chunks * n;
    const int P = n_chunks * n;
    const int nb = qn ? qn[b] : n;
    for (int s = nb + lane; s < n; s += 32) out[s] = 0ull;
    u64 bound = ~0ull;
    for (int r = 0; r < nb; ++r) {
        u64 best = 0ull;
        for (int i = lane; i < P; i += 32) {
            u64 k = in[i];
            if (k < bound && k > best) best = k;
        }
        best = warp_max_u64(best);
        if (lane == 0) out[r] = best;
        if (best == 0ull) {
            for (int s = r + 1 + lane; s < nb; s += 32) out[s] = 0ull;
            break;
        }
        bound = best;
    }
}

// k_cells: one CTA (256 threads) per query: union of the selected centroids, then the threshold
// rule of the variant in use, output ascending.
//   dense   (search.rs:417-425): keep c iff max over ALL query tokens of S[q][c] >= t
//   batched (search.rs:177-199, :226-251): keep c iff final_max[c] >= t, where final_max only
//           records S[q][c] for tokens q whose slab heap c entered at scan time, i.e. fewer than
//           n_probe earlier centroids of the same slab score >= S[q][c] (in the score order).
__global__ void __launch_bounds__(256)
k_cells(const u64 *__restrict__ sel, const float *__restrict__ ST, const int *__restrict__ q_off,
        long long K, int QS, int n, int cells_cap, int has_thr, float thr, int batched,
        long long slab, uint32_t *__restrict__ cells, int *__restrict__ n_cells,
        const unsigned short *__restrict__ cmax16, int n_chunks, int chunk_rows, const float2 *__restrict__ qrange,
        const int *__restrict__ gate) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int b = blockIdx.x;
    const int nq = q_off[b + 1] - q_off[b];
    const int total = nq * n;
    const int P = next_pow2(max(total, 1));
    // chunk maxima of the 16-bit table (threshold-first probe) prune the slab-prefix scan below; not when the
    // probe fell back (flagged query: no valid table)
    const bool use_cmax = cmax16 != nullptr && !(gate && *gate);
    u64 *s = reinterpret_cast<u64 *>(smem_raw);  // [P] sort buffer, then unique list
    int *flags = reinterpret_cast<int *>(s + P);  // [P]
    __shared__ int scan_tmp[33];
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        u64 v = ~0ull;
        if (i < total) {
            u64 k = sel[(size_t)b * QS * n + i];  // rows q < nq are the first nq*n entries
            if (k != 0ull) v = (u64)(uint32_t)(~(uint32_t)k);  // centroid id
        }
        s[i] = v;
    }
    __syncthreads();
    bitonic_sort_u64(s, P);
    // unique
    int nu = 0;
    for (int base = 0; base < P; base += blockDim.x) {
        int i = base + threadIdx.x;
        int f = (i < P && s[i] != ~0ull && (i == 0 || s[i - 1] != s[i])) ? 1 : 0;
        int tot;
        int pos = block_exclusive_scan(f, scan_tmp, &tot);
        u64 v = i < P ? s[i] : 0;
        __syncthreads();
        if (f) reinterpret_cast<uint32_t *>(flags)[nu + pos] = (uint32_t)v;  // stage ids in flags
        nu += tot;
        __syncthreads();
    }
    // move unique ids to the front of s (as u32 in the low half), flags reused below
    for (int i = threadIdx.x; i < nu; i += blockDim.x) s[i] = reinterpret_cast<uint32_t *>(flags)[i];
    __syncthreads();
    // threshold, one warp per unique centroid
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const float *STb = ST + (size_t)b * K * QS;
    for (int u = w; u < nu; u += nwarps) {
        const uint32_t c = (uint32_t)s[u];
        int keep = 1;
        if (has_thr) {
            const float *row = STb + (size_t)c * QS;
            if (!batched) {
                uint32_t best = 0u;
                for (int q = lane; q < nq; q += 32) best = max(best, score_key_asc(row[q]));
#pragma unroll
                for (int m = 16; m >= 1; m >>= 1) best = max(best, __shfl_xor_sync(PB_FULL, best, m));
                // Iterator::max_by keeps the last maximum: all non-finite -> the last token's value
                float mval = best ? key_to_score(best) : (nq > 0 ? row[nq - 1] : -INFINITY);
                keep = (mval >= thr);
            } else {
                // m1 = best finite score among tokens that selected c (they entered their slab heap).
                // Non-finite scores are not tracked here: with NaN/Inf centroid scores only the
                // dense variant's threshold is reproduced exactly (DESIGN.md "Limits").
                uint32_t best = 0u;
                for (int q = lane; q < nq; q += 32) {
                    const u64 *sq = sel + ((size_t)b * QS + q) * n;
                    bool is_sel = false;
                    for (int i = 0; i < n; ++i)
                        if (sq[i] != 0ull && (uint32_t)(~(uint32_t)sq[i]) == c) is_sel = true;
                    if (is_sel) best = max(best, score_key_asc(row[q]));
                }
#pragma unroll
                for (int m = 16; m >= 1; m >>= 1) best = max(best, __shfl_xor_sync(PB_FULL, best, m));
                float m1 = best ? key_to_score(best) : -INFINITY;
                keep = (m1 >= thr);
                if (!keep) {
                    // another token may have recorded a score >= thr for c while scanning its slab
                    const long long s0 = (long long)(c / slab) * slab;
                    for (int q = 0; q < nq && !keep; ++q) {
                        const float v = row[q];
                        const uint32_t kv = score_key_asc(v);
                        if (!(kv != 0u && v >= thr)) continue;  // finite and over the threshold
                        // entered iff fewer than n earlier slab entries are "not worse" than v
                        int cnt = 0;
                        if (use_cmax) {  // a chunk whose largest code is below code(v) holds no entry >= v
                            const float2 rg = qrange[b];
                            const int kv16 = (int)fminf(fmaxf(floorf(__fmaf_rn(v, rg.y, rg.x)), 0.0f), 65535.0f);
                            const long long ch_lo = s0 / chunk_rows, ch_hi = ((long long)c + chunk_rows - 1) / chunk_rows;
                            for (long long ch0 = ch_lo; ch0 < ch_hi; ch0 += 32) {
                                const long long chl = ch0 + lane;
                                const bool need = chl < ch_hi && (int)cmax16[((size_t)b * n_chunks + chl) * QS + q] >= kv16;
                                unsigned todo = __ballot_sync(PB_FULL, need);
                                while (todo) {
                                    const long long ch = ch0 + (__ffs(todo) - 1);
                                    todo &= todo - 1;
                                    const long long r_lo = max(s0, ch * chunk_rows), r_hi = min((long long)c, (ch + 1) * chunk_rows);
                                    for (long long c2 = r_lo + lane; c2 < r_hi; c2 += 32)
                                        cnt += (score_key_asc(STb[(size_t)c2 * QS + q]) >= kv) ? 1 : 0;
                                }
                            }
                        } else
                            for (long long c2 = s0 + lane; c2 < (long long)c; c2 += 32)
                                cnt += (score_key_asc(STb[(size_t)c2 * QS + q]) >= kv) ? 1 : 0;
#pragma unroll
                        for (int m = 16; m >= 1; m >>= 1) cnt += __shfl_xor_sync(PB_FULL, cnt, m);
                        if (cnt < n) keep = 1;
                    }
                }
            }
        }
        if (lane == 0) flags[u] = keep;
    }
    __syncthreads();
    // ordered compaction
    int outn = 0;
    for (int base = 0; base < nu; base += blockDim.x) {
        int i = base + threadIdx.x;
        int f = (i < nu) ? flags[i] : 0;
        int tot;
        int pos = block_exclusive_scan(f, scan_tmp, &tot);
        if (f && outn + pos < cells_cap) cells[(size_t)b * cells_cap + outn + pos] = (uint32_t)s[i];
        outn += tot;
    }
    if (threadIdx.x == 0) n_cells[b] = min(outn, cells_cap);
}
