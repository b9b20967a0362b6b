// k_approx16.cuh -- a5 two-pass form: 16-bit first pass, band select.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ------------------------------------------------------------------------------------------
// a5, two-pass form.  The approximate score only decides WHICH docs make the cut (search.rs:460-469),
// so a first pass ranks every candidate on a 16-bit fixed-point copy of S (half the L2 bytes per
// gather) and only the docs that could still be in the top M -- the M-th largest code sum minus a
// certified band -- get the exact fp32 pass (k_approx).  The cut is therefore EXACTLY the reference's.
//   code(v) = floor(fl(v*scale + R*scale)), monotone in v, |v| <= R = max|c| * max|q| * (1+1e-4)
//   true per-token max in [(code-1)/scale - R, (code+2)/scale - R]; fp32 sum error <= nq*R*2^-18
//   => doc X certainly outranks doc Y when L_X - L_Y > 3.25*nq; band W = 4*nq + 8 code units.
// Queries whose scores leave [-R, R] or are non-finite (qflag) skip the shortcut entirely.
// ------------------------------------------------------------------------------------------
// Per query: the largest token norm, and what the stages derive from it --
//   qrange[b] = (R*scale, scale) of the 16-bit score code, R = max|c| * max|q| * (1 + 1e-4), scale = 65535 / 2R
//   qflag[b]  = 1 when the range is unusable (non-finite or degenerate norms): the query takes the exact paths
//   qexp[b]   = the power of two that brings the largest token norm into [1, 2) (operand scaling of k_scores16_tc)
//   qnmax[b]  = max|q| * (1 + 1e-4), the scale of the MaxSim filter's error bound
// grid = B, 256 threads: a warp per token row.
__global__ void __launch_bounds__(256)
k_query_range(const float *__restrict__ Q, const int *__restrict__ q_off, int dim, float cmax,
              float2 *__restrict__ qrange, int *__restrict__ qflag, int *__restrict__ qexp, float *__restrict__ qnmax) {
    __shared__ float best_s[8];
    __shared__ int bad_s[8];
    const int b = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int r0 = q_off[b], nq = q_off[b + 1] - r0;
    float best = 0.0f;
    bool bad = false;
    for (int r = w; r < nq; r += 8) {
        float p = 0.0f;
        for (int j = lane; j < dim; j += 32) {
            const float v = Q[(size_t)(r0 + r) * dim + j];
            p = fmaf(v, v, p);
        }
        for (int m = 16; m >= 1; m >>= 1) p += __shfl_xor_sync(PB_FULL, p, m);
        bad |= !(p <= 3.0e38f);
        best = fmaxf(best, p == p ? p : INFINITY);
    }
    if (lane == 0) {
        best_s[w] = best;
        bad_s[w] = bad ? 1 : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 8; ++i) {
            best = fmaxf(best, best_s[i]);
            bad |= bad_s[i] != 0;
        }
        float R = cmax * sqrtf(best) * 1.0001f;
        int kq = 0, flag = 0;
        if (!(R > 1e-30f) || !(R < 1e30f) || bad) {
            R = 1.0f;
            flag = nq > 0 ? 1 : 0;
        } else kq = -ilogbf(sqrtf(best));
        const float scale = 65535.0f / (2.0f * R);
        if (qrange) qrange[b] = make_float2(R * scale, scale);
        if (qflag) qflag[b] = flag;
        if (qexp) qexp[b] = kq;
        if (qnmax) qnmax[b] = sqrtf(best) * 1.0001f;
    }
}

__global__ void k_max_row_norm(const float *__restrict__ C, long long K, int dim, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    float best = 0.0f;
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < K; c += nw) {
        float p = 0.0f;
        for (int j = lane; j < dim; j += 32) {
            const float v = C[(size_t)c * dim + j];
            p = fmaf(v, v, p);
        }
        for (int m = 16; m >= 1; m >>= 1) p += __shfl_xor_sync(PB_FULL, p, m);
        best = fmaxf(best, p == p ? p : 3.4e38f);
    }
    if (lane == 0) atomicMax(reinterpret_cast<int *>(out), __float_as_int(best));  // best >= 0
}

// First-pass kernel.  The gather stage is bound by load-instruction / L2 request rate, not bytes, so one
// load instruction fetches FOUR table rows: lane = 8*r + s reads the 8 bytes (4 query tokens) s of the
// row of code r of each group of four codes; maxima stay packed (u16x2 SIMD max).
PB_DEV uint32_t pick4(const uint4 &c, int r) { return r == 0 ? c.x : (r == 1 ? c.y : (r == 2 ? c.z : c.w)); }

PB_DEV uint4 gather16(const char *p) { return *reinterpret_cast<const uint4 *>(p); }
// LPR = lanes per row: 4 (rows up to 64 bytes: nq <= 32, eight rows per load instruction) or 8 (up to 128 bytes:
// nq <= 64 in ONE pass over the codes, four rows per instruction).  Longer queries loop over 8*LPR-token column blocks.
template <int LPR>
__global__ void __launch_bounds__(256, LPR == 4 ? 4 : 2)
k_approx16(const unsigned short *__restrict__ ST16, const int *__restrict__ q_off, long long K, int QS,
           const uint32_t *__restrict__ ucodes, const long long *__restrict__ udoc_off,
           const uint32_t *__restrict__ cand, long long cand_cap, const int *__restrict__ n_cand,
           const int *__restrict__ n_skip, uint32_t *__restrict__ lsum, unsigned long long *__restrict__ tok_counter) {
    constexpr int RG = 32 / LPR;   // row groups of a warp = rows per load instruction
    constexpr int QB = 8 * LPR;    // query tokens covered by one pass
    constexpr int NI = 64 / RG;    // load instructions per 64 codes
    const int b = blockIdx.y;
    const int nq = q_off[b + 1] - q_off[b];
    const int n = n_cand[b];
    const int lane = threadIdx.x & 31, r = lane / LPR, sl = lane % LPR;
    const int warps_per_grid = gridDim.x * (blockDim.x >> 5);
    const char *STb = reinterpret_cast<const char *>(ST16 + (size_t)b * K * QS);
    const unsigned rowb = (unsigned)QS * 2u;
    unsigned long long my_tokens = 0;
    // entries [n_skip[b], n_cand[b]) of the list (n_skip: a5's pruned second round appends to its first)
    int i = (n_skip ? n_skip[b] : 0) + blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    uint32_t d = 0;
    long long t0 = 0, t1 = 0;
    if (i < n) {
        d = cand[(size_t)b * cand_cap + i];
        t0 = udoc_off[d];
        t1 = udoc_off[d + 1];
    }
    for (; i < n; i += warps_per_grid) {
        const int i2 = i + warps_per_grid;
        uint32_t dn = 0;
        long long t0n = 0, t1n = 0;
        if (i2 < n) {
            dn = cand[(size_t)b * cand_cap + i2];
            t0n = udoc_off[dn];
            t1n = udoc_off[dn + 1];
        }
        my_tokens += (unsigned long long)(t1 - t0);
        uint32_t total = 0;
        for (int qc = 0; qc < nq; qc += QB) {
            const bool in_row = qc + 8 * sl < QS;  // QS is a multiple of 8: groups past the row are skipped
            const char *col = STb + (in_row ? (qc + 8 * sl) * 2 : 0);
            uint32_t m0 = 0, m1 = 0, m2 = 0, m3 = 0;  // packed maxima of query tokens qc + 8 sl .. + 7
            // 64 codes per step: two coalesced loads (lane = code), handed to the row groups by shuffle.  (Lists are
            // padded to 8 with the last code; indices past the end repeat it, a max does not care.)
            for (long long t = t0; t < t1; t += 64) {
                const uint32_t cl0 = ucodes[min(t + lane, t1 - 1)], cl1 = ucodes[min(t + 32 + lane, t1 - 1)];
                if (t + 64 <= t1) {
                    uint4 v[NI];
#pragma unroll
                    for (int e = 0; e < NI; ++e)
                        v[e] = gather16(col + (size_t)__shfl_sync(PB_FULL, e < NI / 2 ? cl0 : cl1, RG * (e % (NI / 2)) + r) * rowb);
#pragma unroll
                    for (int e = 0; e < NI; ++e) {
                        m0 = __vmaxu2(m0, v[e].x);
                        m1 = __vmaxu2(m1, v[e].y);
                        m2 = __vmaxu2(m2, v[e].z);
                        m3 = __vmaxu2(m3, v[e].w);
                    }
                } else {
                    const int ne = (int)((t1 - t + RG - 1) / RG);
                    for (int e = 0; e < ne; ++e) {
                        const uint4 va = gather16(col + (size_t)__shfl_sync(PB_FULL, e < NI / 2 ? cl0 : cl1, RG * (e % (NI / 2)) + r) * rowb);
                        m0 = __vmaxu2(m0, va.x);
                        m1 = __vmaxu2(m1, va.y);
                        m2 = __vmaxu2(m2, va.z);
                        m3 = __vmaxu2(m3, va.w);
                    }
                }
            }
            // combine the row groups, then add up this lane's (real) query tokens
#pragma unroll
            for (int m = LPR; m < 32; m <<= 1) {
                m0 = __vmaxu2(m0, __shfl_xor_sync(PB_FULL, m0, m));
                m1 = __vmaxu2(m1, __shfl_xor_sync(PB_FULL, m1, m));
                m2 = __vmaxu2(m2, __shfl_xor_sync(PB_FULL, m2, m));
                m3 = __vmaxu2(m3, __shfl_xor_sync(PB_FULL, m3, m));
            }
            const int q0 = qc + 8 * sl;
            uint32_t part = 0;
            if (in_row && r == 0) {
                const uint32_t mm[4] = {m0, m1, m2, m3};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (q0 + 2 * j < nq) part += mm[j] & 0xffffu;
                    if (q0 + 2 * j + 1 < nq) part += mm[j] >> 16;
                }
            }
            total += __reduce_add_sync(PB_FULL, part);
        }
        if (lane == 0) lsum[(size_t)b * cand_cap + i] = total;
        d = dn;
        t0 = t0n;
        t1 = t1n;
    }
    if (lane == 0 && my_tokens && tok_counter) atomicAdd(tok_counter, my_tokens);
}

// ------------------------------------------------------------------------------------------
// a5 with pruning: bound every candidate's first-pass score from the score-table rows that can matter, and run
// k_approx16 only on the docs that can still reach the band around the cut.
//
// Per query token q a floor f_q (code units, k_a5_floor); a centroid c is LIVE when code[c][q] >= f_q for some
// q < nq (k_a5_live, one bit per centroid).  Every entry of a dead row is <= f_q - 1 in its column, so in exact
// integer arithmetic
//     L(d) = sum_q max_{c in codes(d)} code[c][q]  <=  U(d) = sum_q max(m_live(d, q), f_q - 1)
// (m_live = the maximum over d's live codes, 0 when none; f_q - 1 read as 0 when f_q = 0).  k_a5_bound computes U
// with live-row gathers only.  With W the band of the final select and M the cut:
//   round 1: theta1 = the M1-th largest U (M1 >= M), R1 = {U >= theta1} (ties at theta1 all join), L on R1 by
//            k_approx16, tau1 = the M-th largest L over R1;
//   round 2: R2 = {tau1 - W <= U < theta1}, L on R2 by k_approx16, appended after R1;
//   band:    the select of the dense form, unchanged, over R1 + R2.
// Exact: tau1 <= tau (the M-th largest L over all candidates) since R1 is a subset of them; every doc with
// L >= tau - W >= tau1 - W has U >= L >= tau1 - W, so it is in R1 or R2; there are at least M such docs, so the
// M-th largest L over R1 + R2 is tau and the band set {L >= tau - W} is the dense form's, doc for doc.  A query
// with fewer than M1 candidates, or a flagged one, keeps every candidate in round 1 (theta1 = 0: R2 is empty) and is
// the dense form.  Any floor is exact: f_q = 0 makes every row live and U = L; a floor above every code makes none
// live and U the same for every doc, so R1 takes them all.  The floor only decides the speed.
// ------------------------------------------------------------------------------------------
// floor[b][q]: about the n_live-th largest code of token q, from a histogram of the high byte over a sample of
// S = min(K, 8192) evenly spaced rows: the low edge of the highest bin with at least ceil(n_live * S / K) sampled
// codes at or above it.  n_live = 0: 65536 (nothing live); n_live >= K: 0 (everything live); padding tokens 65536.
// grid = (QS / 8, B), 256 threads; a CTA covers 8 query tokens, one 16-byte group of each sampled row.
__global__ void __launch_bounds__(256)
k_a5_floor(const unsigned short *__restrict__ ST16, const int *__restrict__ q_off, long long K, int QS, long long n_live,
           uint32_t *__restrict__ floor_out) {
    __shared__ int hist[8][256];
    const int g = blockIdx.x, b = blockIdx.y, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nq = q_off[b + 1] - q_off[b];
    const int S = (int)min(K, 8192ll);
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) (&hist[0][0])[i] = 0;
    __syncthreads();
    const uint4 *base = reinterpret_cast<const uint4 *>(ST16 + (size_t)b * K * QS) + g;
    const int GQ = QS >> 3;
    for (int j = threadIdx.x; j < S; j += blockDim.x) {
        const uint4 v = __ldg(base + (size_t)(j * K / S) * GQ);
        const uint32_t p[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            atomicAdd(&hist[2 * k][(p[k] >> 8) & 255u], 1);
            atomicAdd(&hist[2 * k + 1][p[k] >> 24], 1);
        }
    }
    __syncthreads();
    const int q = 8 * g + w;  // warp w picks token w's floor
    uint32_t f;
    if (q >= nq || n_live <= 0) f = 65536u;
    else if (n_live >= K) f = 0u;
    else {
        const int need = (int)min((long long)S, max(1ll, (n_live * S + K - 1) / K));
        // lane l owns bins 8 (31 - l) + 7 .. 8 (31 - l): the inclusive prefix over lanes counts the codes >= 8 (31 - l)
        int loc[8], sum = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            loc[k] = hist[w][8 * (31 - lane) + 7 - k];
            sum += loc[k];
        }
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(PB_FULL, incl, o);
            if (lane >= o) incl += y;
        }
        const unsigned reach = __ballot_sync(PB_FULL, incl >= need);  // lane 31 always reaches it (need <= S)
        const int hit = __ffs(reach) - 1;
        int bin = 0;
        if (lane == hit) {
            int cum = incl - sum, k = 0;
            for (; k < 7; ++k) {
                if (cum + loc[k] >= need) break;
                cum += loc[k];
            }
            bin = 8 * (31 - lane) + 7 - k;
        }
        f = (uint32_t)__shfl_sync(PB_FULL, bin, hit) << 8;
    }
    if (w < 8 && lane == 0 && q < QS) floor_out[(size_t)b * QS + q] = f;
}

// live[b * stride + c / 32] bit c % 32: row c has a code >= floor in some real query token.  Every word below
// (K + 31) / 32 is written; stride rounds that up to a multiple of 4 words, so that k_a5_bound can bulk-copy a query's
// bitmap (16-byte aligned rows).
// grid = (any, B), 256 threads; a warp takes 32 rows at a time (coalesced 16-byte loads, GQ = QS / 8 <= 8 per row).
__global__ void __launch_bounds__(256)
k_a5_live(const unsigned short *__restrict__ ST16, long long K, int QS, const uint32_t *__restrict__ floor_in,
          uint32_t *__restrict__ live, long long stride) {
    __shared__ uint32_t t2_s[32], m2_s[32];  // packed floors / real-token masks of token pairs (QS <= 64)
    __shared__ uint32_t word_s[8];
    const int b = blockIdx.y, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int GQ = QS >> 3;
    if (threadIdx.x < QS / 2) {
        const uint32_t a = floor_in[(size_t)b * QS + 2 * threadIdx.x], c = floor_in[(size_t)b * QS + 2 * threadIdx.x + 1];
        t2_s[threadIdx.x] = min(a, 65535u) | (min(c, 65535u) << 16);
        m2_s[threadIdx.x] = (a < 65536u ? 0xffffu : 0u) | (c < 65536u ? 0xffff0000u : 0u);
    }
    __syncthreads();
    const long long n_words = (K + 31) / 32;
    const uint4 *STb = reinterpret_cast<const uint4 *>(ST16 + (size_t)b * K * QS);
    for (long long wd = (long long)blockIdx.x * 8 + w; wd < n_words; wd += (long long)gridDim.x * 8) {
        const int rows = (int)min(32ll, K - wd * 32), total = rows * GQ;
        const uint4 *base = STb + (size_t)wd * 32 * GQ;
        if (lane == 0) word_s[w] = 0u;
        __syncwarp();
        uint4 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k < GQ && lane + 32 * k < total) v[k] = __ldg(base + lane + 32 * k);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int idx = lane + 32 * k;
            if (k >= GQ || idx >= total) continue;
            const int g = idx % GQ;
            const uint32_t h = (__vcmpgeu2(v[k].x, t2_s[4 * g]) & m2_s[4 * g]) |
                               (__vcmpgeu2(v[k].y, t2_s[4 * g + 1]) & m2_s[4 * g + 1]) |
                               (__vcmpgeu2(v[k].z, t2_s[4 * g + 2]) & m2_s[4 * g + 2]) |
                               (__vcmpgeu2(v[k].w, t2_s[4 * g + 3]) & m2_s[4 * g + 3]);
            if (h) atomicOr(&word_s[w], 1u << (idx / GQ));
        }
        __syncwarp();
        if (lane == 0) live[(size_t)b * stride + wd] = word_s[w];
        __syncwarp();
    }
}

// U(d) of every candidate (bound above).  Each warp streams its docs' distinct-code lists into its own ring of shared
// memory slots with TMA 1-D bulk copies, PB_A5_SPW slots ahead of the doc it bounds.  (The one-warp-per-doc form loaded
// the codes itself and waited on HBM latency for every doc: cand -> offsets -> codes -> live bits -> rows.)
//   CTA (x, b): the contiguous range [lo, hi) = [n x / X, n (x + 1) / X) of query b's candidate list (ascending doc ids,
//   so the code lists are read in ascending address order).  Warp w bounds docs lo + w, lo + w + 8, ...
//   Offsets: the warp loads 32 of its docs' candidate ids and udoc_off pairs at once (one doc per lane), the next 32
//   while it works through these.
//   Staging: lane 0 issues one cp.async.bulk per slot of PB_A5_SLOT codes (1 KiB), the warp's chunk sequence being its
//   docs' lists in order, each cut into slots (a list longer than a slot -- more than 256 distinct codes, or a doc
//   above PB_UCODE_MAX tokens with its raw list -- fills consecutive slots).  A slot holds its size word (codes, bit 31
//   = the doc's last slot) and a full mbarrier, armed with expect_tx and completed by the copy's bytes.  The warp
//   refills a slot as soon as it has read it, so no other warp's pace holds it up (a producer warp feeding all eight,
//   one lane per consumer, reconverged after every wait and so waited on the slowest of them: DESIGN.md 4b).
//   Bounding, per slot: the live test against the bitmap, the ballot compaction into the warp's buffer, then the
//   gather of those rows with k_approx16's row groups, 32 rows per round of independent loads.  QS <= 8 * LPR: one
//   column pass.  The packed maxima start at the dead-row floor f_q - 1 and are summed over the real tokens.
// Bulk-copy condition: source 16-byte aligned, size a multiple of 16.  Every list satisfies it because k_unique_codes
// pads lists to a multiple of 8 codes and udoc_off is the scan of those padded lengths from 0 -- at index open, on
// append (new lists start at the old total), after delete (whole lists compacted, offsets rescanned) and after a
// rebalance (offsets scanned from the arrived padded lengths) -- so a list starts 32-byte aligned and every slot of it
// is a multiple of 32 bytes.
// Counts the doc codes read (tok_counter) and the rows gathered (live_counter), as the dense pass does.
// bits_in_smem: the query's bitmap (live_stride words, a multiple of 4) is bulk-copied into shared memory at CTA start
// (K <= 2^19: up to 64 KiB); for larger K the bits are tested from global memory through L1.
// Dynamic shared memory: a5_bound_smem().
#define PB_A5_SLOT 256  // codes per ring slot (1 KiB): an average list (~212 distinct codes at 300 tokens) fits one
#define PB_A5_SPW 4     // ring slots per warp: 32 KiB of codes in flight per CTA
constexpr int PB_A5_RING = 8 * PB_A5_SPW;
// shared-memory layout: ring [PB_A5_RING][PB_A5_SLOT] u32, live buffers [8][PB_A5_SLOT] u32, slot sizes [PB_A5_RING] u32,
// full mbarriers [PB_A5_RING] + the bitmap's, then the bitmap from PB_A5_BITS_AT (16-byte aligned for its bulk copy)
constexpr size_t PB_A5_BITS_AT = 41 * 1024;
static_assert((size_t)(PB_A5_RING + 8) * PB_A5_SLOT * 4 + PB_A5_RING * 4 + (PB_A5_RING + 1) * 8 <= PB_A5_BITS_AT,
              "k_a5_bound: ring, buffers, sizes and mbarriers overrun the bitmap");
static_assert(PB_A5_BITS_AT % 16 == 0 && (PB_A5_RING * PB_A5_SLOT * 4 + 8 * PB_A5_SLOT * 4 + PB_A5_RING * 4) % 8 == 0,
              "k_a5_bound: misaligned shared-memory layout");
static inline size_t a5_bound_smem(long long live_stride, bool bits_in_smem) {
    return PB_A5_BITS_AT + (bits_in_smem ? (size_t)live_stride * 4 : 0);
}
template <int LPR>
__global__ void __launch_bounds__(256, LPR == 4 ? 3 : 2)  // (sm_90a: 80 / 112 registers, no spills)
k_a5_bound(const unsigned short *__restrict__ ST16, const int *__restrict__ q_off, long long K, int QS,
           const uint32_t *__restrict__ ucodes, const long long *__restrict__ udoc_off,
           const uint32_t *__restrict__ cand, long long cand_cap, const int *__restrict__ n_cand,
           const uint32_t *__restrict__ floor_in, const uint32_t *__restrict__ live, long long live_stride,
           bool bits_in_smem, uint32_t *__restrict__ ubound, unsigned long long *__restrict__ tok_counter,
           unsigned long long *__restrict__ live_counter) {
    constexpr int RG = 32 / LPR;  // rows per load instruction
    constexpr int NE = 32 / RG;   // load instructions per round of 32 rows
    extern __shared__ __align__(128) unsigned char smem_a5[];
    uint32_t *ring = reinterpret_cast<uint32_t *>(smem_a5);  // [PB_A5_RING][PB_A5_SLOT]
    uint32_t *bufs = ring + PB_A5_RING * PB_A5_SLOT;           // [8][PB_A5_SLOT]
    uint32_t *slot_n = bufs + 8 * PB_A5_SLOT;                  // [PB_A5_RING]
    uint64_t *full = reinterpret_cast<uint64_t *>(slot_n + PB_A5_RING), *bits_bar = full + PB_A5_RING;
    uint32_t *bits_s = reinterpret_cast<uint32_t *>(smem_a5 + PB_A5_BITS_AT);
    const int b = blockIdx.y, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long n = n_cand[b];
    const int lo = (int)(n * blockIdx.x / gridDim.x), hi = (int)(n * (blockIdx.x + 1) / gridDim.x);
    if (lo >= hi) return;  // (the whole CTA)
    const uint32_t *liveb = live + (size_t)b * live_stride;
    if (threadIdx.x == 0) {
        for (int s = 0; s < PB_A5_RING; ++s) mbar_init(&full[s], 1);
        mbar_init(bits_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (bits_in_smem && threadIdx.x == 0) {
        mbar_expect_tx(bits_bar, (uint32_t)live_stride * 4u);
        bulk_g2s(bits_s, liveb, (uint32_t)live_stride * 4u, bits_bar);
    }

    // ---- this warp's docs j = lo + w + 8 k, k < nd, and their staging ----
    const int nd = hi - lo > w ? (hi - lo - w + 7) / 8 : 0;
    const uint32_t *cl = cand + (size_t)b * cand_cap + lo + w;
    long long ta = 0, tb = 0, na = 0, nb = 0;  // lane l: offsets of doc k = 32 p + l (this batch) and of the next batch
    if (lane < nd) {
        const uint32_t d = cl[8 * lane];
        ta = udoc_off[d];
        tb = udoc_off[d + 1];
    }
    if (32 + lane < nd) {
        const uint32_t d = cl[8 * (32 + lane)];
        na = udoc_off[d];
        nb = udoc_off[d + 1];
    }
    // the fill position (warp-uniform): doc fk, codes [ft, fe) of it still to stage; slots issued / consumed so far
    int fk = 0;
    long long ft = (long long)shfl_u64((u64)ta, 0), fe = (long long)shfl_u64((u64)tb, 0);
    uint32_t issued = 0, seq = 0;
    auto stage = [&]() {
        while (fk < nd && issued - seq < PB_A5_SPW) {
            const int nc = (int)min((long long)PB_A5_SLOT, fe - ft);
            const int s = w * PB_A5_SPW + (int)(issued % PB_A5_SPW);
            if (lane == 0) {
                slot_n[s] = (uint32_t)nc | (ft + nc >= fe ? 0x80000000u : 0u);
                if (nc > 0) {
                    mbar_expect_tx(&full[s], (uint32_t)nc * 4u);
                    bulk_g2s(ring + s * PB_A5_SLOT, ucodes + ft, (uint32_t)nc * 4u, &full[s]);
                } else
                    mbar_arrive(&full[s]);  // (an empty list: no codes, the bound is the dead-row floor)
            }
            ++issued;
            ft += nc;
            if (ft >= fe && ++fk < nd) {
                if ((fk & 31) == 0) {  // the next batch of offsets becomes current; load the one after it
                    ta = na;
                    tb = nb;
                    na = nb = 0;
                    if (fk + 32 + lane < nd) {
                        const uint32_t d = cl[8 * (fk + 32 + lane)];
                        na = udoc_off[d];
                        nb = udoc_off[d + 1];
                    }
                }
                ft = (long long)shfl_u64((u64)ta, fk & 31);
                fe = (long long)shfl_u64((u64)tb, fk & 31);
            }
        }
    };
    stage();

    const int nq = q_off[b + 1] - q_off[b];
    const int r = lane / LPR, sl = lane % LPR;
    const bool in_row = 8 * sl < QS;
    const char *col = reinterpret_cast<const char *>(ST16 + (size_t)b * K * QS) + (in_row ? 16 * sl : 0);
    const unsigned rowb = (unsigned)QS * 2u;
    uint32_t *buf = bufs + w * PB_A5_SLOT;
    // this lane's dead-row maxima f_q - 1 (0 for f_q = 0), packed as the maxima are
    uint32_t dm[4] = {0u, 0u, 0u, 0u};
    if (in_row)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t f = floor_in[(size_t)b * QS + 8 * sl + j];
            dm[j >> 1] |= (f ? min(f - 1u, 65535u) : 0u) << (16 * (j & 1));
        }
    if (bits_in_smem) mbar_wait(bits_bar, 0u);
    unsigned long long my_tokens = 0, my_live = 0;
    for (int k = 0; k < nd; ++k) {
        uint32_t m0 = dm[0], m1 = dm[1], m2 = dm[2], m3 = dm[3];
        bool last;
        do {
            const int s = w * PB_A5_SPW + (int)(seq % PB_A5_SPW);
            mbar_wait(&full[s], (seq / PB_A5_SPW) & 1u);
            const uint32_t sz = slot_n[s];
            const int nc = (int)(sz & 0xffffu);
            last = (sz >> 31) != 0u;
            const uint32_t *codes = ring + s * PB_A5_SLOT;
            uint32_t cc[PB_A5_SLOT / 32];
#pragma unroll
            for (int j = 0; j < PB_A5_SLOT / 32; ++j) cc[j] = 32 * j + lane < nc ? codes[32 * j + lane] : 0u;
            int cnt = 0;
#pragma unroll
            for (int j = 0; j < PB_A5_SLOT / 32; ++j) {
                const uint32_t c = cc[j];
                const uint32_t word = bits_in_smem ? bits_s[c >> 5] : __ldg(liveb + (c >> 5));
                const bool lv = 32 * j + lane < nc && ((word >> (c & 31)) & 1u);
                const unsigned bal = __ballot_sync(PB_FULL, lv);
                if (lv) buf[cnt + __popc(bal & ((1u << lane) - 1u))] = c;
                cnt += __popc(bal);
            }
            __syncwarp();
            ++seq;
            // the slot is read: order those reads before the copy that refills it (async proxy), then refill
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            stage();
            for (int base = 0; base < cnt; base += 32) {
                uint4 v[NE];
#pragma unroll
                for (int e = 0; e < NE; ++e)
                    if (base + RG * e + r < cnt)
                        v[e] = *reinterpret_cast<const uint4 *>(col + (size_t)buf[base + RG * e + r] * rowb);
#pragma unroll
                for (int e = 0; e < NE; ++e)
                    if (base + RG * e + r < cnt) {
                        m0 = __vmaxu2(m0, v[e].x);
                        m1 = __vmaxu2(m1, v[e].y);
                        m2 = __vmaxu2(m2, v[e].z);
                        m3 = __vmaxu2(m3, v[e].w);
                    }
            }
            my_tokens += (unsigned long long)nc;
            my_live += (unsigned long long)cnt;
            __syncwarp();
        } while (!last);
#pragma unroll
        for (int m = LPR; m < 32; m <<= 1) {
            m0 = __vmaxu2(m0, __shfl_xor_sync(PB_FULL, m0, m));
            m1 = __vmaxu2(m1, __shfl_xor_sync(PB_FULL, m1, m));
            m2 = __vmaxu2(m2, __shfl_xor_sync(PB_FULL, m2, m));
            m3 = __vmaxu2(m3, __shfl_xor_sync(PB_FULL, m3, m));
        }
        const int q0 = 8 * sl;
        uint32_t part = 0;
        if (in_row && r == 0) {
            const uint32_t mm[4] = {m0, m1, m2, m3};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (q0 + 2 * j < nq) part += mm[j] & 0xffffu;
                if (q0 + 2 * j + 1 < nq) part += mm[j] >> 16;
            }
        }
        const uint32_t total = __reduce_add_sync(PB_FULL, part);
        if (lane == 0) ubound[(size_t)b * cand_cap + lo + w + 8 * k] = total;
    }
    if (lane == 0) {
        if (my_tokens) atomicAdd(tok_counter, my_tokens);
        if (my_live) atomicAdd(live_counter, my_live);
    }
}

// "N-th largest with a band" selection.  Per query:
//   tau = N-th largest of sel_keys[0..sel_n) (0 when sel_n < N or the query is flagged),
//   thr = tau - (band_per_q * nq + 8) (thr = tau when band_per_q <= 0), and the output is every
//   entry of filt_list whose filt_key >= thr (unordered).  grid = B, 1024 threads.
// The pruned a5 rounds use the optional arguments: thr_out[b] = thr; filt_hi[b] also caps the key (filt_key <
// filt_hi[b]); the output goes after out_base[b] entries and out_n[b] counts them too; tally adds up the out_n.
// qN: each query's own N (DESIGN.md 4l), or null.
__global__ void __launch_bounds__(1024)
k_select_u32(const uint32_t *__restrict__ sel_keys, const int *__restrict__ sel_n, int N, int band_per_q,
             const uint32_t *__restrict__ filt_keys, const uint32_t *__restrict__ filt_list,
             const int *__restrict__ filt_n, long long stride, const int *__restrict__ q_off,
             const int *__restrict__ qflag, uint32_t *__restrict__ out_list, int *__restrict__ out_n,
             uint32_t *__restrict__ thr_out = nullptr, const uint32_t *__restrict__ filt_hi = nullptr,
             const int *__restrict__ out_base = nullptr, unsigned long long *__restrict__ tally = nullptr,
             const int *__restrict__ qN = nullptr) {
    // one histogram per warp: the keys of a query share their high digits (sums of nq 16-bit codes), so a single
    // histogram serialises every thread of the CTA on one or two shared-memory words (0.15 ms); a warp whose 32 keys
    // fall in one bin adds 32 with one atomic
    __shared__ int hist[32][256];
    __shared__ uint32_t prefix_s, mask_s;
    __shared__ int remaining_s, fill_s;
    const int b = blockIdx.x;
    const int ns = sel_n[b], nf = filt_n[b];
    if (qN) N = qN[b];
    const int nq = q_off[b + 1] - q_off[b];
    const uint32_t *L = sel_keys + (size_t)b * stride;
    const uint32_t *F = filt_keys + (size_t)b * stride;
    const uint32_t *cin = filt_list + (size_t)b * stride;
    uint32_t *cout = out_list + (size_t)b * stride;
    const int wv = threadIdx.x >> 5, ln = threadIdx.x & 31;
    uint32_t thr = 0;  // keep everything
    if (ns >= N && N > 0 && !qflag[b]) {
        if (threadIdx.x == 0) {
            prefix_s = 0u;
            mask_s = 0u;
            remaining_s = N;
        }
        for (int pass = 3; pass >= 0; --pass) {  // N-th smallest of ~L == N-th largest of L
            const int shift = pass * 8;
            for (int i = threadIdx.x; i < 32 * 256; i += blockDim.x) (&hist[0][0])[i] = 0;
            __syncthreads();
            const uint32_t prefix = prefix_s, mask = mask_s;
            for (int i0 = 0; i0 < ns; i0 += blockDim.x * 8) {  // 8 independent loads per thread, then the histogram updates
                uint32_t kk[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int i = i0 + j * (int)blockDim.x + (int)threadIdx.x;
                    kk[j] = i < ns ? ~L[i] : 0u;
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int i = i0 + j * (int)blockDim.x + (int)threadIdx.x;
                    const uint32_t k = kk[j];
                    const bool in = i < ns && (k & mask) == prefix;
                    const uint32_t dg = (k >> shift) & 255u;
                    const unsigned act = __ballot_sync(PB_FULL, in);
                    if (!act) continue;
                    const uint32_t d0 = __shfl_sync(PB_FULL, dg, __ffs(act) - 1);
                    if (__all_sync(PB_FULL, !in || dg == d0)) {
                        if (ln == 0) hist[wv][d0] += __popc(act);  // (this warp's own histogram: no atomic needed)
                    } else if (in) atomicAdd(&hist[wv][dg], 1);
                    __syncwarp();
                }
            }
            __syncthreads();
            if (threadIdx.x < 256) {
                int tot = 0;
#pragma unroll 8
                for (int w2 = 0; w2 < 32; ++w2) tot += hist[w2][threadIdx.x];
                hist[0][threadIdx.x] = tot;  // (only this thread touches column threadIdx.x here)
            }
            __syncthreads();
            if (wv == 0) {  // the digit whose cumulative count reaches `remaining`: 8 bins per lane, warp prefix
                int loc[8], sum = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    loc[j] = hist[0][8 * ln + j];
                    sum += loc[j];
                }
                int incl = sum;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int y = __shfl_up_sync(PB_FULL, incl, o);
                    if (ln >= o) incl += y;
                }
                const int rem = remaining_s;
                const unsigned reach = __ballot_sync(PB_FULL, incl >= rem);
                const int hit = reach ? __ffs(reach) - 1 : 31;  // (ns >= N: some lane always reaches it)
                if (ln == hit) {
                    int cum = incl - sum, d = 0;
                    for (; d < 7; ++d) {
                        if (cum + loc[d] >= rem) break;
                        cum += loc[d];
                    }
                    remaining_s = rem - cum;
                    prefix_s = prefix | ((uint32_t)(8 * ln + d) << shift);
                    mask_s = mask | (255u << shift);
                }
            }
            __syncthreads();
        }
        const uint32_t tau = ~prefix_s;
        const uint32_t W = band_per_q > 0 ? (uint32_t)band_per_q * (uint32_t)nq + 8u : 0u;
        thr = tau > W ? tau - W : 0u;
    }
    const int base0 = out_base ? out_base[b] : 0;
    const uint32_t hi = filt_hi ? filt_hi[b] : 0xffffffffu;
    if (threadIdx.x == 0) {
        fill_s = 0;
        if (thr_out) thr_out[b] = thr;
    }
    cout += base0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int base = 0; base < nf; base += blockDim.x * 8) {
        uint32_t fv[8], cv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = base + j * (int)blockDim.x + (int)threadIdx.x;
            fv[j] = i < nf ? F[i] : 0u;
            cv[j] = i < nf ? cin[i] : 0u;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = base + j * (int)blockDim.x + (int)threadIdx.x;
            const bool keep = i < nf && fv[j] >= thr && (!filt_hi || fv[j] < hi);
            const unsigned bal = __ballot_sync(PB_FULL, keep);
            if (!bal) continue;
            int off = 0;
            if (lane == 0) off = atomicAdd(&fill_s, __popc(bal));
            off = __shfl_sync(PB_FULL, off, 0);
            if (keep) cout[off + __popc(bal & ((1u << lane) - 1u))] = cv[j];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        out_n[b] = base0 + fill_s;
        if (tally) atomicAdd(tally, (unsigned long long)(base0 + fill_s));
    }
}

