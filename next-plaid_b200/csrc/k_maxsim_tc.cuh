// k_maxsim_tc.cuh -- a7'/a8: the linear tensor-core MaxSim estimate as a warp-specialised pipeline, and the exact
// stage reduced to the (token, query token) pairs that can hold a per-token maximum.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ==========================================================================================
// k_maxsim_tc estimates every similarity of a kept doc's tokens as sim~ = (q.w + s~(code)) / |v| (residual part on the
// tensor cores from the query scaled by 2^qexp, centroid score from the 16-bit table, stored norm; bound
// eps_q = |q|max * filter_eps_unit2 on every similarity, DESIGN.md 4c), with the producer and consumer phases of a 128-token chunk on different warpgroups so that
// they overlap inside one CTA:
//   warps 4-7  producers: locate the chunk's tokens, read the packed residuals, expand them to fp16 straight
//              into a 2-stage operand ring (thread = token row);
//   warps 0-3  consumers: the KSTEPS wgmma of a chunk (two M = 64 slabs), staged to a shared fp32 tile; then the
//              epilogue (thread = token = tile row): add the centroid score of the token's code (one 16-bit
//              score-table row per token, fetched one chunk ahead), scale by 1/|v|, reduce per doc.
// Token metadata travels from the producers to the epilogue through a 4-deep ring: the producer of chunk i writes
// slot i % 4 after it finished the tile of chunk i-1, which it could only start once the MMA of chunk i-3 had
// completed, which the consumers issue after the epilogue of chunk i-4 -- and they had read the metadata of chunk
// i-4 before the epilogue of chunk i-5.
//
// EMIT = false (pass 1, every kept doc): per (doc, query token) maxima of the estimate -> maxkey.
// EMIT = true  (pass 2, the filter's survivors): a doc's exact MaxSim needs, per query token, only the tokens whose
//   estimate is within 2 eps_q of that (doc, query token) maximum estimate -- sim(t) >= sim~(t) - eps_q and the
//   exact maximum is >= max sim~ - eps_q, so a token further below cannot hold the maximum.  Those (token, q)
//   pairs (a little over one per (doc, q)) are listed; k_pair_exact decompresses each token and evaluates the dot
//   in the pinned order (codec.rs:443-467, maxsim.rs:281): the same per-token maxima as k_exact, from ~1/250 of
//   the arithmetic.  A query whose list overflows is left to k_exact (per-query flag).
// Residual operand tile: canonical K-major fp16, element (token row r, 8-wide K chunk kc) at
// kc * LBO + (r/8) * 128 + (r%8) * 16 = kc * LBO + 16 r, with LBO = 2048 + 32 bytes between K chunks.
// A stage is the DIM / 8 chunks rounded up to 128 bytes (PB_XTC_STAGE), so that the second stage and the query tile
// behind the ring start on 128-byte boundaries like every other operand base here (the no-swizzle descriptors need
// 16).  The rounding is the identity when DIM % 32 == 0 and adds 64 bytes at DIM = 48 (6 chunks = 12480 bytes).
// ==========================================================================================
#define PB_XTC_LBO 2080u
#define PB_XTC_STAGE(dim) ((((unsigned)(dim) / 8u) * PB_XTC_LBO + 127u) & ~127u)

struct MsMeta {
    long long g;
    int r;
    uint32_t code;
};

PB_DEV void ms_arrive(uint64_t *bar) { mbar_arrive(bar); }

// warp maximum of a float with NaN ignored (all NaN -> NaN), +0 above -0: one redux.sync on the order-preserving int
// image of the float (x ^ ((x >> 31) & 0x7fffffff), its own inverse)
PB_DEV float warp_max_f32(float x) {
    const int i = __float_as_int(x);
    const int m = __reduce_max_sync(PB_FULL, x == x ? i ^ ((i >> 31) & 0x7fffffff) : (int)0x80000000);
    return __int_as_float(m ^ ((m >> 31) & 0x7fffffff));
}

// the consumer warpgroup's own barrier (the producers do not take part)
PB_DEV void consumer_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// gbase[b][r] = first token of kept doc r minus its offset in the query's kept-token stream: token s of the stream is
// index token gbase[r] + s (one dependent load after the prefix search instead of kept -> doc_off)
__global__ void k_doc_gbase(const uint32_t *__restrict__ kept, const int *__restrict__ n_kept, const long long *__restrict__ tok_prefix,
                            const long long *__restrict__ doc_off, int Mcap, long long *__restrict__ gbase) {
    const int b = blockIdx.y, r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n_kept[b]) gbase[(size_t)b * Mcap + r] = doc_off[kept[(size_t)b * Mcap + r]] - tok_prefix[(size_t)b * (Mcap + 1) + r];
}

// locate_token through gbase: (rank, index token, code) of stream position s; the code is loaded here but first used
// one chunk later (when the producer publishes the chunk's metadata), so its latency is off the critical path
PB_DEV TokMeta ms_locate(long long s, long long T, int r_lo, int nk, const long long *__restrict__ tp,
                         const long long *__restrict__ gb, const uint32_t *__restrict__ codes) {
    TokMeta m;
    m.r = -1;
    m.g = 0;
    m.code = 0;
    if (s < T) {
        int lo = r_lo, hi = nk, step = 1;
        while (lo + step < nk) {
            if (tp[lo + step] <= s) {
                lo += step;
                step <<= 1;
            } else {
                hi = lo + step;
                break;
            }
        }
        while (hi - lo > 1) {
            int mid = (lo + hi) >> 1;
            if (tp[mid] <= s) lo = mid; else hi = mid;
        }
        m.r = lo;
        m.g = gb[lo] + s;
        m.code = __ldg(codes + m.g);
    }
    return m;
}

template <int DIM, int NBITS, int NQT, bool EMIT>
__global__ void __launch_bounds__(256, NQT == 32 ? 2 : 1)  // NQT = 64: ~129 KB of shared memory, one CTA per SM
k_maxsim_tc(const float *__restrict__ Q, const int *__restrict__ q_off, int QS, const int *__restrict__ qexp,
            const unsigned short *__restrict__ ST16,
            long long K, const float2 *__restrict__ qrange, const int *__restrict__ qflag, const float *__restrict__ w_rev,
            const uint32_t *__restrict__ codes, const uint8_t *__restrict__ residuals, const float *__restrict__ inv_norm,
            const long long *__restrict__ gbase, const int *__restrict__ n_kept,
            const long long *__restrict__ tok_prefix, int Mcap, uint32_t *__restrict__ maxkey,
            const uint32_t *__restrict__ src_rank, const float *__restrict__ qnmax, float band_unit,
            u64 *__restrict__ pairs, int *__restrict__ n_pairs, int pair_cap) {
    extern __shared__ __align__(128) unsigned char smem_x[];
    constexpr int KC = DIM / 8, KSTEPS = DIM / 16;
    static_assert(NQT == 32 || NQT == 64, "k_maxsim_tc: N = 32 or 64");
    static_assert(DIM % 16 == 0, "k_maxsim_tc: whole wgmma K steps");
    constexpr uint32_t LBO_A = PB_XTC_LBO, A_BYTES = PB_XTC_STAGE(DIM), QB_BYTES = NQT * DIM * 2;
    constexpr uint32_t LBO_B = (NQT / 8) * 128, SBO = 128;
    constexpr int PACKED = DIM * NBITS / 8, NW = PACKED / 4;
    static_assert(PACKED % 4 == 0, "k_maxsim_tc: packed rows are read in 32-bit words");
    constexpr int VB = 8 / NBITS;
    // the 4-bit table (256 entries x 4 B) is kept in TR copies, lane l reads copy l % TR: 32 random lookups of one copy hit
    // the worst bank ~3.5 times, 8 lookups spread over a copy's 8 banks ~2.3 times (the kernel sits on the LSU pipe)
    constexpr int TR = NBITS == 4 ? 4 : 1;
    constexpr int SW = NQT / 2;  // 32-bit words of a score-table row
    unsigned char *As = smem_x;                                   // [2][A_BYTES] fp16 residual tiles
    unsigned char *Qb = As + 2 * A_BYTES;                         // [NQT query rows] fp16 operand tile
    __half *Th = reinterpret_cast<__half *>(Qb + QB_BYTES);       // [256][TR][VB]: fp16 bucket weights of the fields of a byte
    MsMeta *meta = reinterpret_cast<MsMeta *>(Th + 256 * VB * TR); // [4][128]
    uint64_t *bars = reinterpret_cast<uint64_t *>(meta + 4 * 128);
    uint64_t *a_full = bars, *a_empty = bars + 2, *m_full = bars + 4;  // 2,2,4
    float *Acc = reinterpret_cast<float *>(bars + 8);                  // [128 tokens][ACC_LD(NQT)] similarities of the chunk
    const int b = blockIdx.y;
    const int nk = n_kept[b];
    const long long *tp = tok_prefix + (size_t)b * (Mcap + 1);
    const long long *gb = gbase + (size_t)b * Mcap;
    const long long T = tp[nk];
    const int r0q = q_off[b], nq = q_off[b + 1] - r0q;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long n_chunks = (T + 127) / 128;
    const long long per = (n_chunks + gridDim.x - 1) / gridDim.x;
    const long long c_lo = (long long)blockIdx.x * per, c_hi = min(n_chunks, c_lo + per);
    if (c_lo >= c_hi || nq == 0 || qflag[b]) return;
    const int n = (int)(c_hi - c_lo);
    // the query enters the tensor cores scaled by 2^qexp[b] (largest row norm in [1, 2): no fp16 overflow, no
    // subnormal coordinates of the rows that matter) and the products leave scaled by 2^-qexp[b]; both exact
    const float q_up = ldexpf(1.0f, qexp[b]), q_down = ldexpf(1.0f, -qexp[b]);
    for (int i = threadIdx.x; i < 256 * VB * TR; i += blockDim.x) {
        const int byte = i / (VB * TR), j = i % VB;
        Th[i] = __float2half_rn(w_rev[(byte >> (8 - NBITS * (j + 1))) & ((1 << NBITS) - 1)]);
    }
    for (int idx = threadIdx.x; idx < NQT * KC; idx += blockDim.x) {
        const int r = idx / KC, kc = idx - r * KC;
        __half v8[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v8[e] = __float2half_rn(r < nq ? Q[(size_t)(r0q + r) * DIM + kc * 8 + e] * q_up : 0.0f);
        *reinterpret_cast<uint4 *>(Qb + (kc * (NQT / 8) + (r >> 3)) * 128 + (r & 7) * 16) = *reinterpret_cast<uint4 *>(v8);
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) {
            mbar_init(&a_full[s], 128);
            mbar_init(&a_empty[s], 4);  // one arrival per consumer warp
        }
        for (int s = 0; s < 4; ++s) mbar_init(&m_full[s], 128);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // Qb is read by the async proxy
    __syncthreads();

    if (w >= 4) {
        // ================= producers =================
        const int t = threadIdx.x - 128;
        auto load_packed = [&](const TokMeta &m, uint32_t (&pw)[NW]) __attribute__((always_inline)) {
            if (m.r >= 0) {
                const uint8_t *src = residuals + (size_t)m.g * PACKED;
                if (PACKED % 16 == 0) {
#pragma unroll
                    for (int pc = 0; pc < PACKED / 16; ++pc) {
                        const uint4 t4 = __ldg(reinterpret_cast<const uint4 *>(src) + pc);
                        pw[4 * pc] = t4.x;
                        pw[4 * pc + 1] = t4.y;
                        pw[4 * pc + 2] = t4.z;
                        pw[4 * pc + 3] = t4.w;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < NW; ++i) pw[i] = __ldg(reinterpret_cast<const uint32_t *>(src) + i);
                }
            } else {
#pragma unroll
                for (int i = 0; i < NW; ++i) pw[i] = 0u;
            }
        };
        auto step = [&](int i, const TokMeta &cur, const uint32_t (&pw)[NW], TokMeta &nxt, uint32_t (&pwn)[NW])
                        __attribute__((always_inline)) {
            const int s = i & 1, ms = i & 3;
            MsMeta mm;
            mm.g = cur.g;
            mm.r = cur.r;
            mm.code = cur.code;
            meta[ms * 128 + t] = mm;
            ms_arrive(&m_full[ms]);
            nxt.r = -1;
            nxt.g = 0;
            nxt.code = 0;
            if (i + 1 < n) {
                const int r_lo = max(__shfl_sync(PB_FULL, cur.r, 0), 0);
                nxt = ms_locate((c_lo + i + 1) * 128 + t, T, r_lo, nk, tp, gb, codes);
            }
            load_packed(nxt, pwn);
            mbar_wait(&a_empty[s], ((uint32_t)(i >> 1) & 1u) ^ 1u);
            unsigned char *A = As + (size_t)s * A_BYTES;
#pragma unroll
            for (int kc = 0; kc < KC; ++kc) {
                uint32_t wv[4];
                if (NBITS == 4) {
                    const uint32_t x = pw[kc];
                    const uint32_t *T32 = reinterpret_cast<const uint32_t *>(Th) + (t & (TR - 1));
#pragma unroll
                    for (int j = 0; j < 4; ++j) wv[j] = T32[((x >> (8 * j)) & 255u) * TR];
                } else if (NBITS == 2) {
                    const uint32_t x = pw[kc >> 1] >> (16 * (kc & 1));
                    const uint2 *T64 = reinterpret_cast<const uint2 *>(Th);
                    const uint2 a = T64[x & 255u], c = T64[(x >> 8) & 255u];
                    wv[0] = a.x;
                    wv[1] = a.y;
                    wv[2] = c.x;
                    wv[3] = c.y;
                } else if (NBITS == 1) {
                    const uint4 a = reinterpret_cast<const uint4 *>(Th)[(pw[kc >> 2] >> (8 * (kc & 3))) & 255u];
                    wv[0] = a.x;
                    wv[1] = a.y;
                    wv[2] = a.z;
                    wv[3] = a.w;
                } else {
                    const unsigned short *T16 = reinterpret_cast<const unsigned short *>(Th);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t x = pw[2 * kc + (j >> 1)] >> (16 * (j & 1));
                        wv[j] = (uint32_t)T16[x & 255u] | ((uint32_t)T16[(x >> 8) & 255u] << 16);
                    }
                }
                if (cur.r < 0) wv[0] = wv[1] = wv[2] = wv[3] = 0u;
                *reinterpret_cast<uint4 *>(A + kc * LBO_A + t * 16) = make_uint4(wv[0], wv[1], wv[2], wv[3]);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            ms_arrive(&a_full[s]);
        };
        TokMeta mA = ms_locate(c_lo * 128 + t, T, 0, nk, tp, gb, codes), mB;
        uint32_t pA[NW], pB[NW];
        load_packed(mA, pA);
        for (int i = 0; i < n; i += 2) {
            step(i, mA, pA, mB, pB);
            if (i + 1 < n) step(i + 1, mB, pB, mA, pA);
        }
    } else {
        // ================= consumers: MMA + epilogue =================
        const int t = threadIdx.x;
        const float2 rg = qrange[b];
        const float inv_scale0 = 1.0f / rg.y, s_bias = (0.5f - rg.x) / rg.y;
        // code -> score without an int-to-float conversion: PRMT puts the 16-bit code under the exponent of 2^23
        // (float 2^23 + code, exact) and one FFMA applies scale and bias; 2^23 * inv_scale is exact, the folded
        // constant is rounded once (<= half an ulp of ~2^8: 1.6e-5, a per-query constant that filter_eps_unit2 carries).
        // The centroid score joins the scaled accumulator scaled by 2^qexp too, and 1/|v| carries the 2^-qexp back:
        // every step is the unscaled one times a power of two
        const float inv_scale = inv_scale0 * q_up, s_bias23 = (s_bias - 8388608.0f * inv_scale0) * q_up;
        const char *STb = reinterpret_cast<const char *>(ST16 + (size_t)b * K * QS);
        const unsigned rowb = (unsigned)QS * 2u;
        const float band = EMIT ? 2.0f * band_unit * qnmax[b] + 1e-6f : 0.0f;
        // pass 2: the threshold keys of the token's doc for query tokens lane, lane + 32 (what a warp whose 32 tokens share
        // their doc needs), fetched with the side loads so that src_rank -> maxkey is off the epilogue's critical path
        auto load_thr = [&](const MsMeta &m, uint32_t (&tk)[NQT / 32]) __attribute__((always_inline)) {
#pragma unroll
            for (int h = 0; h < NQT / 32; ++h) tk[h] = 0u;
            if (EMIT && m.r >= 0) {
                const uint32_t *trow = maxkey + ((size_t)b * Mcap + src_rank[(size_t)b * Mcap + m.r]) * QS;
#pragma unroll
                for (int h = 0; h < NQT / 32; ++h)
                    if (32 * h + lane < nq) tk[h] = trow[32 * h + lane];
            }
        };
        auto load_side = [&](const MsMeta &m, uint32_t (&sw)[SW], float &inv) __attribute__((always_inline)) {
            inv = 1.0f;  // (a token slot past the stream: its bias is -inf, the product must stay -inf)
            if (m.r >= 0) {
                const uint4 *srow = reinterpret_cast<const uint4 *>(STb + (size_t)m.code * rowb);  // 16-byte aligned (QS % 8 == 0)
#pragma unroll
                for (int i = 0; i < SW / 4; ++i) {
                    uint4 t4 = make_uint4(0, 0, 0, 0);
                    if (8 * i < QS) t4 = srow[i];
                    sw[4 * i] = t4.x;
                    sw[4 * i + 1] = t4.y;
                    sw[4 * i + 2] = t4.z;
                    sw[4 * i + 3] = t4.w;
                }
                inv = inv_norm[m.g] * q_down;
            } else {
#pragma unroll
                for (int i = 0; i < SW; ++i) sw[i] = 0u;
            }
        };
        auto step = [&](int i, const MsMeta &cur, const uint32_t (&sw)[SW], float inv, const uint32_t (&tk)[NQT / 32], MsMeta &nxt,
                        uint32_t (&swn)[SW], float &invn, uint32_t (&tkn)[NQT / 32]) __attribute__((always_inline)) {
            nxt.r = -1;
            nxt.g = 0;
            nxt.code = 0;
            if (i + 1 < n) {
                const int ms = (i + 1) & 3;
                mbar_wait(&m_full[ms], (uint32_t)((i + 1) >> 2) & 1u);
                nxt = meta[ms * 128 + t];
            }
            load_side(nxt, swn, invn);
            load_thr(nxt, tkn);
            const int s = i & 1;
            mbar_wait(&a_full[s], (uint32_t)(i >> 1) & 1u);
            consumer_sync();  // every thread has read the previous chunk's similarities
            {
                const uint32_t a0 = smem_u32(As + (size_t)s * A_BYTES), b0 = smem_u32(Qb);
#pragma unroll
                for (int p = 0; p < 2; ++p) {  // M = 64 slabs: tokens 64 p.. (64 rows = 1024 bytes of the tile)
                    float d[NQT / 2] = {};
                    wg_fence();
#pragma unroll
                    for (int k = 0; k < KSTEPS; ++k)
                        wg_mma_f16<NQT>(d, wg_desc(a0 + p * 1024 + k * 2 * LBO_A, LBO_A, SBO), wg_desc(b0 + k * 2 * LBO_B, LBO_B, SBO),
                                        k > 0 ? 1u : 0u);
                    wg_commit();
                    wg_wait_all(d);
                    wg_stage<NQT>(Acc + p * 64 * ACC_LD(NQT), d);
                }
                __syncwarp();
                if (lane == 0) ms_arrive(&a_empty[s]);  // operand stage free
            }
            consumer_sync();  // the chunk's similarities are staged
            const float *arow = Acc + t * ACC_LD(NQT);
            const int rank = cur.r;
            const unsigned grp = __match_any_sync(PB_FULL, rank);
#pragma unroll
            for (int h = 0; h < NQT / 32; ++h) {
                if (32 * h >= nq) continue;  // (uniform) nothing to read in this half
                if (!EMIT) {
                    // per-doc maxima, 16 query tokens at a time (16 accumulator registers live): one pass per doc
                    // present in the warp's 32 tokens (one, unless a doc boundary falls inside them).  Tokens outside
                    // the doc take bias -inf, so they never win the warp maximum; lane q keeps the maximum of query
                    // token q and publishes it (one atomic instruction per doc and half).
                    const unsigned valid = __ballot_sync(PB_FULL, rank >= 0);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        uint32_t r16[16];
                        acc_row(arow + 32 * h + 16 * hh, r16);
                        unsigned done = 0u;
                        while (valid & ~done) {
                            const int leader = __ffs(valid & ~done) - 1;
                            const int segrank = __shfl_sync(PB_FULL, rank, leader);
                            const bool inseg = rank == segrank;
                            const float bias_l = inseg ? s_bias23 : -INFINITY;
                            float mine = 0.0f;
#pragma unroll
                            for (int q = 0; q < 16; ++q) {
                                const uint32_t f = __byte_perm(sw[16 * h + 8 * hh + (q >> 1)], 0x4B000000u, (q & 1) ? 0x7632 : 0x7610);
                                const float sim = (__uint_as_float(r16[q]) + __fmaf_rn(__uint_as_float(f), inv_scale, bias_l)) * inv;
                                const float m = warp_max_f32(sim);
                                if (lane == 16 * hh + q) mine = m;
                            }
                            const uint32_t key = score_key_asc(mine);
                            const int qq = 32 * h + lane;
                            if ((lane >> 4) == hh && qq < nq && key) atomicMax(&maxkey[((size_t)b * Mcap + segrank) * QS + qq], key);
                            done |= __ballot_sync(PB_FULL, inseg);
                        }
                    }
                    continue;
                }
                uint32_t rr[32];
                acc_row(arow + 32 * h, rr);
                if (EMIT) {
                    // thresholds of the warp's doc: lane = query token (a warp that straddles docs reads per token)
                    const bool uni = grp == PB_FULL;
                    float thr_l = -INFINITY;
                    if (uni && rank >= 0 && 32 * h + lane < nq && tk[h]) thr_l = key_to_score(tk[h]) - band;
                    const uint32_t *trow = nullptr;
                    if (!uni && rank >= 0) trow = maxkey + ((size_t)b * Mcap + src_rank[(size_t)b * Mcap + rank]) * QS + 32 * h;
#pragma unroll
                    for (int q = 0; q < 32; ++q) {
                        const uint32_t f = __byte_perm(sw[16 * h + (q >> 1)], 0x4B000000u, (q & 1) ? 0x7632 : 0x7610);
                        const float sim = (__uint_as_float(rr[q]) + __fmaf_rn(__uint_as_float(f), inv_scale, s_bias23)) * inv;
                        float thr = __shfl_sync(PB_FULL, thr_l, q);
                        if (!uni && rank >= 0 && 32 * h + q < nq) {
                            const uint32_t k = trow[q];
                            thr = k ? key_to_score(k) - band : -INFINITY;
                        }
                        if (rank >= 0 && 32 * h + q < nq && !(sim < thr)) {
                            const int at = atomicAdd(&n_pairs[b], 1);
                            if (at < pair_cap)
                                pairs[(size_t)b * pair_cap + at] = ((u64)cur.g << 24) | ((u64)(32 * h + q) << 16) | (u64)rank;
                        }
                    }
                }
            }
        };
        MsMeta mA, mB;
        uint32_t sA[SW], sB[SW], kA[NQT / 32], kB[NQT / 32];
        float iA, iB;
        mbar_wait(&m_full[0], 0u);
        mA = meta[t];
        load_side(mA, sA, iA);
        load_thr(mA, kA);
        for (int i = 0; i < n; i += 2) {
            step(i, mA, sA, iA, kA, mB, sB, iB, kB);
            if (i + 1 < n) step(i + 1, mB, sB, iB, kB, mA, sA, iA, kA);
        }
    }
}

// ------------------------------------------------------------------------------------------
// exact similarity of the listed (token, query token) pairs.  grid = (a few CTAs, B), 256 threads, dynamic smem =
// ((nq + 256) * (DIM + 1) + 256) floats (staging the query is the fixed cost of a CTA: few CTAs, each loops).  A warp takes 32 pairs at a time: the 32 tokens are decompressed by the whole
// warp exactly as decompress_token does (lane = float4 group, pinned sum-of-squares butterfly, IEEE division) into
// a padded shared-memory tile, then every lane runs its own pair's sequential FMA chain.
// pair = token index << 24 | query token << 16 | rank among the kept docs.
// ------------------------------------------------------------------------------------------
template <int DIM>
__global__ void __launch_bounds__(256)
k_pair_exact(const u64 *__restrict__ pairs, const int *__restrict__ n_pairs, int pair_cap, const float *__restrict__ Q,
             const int *__restrict__ q_off, int QS, const float *__restrict__ C, const float *__restrict__ w_rev, int nbits,
             const uint32_t *__restrict__ codes, const uint8_t *__restrict__ residuals, int Mcap,
             uint32_t *__restrict__ maxkey) {
    static_assert(DIM <= 128, "k_pair_exact: one float4 group per lane");
    extern __shared__ __align__(16) float smem_pe[];
    constexpr int LD = DIM + 1, G = DIM / 4;
    const int b = blockIdx.y;
    const int n = n_pairs[b];
    if (n > pair_cap || (long long)blockIdx.x * 256 >= n) return;  // overflow: k_exact scores this query
    const int nq = q_off[b + 1] - q_off[b];
    const int packed = DIM * nbits / 8;
    float *Qs = smem_pe;                                             // [nq][LD]
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *rows = smem_pe + (size_t)nq * LD + (size_t)w * 32 * LD;   // [32][LD] of this warp
    float *wr = smem_pe + (size_t)(nq + 256) * LD;                   // [256]
    for (int i = threadIdx.x; i < (1 << nbits); i += blockDim.x) wr[i] = w_rev[i];
    const float *Qb = Q + (size_t)q_off[b] * DIM;
    for (int idx = threadIdx.x; idx < nq * DIM; idx += blockDim.x) Qs[(idx / DIM) * LD + idx % DIM] = Qb[idx];
    __syncthreads();
    const u64 *plist = pairs + (size_t)b * pair_cap;
    for (int j0 = (blockIdx.x * 8 + w) * 32; j0 < n; j0 += gridDim.x * 256) {
        const int j = j0 + lane;
        const u64 pr = j < n ? plist[j] : 0ull;
        const long long g = (long long)(pr >> 24);
        const uint32_t code = j < n ? codes[g] : 0u;
        __syncwarp();
        for (int r0 = 0; r0 < 32; r0 += 8) {  // 8 tokens in flight
            float4 c[8];
            uint32_t f[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const long long ge = (long long)shfl_u64((u64)g, r0 + e);
                const uint32_t ce = __shfl_sync(PB_FULL, code, r0 + e);
                c[e] = make_float4(0.f, 0.f, 0.f, 0.f);
                f[e] = 0u;
                if (lane < G) {
                    c[e] = __ldg(reinterpret_cast<const float4 *>(C + (size_t)ce * DIM) + lane);
                    f[e] = load_fields4(residuals + (size_t)ge * packed, lane, nbits);
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                float p = 0.0f;
                if (lane < G) {
                    v.x = __fadd_rn(c[e].x, wr[f[e] & 255u]);
                    v.y = __fadd_rn(c[e].y, wr[(f[e] >> 8) & 255u]);
                    v.z = __fadd_rn(c[e].z, wr[(f[e] >> 16) & 255u]);
                    v.w = __fadd_rn(c[e].w, wr[f[e] >> 24]);
                    p = __fmaf_rn(v.x, v.x, p);
                    p = __fmaf_rn(v.y, v.y, p);
                    p = __fmaf_rn(v.z, v.z, p);
                    p = __fmaf_rn(v.w, v.w, p);
                }
#pragma unroll
                for (int m = 16; m >= 1; m >>= 1) p = __fadd_rn(p, __shfl_xor_sync(PB_FULL, p, m));
                float norm = __fsqrt_rn(p);
                if (!(norm >= 1e-12f)) norm = 1e-12f;  // f32::max(1e-12)
                if (lane < G) {
                    float *dst = rows + (size_t)(r0 + e) * LD + 4 * lane;
                    // the hoisted form of the IEEE division (k_exact.cuh: div_setup / div_fast) where it is exact
                    const uint32_t a0 = __float_as_uint(v.x) & 0x7fffffffu, a1 = __float_as_uint(v.y) & 0x7fffffffu;
                    const uint32_t a2 = __float_as_uint(v.z) & 0x7fffffffu, a3 = __float_as_uint(v.w) & 0x7fffffffu;
                    const uint32_t nb = __float_as_uint(norm);
                    if (div_range_ok(min(min(min(a0, a1), min(a2, a3)), nb), max(max(max(a0, a1), max(a2, a3)), nb))) {
                        const float yr = div_setup(norm);
                        dst[0] = div_fast(v.x, norm, yr);
                        dst[1] = div_fast(v.y, norm, yr);
                        dst[2] = div_fast(v.z, norm, yr);
                        dst[3] = div_fast(v.w, norm, yr);
                    } else {
                        dst[0] = __fdiv_rn(v.x, norm);
                        dst[1] = __fdiv_rn(v.y, norm);
                        dst[2] = __fdiv_rn(v.z, norm);
                        dst[3] = __fdiv_rn(v.w, norm);
                    }
                }
            }
        }
        __syncwarp();
        if (j < n) {
            const uint32_t q = (uint32_t)(pr >> 16) & 255u, r = (uint32_t)pr & 0xffffu;
            const float *qr = Qs + (size_t)q * LD, *vr = rows + (size_t)lane * LD;
            float s = 0.0f;
#pragma unroll 8
            for (int d = 0; d < DIM; ++d) s = __fmaf_rn(qr[d], vr[d], s);
            const uint32_t key = score_key_asc(s);
            if (key) atomicMax(&maxkey[((size_t)b * Mcap + r) * QS + q], key);
        }
    }
}

// per-query switch of the classic exact kernel: 1 = the pair list of this query overflowed (or the query published no
// estimate), k_exact scores its survivors
__global__ void k_pair_overflow(const int *__restrict__ n_pairs, int pair_cap, const int *__restrict__ qflag, int B,
                                int *__restrict__ need_exact) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x)
        need_exact[b] = (n_pairs[b] > pair_cap || qflag[b]) ? 1 : 0;
}
