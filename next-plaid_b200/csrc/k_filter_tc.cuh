// k_filter_tc.cuh -- a7' tensor-core fp16 certified filter in front of the exact stage.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ==========================================================================================
// Tensor-core (wgmma) certified filter in front of the exact stage (search path).
//
// Only the top_k docs of the M kept ones need exact scores (search.rs:496-515).  k_exact_tc
// estimates every kept doc's MaxSim on the tensor cores: tokens are decompressed approximately from an
// fp16 copy of the centroids straight into the MMA operand tile (canonical K-major layout, fp16),
// the query is the N = 32 operand, sims are staged to shared memory, the epilogue takes per-doc column maxima.
// fp16 rather than bf16: every operand is a unit-scale vector, and 11 significand bits make the certified
// band 8x narrower.  With D the exact decompressed token, D~ its estimate, u = 2^-11 the unit roundoff and
// v = c + w the token before normalisation, v~ = h(h(c) + h(w)) what the tile holds (one fp16 add of fp16 operands),
//     |v - v~| <= u (|c| + |w| + |v|) (1 + 2u)  =>  rho = |v - v~| / |v| <= u ((max|c| + max|w|) / min|v| + 1) (1 + 2u)
//     |D - D~| <= rho / (1 - rho / 2)             (Dunkl-Williams; min|v| and max|w| are measured at index open)
//     |q.D - h(q).D~| <= u |q| + (1 + u) |q| |D - D~| + slack               (slack: fp16 subnormals, fp32 sums)
// with h(q) = 2^-qexp h(2^qexp q): the query enters scaled so that its largest row norm is in [1, 2) (qexp from
// k_query_range), which keeps the subnormal slack relative to |q|max and rules out fp16 overflow at any query scale
// so eps_q = |q|max * eps_unit (filter_eps_unit in engine.cu) bounds every similarity and nq * eps_q every
// doc score.  k_tc_select keeps the docs whose estimate is within 2*nq*eps_q (+ slack) of the
// top_k-th best estimate -- a superset of the true top_k -- and only those get k_exact.  Non-finite
// estimates disable the filter for that query.
// Operand tile: element (row r, 8-wide K chunk kc) at kc * LBO + (r/8) * 128 + (r%8) * 16 with
// LBO = 2048 + 32, i.e. at kc * LBO + 16 r: the 32-byte skew makes the 16-byte cp.async scatter of a centroid
// row bank-conflict free, and one thread decompresses one token (= its accumulator row in the epilogue): the token is
// stored unnormalised (h(v), same relative rounding as h(v/|v|)) and 1/|v| scales the 32 similarities instead.
// grid = (CTAs per query, B), 128 threads = one warpgroup (~70 KB smem with NQT = 32, of which 18 KB staged similarities).
// ==========================================================================================
#define PB_XTC_LBO 2080u

__global__ void k_rows_to_f16_plain(const float *__restrict__ X, long long n_elems, __half *__restrict__ Xh) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_elems; i += (long long)gridDim.x * blockDim.x)
        Xh[i] = __float2half_rn(X[i]);
}

// out[0] = min over all tokens of |c + w| (the pre-normalisation norm), out[1] = max over all tokens of |w|:
// the two data-dependent constants of the error bounds; inv_norm[t] = 1 / |c + w| of every token
template <int DIM>
__global__ void __launch_bounds__(256)
k_min_vnorm(const float *__restrict__ C, const float *__restrict__ w_rev, int nbits, const uint32_t *__restrict__ codes,
            const uint8_t *__restrict__ residuals, long long N, float *__restrict__ out, float *__restrict__ inv_norm) {
    __shared__ float wr[256];
    for (int i = threadIdx.x; i < (1 << nbits); i += blockDim.x) wr[i] = w_rev[i];
    __syncthreads();
    constexpr int G = DIM / 4;
    const int packed = DIM * nbits / 8;
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    float best = 3.0e38f, wbest = 0.0f;
    for (long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < N; t += nw) {
        const float *cen = C + (size_t)codes[t] * DIM;
        const uint8_t *prow = residuals + (size_t)t * packed;
        float p = 0.0f, pw = 0.0f;
        for (int g = lane; g < G; g += 32) {
            const float4 c = reinterpret_cast<const float4 *>(cen)[g];
            const uint32_t f = load_fields4(prow, g, nbits);
            const float w0 = wr[f & 255u], w1 = wr[(f >> 8) & 255u], w2 = wr[(f >> 16) & 255u], w3 = wr[f >> 24];
            const float a = c.x + w0, b2 = c.y + w1, c2 = c.z + w2, d2 = c.w + w3;
            p += a * a + b2 * b2 + c2 * c2 + d2 * d2;
            pw += w0 * w0 + w1 * w1 + w2 * w2 + w3 * w3;
        }
        for (int m = 16; m >= 1; m >>= 1) {
            p += __shfl_xor_sync(PB_FULL, p, m);
            pw += __shfl_xor_sync(PB_FULL, pw, m);
        }
        const float nrm = sqrtf(p), wn = sqrtf(pw);
        if (inv_norm && lane == 0) inv_norm[t] = 1.0f / fmaxf(nrm, 1e-12f);  // operand of k_maxsim_tc
        best = fminf(best, nrm == nrm ? nrm : 0.0f);
        wbest = fmaxf(wbest, wn == wn ? wn : 3.0e38f);
    }
    if (lane == 0) {  // non-negative floats order as ints
        atomicMin(reinterpret_cast<int *>(out), __float_as_int(fmaxf(best, 0.0f)));
        atomicMax(reinterpret_cast<int *>(out + 1), __float_as_int(fmaxf(wbest, 0.0f)));
    }
}

// NQT = query rows of the N operand: 32 (nq <= 32, 4 CTAs/SM) or 64 (nq <= 64, e.g. the 48-token default of the
// reference's ONNX encoder; 3 CTAs/SM)
template <int DIM, int NBITS, int NQT>
__global__ void __launch_bounds__(128, NQT == 32 ? 4 : 3)
k_exact_tc(const float *__restrict__ Q, const int *__restrict__ q_off, int QS, const int *__restrict__ qexp,
           const __half *__restrict__ Ch,
           const float *__restrict__ w_rev, const uint32_t *__restrict__ codes,
           const uint8_t *__restrict__ residuals, const long long *__restrict__ doc_off,
           const uint32_t *__restrict__ kept, const int *__restrict__ n_kept, const long long *__restrict__ tok_prefix,
           int Mcap, uint32_t *__restrict__ maxkey) {
    extern __shared__ __align__(128) unsigned char smem_x[];
    constexpr int KC = DIM / 8, KSTEPS = DIM / 16;
    static_assert(KC <= 16 && DIM % 16 == 0, "k_exact_tc: one half-warp stages one centroid row");
    static_assert(NQT == 32 || NQT == 64, "k_exact_tc: N = 32 or 64");
    constexpr uint32_t LBO_A = PB_XTC_LBO, A_BYTES = KC * LBO_A, QB_BYTES = NQT * DIM * 2;
    constexpr uint32_t LBO_B = (NQT / 8) * 128, SBO = 128;
    constexpr int PACKED = DIM * NBITS / 8, NW = PACKED / 4;
    static_assert(PACKED % 4 == 0, "k_exact_tc: packed rows are read in 32-bit words");
    constexpr bool PIECES = PACKED % 16 == 0;  // packed rows are read straight into registers, 16 bytes at a time
    constexpr int P = PIECES ? PACKED / 16 : 1;
    unsigned char *As = smem_x;                        // [128 tokens] fp16 operand tile: element (r, kc) at kc*LBO + 16 r
    unsigned char *Qb = As + A_BYTES;                  // [32 query rows] fp16 operand tile
    // Th[byte] = the fp16 bucket weights of the 8/NBITS fields packed in that byte, first field first
    constexpr int VB = 8 / NBITS;
    __half *Th = reinterpret_cast<__half *>(Qb + QB_BYTES);  // [256][VB]
    float *Acc = reinterpret_cast<float *>(Th + 256 * VB);    // [128 tokens][ACC_LD(NQT)] similarities of the chunk
    const int b = blockIdx.y;
    const int nk = n_kept[b];
    const long long *tp = tok_prefix + (size_t)b * (Mcap + 1);
    const uint32_t *kp = kept + (size_t)b * Mcap;
    const long long T = tp[nk];
    const int r0q = q_off[b], nq = q_off[b + 1] - r0q;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long n_chunks = (T + 127) / 128;
    const long long per = (n_chunks + gridDim.x - 1) / gridDim.x;
    const long long c_lo = (long long)blockIdx.x * per, c_hi = min(n_chunks, c_lo + per);
    if (c_lo >= c_hi || nq == 0) return;
    // the query enters the tensor cores scaled by 2^qexp[b] and the similarities leave scaled by 2^-qexp[b] (exact)
    const float q_up = ldexpf(1.0f, qexp[b]), q_down = ldexpf(1.0f, -qexp[b]);
    for (int i = threadIdx.x; i < 256 * VB; i += blockDim.x) {
        const int byte = i / VB, j = i - byte * VB;
        Th[i] = __float2half_rn(w_rev[(byte >> (8 - NBITS * (j + 1))) & ((1 << NBITS) - 1)]);
    }
    // query * 2^qexp -> fp16, canonical layout (kc * 4 + r/8) * 128 + (r%8) * 16 + 2e; rows >= nq are zero
    for (int idx = threadIdx.x; idx < NQT * KC; idx += blockDim.x) {
        const int r = idx / KC, kc = idx - r * KC;
        __half v8[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v8[e] = __float2half_rn(r < nq ? Q[(size_t)(r0q + r) * DIM + kc * 8 + e] * q_up : 0.0f);
        *reinterpret_cast<uint4 *>(Qb + (kc * (NQT / 8) + (r >> 3)) * 128 + (r & 7) * 16) = *reinterpret_cast<uint4 *>(v8);
    }
    const int hl = lane >> 4, kcl = lane & 15;  // staging: one lane per 8-wide K chunk, two centroid rows per instruction
    const int row = threadIdx.x;                // decompression and epilogue: one thread per token (= accumulator row)
    TokMeta cur = locate_token<false>(c_lo * 128 + threadIdx.x, T, 0, nk, tp, kp, doc_off, codes);
    for (long long chunk = c_lo; chunk < c_hi; ++chunk) {
        __syncthreads();  // previous chunk: similarities read out, operand tile free
        // ---- loads: each thread its own token's packed row, into registers (read once, from HBM); 16 lanes x 16 B =
        //      one fp16 centroid row, straight to its place in the operand tile ----
        uint32_t pw[NW];
        if (cur.r >= 0) {
            const uint8_t *src = residuals + (size_t)cur.g * PACKED;
            if (PIECES) {
#pragma unroll
                for (int pc = 0; pc < P; ++pc) {
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
        const int nvalid = __popc(__ballot_sync(PB_FULL, cur.r >= 0));
        for (int k = 0; k < nvalid; k += 2) {
            const int kk = k + hl;
            const uint32_t ck = __shfl_sync(PB_FULL, cur.code, kk);
            if (kcl < KC && kk < nvalid) cp_async16(As + kcl * LBO_A + (w * 32 + kk) * 16, Ch + (size_t)ck * DIM + kcl * 8);
        }
        TokMeta nxt;
        nxt.r = -1;
        nxt.g = 0;
        nxt.code = 0;
        if (chunk + 1 < c_hi) {
            const int r_lo = max(__shfl_sync(PB_FULL, cur.r, 0), 0);
            nxt = locate_token<false>((chunk + 1) * 128 + threadIdx.x, T, r_lo, nk, tp, kp, doc_off, codes);
        }
        cp_async_wait_all();
        __syncwarp();
        // ---- approximate decompression in place: v = c + w per thread (= token), stored unnormalised as fp16;
        //      1/|v| is applied to the similarities in the epilogue ----
        float inv = 0.0f;
        if (cur.r >= 0) {
            float p = 0.0f;
#pragma unroll
            for (int kc = 0; kc < KC; ++kc) {
                unsigned char *cell = As + kc * LBO_A + row * 16;
                const uint4 raw = *reinterpret_cast<const uint4 *>(cell);
                const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
                uint32_t wv[4], ow[4];  // the chunk's 8 weights / 8 results as half2 words
                // the chunk's fields are bytes [kc*NBITS, (kc+1)*NBITS) of the row (codec.rs:300-340, first field
                // in the high bits): one table read per byte
                if (NBITS == 4) {
                    const uint32_t x = pw[kc];
                    const uint32_t *T32 = reinterpret_cast<const uint32_t *>(Th);
#pragma unroll
                    for (int j = 0; j < 4; ++j) wv[j] = T32[(x >> (8 * j)) & 255u];
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
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const __half2 v2 = __hadd2(*reinterpret_cast<const __half2 *>(&rw[j]), *reinterpret_cast<const __half2 *>(&wv[j]));
                    const float2 f = __half22float2(v2);
                    p = fmaf(f.x, f.x, p);
                    p = fmaf(f.y, f.y, p);
                    ow[j] = *reinterpret_cast<const uint32_t *>(&v2);
                }
                *reinterpret_cast<uint4 *>(cell) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
            }
            inv = rsqrtf(fmaxf(p, 1e-24f)) * q_down;
        } else {
#pragma unroll
            for (int kc = 0; kc < KC; ++kc) *reinterpret_cast<uint4 *>(As + kc * LBO_A + row * 16) = make_uint4(0, 0, 0, 0);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the tiles are read by the async proxy
        __syncthreads();
        {
            // the CTA is one warpgroup: two M = 64 slabs of tokens (64 rows = 1024 bytes of the tile), staged to Acc
            const uint32_t a0 = smem_u32(As), b0 = smem_u32(Qb);
#pragma unroll
            for (int p = 0; p < 2; ++p) {
                float d[NQT / 2] = {};
                wg_fence();
#pragma unroll
                for (int s = 0; s < KSTEPS; ++s)
                    wg_mma_f16<NQT>(d, wg_desc(a0 + p * 1024 + s * 2 * LBO_A, LBO_A, SBO), wg_desc(b0 + s * 2 * LBO_B, LBO_B, SBO),
                                    s > 0 ? 1u : 0u);
                wg_commit();
                wg_wait_all(d);
                wg_stage<NQT>(Acc + p * 64 * ACC_LD(NQT), d);
            }
        }
        __syncthreads();
        // ---- epilogue: thread = token, 32 similarities per pass; per-doc maxima ----
        const int rank = cur.r;
        const unsigned grp = __match_any_sync(PB_FULL, rank);
#pragma unroll 1
        for (int h = 0; h < NQT / 32; ++h) {
            if (32 * h >= nq) break;
            uint32_t rr[32];
            acc_row(Acc + row * ACC_LD(NQT) + 32 * h, rr);
            // maxima are taken on the order-preserving int image of the float (x ^ ((x >> 31) & 0x7fffffff), its own
            // inverse); only the publishing lane converts to the score key.  +inf / +NaN win the max and map to key 0 =
            // "no estimate" (filter off for the query); -NaN loses, like every non-finite value in the exact path.
            if (grp == PB_FULL) {
                if (rank >= 0) {  // the warp's 32 tokens belong to one doc: one 32-lane atomic (lane = query token)
                    int mine = 0;
#pragma unroll
                    for (int q = 0; q < 32; ++q) {
                        const int x = __float_as_int(__uint_as_float(rr[q]) * inv);
                        const int m = __reduce_max_sync(PB_FULL, x ^ ((x >> 31) & 0x7fffffff));
                        if (lane == q) mine = m;
                    }
                    const uint32_t key = score_key_asc(__int_as_float(mine ^ ((mine >> 31) & 0x7fffffff)));
                    if (32 * h + lane < nq && key) atomicMax(&maxkey[((size_t)b * Mcap + rank) * QS + 32 * h + lane], key);
                }
            } else if (rank >= 0) {  // doc boundary inside the warp: reduce per group, the group's first lane publishes
                const int leader = __ffs(grp) - 1;
                uint32_t *mrow = &maxkey[((size_t)b * Mcap + rank) * QS + 32 * h];
#pragma unroll
                for (int q = 0; q < 32; ++q) {  // unrolled: rr stays in registers
                    const int x = __float_as_int(__uint_as_float(rr[q]) * inv);
                    const int m = __reduce_max_sync(grp, x ^ ((x >> 31) & 0x7fffffff));
                    const uint32_t key = score_key_asc(__int_as_float(m ^ ((m >> 31) & 0x7fffffff)));
                    if (lane == leader && 32 * h + q < nq && key) atomicMax(mrow + q, key);
                }
            }
        }
        cur = nxt;
    }
}

// ------------------------------------------------------------------------------------------
// The same filter through the linearity of the dot product (the default): a decompressed token is
// D = (c + w) / |c + w|, so  q.D = (q.c + q.w) / |v|.  q.c is the centroid score the path already has for every
// (query token, centroid) -- one 2*QS-byte row of the 16-bit table per token, the row a5 gathers -- |v| is a
// per-token constant stored at index open, and only q.w, the residual part, goes through the tensor cores: the A
// tile holds the fp16 bucket weights of the token's packed residual (one table read per byte, no centroid row, no
// add, no norm), the epilogue adds the decoded centroid score and scales.  Against k_exact_tc: a quarter of the L2
// traffic per token (64-byte table row instead of a 256-byte fp16 centroid row), about half the instructions,
// and a tighter certificate, because the centroid part is known to a 16-bit code instead of fp16 rounding:
//     |q.c - s~|           <= (E + 1.01) * 2R / 65535          (s~ = centre of the code; E = 0 for the exact table)
//     |q.w - h(q).h(w)|    <= |q| max|w| (2u + u^2 + 2^-15)    (u = 2^-11; products exact, fp32 accumulation;
//                                                               h(q) = 2^-qexp h(2^qexp q) as above, so the 2^-15 of
//                                                               subnormals and fp32 sums holds at every query scale)
//     |1/|v| - inv|        <= 2^-20 / |v|
// so |q.D - est| <= |q|max * eps_unit2 with eps_unit2 = ((E + 1.01) 2 cmax 1.0001 / 65535 + wmax (2u + u^2 + 2^-15)) / vmin
// + 8e-6 (filter_eps_unit2 in engine.cu).  Flagged queries (no valid table) publish nothing -> no estimate -> every
// kept doc survives.  Same grid / block / accumulator layout as k_exact_tc.
// ------------------------------------------------------------------------------------------
// estimate[b][r] = sum over q of the per-token maxima (any order); resets maxkey.  one warp per kept doc.
__global__ void __launch_bounds__(256)
k_tc_finalize(uint32_t *__restrict__ maxkey, const int *__restrict__ q_off, int QS, const int *__restrict__ n_kept, int Mcap,
              const long long *__restrict__ tok_prefix, float *__restrict__ est, int reset) {
    const int b = blockIdx.y, lane = threadIdx.x & 31;
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= n_kept[b]) return;
    const int nq = q_off[b + 1] - q_off[b];
    uint32_t *row = maxkey + ((size_t)b * Mcap + r) * QS;
    float tot = 0.0f;
    bool bad = false;
    for (int q = lane; q < nq; q += 32) {
        const uint32_t k = row[q];
        if (reset) row[q] = 0u;
        if (k) tot += key_to_score(k);
        else bad = true;  // no finite similarity for this query token: do not trust the estimate
    }
    for (int m = 16; m >= 1; m >>= 1) tot += __shfl_xor_sync(PB_FULL, tot, m);
    bad = __any_sync(PB_FULL, bad);
    const long long *tp = tok_prefix + (size_t)b * (Mcap + 1);
    if (tp[r + 1] == tp[r]) {  // a doc without tokens scores exactly 0 (maxsim.rs:284-291 adds nothing)
        bad = false;
        tot = 0.0f;
    }
    if (lane == 0) est[(size_t)b * Mcap + r] = bad ? NAN : tot;
}

// PB_FILTER_DIAG: the pass-1 estimate of every (kept doc, query token) maximum (est) against the exact maximum of the
// same pair (exact, k_exact's keys), in units of the certified bound qnmax[b] * eps_unit.  out[0] = ceil(1e6 * the
// largest ratio) (INT64_MAX: a non-finite estimate of a finite maximum), out[1] += the pairs compared.  A doc without
// tokens has no maximum; a flagged query (qflag: no estimate by design, the filter keeps all its docs) is skipped.
__global__ void __launch_bounds__(256)
k_filter_diag(const uint32_t *__restrict__ est, const uint32_t *__restrict__ exact, const int *__restrict__ q_off, int QS,
              const int *__restrict__ n_kept, int Mcap, const float *__restrict__ qnmax, const int *__restrict__ qflag,
              float eps_unit, unsigned long long *__restrict__ out) {
    const int b = blockIdx.y;
    if (qflag && qflag[b]) return;
    const int nq = q_off[b + 1] - q_off[b];
    const long long n = (long long)n_kept[b] * nq;
    const double unit = (double)qnmax[b] * (double)eps_unit;
    const unsigned long long sat = 0x7fffffffffffffffull;
    unsigned long long worst = 0ull, cnt = 0ull;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const size_t at = ((size_t)b * Mcap + (size_t)(i / nq)) * QS + (size_t)(i % nq);
        const uint32_t xk = exact[at], ek = est[at];
        if (!xk) continue;
        ++cnt;
        unsigned long long v = sat;
        if (ek) {
            const double d = fabs((double)key_to_score(ek) - (double)key_to_score(xk));
            const double r = unit > 0.0 ? ceil(1e6 * d / unit) : (d == 0.0 ? 0.0 : 1e300);
            v = r < 9.0e18 ? (unsigned long long)r : sat;
        }
        worst = v > worst ? v : worst;
    }
    for (int m = 16; m >= 1; m >>= 1) {
        const unsigned long long ow = __shfl_xor_sync(PB_FULL, worst, m), oc = __shfl_xor_sync(PB_FULL, cnt, m);
        worst = ow > worst ? ow : worst;
        cnt += oc;
    }
    if ((threadIdx.x & 31) == 0 && cnt) {
        atomicMax(out, worst);
        atomicAdd(out + 1, cnt);
    }
}

// survivors of the filter, in approximate-rank order.  grid = B, 1024 threads, smem = pow2(n_kept) * 8.
__global__ void __launch_bounds__(1024)
k_tc_select(const float *__restrict__ est, const uint32_t *__restrict__ kept, const uint32_t *__restrict__ krank,
            const int *__restrict__ n_kept, int Mcap, int top_k, const int *__restrict__ q_off,
            const float *__restrict__ qnmax, float eps_unit, const long long *__restrict__ doc_off,
            uint32_t *__restrict__ kept2, uint32_t *__restrict__ krank2, int *__restrict__ n_kept2,
            long long *__restrict__ tok_prefix2, long long *__restrict__ kept_tokens2, uint32_t *__restrict__ src_rank2) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64 *sk = reinterpret_cast<u64 *>(smem_raw);
    __shared__ int scan_tmp[33];
    __shared__ int any_bad;
    const int b = blockIdx.x;
    const int nk = n_kept[b];
    const int nq = q_off[b + 1] - q_off[b];
    const float *e = est + (size_t)b * Mcap;
    if (threadIdx.x == 0) any_bad = 0;
    __syncthreads();
    float thr = -INFINITY;  // keep everything
    if (nk > top_k && top_k > 0) {
        const int P = next_pow2(nk);
        for (int i = threadIdx.x; i < P; i += blockDim.x) {
            u64 k = ~0ull;
            if (i < nk) {
                const uint32_t sk32 = score_key_asc(e[i]);
                if (!sk32) any_bad = 1;
                k = ((u64)(~sk32) << 32) | (uint32_t)i;  // ascending = best first
            }
            sk[i] = k;
        }
        __syncthreads();
        bitonic_sort_u64(sk, P);
        if (!any_bad) {
            const float tau = key_to_score(~(uint32_t)(sk[top_k - 1] >> 32));
            thr = tau - (2.0f * (float)nq * qnmax[b] * eps_unit + 1e-3f);
        }
        __syncthreads();
    }
    long long run = 0;
    int outn = 0;
    for (int base = 0; base < nk; base += blockDim.x) {
        const int i = base + threadIdx.x;
        int f = 0, len = 0;
        uint32_t d = 0;
        if (i < nk && !(e[i] < thr)) {  // NaN estimates survive
            f = 1;
            d = kept[(size_t)b * Mcap + i];
            len = (int)(doc_off[d + 1] - doc_off[d]);
        }
        int tot, ttot;
        const int pos = block_exclusive_scan(f, scan_tmp, &tot);
        const int tpos = block_exclusive_scan(len, scan_tmp, &ttot);
        if (f) {
            kept2[(size_t)b * Mcap + outn + pos] = d;
            krank2[(size_t)b * Mcap + outn + pos] = krank ? krank[(size_t)b * Mcap + i] : (uint32_t)i;
            tok_prefix2[(size_t)b * (Mcap + 1) + outn + pos] = run + tpos;
            if (src_rank2) src_rank2[(size_t)b * Mcap + outn + pos] = (uint32_t)i;
        }
        outn += tot;
        run += ttot;
    }
    if (threadIdx.x == 0) {
        tok_prefix2[(size_t)b * (Mcap + 1) + outn] = run;
        n_kept2[b] = outn;
        kept_tokens2[b] = run;
    }
}
