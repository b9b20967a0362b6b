// k_filter_tc.cuh -- a7' tensor-core fp16 certified filter in front of the exact stage: the token norms it rests on,
// the per-doc estimate and the survivors.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ==========================================================================================
// Tensor-core (wgmma) certified filter in front of the exact stage (search path).
//
// Only the top_k docs of the M kept ones need exact scores (search.rs:496-515).  k_maxsim_tc (k_maxsim_tc.cuh)
// estimates every kept doc's MaxSim on the tensor cores through the linearity of the dot product: a decompressed token
// is D = (c + w) / |c + w|, so  q.D = (q.c + q.w) / |v|.  q.c is the centroid score the path already has for every
// (query token, centroid) -- one 2*QS-byte row of the 16-bit table per token, the row a5 gathers -- |v| is a
// per-token constant stored at index open (k_min_vnorm), and only q.w, the residual part, goes through the tensor
// cores: the A tile holds the fp16 bucket weights of the token's packed residual (one table read per byte), the
// epilogue adds the decoded centroid score and scales.  fp16 rather than bf16: every operand is a unit-scale vector,
// and 11 significand bits make the certified band 8x narrower.  The query enters as h(q) = 2^-qexp h(2^qexp q): scaled
// so that its largest row norm is in [1, 2) (qexp from k_query_range), which keeps the subnormal slack relative to
// |q|max and rules out fp16 overflow at any query scale.  With u = 2^-11 the unit roundoff,
//     |q.c - s~|           <= (E + 1.01) * 2R / 65535          (s~ = centre of the code; E = 0 for the exact table)
//     |q.w - h(q).h(w)|    <= |q| max|w| (2u + u^2 + 2^-15)    (products exact, fp32 accumulation; 2^-15 covers
//                                                               subnormals and fp32 sums at every query scale)
//     |1/|v| - inv|        <= 2^-20 / |v|
// so eps_q = |q|max * eps_unit2 bounds every similarity and nq * eps_q every doc score, with
// eps_unit2 = ((E + 1.01) 2 cmax 1.0001 / 65535 + wmax (2u + u^2 + 2^-15)) / vmin + 8e-6 (filter_eps_unit2 in
// engine.cu; vmin = min|v| and wmax = max|w| are measured at index open).  k_tc_select keeps the docs whose estimate
// is within 2*nq*eps_q (+ slack) of the top_k-th best estimate -- a superset of the true top_k -- and only those get
// exact scores.  Flagged queries (no valid table) publish nothing -> no estimate -> every kept doc survives; so do
// the docs of a query with a non-finite estimate.
// ==========================================================================================

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

// survivors of the filter, in approximate-rank order.  qtopk: each query's own top_k (or null: top_k); a query whose
// top_k reaches its kept count keeps every kept doc.  grid = B, 1024 threads, smem = pow2(n_kept) * 8.
__global__ void __launch_bounds__(1024)
k_tc_select(const float *__restrict__ est, const uint32_t *__restrict__ kept, const uint32_t *__restrict__ krank,
            const int *__restrict__ n_kept, int Mcap, int top_k, const int *__restrict__ q_off,
            const float *__restrict__ qnmax, float eps_unit, const long long *__restrict__ doc_off,
            uint32_t *__restrict__ kept2, uint32_t *__restrict__ krank2, int *__restrict__ n_kept2,
            long long *__restrict__ tok_prefix2, long long *__restrict__ kept_tokens2, uint32_t *__restrict__ src_rank2,
            const int *__restrict__ qtopk) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64 *sk = reinterpret_cast<u64 *>(smem_raw);
    __shared__ int scan_tmp[33];
    __shared__ int any_bad;
    const int b = blockIdx.x;
    const int nk = n_kept[b];
    const int nq = q_off[b + 1] - q_off[b];
    if (qtopk) top_k = qtopk[b];
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
