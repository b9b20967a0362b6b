// k_scores.cuh -- a2 centroid scores: tile_dots (scalar / paired rows), tile loads, k_centroid_scores.
// Part of kernels.cuh (included from there, in order; not a standalone header).

#define PB_TOK_TILE 128          // doc tokens (or centroids) per CTA tile
#define PB_Q_TILE 32             // query tokens per pass
#define PB_PROBE_CHUNK 4096      // centroids scanned by one CTA of k_topn_partial (1024 per warp)

// ------------------------------------------------------------------------------------------
// shared compute core: 8 query rows x 4 vectors per lane, pinned sequential-j fma order
// ------------------------------------------------------------------------------------------
template <int DIM>
PB_DEV void tile_dots(const float *__restrict__ Qs, const float *__restrict__ Vs, float (&acc)[8][4]) {
    // (An explicit two-register-set software pipeline of the LDS was measured: 222 registers, no gain.)
    constexpr int LD = DIM + 4;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[i][k] = 0.0f;
#pragma unroll 2
    for (int j = 0; j < DIM; j += 4) {
        float4 q[8], v[4];
#pragma unroll
        for (int i = 0; i < 8; ++i) q[i] = *reinterpret_cast<const float4 *>(Qs + i * LD + j);
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = *reinterpret_cast<const float4 *>(Vs + (32 * k) * LD + j);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float a = acc[i][k];
                a = __fmaf_rn(q[i].x, v[k].x, a);
                a = __fmaf_rn(q[i].y, v[k].y, a);
                a = __fmaf_rn(q[i].z, v[k].z, a);
                a = __fmaf_rn(q[i].w, v[k].w, a);
                acc[i][k] = a;
            }
    }
}

PB_DEV void cp_async16(void *smem_dst, const void *gmem_src) {
    unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src));
}
PB_DEV void cp_async4(void *smem_dst, const void *gmem_src) {
    unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(gmem_src));
}
PB_DEV void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// async variant of load_rows_padded: cp.async for valid rows, zero fill for the rest
template <int DIM>
PB_DEV void load_rows_padded_async(float *__restrict__ dst, const float *__restrict__ src, int n_valid, int rows) {
    constexpr int LD = DIM + 4, G = DIM / 4;
    for (int idx = threadIdx.x; idx < rows * G; idx += blockDim.x) {
        int r = idx / G, g = idx - r * G;
        if (r < n_valid) cp_async16(dst + r * LD + 4 * g, src + (size_t)r * DIM + 4 * g);
        else *reinterpret_cast<float4 *>(dst + r * LD + 4 * g) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// tile_dots on fp32 pairs: two independent IEEE FMAs per pair with a broadcast scalar operand, the same
// sequential-j FMA per dot, hence the same bits.  (sm_90 has no packed fp32 FMA; the pair is two FFMAs, and the
// 8-byte operand loads of the interleaved rows stay.)  Qi holds the 8 query rows as 4 row pairs interleaved
// element-wise, pair p at Qi + p*2*DIM: (q_2p[0], q_2p+1[0], q_2p[1], q_2p+1[1], ...); acc[2p][k] / acc[2p+1][k] come
// out as the halves of one register pair.
PB_DEV u64 fma2_bcast(u64 a_pair, float b, u64 c_pair) {
    const float lo = __fmaf_rn(__uint_as_float((uint32_t)a_pair), b, __uint_as_float((uint32_t)c_pair));
    const float hi = __fmaf_rn(__uint_as_float((uint32_t)(a_pair >> 32)), b, __uint_as_float((uint32_t)(c_pair >> 32)));
    return ((u64)__float_as_uint(hi) << 32) | __float_as_uint(lo);
}
template <int DIM>
PB_DEV void tile_dots_f2(const float *__restrict__ Qi, const float *__restrict__ Vs, float (&acc)[8][4]) {
    constexpr int LD = DIM + 4;
    u64 a2[4][4];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int k = 0; k < 4; ++k) a2[p][k] = 0ull;
#pragma unroll 2
    for (int j = 0; j < DIM; j += 4) {
        ulonglong2 qa[4], qb[4];
        float4 v[4];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            qa[p] = *reinterpret_cast<const ulonglong2 *>(Qi + p * 2 * DIM + 2 * j);      // dims j, j+1
            qb[p] = *reinterpret_cast<const ulonglong2 *>(Qi + p * 2 * DIM + 2 * j + 4);  // dims j+2, j+3
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = *reinterpret_cast<const float4 *>(Vs + (32 * k) * LD + j);
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                u64 a = a2[p][k];
                a = fma2_bcast(qa[p].x, v[k].x, a);
                a = fma2_bcast(qa[p].y, v[k].y, a);
                a = fma2_bcast(qb[p].x, v[k].z, a);
                a = fma2_bcast(qb[p].y, v[k].w, a);
                a2[p][k] = a;
            }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            acc[2 * p][k] = __uint_as_float((uint32_t)a2[p][k]);
            acc[2 * p + 1][k] = __uint_as_float((uint32_t)(a2[p][k] >> 32));
        }
}

// element-wise interleaved copy of the query rows for tile_dots_f2: Qi[b][QS/2][DIM][2], rows >= nq are zero
__global__ void k_interleave_query_rows(const float *__restrict__ Q, const int *__restrict__ q_off, int QS, int dim,
                                        float *__restrict__ Qi) {
    const int b = blockIdx.y, r0 = q_off[b], nq = q_off[b + 1] - r0;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < QS * dim; idx += gridDim.x * blockDim.x) {
        const int r = idx / dim, j = idx - r * dim;
        Qi[(((size_t)b * (QS >> 1) + (r >> 1)) * dim + j) * 2 + (r & 1)] = r < nq ? Q[(size_t)(r0 + r) * dim + j] : 0.0f;
    }
}

// contiguous async copy of n_valid row pairs (2*DIM floats each), zero fill up to `pairs`
template <int DIM>
PB_DEV void load_pairs_async(float *__restrict__ dst, const float *__restrict__ src, int n_valid, int pairs) {
    constexpr int G = 2 * DIM / 4;
    for (int idx = threadIdx.x; idx < pairs * G; idx += blockDim.x) {
        if (idx < n_valid * G) cp_async16(dst + 4 * idx, src + 4 * idx);
        else *reinterpret_cast<float4 *>(dst + 4 * idx) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// copy `rows` x DIM floats (zero rows beyond n_valid) from global to a padded smem tile
template <int DIM>
PB_DEV void load_rows_padded(float *__restrict__ dst, const float *__restrict__ src, int n_valid, int rows) {
    constexpr int LD = DIM + 4, G = DIM / 4;
    for (int idx = threadIdx.x; idx < rows * G; idx += blockDim.x) {
        int r = idx / G, g = idx - r * G;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < n_valid) v = reinterpret_cast<const float4 *>(src)[(size_t)r * G + g];
        *reinterpret_cast<float4 *>(dst + r * LD + 4 * g) = v;
    }
}

// ------------------------------------------------------------------------------------------
// a2: centroid scores.  grid = (ceil(K/128), query groups); 128 threads.
// ------------------------------------------------------------------------------------------
// F2: the query tiles come from the interleaved copy (k_interleave_query_rows) and the dots run on row pairs (tile_dots_f2).
template <int DIM, bool F2>
__global__ void __launch_bounds__(128, 2)
k_centroid_scores(const float *__restrict__ Q, const int *__restrict__ q_off, int B, int QS,
                  const float *__restrict__ C, long long K, float *__restrict__ ST,
                  unsigned short *__restrict__ ST16, const float2 *__restrict__ qrange, int *__restrict__ qflag) {
    extern __shared__ __align__(16) float smem[];
    constexpr int LD = DIM + 4;
    float *Vs = smem;                      // [128][LD] centroid tile, resident for the CTA's lifetime
    float *Qs0 = smem + PB_TOK_TILE * LD;  // 2 x [32][LD] query tiles: the next one streams in (cp.async)
    const long long c0 = (long long)blockIdx.x * PB_TOK_TILE;        // while the current one is used
    const int nv = (int)min((long long)PB_TOK_TILE, K - c0);
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // work items of this CTA: (query b, block of 32 query tokens qb), b = blockIdx.y, += gridDim.y
    int b = blockIdx.y, qb = 0, buf = 0;
    while (b < B && q_off[b + 1] - q_off[b] == 0) b += gridDim.y;
    load_rows_padded_async<DIM>(Vs, C + (size_t)c0 * DIM, nv, PB_TOK_TILE);
    if (b < B) {
        const int r0 = q_off[b], nq = q_off[b + 1] - r0;
        if (F2) load_pairs_async<DIM>(Qs0, Q + (size_t)b * QS * DIM, min(PB_Q_TILE, QS) / 2, PB_Q_TILE / 2);
        else load_rows_padded_async<DIM>(Qs0, Q + (size_t)r0 * DIM, min(PB_Q_TILE, nq), PB_Q_TILE);
    }
    while (b < B) {
        const int r0 = q_off[b], nq = q_off[b + 1] - r0;
        // next work item
        int nb = b, nqb = qb + PB_Q_TILE;
        if (nqb >= nq) {
            nqb = 0;
            nb = b + gridDim.y;
            while (nb < B && q_off[nb + 1] - q_off[nb] == 0) nb += gridDim.y;
        }
        cp_async_wait_all();
        __syncthreads();  // tile `buf` (and Vs) landed; everyone is done with tile buf^1
        if (nb < B) {
            const int nr0 = q_off[nb], nnq = q_off[nb + 1] - nr0;
            if (F2)
                load_pairs_async<DIM>(Qs0 + (buf ^ 1) * PB_Q_TILE * LD, Q + ((size_t)nb * QS + nqb) * DIM,
                                      min(PB_Q_TILE, QS - nqb) / 2, PB_Q_TILE / 2);
            else
                load_rows_padded_async<DIM>(Qs0 + (buf ^ 1) * PB_Q_TILE * LD, Q + (size_t)(nr0 + nqb) * DIM,
                                            min(PB_Q_TILE, nnq - nqb), PB_Q_TILE);
        }
        if (qb + 8 * w < ((nq + 7) & ~7)) {
            float acc[8][4];
            if (F2) tile_dots_f2<DIM>(Qs0 + buf * PB_Q_TILE * LD + 4 * w * 2 * DIM, Vs + lane * LD, acc);
            else tile_dots<DIM>(Qs0 + buf * PB_Q_TILE * LD + 8 * w * LD, Vs + lane * LD, acc);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                long long c = c0 + lane + 32 * k;
                if (c < K) {
                    float4 *dst = reinterpret_cast<float4 *>(ST + ((size_t)b * K + c) * QS + qb + 8 * w);
                    dst[0] = make_float4(acc[0][k], acc[1][k], acc[2][k], acc[3][k]);
                    dst[1] = make_float4(acc[4][k], acc[5][k], acc[6][k], acc[7][k]);
                    if (ST16) {  // 16-bit fixed-point copy for the first approximate pass (k_approx16)
                        const float2 rg = qrange[b];  // (R*scale, scale)
                        uint32_t cd[8];
                        bool bad = false;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            const float t = floorf(__fmaf_rn(acc[i][k], rg.y, rg.x));
                            bad |= !(t >= 0.0f && t <= 65535.0f);  // out of range or NaN
                            cd[i] = (uint32_t)fminf(fmaxf(t, 0.0f), 65535.0f);
                        }
                        if (bad && qb + 8 * w < nq) {
                            // only rows of real query tokens matter (padding rows are zeros: in range)
                            bool real_bad = false;
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                const float t = floorf(__fmaf_rn(acc[i][k], rg.y, rg.x));
                                real_bad |= (qb + 8 * w + i < nq) && !(t >= 0.0f && t <= 65535.0f);
                            }
                            if (real_bad) atomicOr(&qflag[b], 1);
                        }
                        uint4 pk4;
                        pk4.x = cd[0] | (cd[1] << 16);
                        pk4.y = cd[2] | (cd[3] << 16);
                        pk4.z = cd[4] | (cd[5] << 16);
                        pk4.w = cd[6] | (cd[7] << 16);
                        *reinterpret_cast<uint4 *>(ST16 + ((size_t)b * K + c) * QS + qb + 8 * w) = pk4;
                    }
                }
            }
        }
        b = nb;
        qb = nqb;
        buf ^= 1;
    }
    cp_async_wait_all();
}

// plain [n_rows][K] row-major output for the pb_centroid_scores stage entry point
__global__ void k_transpose_scores(const float *__restrict__ ST, long long K, int QS, int nq,
                                   float *__restrict__ S) {
    long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= K) return;
    for (int q = 0; q < nq; ++q) S[(size_t)q * K + c] = ST[(size_t)c * QS + q];
}
