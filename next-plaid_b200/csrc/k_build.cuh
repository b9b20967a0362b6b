// k_build.cuh -- index build: assignment (exact fp32 and tensor-core certified), quantise + pack, k-means.
// Part of kernels.cuh (included from there, in order; not a standalone header).
// ==========================================================================================
// Index-build path (SURVEY 8 a12, secondary): nearest-centroid assignment, residual quantisation
// and bit packing, Lloyd k-means.
// ==========================================================================================

// compress_into_codes (codec.rs:297-343): code = argmax_c dot(x, C_c) in the score order, the LAST
// maximum winning exact ties (Iterator::max_by).  One CTA = 64 tokens resident in shared memory,
// all centroid tiles streamed through a double-buffered 128-row tile (cp.async); 8 warps, each
// 8 tokens x 4 centroids per lane with the pinned sequential-j FMA, running best key
// (score_key << 32 | c) per token row in registers.  `bias` (optional, k-means only) is added to the
// score before ranking: argmin ||x - c||^2 == argmax (x.c - |c|^2 / 2).
template <int DIM>
__global__ void __launch_bounds__(256, 1)
k_assign(const float *__restrict__ X, long long n, const float *__restrict__ C, long long K,
         const float *__restrict__ bias, long long *__restrict__ codes_i64, uint32_t *__restrict__ codes_u32) {
    extern __shared__ __align__(16) float smem[];
    constexpr int LD = DIM + 4;
    constexpr int NB = DIM <= 128 ? 2 : 1;      // the double-buffered tile does not fit at dim 256
    float *Vs0 = smem;                          // NB x [128][LD] centroid tiles
    float *Xs = smem + NB * PB_TOK_TILE * LD;   // [64][LD] tokens
    const long long x0 = (long long)blockIdx.x * 64;
    const int nx = (int)min(64ll, n - x0);
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    load_rows_padded_async<DIM>(Xs, X + (size_t)x0 * DIM, nx, 64);
    const long long n_tiles = (K + PB_TOK_TILE - 1) / PB_TOK_TILE;
    load_rows_padded_async<DIM>(Vs0, C, (int)min((long long)PB_TOK_TILE, K), PB_TOK_TILE);
    u64 best[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) best[i] = 0ull;
    for (long long t = 0; t < n_tiles; ++t) {
        const int buf = NB == 2 ? (int)(t & 1) : 0;
        if (NB == 1 && t > 0) {
            __syncthreads();  // everyone finished with the previous tile
            const long long c1 = t * PB_TOK_TILE;
            load_rows_padded_async<DIM>(Vs0, C + (size_t)c1 * DIM, (int)min((long long)PB_TOK_TILE, K - c1), PB_TOK_TILE);
        }
        cp_async_wait_all();
        __syncthreads();  // tile t (and Xs) landed; everyone finished with tile t-1's buffer
        if (NB == 2 && t + 1 < n_tiles) {
            const long long c1 = (t + 1) * PB_TOK_TILE;
            load_rows_padded_async<DIM>(Vs0 + (buf ^ 1) * PB_TOK_TILE * LD, C + (size_t)c1 * DIM,
                                        (int)min((long long)PB_TOK_TILE, K - c1), PB_TOK_TILE);
        }
        float acc[8][4];
        tile_dots<DIM>(Xs + 8 * w * LD, Vs0 + buf * PB_TOK_TILE * LD + lane * LD, acc);
        const long long c0 = t * PB_TOK_TILE;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const long long c = c0 + lane + 32 * k;
            if (c < K) {
                const float bs = bias ? bias[c] : 0.0f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float sc = bias ? acc[i][k] + bs : acc[i][k];
                    const u64 key = ((u64)score_key_asc(sc) << 32) | (uint32_t)c;
                    best[i] = key >= best[i] ? key : best[i];
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const u64 b = warp_max_u64(best[i]);
        const long long tok = x0 + 8 * w + i;
        if (lane == 0 && tok < n) {
            if (codes_i64) codes_i64[tok] = (long long)(uint32_t)b;
            if (codes_u32) codes_u32[tok] = (uint32_t)b;
        }
    }
}

// residual = x - C[code] (index.rs:17-40), bucket = #{cutoffs < v} (codec.rs:386), bits LSB-first into
// an MSB-first stream (codec.rs:389-395) == per value the bit-reversed bucket, first dim in the high
// bits.  One warp per token, lane = float4 group.
template <int DIM>
__global__ void __launch_bounds__(256)
k_quantize_pack(const float *__restrict__ X, long long n, const float *__restrict__ C,
                const long long *__restrict__ codes, const float *__restrict__ cutoffs, int nbits,
                uint8_t *__restrict__ packed_out, float *__restrict__ residual_out) {
    __shared__ float cut[256];
    const int ncut = (1 << nbits) - 1;
    for (int i = threadIdx.x; i < ncut; i += blockDim.x) cut[i] = cutoffs[i];
    __syncthreads();
    constexpr int G = DIM / 4;
    const int packed = DIM * nbits / 8;
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n; t += nw) {
        const float *cen = C + (size_t)codes[t] * DIM;
        uint8_t *prow = packed_out ? packed_out + (size_t)t * packed : nullptr;
        for (int g0 = 0; g0 < G; g0 += 32) {
            const int g = g0 + lane;
            uint32_t bits = 0;  // this lane's 4*nbits bits, MSB-first
            if (g < G) {
                const float4 x = reinterpret_cast<const float4 *>(X + (size_t)t * DIM)[g];
                const float4 c = reinterpret_cast<const float4 *>(cen)[g];
                float v[4] = {__fsub_rn(x.x, c.x), __fsub_rn(x.y, c.y), __fsub_rn(x.z, c.z), __fsub_rn(x.w, c.w)};
                if (residual_out) reinterpret_cast<float4 *>(residual_out + (size_t)t * DIM)[g] = make_float4(v[0], v[1], v[2], v[3]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    uint32_t bucket = 0;
                    for (int c2 = 0; c2 < ncut; ++c2) bucket += (v[e] > cut[c2]) ? 1u : 0u;
                    uint32_t rev = 0;
                    for (int b2 = 0; b2 < nbits; ++b2) rev |= ((bucket >> b2) & 1u) << (nbits - 1 - b2);
                    bits = (bits << nbits) | rev;
                }
            }
            if (!prow) continue;
            if (nbits == 8) {
                if (g < G) {  // 4 bytes, first dim first
                    prow[4 * g] = (uint8_t)(bits >> 24);
                    prow[4 * g + 1] = (uint8_t)(bits >> 16);
                    prow[4 * g + 2] = (uint8_t)(bits >> 8);
                    prow[4 * g + 3] = (uint8_t)bits;
                }
            } else if (nbits == 4) {
                if (g < G) {
                    prow[2 * g] = (uint8_t)(bits >> 8);
                    prow[2 * g + 1] = (uint8_t)bits;
                }
            } else if (nbits == 2) {
                if (g < G) prow[g] = (uint8_t)bits;
            } else {  // nbits == 1: two lanes share a byte
                const uint32_t other = __shfl_down_sync(PB_FULL, bits, 1);
                if (g < G && (g & 1) == 0) prow[g >> 1] = (uint8_t)((bits << 4) | (other & 15u));
            }
        }
    }
}

// ---- Lloyd k-means (kmeans.rs:261-422 wraps fastkmeans-rs 1.0.8, whose source is not in the
// reference tree: PARITY UNPINNED, statistical tests only) ----
__global__ void k_half_sqnorm(const float *__restrict__ C, long long K, int dim, float *__restrict__ bias) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < K; c += nw) {
        float p = 0.0f;
        for (int j = lane; j < dim; j += 32) {
            const float v = C[(size_t)c * dim + j];
            p = fmaf(v, v, p);
        }
        for (int m = 16; m >= 1; m >>= 1) p += __shfl_xor_sync(PB_FULL, p, m);
        if (lane == 0) bias[c] = -0.5f * p;
    }
}

__global__ void k_accumulate(const float *__restrict__ X, long long n, int dim, const uint32_t *__restrict__ codes,
                             float *__restrict__ sums, float *__restrict__ counts) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < n; t += nw) {
        const uint32_t c = codes[t];
        for (int j = lane; j < dim; j += 32) atomicAdd(&sums[(size_t)c * dim + j], X[(size_t)t * dim + j]);
        if (lane == 0) atomicAdd(&counts[c], 1.0f);
    }
}

// new centroid = mean of its points; an empty cluster keeps its previous centroid
__global__ void k_update_centroids(float *__restrict__ C, long long K, int dim, const float *__restrict__ sums,
                                   const float *__restrict__ counts) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < K * dim; i += (long long)gridDim.x * blockDim.x) {
        const float cnt = counts[i / dim];
        if (cnt > 0.0f) C[i] = sums[i] / cnt;
    }
}

// row /= max(||row||, 1e-12)  (kmeans.rs:415-419)
__global__ void k_normalize_rows(float *__restrict__ C, long long K, int dim) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < K; c += nw) {
        float p = 0.0f;
        for (int j = lane; j < dim; j += 32) {
            const float v = C[(size_t)c * dim + j];
            p = fmaf(v, v, p);
        }
        for (int m = 16; m >= 1; m >>= 1) p += __shfl_xor_sync(PB_FULL, p, m);
        const float nrm = fmaxf(sqrtf(p), 1e-12f);
        for (int j = lane; j < dim; j += 32) C[(size_t)c * dim + j] /= nrm;
    }
}

__global__ void k_gather_rows(const float *__restrict__ X, const long long *__restrict__ idx, long long K, int dim,
                              float *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < K * dim; i += (long long)gridDim.x * blockDim.x)
        out[i] = X[(size_t)idx[i / dim] * dim + (i % dim)];
}

// ==========================================================================================
// Tensor-core certified filter for nearest-centroid assignment (index-build path).
//
// The exact kernel above spends 128 fp32 FMAs per (token, centroid) pair.  Here an fp16 wgmma
// (fp32 accumulators in registers) scores every pair and the epilogue keeps the 4 best
// centroids per token.  |s_tc - s_exact| <= eps = (2^-10 + 2^-22) |x| max|c| + 2^-24 sqrt(dim) (|x| + max|c|) + 1e-5
// (two fp16 roundings per product, Cauchy-Schwarz; the absolute spacing of fp16 subnormals; fp32 accumulation
// slack), so if the 4th best tensor-core score is more than 2*eps below the best, the true argmax is among the
// first three; those are re-scored in the pinned fp32 order and ranked with the reference's tie rule.  (bf16
// operands, round 1: eps = 2^-7 |x| max|c| -- on k-means centroids of real data, where a token has several
// centroids within 0.01 of its best, nearly every token failed the certificate: 99.98 % exact fallback on the
// clustered benchmark corpus.  fp16 narrows the band 8x; values past the fp16 range become inf and are flagged.)  Tokens that cannot be certified
// (near ties, non-finite values) go through k_assign.  The result is therefore bit-identical to
// compress_into_codes_cpu while ~98 % of the arithmetic runs on the tensor cores.
//
// One CTA = 256 tokens (two 128-token tiles sharing every 128-centroid tile), 288 threads: warps
// 0-7 two warpgroups that issue the MMAs and rank their tokens, warp 8 loader (bulk copies, 3-stage ring).
// Operands sit in shared memory in the canonical K-major no-swizzle layout (8 rows x 16 bytes core
// matrices; SBO = 128 B between row groups, LBO = rows/8 * 128 B between the two 8-element K
// chunks of one MMA).
// ==========================================================================================
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#define PB_TC_M 128
#define PB_TC_N 128
#define PB_TC_STAGES 3

PB_DEV uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
PB_DEV void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
PB_DEV void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
PB_DEV void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done = 0;
    const uint32_t a = smem_u32(bar);
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(done)
                     : "r"(a), "r"(parity)
                     : "memory");
    } while (!done);
}
PB_DEV void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier
PB_DEV void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// ---- Hopper warpgroup MMA (wgmma) ----
// The 128 threads of a warpgroup issue one m64nNk16 product together (fp16 operands from shared memory, fp32
// accumulator in registers).  Fragment of thread t of the warpgroup: d[4i + 2h + j] = element (row 16 (t/32) +
// (t%32)/4 + 8h, column 8i + 2 (t%4) + j).
// shared-memory matrix descriptor, K-major, no swizzle: start>>4 [0,14), LBO>>4 [16,30) = byte stride between the
// 8-element K chunks, SBO>>4 [32,46) = byte stride between 8-row groups, layout type 0 [62,64)
PB_DEV u64 wg_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (u64)((saddr >> 4) & 0x3fffu) | ((u64)((lbo_bytes >> 4) & 0x3fffu) << 16) |
           ((u64)((sbo_bytes >> 4) & 0x3fffu) << 32);
}
PB_DEV void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
PB_DEV void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// waits for every committed group, then pins the accumulator registers behind the wait (the compiler must not read
// them earlier)
template <int R> PB_DEV void wg_wait_all(float (&d)[R]) {
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// d (+)= A B^T, A = 64 rows x 16 (descriptor da), B = N rows x 16 (descriptor db); accumulate = 0 overwrites d
template <int N> PB_DEV void wg_mma_f16(float (&d)[N / 2], u64 da, u64 db, uint32_t accumulate);
template <> PB_DEV void wg_mma_f16<32>(float (&d)[16], u64 da, u64 db, uint32_t accumulate) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(accumulate));
}
template <> PB_DEV void wg_mma_f16<64>(float (&d)[32], u64 da, u64 db, uint32_t accumulate) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(accumulate));
}
template <> PB_DEV void wg_mma_f16<128>(float (&d)[64], u64 da, u64 db, uint32_t accumulate) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(accumulate));
}
// The filters' epilogues work per token (thread = accumulator row).  Their warpgroup stages its m64nN fragment into a
// row-major fp32 tile of ACC_LD(N) floats per row (+4: conflict-free 16-byte row reads) ...
#define ACC_LD(N) ((N) + 4)
template <int N> PB_DEV void wg_stage(float *tile, const float (&d)[N / 2]) {
    const int t = threadIdx.x & 127;
    float *p = tile + (16 * (t >> 5) + ((t & 31) >> 2)) * ACC_LD(N) + 2 * (t & 3);
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
        *reinterpret_cast<float2 *>(p + 8 * i) = make_float2(d[4 * i], d[4 * i + 1]);
        *reinterpret_cast<float2 *>(p + 8 * ACC_LD(N) + 8 * i) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
}
// ... and reads R consecutive columns of its own row back
template <int R> PB_DEV void acc_row(const float *p, uint32_t (&r)[R]) {
#pragma unroll
    for (int i = 0; i < R / 4; ++i) {
        const uint4 v = reinterpret_cast<const uint4 *>(p)[i];
        r[4 * i] = v.x;
        r[4 * i + 1] = v.y;
        r[4 * i + 2] = v.z;
        r[4 * i + 3] = v.w;
    }
}

// f32 rows -> fp16 (round to nearest even; the array type says bf16 for history, the bits are fp16) in MMA tile order
// + the L2 norm of every row.
// Tile order: blocks of 128 rows, each block stored exactly as the kernel wants it in shared memory --
// K-major canonical no-swizzle layout, byte (kc*16 + r/8)*128 + (r%8)*16 + 2*e for row r, 16-byte K chunk
// kc, element e -- so one cp.async.bulk (TMA 1-D copy) moves a whole operand tile.  The array is padded
// with zero rows to a multiple of 128.
__global__ void k_rows_to_bf16(const float *__restrict__ X, long long n, int dim, __nv_bfloat16 *__restrict__ Xb,
                               float *__restrict__ norms) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    const size_t tile_elems = (size_t)128 * dim;
    for (long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nw) {
        float p = 0.0f;
        const size_t tbase = (size_t)(r >> 7) * tile_elems;
        const int rr = (int)(r & 127);
        for (int j = lane; j < dim; j += 32) {
            const float v = X[(size_t)r * dim + j];
            const int kc = j >> 3, e = j & 7;
            reinterpret_cast<__half *>(Xb)[tbase + (size_t)(kc * 16 + (rr >> 3)) * 64 + (rr & 7) * 8 + e] = __float2half_rn(v);
            p = fmaf(v, v, p);
        }
        for (int m = 16; m >= 1; m >>= 1) p += __shfl_xor_sync(PB_FULL, p, m);
        if (lane == 0) norms[r] = sqrtf(p);
    }
}

// BIAS: rank x.c + bias[c] instead of x.c (k-means: bias = -|c|^2 / 2 turns the maximum into the L2-nearest centroid);
// the encode path instantiates BIAS = false.
template <int DIM, bool BIAS>
__global__ void __launch_bounds__(288, 1)
k_assign_tc(const __nv_bfloat16 *__restrict__ Xb, long long n, const __nv_bfloat16 *__restrict__ Cb, long long K,
            float *__restrict__ top_s /* [n][4] */, uint32_t *__restrict__ top_i /* [n][4] */,
            const float *__restrict__ bias /* [ceil(K/128)*128] or NULL */) {
    // 256 tokens per CTA = two 128-token operand tiles that share every centroid tile (halves the L2 traffic per
    // token); N = 128 centroids per tile.  warps 0-7: two consumer warpgroups (warpgroup h = token tile h, as two
    // M = 64 slabs), warp 8: loader.
    extern __shared__ __align__(1024) unsigned char smem_tc[];
    constexpr int KSTEPS = DIM / 16;       // wgmma K = 16 for fp16
    constexpr uint32_t A_BYTES = PB_TC_M * DIM * 2, B_BYTES = PB_TC_N * DIM * 2;   // per 128-row tile
    constexpr uint32_t LBO = (128 / 8) * 128, SBO = 128;
    unsigned char *As = smem_tc;                 // 2 tiles (token halves)
    unsigned char *Bs = smem_tc + 2 * A_BYTES;   // PB_TC_STAGES tiles
    uint64_t *bars = reinterpret_cast<uint64_t *>(Bs + PB_TC_STAGES * B_BYTES);
    uint64_t *full = bars, *empty = bars + PB_TC_STAGES, *abar = bars + 2 * PB_TC_STAGES;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long x0 = (long long)blockIdx.x * (2 * PB_TC_M);
    const long long n_tiles = (K + PB_TC_N - 1) / PB_TC_N;

    if (threadIdx.x == 0) {
        for (int i = 0; i < PB_TC_STAGES; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8);  // one arrival per consumer warp
        }
        mbar_init(abar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (w == 8) {
        // ---------------- loader: one elected lane, one bulk copy per token tile and per centroid tile ----------------
        if (lane == 0) {
            // A tiles: this CTA's two 128-token tiles (the fp16 array is stored in tile order)
            mbar_expect_tx(abar, 2 * A_BYTES);
            bulk_g2s(As, reinterpret_cast<const unsigned char *>(Xb) + (size_t)(2 * blockIdx.x) * A_BYTES, A_BYTES, abar);
            bulk_g2s(As + A_BYTES, reinterpret_cast<const unsigned char *>(Xb) + (size_t)(2 * blockIdx.x + 1) * A_BYTES, A_BYTES, abar);
            for (long long t = 0; t < n_tiles; ++t) {
                const int st = (int)(t % PB_TC_STAGES);
                mbar_wait(&empty[st], (uint32_t)(((t / PB_TC_STAGES) & 1) ^ 1));
                mbar_expect_tx(&full[st], B_BYTES);
                bulk_g2s(Bs + (size_t)st * B_BYTES, reinterpret_cast<const unsigned char *>(Cb) + (size_t)t * B_BYTES, B_BYTES,
                         &full[st]);
            }
        }
    } else {
        // ---------------- consumers: MMA, then a running top-4 per token row ----------------
        // thread row (slab p, half h) = token 64 p + 16 (w%4) + lane/4 + 8 h of the warpgroup's tile; its 32 columns of
        // a centroid tile are 8 i + 2 (lane%4) + j, visited in ascending order, so strict '>' keeps the lowest index
        // among equal scores exactly as a scan over all columns would; the quad's four lists are merged at the end.
        const int half = w >> 2;
        float s[4][4];
        uint32_t ix[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s[r][k] = -INFINITY;
                ix[r][k] = 0xffffffffu;
            }
        float d[PB_TC_N / 2];
#pragma unroll
        for (int i = 0; i < PB_TC_N / 2; ++i) d[i] = 0.0f;
        mbar_wait(abar, 0);  // token tiles landed
        for (long long t = 0; t < n_tiles; ++t) {
            const int st = (int)(t % PB_TC_STAGES);
            mbar_wait(&full[st], (uint32_t)((t / PB_TC_STAGES) & 1));
            const long long c0 = t * PB_TC_N;
            const bool edge = c0 + PB_TC_N > K;  // the (zero-filled) columns past K must not be ranked
            const uint32_t b0 = smem_u32(Bs + (size_t)st * B_BYTES);
#pragma unroll
            for (int p = 0; p < 2; ++p) {
                const uint32_t a0 = smem_u32(As + half * A_BYTES) + p * 1024;  // 64 rows = 8 row groups of 128 B
                wg_fence();
#pragma unroll
                for (int k = 0; k < KSTEPS; ++k)
                    wg_mma_f16<PB_TC_N>(d, wg_desc(a0 + k * 2 * LBO, LBO, SBO), wg_desc(b0 + k * 2 * LBO, LBO, SBO), k > 0 ? 1u : 0u);
                wg_commit();
                wg_wait_all(d);
                if (p == 1) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[st]);  // B tile consumed
                }
                if (BIAS) {  // bias of column 8 i + 2 (lane%4) + j
#pragma unroll
                    for (int i = 0; i < PB_TC_N / 8; ++i) {
                        const float2 bb = __ldg(reinterpret_cast<const float2 *>(bias + c0 + 8 * i + 2 * (lane & 3)));
                        d[4 * i] += bb.x;
                        d[4 * i + 1] += bb.y;
                        d[4 * i + 2] += bb.x;
                        d[4 * i + 3] += bb.y;
                    }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = 2 * p + h;
                    float s0 = s[r][0], s1 = s[r][1], s2 = s[r][2], s3 = s[r][3];
                    uint32_t i0 = ix[r][0], i1 = ix[r][1], i2 = ix[r][2], i3 = ix[r][3];
                    // one max tree per row; the insertion path runs only when the tile can matter
                    float m = d[2 * h];
#pragma unroll
                    for (int i = 0; i < PB_TC_N / 8; ++i) m = fmaxf(m, fmaxf(d[4 * i + 2 * h], d[4 * i + 2 * h + 1]));
                    if (m > s3 || edge) {
#pragma unroll
                        for (int i = 0; i < PB_TC_N / 8; ++i)
#pragma unroll
                            for (int j = 0; j < 2; ++j) {
                                const float v = d[4 * i + 2 * h + j];
                                const uint32_t c = (uint32_t)(c0 + 8 * i + 2 * (lane & 3) + j);
                                if (v > s3 && c < (uint32_t)K) {  // NaN never enters
                                    if (v > s0) { s3 = s2; i3 = i2; s2 = s1; i2 = i1; s1 = s0; i1 = i0; s0 = v; i0 = c; }
                                    else if (v > s1) { s3 = s2; i3 = i2; s2 = s1; i2 = i1; s1 = v; i1 = c; }
                                    else if (v > s2) { s3 = s2; i3 = i2; s2 = v; i2 = c; }
                                    else { s3 = v; i3 = c; }
                                }
                            }
                    }
                    s[r][0] = s0; s[r][1] = s1; s[r][2] = s2; s[r][3] = s3;
                    ix[r][0] = i0; ix[r][1] = i1; ix[r][2] = i2; ix[r][3] = i3;
                }
            }
        }
        // merge the quad's lists: order (score descending, index ascending), the order the scan above produces
#pragma unroll
        for (int r = 0; r < 4; ++r) {
#pragma unroll
            for (int mask = 1; mask <= 2; mask <<= 1) {
                float os[4];
                uint32_t oi[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    os[k] = __shfl_xor_sync(PB_FULL, s[r][k], mask);
                    oi[k] = __shfl_xor_sync(PB_FULL, ix[r][k], mask);
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float v = os[k];
                    const uint32_t c = oi[k];
                    auto before = [&](float a, uint32_t ia) { return v > a || (v == a && c < ia); };
                    if (c == 0xffffffffu || !before(s[r][3], ix[r][3])) continue;  // empty slot, or not in the top 4
                    if (before(s[r][0], ix[r][0])) {
                        s[r][3] = s[r][2]; ix[r][3] = ix[r][2]; s[r][2] = s[r][1]; ix[r][2] = ix[r][1];
                        s[r][1] = s[r][0]; ix[r][1] = ix[r][0]; s[r][0] = v; ix[r][0] = c;
                    } else if (before(s[r][1], ix[r][1])) {
                        s[r][3] = s[r][2]; ix[r][3] = ix[r][2]; s[r][2] = s[r][1]; ix[r][2] = ix[r][1]; s[r][1] = v; ix[r][1] = c;
                    } else if (before(s[r][2], ix[r][2])) {
                        s[r][3] = s[r][2]; ix[r][3] = ix[r][2]; s[r][2] = v; ix[r][2] = c;
                    } else {
                        s[r][3] = v; ix[r][3] = c;
                    }
                }
            }
            const long long tok = x0 + half * PB_TC_M + 64 * (r >> 1) + 16 * (w & 3) + (lane >> 2) + 8 * (r & 1);
            if ((lane & 3) == 0 && tok < n) {
                reinterpret_cast<float4 *>(top_s)[tok] = make_float4(s[r][0], s[r][1], s[r][2], s[r][3]);
                reinterpret_cast<uint4 *>(top_i)[tok] = make_uint4(ix[r][0], ix[r][1], ix[r][2], ix[r][3]);
            }
        }
    }
}

// certification + exact re-scoring of the shortlist; uncertified tokens are flagged for k_assign
__global__ void k_assign_certify(const float *__restrict__ X, long long n, int dim, const float *__restrict__ C,
                                 const float *__restrict__ xnorm, float cmax, int c_finite,
                                 const float *__restrict__ top_s, const uint32_t *__restrict__ top_i,
                                 long long *__restrict__ codes, int *__restrict__ n_fallback,
                                 long long *__restrict__ fallback_list) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const float4 s = reinterpret_cast<const float4 *>(top_s)[t];
        const uint4 id = reinterpret_cast<const uint4 *>(top_i)[t];
        const float xn = xnorm[t];
        // (2^-10 + 2^-22) |x| max|c| (fp16 unit roundoff 2^-11, twice) + subnormal spacing + accumulation slack
        const float eps = 0.00097680f * xn * cmax + 5.9604645e-8f * sqrtf((float)dim) * (xn + cmax) + 1e-5f;
        // certified iff everything is finite, four candidates exist and the 4th is out of the band
        bool ok = c_finite && xn < 1e18f && (s.x > -1e30f) && (s.x < 1e30f) && id.w != 0xffffffffu && (s.w < s.x - 2.0f * eps);
        if (ok) {
            const float sv[3] = {s.x, s.y, s.z};
            const uint32_t iv[3] = {id.x, id.y, id.z};
            u64 best = 0ull;
            for (int j = 0; j < 3; ++j) {
                if (sv[j] < s.x - 2.0f * eps) continue;  // cannot be the argmax
                const float *c = C + (size_t)iv[j] * dim;
                const float *x = X + (size_t)t * dim;
                float acc = 0.0f;
                for (int d = 0; d < dim; ++d) acc = __fmaf_rn(x[d], c[d], acc);  // pinned order
                const u64 key = ((u64)score_key_asc(acc) << 32) | iv[j];
                best = key >= best ? key : best;
            }
            codes[t] = (long long)(uint32_t)best;
        } else {
            const int slot = atomicAdd(n_fallback, 1);
            fallback_list[slot] = t;
        }
    }
}

__global__ void k_gather_rows_i64(const float *__restrict__ X, const long long *__restrict__ idx, long long m, int dim,
                                  float *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m * dim; i += (long long)gridDim.x * blockDim.x)
        out[i] = X[(size_t)idx[i / dim] * dim + (i % dim)];
}
__global__ void k_scatter_codes(const long long *__restrict__ src, const long long *__restrict__ idx, long long m,
                                long long *__restrict__ dst) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x)
        dst[idx[i]] = src[i];
}

// ------------------------------------------------------------------------------------------
// Inverted file from the codes (index.rs:850-873: code -> sorted unique doc ids).  The per-doc distinct code lists
// (ucodes, built by k_unique_codes for a5) already hold the (doc, code) relation; k_ivf_pairs emits one 64-bit key
// (code << 32 | doc) per distinct pair -- entries equal to their predecessor are the padding -- a radix sort on
// the keys orders them by centroid, then doc id; duplicates (docs longer than PB_UCODE_MAX keep a raw code list) are
// dropped by a unique pass.  Offsets = one lower_bound per centroid.
// ------------------------------------------------------------------------------------------
__global__ void k_ivf_pairs(const uint32_t *__restrict__ ucodes, const long long *__restrict__ udoc_off, long long D,
                            u64 *__restrict__ keys, unsigned long long *__restrict__ n_keys) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long d = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); d < D; d += nw) {
        const long long t0 = udoc_off[d], t1 = udoc_off[d + 1];
        for (long long t = t0; t < t1; t += 32) {
            const long long i = t + lane;
            const bool real = i < t1 && (i == t0 || ucodes[i] != ucodes[i - 1]);
            const unsigned bal = __ballot_sync(PB_FULL, real);
            unsigned long long base = 0;
            if (lane == 0 && bal) base = atomicAdd(n_keys, (unsigned long long)__popc(bal));
            base = shfl_u64(base, 0);
            if (real) keys[base + __popc(bal & ((1u << lane) - 1u))] = ((u64)ucodes[i] << 32) | (uint32_t)d;
        }
    }
}

__global__ void k_ivf_from_keys(const u64 *__restrict__ keys, long long n, uint32_t *__restrict__ ivf) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        ivf[i] = (uint32_t)keys[i];
}

// ivf_off[c] = first position whose key has centroid >= c (c = 0..K)
__global__ void k_ivf_offsets(const u64 *__restrict__ keys, long long n, long long K, long long *__restrict__ ivf_off) {
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c <= K; c += (long long)gridDim.x * blockDim.x) {
        const u64 want = (u64)c << 32;
        long long lo = 0, hi = n;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (keys[mid] < want) lo = mid + 1; else hi = mid;
        }
        ivf_off[c] = lo;
    }
}

// export in the reference's dtypes: ivf.npy <i8 (global doc ids), ivf_lengths.npy <i4
__global__ void k_ivf_export(const uint32_t *__restrict__ ivf, const long long *__restrict__ ivf_off, long long n, long long K,
                             long long doc_id_base, long long *__restrict__ out_ivf, int *__restrict__ out_len) {
    const long long stride = (long long)gridDim.x * blockDim.x, i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (out_ivf)
        for (long long i = i0; i < n; i += stride) out_ivf[i] = (long long)ivf[i] + doc_id_base;
    if (out_len)
        for (long long c = i0; c < K; c += stride) out_len[c] = (int)(ivf_off[c + 1] - ivf_off[c]);
}

// ------------------------------------------------------------------------------------------
// Incremental append (pb_index_append): the merged inverted file is, per centroid, sort + dedup(old list + new pids)
// (update.rs:1000-1067).  The new docs' ids exceed every old id and both parts are ascending and unique, so that is the
// old list followed by the centroid's sorted new pairs.  add_before[c] = number of new pairs whose centroid is < c (the
// lower bound of c << 32 in the sorted new keys, k_ivf_offsets).  Out of place, into the spare half of the ping-pong:
// old entry j of centroid c goes to old_off[c] + add_before[c] + j, one warp per centroid (coalesced on both sides);
// new_off[c] = old_off[c] + add_before[c] for c = 0..K.
// ------------------------------------------------------------------------------------------
__global__ void k_ivf_merge_old(const uint32_t *__restrict__ ivf, const long long *__restrict__ old_off,
                                const long long *__restrict__ add_before, long long K, uint32_t *__restrict__ out,
                                long long *__restrict__ new_off) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c <= K; c += nw) {
        const long long o0 = old_off[c], dst = o0 + add_before[c];
        if (lane == 0) new_off[c] = dst;
        if (c == K) continue;
        const long long n = old_off[c + 1] - o0;
        for (long long j = lane; j < n; j += 32) out[dst + j] = ivf[o0 + j];
    }
}

// the j-th sorted new key (centroid c, doc local to the appended batch) lands right after c's old list:
// new_off[c] + old_len[c] + (j - add_before[c]) = old_off[c + 1] + j; the doc id is offset by the old D
__global__ void k_ivf_merge_new(const u64 *__restrict__ keys, long long m, const long long *__restrict__ old_off,
                                uint32_t doc_base, uint32_t *__restrict__ out) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (long long)gridDim.x * blockDim.x) {
        const u64 k = keys[j];
        out[old_off[(k >> 32) + 1] + j] = (uint32_t)k + doc_base;
    }
}

// *flag = 1 when the two arrays differ in any bit (the codec of an append must hold the index's centroids exactly)
__global__ void k_words_differ(const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, long long n, int *__restrict__ flag) {
    bool d = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        d |= a[i] != b[i];
    if (__syncthreads_or(d) && threadIdx.x == 0) *flag = 1;
}

// ------------------------------------------------------------------------------------------
// Incremental delete (pb_index_delete, delete.rs:43-273).  The deleted docs are one bit each in `bits` [ceil(D/32)];
// word_pre[w] = deleted docs in words < w (exclusive scan of the per-word popcounts).  rank(d), the number of deleted
// docs below d, is word_pre[d / 32] + the popcount of the bits below d in its word; a survivor's new id is d - rank(d)
// (delete.rs:224-226), so the survivors keep their order.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ bool del_bit(const uint32_t *__restrict__ bits, uint32_t d) { return (bits[d >> 5] >> (d & 31)) & 1u; }
__device__ __forceinline__ long long del_rank(const uint32_t *__restrict__ bits, const long long *__restrict__ word_pre, uint32_t d) {
    return word_pre[d >> 5] + __popc(bits[d >> 5] & ((1u << (d & 31)) - 1u));
}

// ids are global (doc_id_base + local); negative, out-of-range and repeated ids set no new bit
__global__ void k_del_mark(const long long *__restrict__ ids, long long n, long long base, long long D, uint32_t *__restrict__ bits) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long id = ids[i];
        if (id >= base && id - base < D) {
            const long long d = id - base;
            atomicOr(&bits[d >> 5], 1u << (d & 31));
        }
    }
}

// cnt[w] = deleted docs in word w (w < nw), cnt[nw] = 0: scanned into word_pre[0..nw], word_pre[nw] = all deleted docs
__global__ void k_del_popc(const uint32_t *__restrict__ bits, long long nw, long long *__restrict__ cnt) {
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w <= nw; w += (long long)gridDim.x * blockDim.x)
        cnt[w] = w < nw ? __popc(bits[w]) : 0;
}

// survivor j = d - rank(d): kept[j] = d and its token / distinct-code counts, scanned into the new doc_off / udoc_off
__global__ void k_del_kept(const uint32_t *__restrict__ bits, const long long *__restrict__ word_pre, long long D,
                           const long long *__restrict__ doc_off, const long long *__restrict__ udoc_off,
                           long long *__restrict__ kept, long long *__restrict__ tlen, long long *__restrict__ ulen) {
    for (long long d = (long long)blockIdx.x * blockDim.x + threadIdx.x; d < D; d += (long long)gridDim.x * blockDim.x) {
        if (del_bit(bits, (uint32_t)d)) continue;
        const long long j = d - del_rank(bits, word_pre, (uint32_t)d);
        kept[j] = d;
        tlen[j] = doc_off[d + 1] - doc_off[d];
        ulen[j] = udoc_off[d + 1] - udoc_off[d];
    }
}

// Inverted file, delete.rs:196-237: each centroid's list without the deleted ids, survivors renumbered.  One warp per
// centroid; cnt[c] = its survivors (cnt[K] = 0), scanned into the new offsets.
__global__ void k_ivf_delete_count(const uint32_t *__restrict__ ivf, const long long *__restrict__ off, long long K,
                                   const uint32_t *__restrict__ bits, long long *__restrict__ cnt) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c <= K; c += nw) {
        if (c == K) {
            if (lane == 0) cnt[K] = 0;
            continue;
        }
        const long long o0 = off[c], n = off[c + 1] - o0;
        long long kept = 0;
        for (long long b = 0; b < n; b += 32) {
            const long long i = b + lane;
            kept += __popc(__ballot_sync(PB_FULL, i < n && !del_bit(bits, ivf[o0 + i])));
        }
        if (lane == 0) cnt[c] = kept;
    }
}

// the survivors of centroid c, in order, at new_off[c]..: compacted with a ballot, written as id - rank(id)
__global__ void k_ivf_delete_write(const uint32_t *__restrict__ ivf, const long long *__restrict__ off, long long K,
                                   const uint32_t *__restrict__ bits, const long long *__restrict__ word_pre,
                                   const long long *__restrict__ new_off, uint32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < K; c += nw) {
        const long long o0 = off[c], n = off[c + 1] - o0;
        long long dst = new_off[c];
        for (long long b = 0; b < n; b += 32) {
            const long long i = b + lane;
            const uint32_t id = i < n ? ivf[o0 + i] : 0u;
            const bool keep = i < n && !del_bit(bits, id);
            const unsigned bal = __ballot_sync(PB_FULL, keep);
            if (keep) out[dst + __popc(bal & ((1u << lane) - 1u))] = id - (uint32_t)del_rank(bits, word_pre, id);
            dst += __popc(bal);
        }
    }
}

// ------------------------------------------------------------------------------------------
// The inverted file of a doc range [b, e) of a directory (pb_index_load_range): each list of ivf.npy filtered to the
// range, in file order, ids minus b.  The file (i64, global ids) arrives in slabs: slab holds its entries [s0, s0 + m),
// off [K + 1] are the file's list offsets, and the centroids c0 <= c < c1 are those whose list overlaps the slab (a list
// may straddle slabs).  One warp per centroid; slabs go in order on one stream, so cnt[c] / cur[c] need no atomics.
// Every entry outside [0, limit) sets *bad.  With a deleted set (bits, word_pre over the directory's docs, b = 0) its
// ids leave the lists too and a survivor is written as id - rank(id): delete.rs:196-237 on the file.  bits = nullptr
// is the plain range.
// ------------------------------------------------------------------------------------------
__global__ void k_ivf_range_count(const long long *__restrict__ slab, long long s0, long long m,
                                  const long long *__restrict__ off, long long c0, long long c1, long long limit,
                                  long long b, long long e, const uint32_t *__restrict__ bits,
                                  long long *__restrict__ cnt, int *__restrict__ bad) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    bool oob = false;
    for (long long c = c0 + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < c1; c += nw) {
        const long long i0 = max(off[c], s0) - s0, i1 = min(off[c + 1], s0 + m) - s0;
        long long kept = 0;
        for (long long i = i0 + lane; i - lane < i1; i += 32) {
            const long long id = i < i1 ? slab[i] : -1;
            oob |= i < i1 && (id < 0 || id >= limit);
            kept += __popc(__ballot_sync(PB_FULL, id >= b && id < e && !(bits && del_bit(bits, (uint32_t)id))));
        }
        if (lane == 0) cnt[c] += kept;
    }
    if (oob) *bad = 1;
}

// the kept entries of the slab's part of list c at cur[c].., compacted with a ballot, as id - b; cur[c] advances
__global__ void k_ivf_range_write(const long long *__restrict__ slab, long long s0, long long m,
                                  const long long *__restrict__ off, long long c0, long long c1, long long b,
                                  long long e, const uint32_t *__restrict__ bits, const long long *__restrict__ word_pre,
                                  long long *__restrict__ cur, uint32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = c0 + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < c1; c += nw) {
        const long long i0 = max(off[c], s0) - s0, i1 = min(off[c + 1], s0 + m) - s0;
        long long dst = cur[c];
        for (long long i = i0 + lane; i - lane < i1; i += 32) {
            const long long id = i < i1 ? slab[i] : -1;
            const bool keep = id >= b && id < e && !(bits && del_bit(bits, (uint32_t)id));
            const unsigned bal = __ballot_sync(PB_FULL, keep);
            if (keep)
                out[dst + __popc(bal & ((1u << lane) - 1u))] =
                    (uint32_t)(id - b - (bits ? del_rank(bits, word_pre, (uint32_t)id) : 0));
            dst += __popc(bal);
        }
        if (lane == 0) cur[c] = dst;
    }
}

// In-place compaction of a per-token (or per-distinct-code) array, one window of survivors [j0, j1) at a time: survivor
// j's rows old_off[kept[j]] .. old_off[kept[j] + 1] go to staging at new_off[j] - new_off[j0], and the caller then
// copies the staging to new_off[j0].  One warp per doc, V-wide accesses (row_bytes * every offset is a multiple of
// sizeof(V)).
// Invariant: new_off[j] <= old_off[kept[j]] for every j (a survivor only moves down), so a window's writes end at
// new_off[j1] <= old_off[kept[j1]], where the next window's reads begin: windows in ascending order never read rows an
// earlier window overwrote, and the staging is never more than one window.
template <class V>
__global__ void k_compact_gather(const uint8_t *__restrict__ src, const long long *__restrict__ old_off,
                                 const long long *__restrict__ kept, const long long *__restrict__ new_off, long long j0,
                                 long long j1, int row_bytes, uint8_t *__restrict__ stage) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    const long long s0 = new_off[j0];
    for (long long j = j0 + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < j1; j += nw) {
        const long long d = kept[j], o = old_off[d];
        const long long nv = (old_off[d + 1] - o) * row_bytes / (long long)sizeof(V);
        const V *in = reinterpret_cast<const V *>(src + o * row_bytes);
        V *out = reinterpret_cast<V *>(stage + (new_off[j] - s0) * row_bytes);
        for (long long k = lane; k < nv; k += 32) out[k] = in[k];
    }
}

// ------------------------------------------------------------------------------------------
// Rebalance of a doc-sharded deployment (pb_index_rebalance_sharded).  A sender's local ids [0, D) split into W
// destination pieces by the bounds q [W + 1] (q[0] = 0, q[W] = D, non-decreasing; piece r = ids [q[r], q[r + 1])).
// Each list is partitioned stably: per 32 entries the lanes bound for one piece form a __match_any_sync group whose
// lowest lane owns that piece's counter / cursor.  cnt and cur are [W][K + 1], entry r (K + 1) + c for piece r and
// centroid c; one warp per centroid, so neither needs atomics.  cnt[r (K + 1) + K] stays 0, so one exclusive scan of
// cnt gives every piece's list offsets in one buffer, the pieces in destination order.
// ------------------------------------------------------------------------------------------
// the piece of local id `id`: the last r with q[r] <= id (empty pieces have q[r] = q[r + 1] and are skipped)
__device__ __forceinline__ int split_piece(const long long *__restrict__ q, int W, uint32_t id) {
    int lo = 0, hi = W - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (q[mid] <= (long long)id) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// cnt[r (K + 1) + c] += entries of list c bound for piece r (cnt zeroed by the caller)
__global__ void k_ivf_split_count(const uint32_t *__restrict__ ivf, const long long *__restrict__ off, long long K,
                                  const long long *__restrict__ q, int W, long long *__restrict__ cnt) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < K; c += nw) {
        const long long o0 = off[c], n = off[c + 1] - o0;
        for (long long b = 0; b < n; b += 32) {
            const long long i = b + lane;
            const int r = i < n ? split_piece(q, W, ivf[o0 + i]) : W;
            const unsigned same = __match_any_sync(PB_FULL, r);
            if (r < W && lane == __ffs(same) - 1) cnt[r * (K + 1) + c] += __popc(same);
        }
    }
}

// the entries of list c bound for piece r, in list order, at cur[r (K + 1) + c].., as id - q[r]; cur advances
__global__ void k_ivf_split_write(const uint32_t *__restrict__ ivf, const long long *__restrict__ off, long long K,
                                  const long long *__restrict__ q, int W, long long *__restrict__ cur,
                                  uint32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < K; c += nw) {
        const long long o0 = off[c], n = off[c + 1] - o0;
        for (long long b = 0; b < n; b += 32) {
            const long long i = b + lane;
            const uint32_t id = i < n ? ivf[o0 + i] : 0u;
            const int r = i < n ? split_piece(q, W, id) : W;
            const unsigned same = __match_any_sync(PB_FULL, r);
            const int leader = __ffs(same) - 1;
            long long base = 0;
            if (r < W && lane == leader) base = cur[r * (K + 1) + c];
            base = __shfl_sync(PB_FULL, base, leader);
            if (r < W) out[base + __popc(same & ((1u << lane) - 1u))] = id - (uint32_t)q[r];
            if (r < W && lane == leader) cur[r * (K + 1) + c] = base + __popc(same);
        }
    }
}

// Receiver side.  O [W][K + 1] holds each source's piece offsets as its sender scanned them (zeros for a source that
// sends nothing); source s's entries arrived at seg[segbase[s]..].  len[c] = the new length of list c (len[K] = 0), the
// sum over the sources, scanned by the caller into new_off.
__global__ void k_ivf_rebalance_count(const long long *__restrict__ O, int W, long long K, long long *__restrict__ len) {
    for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c <= K; c += (long long)gridDim.x * blockDim.x) {
        long long n = 0;
        if (c < K)
            for (int s = 0; s < W; ++s) n += O[s * (K + 1) + c + 1] - O[s * (K + 1) + c];
        len[c] = n;
    }
}

// new list c = the sources' segments of list c concatenated in source order, ids + idoff[s] (the piece's first doc in
// the receiver's range).  One warp per centroid, coalesced on both sides.
__global__ void k_ivf_rebalance_merge(const uint32_t *__restrict__ seg, const long long *__restrict__ O,
                                      const long long *__restrict__ segbase, const long long *__restrict__ idoff, int W,
                                      long long K, const long long *__restrict__ new_off, uint32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < K; c += nw) {
        long long dst = new_off[c];
        for (int s = 0; s < W; ++s) {
            const long long *o = O + s * (K + 1);
            const long long src = segbase[s] + o[c] - o[0], n = o[c + 1] - o[c];
            const uint32_t add = (uint32_t)idoff[s];
            for (long long j = lane; j < n; j += 32) out[dst + j] = seg[src + j] + add;
            dst += n;
        }
    }
}

// tlen[d] / ulen[d]: the tokens and distinct-code entries of doc d, the per-doc rows a rebalance moves with the doc
__global__ void k_doc_lengths(const long long *__restrict__ doc_off, const long long *__restrict__ udoc_off, long long D,
                              long long *__restrict__ tlen, long long *__restrict__ ulen) {
    for (long long d = (long long)blockIdx.x * blockDim.x + threadIdx.x; d < D; d += (long long)gridDim.x * blockDim.x) {
        tlen[d] = doc_off[d + 1] - doc_off[d];
        ulen[d] = udoc_off[d + 1] - udoc_off[d];
    }
}

// codec training (index.rs:240-258): L2 norm of every residual row; per-dimension mean of |residual|
__global__ void k_residual_stats(const float *__restrict__ R, long long n, int dim, float *__restrict__ norms) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += nw) {
        float p = 0.0f;
        for (int j = lane; j < dim; j += 32) {
            const float v = R[(size_t)r * dim + j];
            p = fmaf(v, v, p);
        }
        for (int m = 16; m >= 1; m >>= 1) p += __shfl_xor_sync(PB_FULL, p, m);
        if (lane == 0) norms[r] = sqrtf(p);
    }
}
__global__ void k_column_abs_mean(const float *__restrict__ R, long long n, int dim, float *__restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= dim) return;
    double acc = 0.0;  // one thread per dimension, rows in order: deterministic
    for (long long r = 0; r < n; ++r) acc += (double)fabsf(R[(size_t)r * dim + j]);
    out[j] = n > 0 ? (float)(acc / (double)n) : 0.0f;
}

// out[i] = stage[0][i] + stage[1][i] + ... in rank order (the in-process all-reduce: identical bits on every rank)
__global__ void k_sum_ranks(const float *__restrict__ stage, int world, long long count, float *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
        float acc = stage[i];
        for (int r = 1; r < world; ++r) acc += stage[(size_t)r * count + i];
        out[i] = acc;
    }
}

// k-means assignment from the tensor-core shortlist: the best (score + bias) wins, no exact re-score (the iteration is
// parity-unpinned; bf16 rounding only moves points that sit between two centroids)
__global__ void k_take_top1(const uint32_t *__restrict__ top_i, long long n, uint32_t *__restrict__ codes) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const uint32_t c = top_i[4 * t];
        codes[t] = c == 0xffffffffu ? 0u : c;
    }
}
// bias[c] = -|c|^2 / 2 for c < K, 0 for the padding columns of the last tile
__global__ void k_half_sqnorm_padded(const float *__restrict__ C, long long K, long long Kpad, int dim, float *__restrict__ bias) {
    const int lane = threadIdx.x & 31;
    const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long c = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < Kpad; c += nw) {
        float p = 0.0f;
        if (c < K)
            for (int j = lane; j < dim; j += 32) {
                const float v = C[(size_t)c * dim + j];
                p = fmaf(v, v, p);
            }
        for (int m = 16; m >= 1; m >>= 1) p += __shfl_xor_sync(PB_FULL, p, m);
        if (lane == 0) bias[c] = -0.5f * p;
    }
}
