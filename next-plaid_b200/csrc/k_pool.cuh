// k_pool.cuh -- pool_document_embeddings (next-plaid-onnx lib.rs:1632) on the device: token 0 kept, tokens 1..n-1
// clustered by Ward's nearest-neighbour chain (hierarchy.rs:128-284), cut after the first t-k merges in chain order
// (fcluster_maxclust, hierarchy.rs:426-504) and averaged (lib.rs:2286-2314).  DESIGN.md §4p.
//
// Every operation whose rounding decides the result is written with an explicit _rn intrinsic: the library is built
// without -fmad=false, and a contracted a*b+c would round differently from the reference's separate operations.
// The one FMA is the f64 dot/norm chain: a product of two f32 values is exact in f64, so fma(a, b, s) rounds exactly as
// the reference's s + a*b does -- provided the chain runs in k order, which every thread here does.
#pragma once
#include "common.cuh"

#include <climits>

// One document of a pb_pool_embeddings call.  k == 0: returned unchanged (pass-through).  Otherwise t = n - 1 tokens
// are clustered into k clusters; ws_off / par_off locate its t*t f64 d^2 matrix and its t-int merge forest in the
// wave's workspace.
struct PoolDoc {
    long long in_off, out_off;    // first row of the document in the input / output
    long long ws_off, par_off;
    int n, k;
};

constexpr int PB_POOL_TILE = 64;     // k_pool_dist: 64 x 64 token pairs per CTA
constexpr int PB_POOL_KC = 16;       // features staged per step (divides every built dim)
constexpr int PB_POOL_MAX_T = 8192;  // clustered tokens per document: k_pool_chain keeps 24 B per token in shared memory

// err[0] bits: 1 = an input value is not finite; 2 = a nearest-neighbour chain revisited a cluster (the reference loops
// forever there); 4 = a cut did not give k clusters
__global__ void k_pool_finite(const float *__restrict__ x, long long n, int *__restrict__ err) {
    bool bad = false;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        bad |= !isfinite(x[i]);
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(err, 1);
}

// pdist_cosine (hierarchy.rs:599-653) of one 64 x 64 tile of a document's token pairs, written as d^2 (linkage_ward's
// dist_sq, hierarchy.rs:137-145) to both halves of the document's t x t matrix.  items[b] = (doc, I, J) with I <= J.
// 256 threads, each 4 x 4 pairs; the features are staged in f64 KC at a time, the row norms accumulated alongside.
template <int DIM>
__global__ void __launch_bounds__(256) k_pool_dist(const float *__restrict__ x, const PoolDoc *__restrict__ docs,
                                                   const int4 *__restrict__ items, double *__restrict__ ws) {
    static_assert(DIM % PB_POOL_KC == 0, "KC must divide DIM");
    constexpr int TL = PB_POOL_TILE, TLP = TL + 1;   // the padded stride keeps the staging stores off one bank
    __shared__ double buf[TL * TLP];   // staging (2 x KC x TLP), then the d^2 tile (TL x TLP)
    __shared__ double nrm[2][TL];
    const int4 it = items[blockIdx.x];
    const PoolDoc d = docs[it.x];
    const int t = d.n - 1;
    const float *base = x + (d.in_off + 1) * DIM;
    const int i0 = it.y * TL, j0 = it.z * TL;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    double *As = buf, *Bs = buf + PB_POOL_KC * TLP;
    double acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
    double ns = 0.0;   // threads 0..127: the norm^2 of row (tid & 63) of tile A (tid < 64) or B
    for (int k0 = 0; k0 < DIM; k0 += PB_POOL_KC) {
        for (int e = tid; e < 2 * TL * PB_POOL_KC; e += 256) {
            const int which = e / (TL * PB_POOL_KC), r = (e / PB_POOL_KC) % TL, kk = e % PB_POOL_KC;
            const int row = (which ? j0 : i0) + r;
            const float v = row < t ? base[(long long)row * DIM + k0 + kk] : 0.f;
            (which ? Bs : As)[kk * TLP + r] = (double)v;
        }
        __syncthreads();
        if (tid < 2 * TL) {
            const double *S = (tid < TL ? As : Bs) + (tid & (TL - 1));
#pragma unroll
            for (int kk = 0; kk < PB_POOL_KC; ++kk) ns = __fma_rn(S[kk * TLP], S[kk * TLP], ns);
        }
#pragma unroll
        for (int kk = 0; kk < PB_POOL_KC; ++kk) {
            double a[4], b[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) a[r] = As[kk * TLP + ty + 16 * r];
#pragma unroll
            for (int c = 0; c < 4; ++c) b[c] = Bs[kk * TLP + tx + 16 * c];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = __fma_rn(a[r], b[c], acc[r][c]);
        }
        __syncthreads();
    }
    if (tid < 2 * TL) nrm[tid / TL][tid & (TL - 1)] = __dsqrt_rn(ns);
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const double ni = nrm[0][ty + 16 * r], nj = nrm[1][tx + 16 * c];
            const double cs = (ni > 0.0 && nj > 0.0) ? __ddiv_rn(acc[r][c], __dmul_rn(ni, nj)) : 0.0;
            const double dist = fmin(fmax(__dsub_rn(1.0, cs), 0.0), 2.0);
            buf[(ty + 16 * r) * TLP + tx + 16 * c] = __dmul_rn(dist, dist);
        }
    __syncthreads();
    double *D = ws + d.ws_off;
    for (int e = tid; e < TL * TL; e += 256) {
        const int r = e / TL, c = e % TL;
        if (i0 + r < t && j0 + c < t) D[(long long)(i0 + r) * t + j0 + c] = buf[r * TLP + c];
        if (j0 + r < t && i0 + c < t) D[(long long)(j0 + r) * t + i0 + c] = buf[c * TLP + r];
    }
}

// lexicographic min of (d, p) over the warp; every lane gets it
__device__ __forceinline__ void pool_warp_argmin(double &d, int &p) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, d, o);
        const int op = __shfl_xor_sync(0xffffffffu, p, o);
        if (od < d || (od == d && op < p)) {
            d = od;
            p = op;
        }
    }
}

// find_nearest_neighbor (hierarchy.rs:263-284): the first strictly smaller d^2 in active-list order
__device__ __forceinline__ void pool_find_nn(const double *__restrict__ D, int t, int i, const int *act, int nact,
                                             int &nn, double &nd) {
    const int lane = threadIdx.x & 31;
    double best = __longlong_as_double(0x7ff0000000000000LL);   // +inf
    int bp = INT_MAX;
    const double *row = D + (long long)i * t;
    for (int p = lane; p < nact; p += 32) {
        const int j = act[p];
        if (j == i) continue;
        const double v = row[j];
        if (v < best) {
            best = v;
            bp = p;
        }
    }
    pool_warp_argmin(best, bp);
    nn = bp == INT_MAX ? -1 : act[bp];
    nd = best;
}

// linkage_ward (hierarchy.rs:128-259), one warp per document, stopped after the t - k merges the cut applies.  Slot s
// holds the cluster that contains token s: a merge of chain top a with b puts the new cluster in a's slot and retires
// b's, so the d^2 matrix is t x t (not the reference's (2t-1)^2) and the merge forest is par[b] = a.  Tie order comes
// from the active list, which keeps the reference's order (retain, then append), never from slot numbers.  The chain,
// sizes, NN cache and active list live in shared memory (24 B per token); d^2 in the wave's workspace.
__global__ void __launch_bounds__(32) k_pool_chain(const PoolDoc *__restrict__ docs, const int *__restrict__ pooled,
                                                   double *__restrict__ ws, int *__restrict__ par, int *__restrict__ err) {
    extern __shared__ double smd[];
    const PoolDoc d = docs[pooled[blockIdx.x]];
    const int t = d.n - 1, M = t - d.k, lane = threadIdx.x;
    double *D = ws + d.ws_off;
    int *P = par + d.par_off;
    double *cd = smd;                      // NN cache distance
    int *act = reinterpret_cast<int *>(cd + t), *sz = act + t, *cnn = sz + t, *chain = cnn + t;
    for (int x = lane; x < t; x += 32) {
        act[x] = x;
        sz[x] = 1;
        P[x] = x;
    }
    // the initial NN cache (hierarchy.rs:158-170): the active list is 0..t-1, so row order is active order
    for (int i = lane; i < t; i += 32) {
        const double *row = D + (long long)i * t;
        double best = __longlong_as_double(0x7ff0000000000000LL);
        int nn = -1;
        for (int j = 0; j < t; ++j) {
            const double v = j == i ? best : row[j];
            if (v < best) {
                best = v;
                nn = j;
            }
        }
        cnn[i] = nn;
        cd[i] = best;
    }
    __syncwarp();
    int nact = t, clen = 0;
    for (int m = 0; m < M; ++m) {
        if (clen == 0) {
            chain[0] = act[0];
            clen = 1;
            __syncwarp();
        }
        for (;;) {
            const int cur = chain[clen - 1];
            int nn = cnn[cur];
            double nd = cd[cur];
            if (nn < 0) {
                pool_find_nn(D, t, cur, act, nact, nn, nd);
                __syncwarp();
                if (lane == 0) {
                    cnn[cur] = nn;
                    cd[cur] = nd;
                }
            }
            if (clen >= 2 && chain[clen - 2] == nn) {
                const int a = cur, b = nn;
                const double dab = nd;
                const int na = sz[a], nb = sz[b];
                clen -= 2;
                // active_list.retain(|&x| x != a && x != b), order kept: a ballot compaction, chunk by chunk
                int w = 0;
                for (int b0 = 0; b0 < nact; b0 += 32) {
                    const int p = b0 + lane;
                    const int v = p < nact ? act[p] : -1;
                    const bool keep = p < nact && v != a && v != b;
                    const unsigned bal = __ballot_sync(0xffffffffu, keep);
                    __syncwarp();
                    if (keep) act[w + __popc(bal & ((1u << lane) - 1))] = v;
                    w += __popc(bal);
                    __syncwarp();
                }
                nact = w;
                // Ward's update for every remaining k (hierarchy.rs:225-242), a's term first, no contraction
                for (int p = lane; p < nact; p += 32) {
                    const int k = act[p];
                    const int nk = sz[k];
                    const double dak = D[(long long)a * t + k], dbk = D[(long long)b * t + k];
                    const double v = __ddiv_rn(__dsub_rn(__dadd_rn(__dmul_rn((double)(na + nk), dak),
                                                                   __dmul_rn((double)(nb + nk), dbk)),
                                                         __dmul_rn((double)nk, dab)),
                                               (double)(na + nb + nk));
                    D[(long long)a * t + k] = v;
                    D[(long long)k * t + a] = v;
                    if (cnn[k] == a || cnn[k] == b) cnn[k] = -1;
                }
                __syncwarp();
                if (lane == 0) {
                    sz[a] = na + nb;
                    act[nact] = a;
                    P[b] = a;
                }
                ++nact;
                __syncwarp();
                int nn2;
                double nd2;
                pool_find_nn(D, t, a, act, nact, nn2, nd2);
                __syncwarp();
                if (lane == 0) {
                    cnn[a] = nn2;
                    cd[a] = nd2;
                }
                __syncwarp();
                break;
            }
            // a chain longer than the active list has revisited a cluster: from there the reference never terminates
            if (clen >= nact) {
                if (lane == 0) atomicOr(err, 2);
                return;
            }
            __syncwarp();
            chain[clen++] = nn;
            __syncwarp();
        }
    }
}

// The cut and the means (fcluster_maxclust's labels, lib.rs:2286-2314), one CTA per document of the wave.  A
// pass-through document is copied; otherwise row 0 is copied and cluster c (numbered by its first token) becomes row
// 1 + c: its f32 sum in token order divided by (f32)count.  Shared memory: 4 t + 2 k ints.
template <int DIM>
__global__ void __launch_bounds__(256) k_pool_means(const float *__restrict__ x, const PoolDoc *__restrict__ docs,
                                                    int d0, const int *__restrict__ par, float *__restrict__ out,
                                                    int *__restrict__ err) {
    extern __shared__ int smi[];
    const PoolDoc d = docs[d0 + blockIdx.x];
    const float *src = x + d.in_off * DIM;
    float *dst = out + d.out_off * DIM;
    if (d.k == 0) {
        for (long long e = threadIdx.x; e < (long long)d.n * DIM; e += blockDim.x) dst[e] = src[e];
        return;
    }
    for (int e = threadIdx.x; e < DIM; e += blockDim.x) dst[e] = src[e];
    const int t = d.n - 1, k = d.k;
    const int *P = par + d.par_off;
    int *root = smi, *lab = root + t, *first = lab + t, *mem = first + t, *cnt = mem + t, *off = cnt + k;
    for (int x0 = threadIdx.x; x0 < t; x0 += blockDim.x) {
        int r = x0;
        while (P[r] != r) r = P[r];
        root[x0] = r;
        first[x0] = -1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        // labels by first token (hierarchy.rs:489-501), then the members of each label in token order
        int nl = 0;
        for (int x0 = 0; x0 < t; ++x0) {
            const int r = root[x0];
            if (first[r] < 0) {
                if (nl < k) cnt[nl] = 0;
                first[r] = nl++;
            }
            lab[x0] = first[r];
            if (lab[x0] < k) ++cnt[lab[x0]];
        }
        if (nl != k) {
            atomicOr(err, 4);
            cnt[0] = -1;
        } else {
            int s = 0;
            for (int c = 0; c < k; ++c) {
                off[c] = s;
                s += cnt[c];
            }
            for (int x0 = 0; x0 < t; ++x0) mem[off[lab[x0]]++] = x0;
            for (int c = 0; c < k; ++c) off[c] -= cnt[c];
        }
    }
    __syncthreads();
    if (cnt[0] < 0) return;
    const float *tok = src + DIM;   // the clustered tokens
    for (int e = threadIdx.x; e < k * DIM; e += blockDim.x) {
        const int c = e / DIM, f = e % DIM;
        float s = 0.f;
        for (int q = off[c]; q < off[c] + cnt[c]; ++q) s = __fadd_rn(s, tok[(long long)mem[q] * DIM + f]);
        dst[(long long)(1 + c) * DIM + f] = __fdiv_rn(s, (float)cnt[c]);
    }
}
