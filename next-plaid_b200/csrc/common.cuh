// common.cuh -- shared device helpers for libplaid_b200 (sm_90a).
//
// Numerics contract (DESIGN.md "Numerics"): every floating-point operation that feeds a ranking
// decision is written with explicit round-to-nearest intrinsics so nvcc can neither fuse nor
// reorder it, and follows the pinned order oracle/plaid_oracle.c documents:
//     dot(a,b)   = acc=+0; for j ascending: acc = fma(a[j], b[j], acc)
//     sumsq(row) = per-lane fma chains over the lane's float4 groups (group g -> lane g%32),
//                  combined by the xor butterfly 16,8,4,2,1
// so results are bit-identical to the CPU restatement of the reference.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define PB_DEV __device__ __forceinline__
#define PB_FULL 0xffffffffu

typedef unsigned long long u64;

// Score order of search.rs:110-133 as an unsigned key: finite values in f32::total_cmp order,
// every non-finite value (NaN, +-Inf) below all finite ones and equal to each other (key 0).
PB_DEV uint32_t score_key_asc(float x) {
    uint32_t b = __float_as_uint(x);
    uint32_t k = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ((b & 0x7f800000u) != 0x7f800000u) ? k : 0u;
}
// inverse for finite keys (key != 0)
PB_DEV float key_to_score(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

// A row array addressed by byte.  FlatRows: one allocation.  SegRows: the pinned host segments of a host-tier handle
// (DESIGN.md 4r), 2^shift bytes each, read over the mapping through the device's segment table: byte b is at
// seg[b >> shift] + (b & (2^shift - 1)).  The segment size is a multiple of 16 and a load unit of V (2, 4 or 16 bytes)
// sits at a multiple of sizeof(V) from the array start, so no unit straddles two segments.
struct FlatRows {
    const uint8_t *p;
    template <class V> PB_DEV const V *at(long long b) const { return reinterpret_cast<const V *>(p + b); }
};
struct SegRows {
    const uint8_t *const *seg;
    int shift;
    template <class V> PB_DEV const V *at(long long b) const {
        return reinterpret_cast<const V *>(seg[b >> shift] + (b & ((1ll << shift) - 1)));
    }
};

PB_DEV u64 shfl_u64(u64 v, int src) {
    uint32_t lo = __shfl_sync(PB_FULL, (uint32_t)v, src);
    uint32_t hi = __shfl_sync(PB_FULL, (uint32_t)(v >> 32), src);
    return ((u64)hi << 32) | lo;
}
PB_DEV u64 shfl_xor_u64(u64 v, int m) {
    uint32_t lo = __shfl_xor_sync(PB_FULL, (uint32_t)v, m);
    uint32_t hi = __shfl_xor_sync(PB_FULL, (uint32_t)(v >> 32), m);
    return ((u64)hi << 32) | lo;
}
PB_DEV u64 warp_max_u64(u64 v) {
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
        u64 o = shfl_xor_u64(v, m);
        v = o > v ? o : v;
    }
    return v;
}

// In-place ascending bitonic sort of n (power of two) 64-bit keys in shared memory by the whole CTA.
PB_DEV void bitonic_sort_u64(u64 *s, int n) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                int ixj = i ^ j;
                if (ixj > i) {
                    u64 a = s[i], b = s[ixj];
                    bool up = ((i & k) == 0);
                    if ((a > b) == up) {
                        s[i] = b;
                        s[ixj] = a;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// ---- shared-memory mbarriers and TMA 1-D bulk copies (k_a5_bound, k_assign_tc, k_scores16_tc, k_maxsim_tc) ----
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
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier.  Source and destination 16-byte
// aligned, bytes a multiple of 16.
PB_DEV void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

PB_DEV int next_pow2(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// Exclusive scan of one int per thread across the CTA (blockDim.x <= 1024). `tmp` needs 33 ints.
PB_DEV int block_exclusive_scan(int v, int *tmp, int *total) {
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(PB_FULL, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) tmp[w] = x;
    __syncthreads();
    if (w == 0) {
        int nw = (blockDim.x + 31) >> 5;
        int t = lane < nw ? tmp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(PB_FULL, t, o);
            if (lane >= o) t += y;
        }
        if (lane < nw) tmp[lane] = t;
        if (lane == 31) tmp[32] = t;
    }
    __syncthreads();
    int base = w > 0 ? tmp[w - 1] : 0;
    if (total) *total = tmp[32];
    int r = base + x - v;
    __syncthreads();
    return r;
}
