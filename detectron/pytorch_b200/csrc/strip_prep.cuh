// strip_prep.cuh -- the parts of the strip forwards' one-kernel prepass that do not depend on the path (roi_align_stream.cu,
// roi_align_strip.cu): the grid barrier, the CSR / cost scan every CTA keeps in shared memory, and the search of the piece
// boundaries in that scan.
//
// Both paths key their fragments by (strip column q, row y): key = colstart[q] + y, the rows of a column are consecutive keys.
// The main kernels walk the linear order (column, 32-channel group, row) and every persistent CTA takes one piece of it.
#pragma once
#include "common.cuh"

namespace b200 {
namespace prepass {

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// Every CTA of the grid arrives once on a zeroed counter and waits for the others.  The grid must be resident (sized by the
// occupancy query), else this never returns: the wait traps after seconds instead of hanging the GPU.
__device__ __forceinline__ void grid_barrier(int* counter) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1);
        unsigned spins = 0;
        while (ld_acquire_gpu(counter) < (int)gridDim.x) {
            __nanosleep(64);
            if (++spins > (1u << 24)) __trap();
        }
    }
    __syncthreads();
}

// Exclusive prefix of the fragment histogram (s_pre) and of the cost (s_cpre, every key costs row_cost on top of its
// fragments) over keys [0, keys], in this CTA's shared memory; s_pre[keys] / s_cpre[keys] are the totals.
// s_ph / s_pc: THREADS words of scratch each.  All THREADS threads of the CTA call it.
template <int THREADS>
__device__ __forceinline__ void scan_keys(const int* hist, const int* cost, unsigned row_cost, int keys, unsigned* s_pre,
                                          unsigned* s_cpre, unsigned* s_ph, unsigned* s_pc) {
    static_assert(THREADS == 128, "one warp scans THREADS / 32 = 4 chunk sums per lane");
    const int t = threadIdx.x;
    for (int k = t; k < keys; k += THREADS) {
        s_pre[k] = (unsigned)__ldcg(&hist[k]);
        s_cpre[k] = (unsigned)__ldcg(&cost[k]) + row_cost;
    }
    __syncthreads();
    const int chunk = ((keys + THREADS - 1) / THREADS) | 1;  // odd: thread-strided chunks do not collide on banks
    const int k0 = min(keys, t * chunk), k1 = min(keys, k0 + chunk);
    {
        unsigned sh = 0, sc = 0;
        for (int k = k0; k < k1; ++k) { sh += s_pre[k]; sc += s_cpre[k]; }
        s_ph[t] = sh; s_pc[t] = sc;
    }
    __syncthreads();
    if (t < 32) {                                             // exclusive scan of the chunk sums by one warp (4 per lane)
        unsigned vh[4], vc[4], th = 0, tc = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) { vh[j] = s_ph[t * 4 + j]; vc[j] = s_pc[t * 4 + j]; th += vh[j]; tc += vc[j]; }
        unsigned ih = th, ic = tc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned uh = __shfl_up_sync(0xffffffffu, ih, d), uc = __shfl_up_sync(0xffffffffu, ic, d);
            if (t >= d) { ih += uh; ic += uc; }
        }
        unsigned rh = ih - th, rc = ic - tc;
#pragma unroll
        for (int j = 0; j < 4; ++j) { s_ph[t * 4 + j] = rh; s_pc[t * 4 + j] = rc; rh += vh[j]; rc += vc[j]; }
        if (t == 31) { s_pre[keys] = rh; s_cpre[keys] = rc; }
    }
    __syncthreads();
    {
        unsigned rh = s_ph[t], rc = s_pc[t];
        for (int k = k0; k < k1; ++k) {
            const unsigned h = s_pre[k], c = s_cpre[k];
            s_pre[k] = rh; s_cpre[k] = rc;
            rh += h; rc += c;
        }
    }
    __syncthreads();
}

// First linear index (column, channel group, row) of piece p of `pieces`: where the cumulative cost over the linear order
// reaches p / pieces of the total.  s_cpre: the cost prefix of scan_keys; colstart[Q] = keys.
__device__ __forceinline__ int piece_start(int p, int pieces, int G, int keys, int Q, const int* colstart, const unsigned* s_cpre) {
    if (p == 0) return 0;
    if (p == pieces) return G * keys;
    const unsigned total = s_cpre[keys];
    const unsigned long long grand = (unsigned long long)total * (unsigned long long)G;
    const unsigned long long target = grand / (unsigned long long)pieces * (unsigned long long)p +
                                      (grand % (unsigned long long)pieces) * (unsigned long long)p / (unsigned long long)pieces;
    int lo = 0, hi = Q - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((unsigned long long)G * (unsigned long long)s_cpre[colstart[mid]] <= target) lo = mid; else hi = mid - 1;
    }
    const int kb = colstart[lo], Hq = colstart[lo + 1] - kb;
    const unsigned c0 = s_cpre[kb];
    const unsigned colsum = s_cpre[kb + Hq] - c0;             // >= row_cost * Hq > 0
    unsigned long long rem = target - (unsigned long long)G * (unsigned long long)c0;
    int gg = (int)(rem / colsum);
    if (gg > G - 1) gg = G - 1;
    rem -= (unsigned long long)gg * colsum;
    int ylo = 0, yhi = Hq - 1;
    while (ylo < yhi) {
        const int mid = (ylo + yhi + 1) >> 1;
        if ((unsigned long long)(s_cpre[kb + mid] - c0) <= rem) ylo = mid; else yhi = mid - 1;
    }
    return G * kb + gg * Hq + ylo;
}

}  // namespace prepass
}  // namespace b200
