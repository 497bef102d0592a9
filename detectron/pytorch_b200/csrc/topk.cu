// topk.cu -- batched top-k of RPN score maps (SURVEY.md 8f N1), replacing torch.topk / torch.sort in the proposal layer.
//
// Reference: lib/modeling/generate_proposals.py:118-131 -- per image and level, np.argpartition + np.argsort of the
// (H, W, A)-flattened scores on the host: "order" = indices of the pre_nms_topN best scores, best first.
// Here every (level, image) score map of a step is one PROBLEM of one batched call (<= 64 problems, k <= 16384):
//   3 histogram passes (radix select on the order-preserving key of the float: 11 + 11 + 10 bits, most significant first;
//     problem-parallel AND chunk-parallel: a CTA per 16 K scores, shared-memory histogram, one global atomic per non-empty bin;
//     from the second pass on every CTA re-derives the digits selected so far from the global histograms -- no host read, no
//     grid barrier, the stream order of the four launches is the only synchronisation),
//   1 collect + sort launch (a CTA per problem): the map is walked in (H, W, A) order; scores above the k-th key and the
//     first ties in that order are compacted into shared memory as (key << 32 | ~index) words and sorted there (bitonic,
//     descending).  The result is exactly np.argsort(-x_hwa, kind="stable")[:k]: equal scores -- also those that straddle
//     the cut -- are taken and returned in ascending (h, w, a) index.  NaN ranks below every number (numpy sorts it last),
//     NaNs among themselves by index, and -0.0 ties with +0.0 (one key each, shared by every pass).
// The maps are read where they lie, in (A, H, W) layout; the returned indices enumerate (H, W, A) like the reference's
// `scores.transpose((1, 2, 0)).reshape((-1, 1))`, so no permuted copy of the scores is made.
#include "common.cuh"
#include <string.h>

namespace b200 {

namespace {

constexpr int kTopkMaxProblems = 64;
constexpr int kTopkMaxK = 16384;
constexpr int kHistThreads = 256;
constexpr int kChunk = 16384;                 // scores per histogram CTA
constexpr int kBins = 2048;
constexpr int kSortThreads = 1024;
constexpr int kCollectUnroll = 4;              // chunks of kSortThreads scores per collect round

typedef unsigned long long u64;

struct TopkBatch {
    int count;
    const float* src[kTopkMaxProblems];       // (A, H*W) score map of the problem
    int A[kTopkMaxProblems], HW[kTopkMaxProblems], k[kTopkMaxProblems];
    int out_off[kTopkMaxProblems];            // first output slot
    int chunk_off[kTopkMaxProblems + 1];      // first histogram CTA
};

// order-preserving key; every NaN gets 0 (below -inf's 0x007fffff: the stable-argsort rank of NaN), -0.0 the key of +0.0
__device__ __forceinline__ unsigned ordered_key(float x) {
    if (x != x) return 0u;
    const unsigned b = __float_as_uint(x == 0.f ? 0.f : x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
template <int PASS> __device__ __forceinline__ unsigned digit_of(unsigned key) {
    return PASS == 0 ? (key >> 21) : PASS == 1 ? ((key >> 10) & 2047u) : (key & 1023u);
}

// Largest bin b with count(bins > b) < need <= count(bins >= b); need_out = need - count(bins > b).  All threads of the CTA
// call it (blockDim.x == T); s_scan: T ints of shared memory.  hist: kBins global ints (complete: written by earlier launches).
template <int T>
__device__ __forceinline__ void select_bin(const int* __restrict__ hist, int need, int* s_scan, int* s_res, int& bin, int& need_out) {
    constexpr int PER = kBins / T;
    const int t = threadIdx.x;
    int v[PER], sum = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) { v[j] = __ldcg(hist + (kBins - 1 - (t * PER + j))); sum += v[j]; }     // descending bins
    s_scan[t] = sum;
    __syncthreads();
    if (t < 32) {                                              // exclusive scan of T sums by one warp
        constexpr int W = T / 32;
        int loc[W], tot = 0;
#pragma unroll
        for (int j = 0; j < W; ++j) { loc[j] = s_scan[t * W + j]; tot += loc[j]; }
        int inc = tot;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(0xffffffffu, inc, d); if (t >= d) inc += u; }
        int run = inc - tot;
#pragma unroll
        for (int j = 0; j < W; ++j) { s_scan[t * W + j] = run; run += loc[j]; }
    }
    __syncthreads();
    int above = s_scan[t];                                     // count of the bins above this thread's first bin
    if (above < need && need <= above + sum) {                 // the crossing lies in this thread's bins (exactly one thread)
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            if (need <= above + v[j]) { s_res[0] = kBins - 1 - (t * PER + j); s_res[1] = need - above; break; }
            above += v[j];
        }
    }
    __syncthreads();
    bin = s_res[0]; need_out = s_res[1];
    __syncthreads();
}

template <int PASS>
__global__ void __launch_bounds__(kHistThreads)
topk_hist_kernel(const __grid_constant__ TopkBatch tb, int* __restrict__ hist) {
    __shared__ int s_hist[kBins];
    __shared__ int s_scan[kHistThreads];
    __shared__ int s_res[2];
    int p = 0;
    {
        int lo = 0, hi = tb.count - 1;
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (tb.chunk_off[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1; }
        p = lo;
    }
    const int n = tb.A[p] * tb.HW[p];
    const int c = (int)blockIdx.x - tb.chunk_off[p];
    for (int b = threadIdx.x; b < kBins; b += kHistThreads) s_hist[b] = 0;
    int b0 = 0, b1 = 0, need = tb.k[p];
    if (PASS >= 1) select_bin<kHistThreads>(hist + ((size_t)p * 3 + 0) * kBins, need, s_scan, s_res, b0, need);
    if (PASS >= 2) select_bin<kHistThreads>(hist + ((size_t)p * 3 + 1) * kBins, need, s_scan, s_res, b1, need);
    __syncthreads();
    const float* src = tb.src[p];
    const int i0 = c * kChunk, i1 = min(n, i0 + kChunk);
    for (int i = i0 + threadIdx.x; i < i1; i += kHistThreads) {
        const unsigned key = ordered_key(__ldg(src + i));
        bool in = true;
        if (PASS >= 1) in = (key >> 21) == (unsigned)b0;
        if (PASS >= 2) in = in && ((key >> 10) & 2047u) == (unsigned)b1;
        if (in) atomicAdd(&s_hist[digit_of<PASS>(key)], 1);
    }
    __syncthreads();
    int* gh = hist + ((size_t)p * 3 + PASS) * kBins;
    for (int b = threadIdx.x; b < kBins; b += kHistThreads) {
        const int v = s_hist[b];
        if (v) atomicAdd(gh + b, v);
    }
}

__global__ void __launch_bounds__(kSortThreads)
topk_collect_sort_kernel(const __grid_constant__ TopkBatch tb, const int* __restrict__ hist, long long* __restrict__ order_out,
                         float* __restrict__ scores_out) {
    extern __shared__ u64 s_items[];                           // [m2] composite words
    __shared__ int s_scan[kSortThreads];
    __shared__ int s_res[2];
    __shared__ int s_warp[32];
    __shared__ int s_count, s_ties;
    const int p = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int A = tb.A[p], HW = tb.HW[p], n = A * HW, k = tb.k[p];
    if (k <= 0) return;
    int b0, b1, b2, need = k;
    select_bin<kSortThreads>(hist + ((size_t)p * 3 + 0) * kBins, need, s_scan, s_res, b0, need);
    select_bin<kSortThreads>(hist + ((size_t)p * 3 + 1) * kBins, need, s_scan, s_res, b1, need);
    select_bin<kSortThreads>(hist + ((size_t)p * 3 + 2) * kBins, need, s_scan, s_res, b2, need);
    const unsigned T = ((unsigned)b0 << 21) | ((unsigned)b1 << 10) | (unsigned)b2;       // the k-th largest key
    const int ties_wanted = need;                              // how many scores equal to T belong to the top k
    int m2 = 1;
    while (m2 < k) m2 <<= 1;
    for (int i = t; i < m2; i += kSortThreads) s_items[i] = 0ull;                         // padding sorts to the end
    if (t == 0) { s_count = 0; s_ties = 0; }
    __syncthreads();
    const float* src = tb.src[p];
    for (int base = 0; base < n; base += kSortThreads * kCollectUnroll) {
        unsigned keys[kCollectUnroll];
#pragma unroll
        for (int j = 0; j < kCollectUnroll; ++j) {             // every load of the round first: several in flight per thread
            const int e = base + j * kSortThreads + t;         // index in (H, W, A) enumeration
            keys[j] = 0u;
            if (e < n) {
                const int cell = e / A, a = e - cell * A;
                keys[j] = ordered_key(__ldg(src + (size_t)a * HW + cell));
            }
        }
#pragma unroll
        for (int j = 0; j < kCollectUnroll; ++j) {
            const int e = base + j * kSortThreads + t;
            const unsigned key = keys[j];
            const bool gt = e < n && key > T, eq = e < n && key == T;
            // ties are admitted in (H, W, A) order: rank of this tie among all ties seen so far.  The block-wide rank is only
            // worked out for a chunk that holds one
            bool take = gt;
            if (__syncthreads_or(eq ? 1 : 0)) {
                const unsigned em = __ballot_sync(0xffffffffu, eq);
                if (lane == 0) s_warp[warp] = __popc(em);
                __syncthreads();
                int rank = s_ties + __popc(em & ((1u << lane) - 1u));
                for (int w = 0; w < warp; ++w) rank += s_warp[w];
                take = gt || (eq && rank < ties_wanted);
                __syncthreads();
                if (t == 0) { int tot = 0; for (int w = 0; w < 32; ++w) tot += s_warp[w]; s_ties += tot; }
            }
            if (take) {
                const int pos = atomicAdd(&s_count, 1);
                if (pos < m2) s_items[pos] = ((u64)key << 32) | (u64)(0xffffffffu - (unsigned)e);
            }
        }
    }
    __syncthreads();
    // bitonic sort, descending
    for (int size = 2; size <= m2; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = t; i < (m2 >> 1); i += kSortThreads) {
                const int lo = 2 * i - (i & (stride - 1));                                // index of the lower element of the pair
                const int hi = lo + stride;
                const bool desc = ((lo & size) == 0);
                const u64 x = s_items[lo], y = s_items[hi];
                if ((x < y) == desc) { s_items[lo] = y; s_items[hi] = x; }
            }
            __syncthreads();
        }
    }
    const int off = tb.out_off[p];
    for (int i = t; i < k; i += kSortThreads) {
        const u64 w = s_items[i];
        order_out[off + i] = (long long)(0xffffffffu - (unsigned)(w & 0xffffffffull));
        scores_out[off + i] = key_to_float((unsigned)(w >> 32));
    }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_topk_batched_workspace_bytes(int num_problems) {
    if (num_problems < 1 || num_problems > kTopkMaxProblems) return 0;
    return (size_t)num_problems * 3 * kBins * sizeof(int);
}

// returns B200_ROI_EWORKSPACE when the batch does not fit the kernel's limits (caller falls back)
int b200_topk_batched(const float* const* scores_dev_ptrs_host, const int* A_host, const int* HW_host, const int* k_host, int num_problems,
                      long long* order_out, float* scores_out, void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    if (num_problems < 1 || !scores_dev_ptrs_host || !A_host || !HW_host || !k_host) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num_problems && p < 64; ++p) {
        if (!scores_dev_ptrs_host[p] || k_host[p] < 0) return B200_ROI_EINVAL;
        total += k_host[p];
    }
    if (total > 0 && (!order_out || !scores_out)) return B200_ROI_EINVAL;
    if (num_problems > kTopkMaxProblems) return B200_ROI_EWORKSPACE;
    if (workspace == nullptr || workspace_bytes < b200_topk_batched_workspace_bytes(num_problems)) return B200_ROI_EWORKSPACE;
    TopkBatch tb;
    memset(&tb, 0, sizeof(tb));
    tb.count = num_problems;
    int off = 0, chunks = 0, kmax = 0;
    for (int p = 0; p < num_problems; ++p) {
        const long long n = (long long)A_host[p] * HW_host[p];
        if (A_host[p] < 1 || HW_host[p] < 1 || n >= (1LL << 30) || k_host[p] < 0 || k_host[p] > n || k_host[p] > kTopkMaxK)
            return B200_ROI_EWORKSPACE;
        tb.src[p] = scores_dev_ptrs_host[p]; tb.A[p] = A_host[p]; tb.HW[p] = HW_host[p]; tb.k[p] = k_host[p];
        tb.out_off[p] = off; off += k_host[p];
        tb.chunk_off[p] = chunks; chunks += (int)((n + kChunk - 1) / kChunk);
        if (k_host[p] > kmax) kmax = k_host[p];
    }
    for (int p = num_problems; p <= kTopkMaxProblems; ++p) tb.chunk_off[p] = chunks;
    if (kmax == 0) return B200_ROI_OK;
    int* hist = (int*)workspace;
    cudaError_t err = cudaMemsetAsync(hist, 0, b200_topk_batched_workspace_bytes(num_problems), stream);
    if (err != cudaSuccess) return (int)err;
    topk_hist_kernel<0><<<chunks, kHistThreads, 0, stream>>>(tb, hist);
    topk_hist_kernel<1><<<chunks, kHistThreads, 0, stream>>>(tb, hist);
    topk_hist_kernel<2><<<chunks, kHistThreads, 0, stream>>>(tb, hist);
    int m2 = 1;
    while (m2 < kmax) m2 <<= 1;
    const size_t smem = (size_t)m2 * sizeof(u64);
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return B200_ROI_EWORKSPACE;
    if (const int rc = smem_opt_in(topk_collect_sort_kernel, kTopkMaxK * sizeof(u64))) return rc;
    topk_collect_sort_kernel<<<num_problems, kSortThreads, smem, stream>>>(tb, hist, order_out, scores_out);
    return finish_launch(4);
}

}  // extern "C"
