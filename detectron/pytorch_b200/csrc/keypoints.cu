// keypoints.cu -- test-time Keypoint R-CNN keypoint extraction (SURVEY.md 8f N3): heatmaps_to_keypoints and nms_oks,
// lib/utils/keypoints.py:103-157 and 225-266 (reference), as keypoint_results (lib/core/test.py:850-866) calls them for the
// detections of one image.
//
// Per detection d and keypoint k: w = max(x2 - x1, 1), map_w = int(max(ceil(w), min_size)) (the same for h); the M x M
// logit map is resized to map_h x map_w with cv2.resize's float32 INTER_CUBIC arithmetic on the K-channel HWC heatmap;
// the result is the first maximum in row-major order (x, y, logit) and the spatial softmax's value there,
// prob = 1 / sum(exp(map - max)).  The resized map is never written anywhere: one CTA per (d, k) recomputes it a column
// tile at a time and keeps a running max / first argmax / sum of exponentials.
//
// Resize arithmetic (cv2 imgproc resize.cpp, float32, every product and sum rounded on its own -- _rn intrinsics, no
// contraction):
//   per axis: scale = 1 / (dst / src) in double, f = float((d + .5) * scale - .5), s = floor(f), f -= s; taps s - 1 ..
//   s + 2 clamped into [0, src - 1], f kept at the borders; interpolateCubic coefficients with A = -0.75.
//   Horizontal pass ((S0 a0 + S1 a1) + S2 a2) + S3 a3.  The vertical pass runs over the flattened row of n = map_w * K
//   floats (channel fastest): its first 4 * floor(n / 4) elements come from cv2's 4-lane vector loop,
//   S0 b0 + (S1 b1 + (S2 b2 + S3 b3)), the rest from its scalar tail, ((S0 b0 + S1 b1) + S2 b2) + S3 b3.  Which one an
//   element takes depends on K, so the kernel needs the real channel count.  A map the size of the source is a copy.
//
// The coordinates follow numpy 2: corr = float32(w / map_w), x = float32(float64(x_int + .5) * float64(corr) + float64(x1)).
// The sum of exponentials is accumulated in double (numpy sums float32 pairwise); prob matches to ~1e-7 relative.
//
// OKS NMS (one CTA): score = float32 mean of the K = 17 logits, summed in numpy's pairwise order; greedy in descending
// score, equal scores the higher index first; OKS against every later candidate in float64 with the COCO sigmas and the
// float32 area (x2 - x1 + 1)(y2 - y1 + 1); a candidate is dropped when OKS > thresh.
#include "common.cuh"
#include <cub/block/block_reduce.cuh>

namespace b200 {

namespace {
constexpr int kKpThreads = 256;
constexpr int kKpTileW = 32;                            // output columns per tile: one warp lane each
constexpr int kKpRowStep = kKpThreads / kKpTileW;       // output rows in flight per tile
constexpr int kKpChunkH = 512;                          // output rows whose vertical taps are staged at once
constexpr int kKpMaxM = 64;
constexpr int kKpMaxSide = 16384;
constexpr int kOksKeypoints = 17;
constexpr int kOksMaxDets = 4096;

struct CubicTap {
    int s[4];
    float c[4];
};

// one axis of cv2's INTER_CUBIC: output index d of dst, source length src
__device__ __forceinline__ CubicTap cubic_tap(int d, int dst, int src) {
    const double scale = __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src));
    float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, .5), scale), .5));
    const float fl = floorf(f);
    const int s = (int)fl;
    f = __fsub_rn(f, fl);
    CubicTap t;
#pragma unroll
    for (int j = 0; j < 4; ++j) t.s[j] = min(max(s - 1 + j, 0), src - 1);
    constexpr float A = -0.75f;
    const float xp = __fadd_rn(f, 1.f);
    t.c[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, xp), 5.f * A), xp), 8.f * A), xp), 4.f * A);
    t.c[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, f), A + 3.f), f), f), 1.f);
    const float g = __fsub_rn(1.f, f);
    t.c[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, g), A + 3.f), g), g), 1.f);
    t.c[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.f, t.c[0]), t.c[1]), t.c[2]);
    return t;
}

// heatmap side for a box side of `len` pixels (already clamped to >= 1); non-finite or huge sides give kKpMaxSide
__device__ __forceinline__ int map_side(float len, int min_size) {
    float c = ceilf(len);
    if (min_size > 0) c = fmaxf(c, (float)min_size);
    return c < (float)kKpMaxSide ? (int)c : kKpMaxSide;
}

struct ArgMax {
    float v;
    long long i;
};
struct ArgMaxOp {        // larger value; equal values: the smaller row-major index
    __device__ ArgMax operator()(const ArgMax& a, const ArgMax& b) const { return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a; }
};

__global__ void __launch_bounds__(kKpThreads)
heatmaps_to_keypoints_kernel(const float* __restrict__ maps, const float* __restrict__ rois, int K, int M, int min_size,
                             float* __restrict__ out) {
    using ReduceMax = cub::BlockReduce<ArgMax, kKpThreads>;
    using ReduceSum = cub::BlockReduce<double, kKpThreads>;
    __shared__ float src[kKpMaxM * kKpMaxM];
    __shared__ float hs[kKpMaxM * kKpTileW];               // horizontal pass of the current column tile, all M rows
    __shared__ CubicTap ytab[kKpChunkH];
    __shared__ union { typename ReduceMax::TempStorage m; typename ReduceSum::TempStorage s; } tmp;
    __shared__ ArgMax best;
    const int d = blockIdx.x / K, k = blockIdx.x % K;
    const float* roi = rois + (size_t)d * 4;
    const float x1 = roi[0], y1 = roi[1];
    const float w = fmaxf(__fsub_rn(roi[2], x1), 1.f), h = fmaxf(__fsub_rn(roi[3], y1), 1.f);
    const int mw = map_side(w, min_size), mh = map_side(h, min_size);
    const bool copy = mw == M && mh == M;
    const float* m = maps + ((size_t)d * K + k) * M * M;
    for (int i = threadIdx.x; i < M * M; i += kKpThreads) src[i] = m[i];
    const int lane = threadIdx.x % kKpTileW, row = threadIdx.x / kKpTileW;
    const long long n_vec = ((long long)mw * K) & ~3LL;    // elements of a resized row that cv2's vector loop writes
    float vmax = -INFINITY;
    long long imax = LLONG_MAX;
    double sum = 0.0;                                      // sum of exp(v - vmax) over this thread's values
    for (int y0 = 0; y0 < mh; y0 += kKpChunkH) {
        const int ny = min(kKpChunkH, mh - y0);
        __syncthreads();
        if (!copy)
            for (int yy = threadIdx.x; yy < ny; yy += kKpThreads) ytab[yy] = cubic_tap(y0 + yy, mh, M);
        for (int x0 = 0; x0 < mw; x0 += kKpTileW) {
            const int x = x0 + lane;
            __syncthreads();
            if (x < mw) {
                if (copy) {
                    for (int r = row; r < M; r += kKpRowStep) hs[r * kKpTileW + lane] = src[r * M + x];
                } else {
                    const CubicTap t = cubic_tap(x, mw, M);
                    for (int r = row; r < M; r += kKpRowStep) {
                        const float* s = src + r * M;
                        hs[r * kKpTileW + lane] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s[t.s[0]], t.c[0]), __fmul_rn(s[t.s[1]], t.c[1])),
                                                                      __fmul_rn(s[t.s[2]], t.c[2])),
                                                            __fmul_rn(s[t.s[3]], t.c[3]));
                    }
                }
            }
            __syncthreads();
            if (x >= mw) continue;
            const bool vec = (long long)x * K + k < n_vec;
            for (int yy = row; yy < ny; yy += kKpRowStep) {
                float v;
                if (copy) {
                    v = hs[(y0 + yy) * kKpTileW + lane];
                } else {
                    const CubicTap& t = ytab[yy];
                    const float p0 = __fmul_rn(hs[t.s[0] * kKpTileW + lane], t.c[0]);
                    const float p1 = __fmul_rn(hs[t.s[1] * kKpTileW + lane], t.c[1]);
                    const float p2 = __fmul_rn(hs[t.s[2] * kKpTileW + lane], t.c[2]);
                    const float p3 = __fmul_rn(hs[t.s[3] * kKpTileW + lane], t.c[3]);
                    v = vec ? __fadd_rn(p0, __fadd_rn(p1, __fadd_rn(p2, p3))) : __fadd_rn(__fadd_rn(__fadd_rn(p0, p1), p2), p3);
                }
                const long long idx = (long long)(y0 + yy) * mw + x;
                if (v > vmax) {
                    sum = __dadd_rn(__dmul_rn(sum, exp((double)vmax - (double)v)), 1.0);
                    vmax = v;
                    imax = idx;
                } else {
                    if (v == vmax && idx < imax) imax = idx;
                    sum = __dadd_rn(sum, (double)expf(__fsub_rn(v, vmax)));
                }
            }
        }
    }
    const ArgMax b = ReduceMax(tmp.m).Reduce(ArgMax{vmax, imax}, ArgMaxOp());
    if (threadIdx.x == 0) best = b;
    __syncthreads();
    const ArgMax g = best;
    const double total = ReduceSum(tmp.s).Sum(sum > 0.0 ? __dmul_rn(sum, exp((double)vmax - (double)g.v)) : 0.0);
    if (threadIdx.x == 0) {
        const long long i = (g.i >= 0 && g.i < (long long)mw * mh) ? g.i : 0;     // no maximum: non-finite logits
        const long long xi = i % mw, yi = i / mw;
        const float cx = __fdiv_rn(w, (float)mw), cy = __fdiv_rn(h, (float)mh);
        float* o = out + (size_t)d * 4 * K + k;
        o[0] = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)xi, .5), (double)cx), (double)x1));
        o[K] = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)yi, .5), (double)cy), (double)y1));
        o[2 * K] = g.v;
        o[3 * K] = __fdiv_rn(1.f, __double2float_rn(total));
    }
}

// numpy's pairwise sum of 17 values (8 accumulators, then the rest)
template <typename T>
__device__ __forceinline__ T sum17(const T* a) {
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j] + a[8 + j];
    const T s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    return s + a[16];
}

__global__ void __launch_bounds__(kKpThreads)
nms_oks_kernel(const float* __restrict__ xy, const float* __restrict__ rois, int D, double thresh, int* __restrict__ keep,
               int* __restrict__ num_keep) {
    constexpr int K = kOksKeypoints;
    __shared__ float score[kOksMaxDets];
    __shared__ int order[kOksMaxDets];
    __shared__ unsigned char dropped[kOksMaxDets];
    __shared__ double var[K];
    __shared__ int kept;
    const double sigmas[K] = {.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89};
    if (threadIdx.x < K) {
        const double s2 = __dmul_rn(__ddiv_rn(sigmas[threadIdx.x], 10.0), 2.0);
        var[threadIdx.x] = __dmul_rn(s2, s2);
    }
    if (threadIdx.x == 0) kept = 0;
    for (int i = threadIdx.x; i < D; i += kKpThreads) {
        const float* l = xy + (size_t)i * 4 * K + 2 * K;
        float a[K];
#pragma unroll
        for (int j = 0; j < K; ++j) a[j] = l[j];
        const float s = __double2float_rn(__ddiv_rn((double)sum17(a), (double)K));
        score[i] = s == s ? s : -INFINITY;
        dropped[i] = 0;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += kKpThreads) {     // rank in descending score, equal scores the higher index first
        const float s = score[i];
        int r = 0;
        for (int j = 0; j < D; ++j) r += (score[j] > s) || (score[j] == s && j > i);
        order[r] = i;
    }
    __syncthreads();
    for (int p = 0; p < D; ++p) {
        const int i = order[p];
        if (dropped[i]) continue;                           // uniform: written before the last barrier
        if (threadIdx.x == 0) keep[kept++] = i;
        const float* a = xy + (size_t)i * 4 * K;
        const float* ra = rois + (size_t)i * 4;
        const float area = __fmul_rn(__fadd_rn(__fsub_rn(ra[2], ra[0]), 1.f), __fadd_rn(__fsub_rn(ra[3], ra[1]), 1.f));
        const double denom = __dadd_rn((double)area, 0x1p-52);                 // np.spacing(1)
        for (int q = p + 1 + threadIdx.x; q < D; q += kKpThreads) {
            const int j = order[q];
            if (dropped[j]) continue;
            const float* b = xy + (size_t)j * 4 * K;
            double e[K];
#pragma unroll
            for (int t = 0; t < K; ++t) {
                const float dx = __fsub_rn(b[t], a[t]), dy = __fsub_rn(b[K + t], a[K + t]);
                const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
                e[t] = exp(-__ddiv_rn(__ddiv_rn(__ddiv_rn((double)d2, var[t]), denom), 2.0));
            }
            if (__ddiv_rn(sum17(e), (double)K) > thresh) dropped[j] = 1;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *num_keep = kept;
}
}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_heatmaps_to_keypoints(const float* maps, const float* rois, int D, int K, int M, int min_size, float* out, b200_stream_t stream) {
    if (!(D >= 0 && K >= 1 && M >= 1 && M <= kKpMaxM && min_size <= kKpMaxSide && (long long)D * K < (1LL << 31)))
        return B200_ROI_EINVAL;
    if (D == 0) return B200_ROI_OK;
    if (!maps || !rois || !out) return B200_ROI_EINVAL;
    heatmaps_to_keypoints_kernel<<<D * K, kKpThreads, 0, stream>>>(maps, rois, K, M, min_size, out);
    return finish_launch();
}

int b200_nms_oks(const float* xy, const float* rois, int D, int K, double thresh, int* keep, int* num_keep, b200_stream_t stream) {
    if (!(D >= 0 && D <= kOksMaxDets && K == kOksKeypoints)) return B200_ROI_EINVAL;
    if (D == 0) return B200_ROI_OK;
    if (!xy || !rois || !keep || !num_keep) return B200_ROI_EINVAL;
    nms_oks_kernel<<<1, kKpThreads, 0, stream>>>(xy, rois, D, thresh, keep, num_keep);
    return finish_launch();
}

}  // extern "C"
