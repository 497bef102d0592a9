// roi_pool.cu -- RoIPool forward (max + int32 argmax) and backward.
//
// Semantics: lib/model/roi_pooling/src/roi_pooling_kernel.cu (reference) ROIPoolForward :24-93,
// ROIPoolBackward :128-203.  Integer/compare work only, so both directions are bit-identical to the
// reference, including its quirks: argmax is a flat int32 index into the WHOLE bottom tensor, the
// first maximum wins, empty bins give 0 / -1, and the backward only credits a cell when it lies
// inside the rounded RoI rectangle and the bin lies in the cell's "feasible" bin range.
//
// Forward: one CTA per (RoI, channel slab); the quantised bin rectangles are computed once per CTA.
// Backward: the reference loops over ALL R RoIs for every input cell (O(N*C*H*W*R)).  Here a CTA
// owns a spatial tile x channel slab, first compacts -- in ascending RoI order, which keeps the fp32
// summation order of the reference -- the RoIs whose rectangle meets the tile, and each cell then
// visits only those.
#include "common.cuh"
#include <float.h>

namespace b200 {

constexpr int kPoolThreads = 256;
constexpr int kPoolBinMax = 1024;

struct PoolRoi {
    int batch, sw, sh, ew, eh;
    float bin_h, bin_w;
};

__device__ __forceinline__ PoolRoi pool_roi(const float* __restrict__ roi, float scale, int PH, int PW) {
    PoolRoi r;
    r.batch = (int)roi[0];
    r.sw = (int)roundf(__fmul_rn(roi[1], scale));
    r.sh = (int)roundf(__fmul_rn(roi[2], scale));
    r.ew = (int)roundf(__fmul_rn(roi[3], scale));
    r.eh = (int)roundf(__fmul_rn(roi[4], scale));
    const int rw = (int)fmaxf((float)(r.ew - r.sw + 1), 1.f);
    const int rh = (int)fmaxf((float)(r.eh - r.sh + 1), 1.f);
    r.bin_h = __fdiv_rn((float)rh, (float)PH);
    r.bin_w = __fdiv_rn((float)rw, (float)PW);
    return r;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

__global__ void __launch_bounds__(kPoolThreads)
roi_pool_forward_kernel(const float* __restrict__ bottom, const float* __restrict__ rois, float* __restrict__ top,
                        int* __restrict__ argmax, float scale, int N, int C, int H, int W, int PH, int PW, int c_per_cta) {
    __shared__ int4 rect[kPoolBinMax];   // hstart, hend, wstart, wend per bin
    const int n = blockIdx.x;
    const int c0 = blockIdx.y * c_per_cta, c1 = min(C, c0 + c_per_cta);
    const PoolRoi r = pool_roi(rois + 5 * (size_t)n, scale, PH, PW);
    const int bins = PH * PW;
    const bool use_tab = bins <= kPoolBinMax;
    auto bin_rect = [&](int b) {
        const int ph = b / PW, pw = b % PW;
        int hs = (int)floorf(__fmul_rn((float)ph, r.bin_h)), ws = (int)floorf(__fmul_rn((float)pw, r.bin_w));
        int he = (int)ceilf(__fmul_rn((float)(ph + 1), r.bin_h)), we = (int)ceilf(__fmul_rn((float)(pw + 1), r.bin_w));
        return make_int4(clampi(hs + r.sh, 0, H), clampi(he + r.sh, 0, H), clampi(ws + r.sw, 0, W), clampi(we + r.sw, 0, W));
    };
    if (use_tab)
        for (int b = threadIdx.x; b < bins; b += kPoolThreads) rect[b] = bin_rect(b);
    __syncthreads();
    const bool batch_ok = r.batch >= 0 && r.batch < N;
    const int total = (c1 - c0) * bins;
    for (int idx = threadIdx.x; idx < total; idx += kPoolThreads) {
        const int c = c0 + idx / bins, b = idx % bins;
        const int4 q = use_tab ? rect[b] : bin_rect(b);
        const bool empty = (q.y <= q.x) || (q.w <= q.z) || !batch_ok;
        float maxval = empty ? 0.f : -FLT_MAX;
        int maxidx = -1;
        if (!empty) {
            const int off = (r.batch * C + c) * H * W;
            for (int h = q.x; h < q.y; ++h)
                for (int w = q.z; w < q.w; ++w) {
                    const float v = __ldg(bottom + off + h * W + w);
                    if (v > maxval) { maxval = v; maxidx = off + h * W + w; }
                }
        }
        const size_t o = ((size_t)n * C + c) * bins + b;
        top[o] = maxval;
        if (argmax != nullptr) argmax[o] = maxidx;
    }
}

// ---- backward -------------------------------------------------------------------------------
constexpr int kPbTileH = 8, kPbTileW = 32;      // 256 cells per CTA tile, one thread per cell
constexpr int kPbListMax = 512;                 // RoIs cached per pass

struct __align__(16) PoolRoiB {
    int sw, sh, ew, eh;
    float bin_h, bin_w;
    int idx, pad;
};

__global__ void __launch_bounds__(kPoolThreads)
roi_pool_backward_kernel(const float* __restrict__ top_diff, const int* __restrict__ argmax,
                         const float* __restrict__ rois, float* __restrict__ bottom_diff, float scale,
                         int N, int R, int C, int H, int W, int PH, int PW, int c_per_cta) {
    __shared__ PoolRoiB list[kPbListMax];
    __shared__ int s_count;
    __shared__ int s_warp_counts[kPoolThreads / 32];

    const int tiles_w = (W + kPbTileW - 1) / kPbTileW;
    const int h0 = (blockIdx.x / tiles_w) * kPbTileH, w0 = (blockIdx.x % tiles_w) * kPbTileW;
    const int n = blockIdx.z;
    const int c0 = blockIdx.y * c_per_cta, c1 = min(C, c0 + c_per_cta);
    const int h = h0 + threadIdx.x / kPbTileW, w = w0 + threadIdx.x % kPbTileW;
    const bool cell_ok = (h < H) && (w < W);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int bins = PH * PW;

    // The RoI list is consumed in chunks of at most kPbListMax entries, in ascending RoI order.  The
    // per-cell partial sum is carried from chunk to chunk through bottom_diff itself (the first
    // chunk starts from 0), so the fp32 summation order equals the reference's single loop.
    int r_next = 0;
    bool first_chunk = true;
    do {
        if (threadIdx.x == 0) s_count = 0;
        __syncthreads();
        while (r_next < R) {
            const int r_idx = r_next + threadIdx.x;
            bool hit = false;
            PoolRoiB e;
            e.sw = e.sh = e.ew = e.eh = 0; e.bin_h = e.bin_w = 1.f; e.idx = 0; e.pad = 0;
            if (r_idx < R) {
                const PoolRoi pr = pool_roi(rois + 5 * (size_t)r_idx, scale, PH, PW);
                hit = (pr.batch == n) && !(pr.ew < w0 || pr.sw >= w0 + kPbTileW || pr.eh < h0 || pr.sh >= h0 + kPbTileH);
                e.sw = pr.sw; e.sh = pr.sh; e.ew = pr.ew; e.eh = pr.eh; e.bin_h = pr.bin_h; e.bin_w = pr.bin_w; e.idx = r_idx;
            }
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) s_warp_counts[warp] = __popc(m);
            __syncthreads();
            const int base_cnt = s_count;
            int before = base_cnt, chunk_total = 0;
            for (int k = 0; k < kPoolThreads / 32; ++k) {
                const int wc = s_warp_counts[k];
                if (k < warp) before += wc;
                chunk_total += wc;
            }
            if (base_cnt + chunk_total > kPbListMax) {   // uniform: list full, consume it first
                __syncthreads();
                break;
            }
            if (hit) list[before + __popc(m & ((1u << lane) - 1u))] = e;
            __syncthreads();
            if (threadIdx.x == 0) s_count = base_cnt + chunk_total;
            __syncthreads();
            r_next += kPoolThreads;
        }
        const int cnt = s_count;
        if (cell_ok) {
            for (int c = c0; c < c1; ++c) {
                const int index = ((n * C + c) * H + h) * W + w;
                float grad = first_chunk ? 0.f : bottom_diff[index];
                for (int k = 0; k < cnt; ++k) {
                    const PoolRoiB e = list[k];
                    if (!(w >= e.sw && w <= e.ew && h >= e.sh && h <= e.eh)) continue;
                    int phs = (int)floorf(__fdiv_rn((float)(h - e.sh), e.bin_h));
                    int phe = (int)ceilf(__fdiv_rn((float)(h - e.sh + 1), e.bin_h));
                    int pws = (int)floorf(__fdiv_rn((float)(w - e.sw), e.bin_w));
                    int pwe = (int)ceilf(__fdiv_rn((float)(w - e.sw + 1), e.bin_w));
                    phs = clampi(phs, 0, PH); phe = clampi(phe, 0, PH);
                    pws = clampi(pws, 0, PW); pwe = clampi(pwe, 0, PW);
                    const size_t off = ((size_t)e.idx * C + c) * bins;
                    for (int ph = phs; ph < phe; ++ph)
                        for (int pw = pws; pw < pwe; ++pw)
                            if (__ldg(argmax + off + ph * PW + pw) == index)
                                grad = __fadd_rn(grad, __ldg(top_diff + off + ph * PW + pw));
                }
                bottom_diff[index] = grad;
            }
        }
        first_chunk = false;
        __syncthreads();
    } while (r_next < R);
}

static int pool_c_per_cta(int R, int C, int bins) {
    int cpc = C;
    while (cpc > 1 && (long)R * ((C + cpc - 1) / cpc) < 8L * kNumSMs && (cpc / 2) * bins >= kPoolThreads) cpc /= 2;
    return cpc;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_roi_pool_forward(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW,
                          const float* rois, float* top, int* argmax, b200_stream_t stream) {
    if (bad_dims(N, R, H, W, C, PH, PW)) return B200_ROI_EINVAL;
    if (R > 0 && C > 0 && (!bottom || !rois || !top)) return B200_ROI_EINVAL;
    if (R == 0 || C == 0) return B200_ROI_OK;
    const int cpc = pool_c_per_cta(R, C, PH * PW);
    dim3 grid(R, (C + cpc - 1) / cpc);
    roi_pool_forward_kernel<<<grid, kPoolThreads, 0, stream>>>(bottom, rois, top, argmax, scale, N, C, H, W, PH, PW, cpc);
    return finish_launch();
}

int b200_roi_pool_backward(const float* top_diff, float scale, int N, int R, int H, int W, int C, int PH, int PW,
                           const float* rois, float* bottom_diff, const int* argmax, b200_stream_t stream) {
    if (bad_dims(N, R, H, W, C, PH, PW)) return B200_ROI_EINVAL;
    if ((size_t)N * C == 0) return B200_ROI_OK;
    if (!bottom_diff || (R > 0 && (!top_diff || !rois || !argmax))) return B200_ROI_EINVAL;
    if (N == 0 || C == 0 || H == 0 || W == 0) return B200_ROI_OK;
    const int tiles = ((H + kPbTileH - 1) / kPbTileH) * ((W + kPbTileW - 1) / kPbTileW);
    int cpc = C;
    while (cpc > 8 && (long)tiles * N * ((C + cpc - 1) / cpc) < 4L * kNumSMs) cpc /= 2;
    dim3 grid(tiles, (C + cpc - 1) / cpc, N);
    roi_pool_backward_kernel<<<grid, kPoolThreads, 0, stream>>>(top_diff, argmax, rois, bottom_diff, scale, N, R, C, H, W, PH, PW, cpc);
    return finish_launch();
}

}  // extern "C"
