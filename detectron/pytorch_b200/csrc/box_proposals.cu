// box_proposals.cu -- proposal recall on the device: the greedy gt-to-proposal assignment of the reference's
// json_dataset_evaluator.evaluate_box_proposals (lib/datasets/json_dataset_evaluator.py:236-317; oracle/box_proposals.py restates it).
//
// One CTA per work item (limit l, area range a, image i); one launch covers every item.  The reference builds the (P x G) IoU matrix of
// the image's first P proposals against its G area-valid ground-truth boxes, then min(P, G) times takes the column with the largest
// maximum (first such column), records that maximum, and masks the winning proposal's row and the column with -1.  Every IoU that is not
// NaN is >= 0 (cython_iou is 0 unless iw > 0 and ih > 0, and then the union is at least the intersection), so a masked cell never wins
// against a live one and the masking is the same as removing the row and the column.  The CTA therefore keeps, per live column, its
// maximum over the unused proposals and the first proposal reaching it (numpy's max / argmax over the column), and after each pick
// recomputes only the columns whose argmax was the proposal just taken: removing any other proposal changes neither value.
//   per-gt state (column maximum, its argmax or a "not live" mark) and the used-proposal bytes live in the caller's workspace, so
//   neither P nor G has a capacity; a warp computes one column (lanes stride over the proposals, shuffle reduction), and the pick is a
//   CTA reduction over the live columns (largest maximum, then lowest index).
//   A proposal with a NaN coordinate has IoU 0 with every gt, as in the compiled Cython; a NaN gt coordinate gives NaN IoUs.
//   A NaN IoU anywhere in the item's matrix fails the reference's `assert gt_ovr >= 0` at its first iteration: the item is flagged and
//   nothing of it is counted.
//   After the matching, the CTA counts its counted gts (matched: the recorded IoU, unmatched: 0) against every threshold, compared in
//   float64 as numpy compares the float64 gt_overlaps array, and adds the counts to the (l, a) row with one atomic per threshold.
#include <climits>
#include <cstdint>

#include "common.cuh"

namespace b200 {

namespace {

constexpr int kBpThreads = 256;
constexpr int kBpWarps = kBpThreads / 32;
constexpr int kNotLive = -1;              // colarg of a gt outside the area range or already matched

struct AreaTable {
    double lo[B200_BOX_PROPOSAL_MAX_AREAS], hi[B200_BOX_PROPOSAL_MAX_AREAS];
};

// (v, i) beats (bv, bi): larger value, then lower index -- numpy's argmax over values that are never NaN here
__device__ __forceinline__ bool beats(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__device__ __forceinline__ void warp_best(float& v, int& i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (beats(ov, oi, v, i)) { v = ov; i = oi; }
    }
}

// The maximum of column q over the unused proposals 0 .. pe - 1 and the first proposal reaching it, in every lane of the warp.
// *nan is set when an IoU is NaN.
__device__ __forceinline__ void column_max(const float4* __restrict__ prop, const unsigned char* used, int pe, float4 q, float& v, int& arg,
                                           bool& nan) {
    const float qarea = cython_area(q.x, q.y, q.z, q.w);
    v = -1.f;
    arg = INT_MAX;
    for (int p = (int)(threadIdx.x & 31); p < pe; p += 32) {
        if (used[p]) continue;
        const float4 b = __ldg(prop + p);
        // The compiled Cython's min / max are `q < b ? q : b` selects, which return the proposal's NaN, so iw or ih is NaN and the
        // IoU 0; fminf / fmaxf would return the gt's value instead.  A NaN in the gt alone gives the same selects either way.
        const bool prop_nan = isnan(b.x) || isnan(b.y) || isnan(b.z) || isnan(b.w);
        const float ov = prop_nan ? 0.f : cython_iou(b.x, b.y, b.z, b.w, q.x, q.y, q.z, q.w, qarea);
        if (isnan(ov)) { nan = true; continue; }
        if (ov > v) { v = ov; arg = p; }        // p grows within a lane: the first maximum of the lane
    }
    warp_best(v, arg);
}

__global__ void __launch_bounds__(kBpThreads)
box_proposal_match_kernel(int num_images, int num_props, int num_gt, int num_areas, int num_thresholds, AreaTable areas,
                          const float4* __restrict__ prop_box, const int* __restrict__ prop_begin, const float4* __restrict__ gt_box,
                          const double* __restrict__ gt_area, const int* __restrict__ gt_begin, const int* __restrict__ prop_count,
                          const double* __restrict__ thresholds, float* colmax, int* colarg, unsigned char* prop_used, float* overlap,
                          unsigned char* excluded, unsigned char* error, unsigned long long* counts) {
    __shared__ float s_v[kBpWarps];
    __shared__ int s_i[kBpWarps];
    __shared__ int s_pick_p, s_nan, s_valid;
    __shared__ unsigned long long s_cnt[kBpWarps];

    const int item = blockIdx.x;
    const int i = item % num_images;
    const int la = item / num_images;                   // l * num_areas + a
    const int a = la % num_areas;
    const int l = la / num_areas;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    const int p0 = prop_begin[i], P = prop_begin[i + 1] - p0;
    const int g0 = gt_begin[i], G = gt_begin[i + 1] - g0;
    const int pe = min(max(prop_count[(size_t)l * num_images + i], 0), P);
    const bool skipped = P == 0;                        // the reference's `continue`: its gts count in num_pos only
    double lo = 0.0, hi = 0.0;
#pragma unroll
    for (int k = 0; k < B200_BOX_PROPOSAL_MAX_AREAS; ++k) {   // constant indices keep the table in the parameter bank
        if (k == a) { lo = areas.lo[k]; hi = areas.hi[k]; }
    }
    const size_t gbase = (size_t)la * num_gt + g0;
    float* cmax = colmax + gbase;
    int* carg = colarg + gbase;
    float* ovr = overlap + gbase;
    unsigned char* used = prop_used + (size_t)la * num_props + p0;
    const float4* prop = prop_box + p0;
    const float4* gt = gt_box + g0;

    if (tid == 0) { s_nan = 0; s_valid = 0; }
    __syncthreads();
    int valid = 0;
    for (int g = tid; g < G; g += kBpThreads) {
        const double ar = __ldg(gt_area + g0 + g);
        const bool in_range = ar >= lo && ar <= hi;
        ovr[g] = 0.f;
        excluded[gbase + g] = (!in_range || skipped) ? 1 : 0;
        carg[g] = in_range ? 0 : kNotLive;
        valid += in_range;
    }
    for (int p = tid; p < pe; p += kBpThreads) used[p] = 0;
    if (valid) atomicAdd(&s_valid, valid);
    __syncthreads();
    const int gv = s_valid;
    if (skipped || gv == 0) {
        if (tid == 0) error[item] = 0;
        return;
    }

    // column maxima over the first pe proposals (none when pe == 0: every valid gt stays at 0)
    const int iters = min(pe, gv);
    if (iters > 0) {
        bool nan = false;
        for (int g = warp; g < G; g += kBpWarps) {
            if (carg[g] == kNotLive) continue;
            float v;
            int arg;
            column_max(prop, used, pe, gt[g], v, arg, nan);
            if (lane == 0) { cmax[g] = v; carg[g] = arg; }
        }
        if (__any_sync(0xffffffffu, nan) && lane == 0) s_nan = 1;
        __syncthreads();
        if (s_nan) {
            if (tid == 0) error[item] = 1;
            return;
        }
    }
    if (tid == 0) error[item] = 0;

    for (int j = 0; j < iters; ++j) {
        // pick: the live column with the largest maximum, lowest index on ties
        float bv = -1.f;
        int bg = INT_MAX;
        for (int g = tid; g < G; g += kBpThreads) {
            if (carg[g] == kNotLive) continue;
            const float v = cmax[g];
            if (v > bv) { bv = v; bg = g; }             // g grows within a thread
        }
        warp_best(bv, bg);
        if (lane == 0) { s_v[warp] = bv; s_i[warp] = bg; }
        __syncthreads();
        if (warp == 0) {
            bv = lane < kBpWarps ? s_v[lane] : -1.f;
            bg = lane < kBpWarps ? s_i[lane] : INT_MAX;
            warp_best(bv, bg);
            if (lane == 0) {
                const int p = carg[bg];
                ovr[bg] = bv;
                carg[bg] = kNotLive;
                used[p] = 1;
                s_pick_p = p;
            }
        }
        __syncthreads();
        if (j + 1 == iters) break;
        // the columns that lost their argmax: maximum over the proposals still unused
        const int taken = s_pick_p;
        bool nan = false;                              // cannot happen: the first pass saw every cell
        for (int g = warp; g < G; g += kBpWarps) {
            if (carg[g] != taken) continue;
            float v;
            int arg;
            column_max(prop, used, pe, gt[g], v, arg, nan);
            if (lane == 0) { cmax[g] = v; carg[g] = arg; }
        }
        __syncthreads();
    }

    // per-threshold counts of this item's counted gts (matched or not), float64 compare of the widened float32 value
    for (int t = 0; t < num_thresholds; ++t) {
        const double thr = __ldg(thresholds + t);
        unsigned long long c = 0;
        for (int g = tid; g < G; g += kBpThreads) {
            const double ar = __ldg(gt_area + g0 + g);
            if (ar >= lo && ar <= hi && (double)ovr[g] >= thr) ++c;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) s_cnt[warp] = c;
        __syncthreads();
        if (tid == 0) {
            unsigned long long sum = 0;
            for (int w = 0; w < kBpWarps; ++w) sum += s_cnt[w];
            if (sum) atomicAdd(counts + (size_t)la * num_thresholds + t, sum);
        }
        __syncthreads();
    }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_box_proposal_match_workspace_bytes(int num_props, int num_gt, int num_areas, int num_limits) {
    if (num_props < 0 || num_gt < 0 || num_areas < 0 || num_limits < 0) return 0;
    const size_t la = (size_t)num_areas * num_limits;
    return la * ((size_t)num_gt * (sizeof(float) + sizeof(int)) + (size_t)num_props) + 16;
}

int b200_box_proposal_match(int num_images, int num_props, int num_gt, int num_areas, int num_limits, int num_thresholds, const float* prop_box,
                            const int* prop_begin, const float* gt_box, const double* gt_area, const int* gt_begin, const int* prop_count,
                            const double* area_range, const double* thresholds, void* workspace, size_t workspace_bytes, float* overlap,
                            unsigned char* excluded, unsigned char* error, long long* counts, b200_stream_t stream) {
    if (num_images < 0 || num_props < 0 || num_gt < 0 || num_areas < 0 || num_areas > B200_BOX_PROPOSAL_MAX_AREAS || num_limits < 0 ||
        num_thresholds < 0)
        return B200_ROI_EINVAL;
    const long long items = (long long)num_images * num_areas * num_limits;
    if (items == 0) return B200_ROI_OK;
    if (items > INT_MAX) return B200_ROI_EINVAL;
    if (!prop_begin || !gt_begin || !prop_count || !area_range || !error) return B200_ROI_EINVAL;
    if (num_props > 0 && !prop_box) return B200_ROI_EINVAL;
    if (num_gt > 0 && (!gt_box || !gt_area || !overlap || !excluded)) return B200_ROI_EINVAL;
    if (num_thresholds > 0 && (!thresholds || !counts)) return B200_ROI_EINVAL;
    if (((uintptr_t)prop_box | (uintptr_t)gt_box) & 15) return B200_ROI_EINVAL;
    if (((uintptr_t)gt_area | (uintptr_t)thresholds | (uintptr_t)counts) & 7) return B200_ROI_EINVAL;
    const size_t need = b200_box_proposal_match_workspace_bytes(num_props, num_gt, num_areas, num_limits);
    if (!workspace || workspace_bytes < need) return B200_ROI_EWORKSPACE;
    AreaTable areas;
    for (int a = 0; a < num_areas; ++a) {
        areas.lo[a] = area_range[2 * a];
        areas.hi[a] = area_range[2 * a + 1];
    }
    const size_t la_g = (size_t)num_areas * num_limits * num_gt;
    char* ws = (char*)(((uintptr_t)workspace + 15) & ~(uintptr_t)15);
    float* colmax = (float*)ws;
    int* colarg = (int*)(ws + la_g * sizeof(float));
    unsigned char* prop_used = (unsigned char*)(ws + la_g * (sizeof(float) + sizeof(int)));
    if (num_thresholds > 0 &&
        cudaMemsetAsync(counts, 0, (size_t)num_areas * num_limits * num_thresholds * sizeof(long long), stream) != cudaSuccess)
        return finish_launch(0);
    box_proposal_match_kernel<<<(unsigned)items, kBpThreads, 0, stream>>>(
        num_images, num_props, num_gt, num_areas, num_thresholds, areas, (const float4*)prop_box, prop_begin, (const float4*)gt_box, gt_area,
        gt_begin, prop_count, thresholds, colmax, colarg, prop_used, overlap, excluded, error, (unsigned long long*)counts);
    return finish_launch(1);
}

}  // extern "C"
