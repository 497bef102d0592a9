// keypoint_targets.cu -- Keypoint R-CNN training targets on the device (the training-time add_keypoint_rcnn_blobs).
//
// The reference does this on the host, per image, inside the training forward:
//   lib/roi_data/keypoint_rcnn.py:33-51     candidates: max_overlaps >= FG_THRESH and some visible keypoint of the box's person
//                                           (gt_inds[box_to_gt_ind_map], numpy indexing) inside the box (_within_box, :99-114)
//   lib/roi_data/keypoint_rcnn.py:53-57     np.random.choice of fg_rois_per_image of them when there are more
//   lib/roi_data/keypoint_rcnn.py:59-82     the sampled boxes' keypoints (all -1 for a negative map entry), heatmap labels
//                                           (utils/keypoints.py:160-211), the rois scaled by im_scale with the batch index
// All images of a step go through two launches with the draw on the host in between:
//   keypoint_candidates_kernel   one CTA per image: the ascending candidate list (ballot + prefix per chunk) and its count
//   keypoint_targets_kernel      one thread per (selected RoI, keypoint): location, weight and (keypoint 0) the RoI row
//
// Numerics: every float32 step of keypoints_to_heatmap_labels is written with an _rn intrinsic (nothing to contract), the
// boundary override comes after the floor, NaN compares false, and the int32 conversion is x86's: truncation for finite
// values, INT_MIN for NaN / +-inf (cvt.rzi would give 0 for NaN).
#include <climits>

#include "common.cuh"

namespace b200 {

constexpr int kKpMaxImages = 64;
constexpr int kKpMaxKeypoints = 64;
constexpr int kKpMaxHeatmap = 4096;       // HS * HS <= 2^24: every linear index is exact in float32

namespace {

constexpr int kCandThreads = 1024;
constexpr int kEmitThreads = 256;

struct KpImages {
    int num_images;
    int box_begin[kKpMaxImages + 1];      // image n's merged boxes (ground truth first, then proposals)
    int gt_begin[kKpMaxImages + 1];       // image n's gt_inds entries
    int person_begin[kKpMaxImages + 1];   // image n's gt_keypoints rows
    int roi_begin[kKpMaxImages + 1];      // image n's selected RoIs (the emit only)
    float im_scale[kKpMaxImages];
    float batch_index[kKpMaxImages];
};

// gt_inds[m] with numpy's wrap of negative indices -> the global keypoint row, or -1 when it is out of range
__device__ __forceinline__ int person_of(const KpImages& im, int n, int m, const int* __restrict__ gt_inds) {
    const int g0 = im.gt_begin[n], G = im.gt_begin[n + 1] - g0;
    const int j = m < 0 ? m + G : m;
    if (j < 0 || j >= G) return -1;
    const int p = __ldg(gt_inds + g0 + j), P = im.person_begin[n + 1] - im.person_begin[n];
    return (p >= 0 && p < P) ? im.person_begin[n] + p : -1;
}

__global__ void __launch_bounds__(kCandThreads)
keypoint_candidates_kernel(const __grid_constant__ KpImages im, const float* __restrict__ boxes, const float* __restrict__ max_overlaps,
                           const int* __restrict__ box_to_gt, const int* __restrict__ gt_inds, const int* __restrict__ keypoints, int K,
                           float fg_thresh, int* __restrict__ candidates, int* __restrict__ counts) {
    __shared__ int s_warp[kCandThreads / 32];
    __shared__ int s_base;
    const int n = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int b0 = im.box_begin[n], b1 = im.box_begin[n + 1];
    if (t == 0) s_base = 0;
    __syncthreads();
    for (int c0 = b0; c0 < b1; c0 += kCandThreads) {
        const int b = c0 + t;
        bool cand = false;
        if (b < b1 && __ldg(max_overlaps + b) >= fg_thresh) {               // b200_roi_select's comparison
            const int p = person_of(im, n, __ldg(box_to_gt + b), gt_inds);
            if (p >= 0) {
                // _within_box: int32 keypoints against float32 boxes, both promoted to double, ends included
                const double x1 = __ldg(boxes + 4 * b), y1 = __ldg(boxes + 4 * b + 1);
                const double x2 = __ldg(boxes + 4 * b + 2), y2 = __ldg(boxes + 4 * b + 3);
                const int* kp = keypoints + (size_t)p * 3 * K;
                for (int k = 0; k < K && !cand; ++k) {
                    if (__ldg(kp + 2 * K + k) <= 0) continue;
                    const double x = (double)__ldg(kp + k), y = (double)__ldg(kp + K + k);
                    cand = x >= x1 && x <= x2 && y >= y1 && y <= y2;
                }
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, cand);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int pos = s_base;
        for (int w = 0; w < warp; ++w) pos += s_warp[w];
        if (cand) candidates[b0 + pos + __popc(m & ((1u << lane) - 1u))] = b - b0;   // np.where: ascending, image-relative
        __syncthreads();
        if (t == 0) {
            int s = 0;
            for (int w = 0; w < kCandThreads / 32; ++w) s += s_warp[w];
            s_base += s;
        }
        __syncthreads();
    }
    if (t == 0) counts[n] = s_base;
}

__global__ void __launch_bounds__(kEmitThreads)
keypoint_targets_kernel(const __grid_constant__ KpImages im, const float* __restrict__ boxes, const int* __restrict__ box_to_gt,
                        const int* __restrict__ gt_inds, const int* __restrict__ keypoints, int K, int HS,
                        const int* __restrict__ candidates, const int* __restrict__ counts, const int* __restrict__ picks, int R,
                        float* __restrict__ rois_out, int* __restrict__ locations_out, float* __restrict__ weights_out) {
    const long long i = (long long)blockIdx.x * kEmitThreads + threadIdx.x;
    if (i >= (long long)R * K) return;
    const int r = (int)(i / K), k = (int)(i - (long long)r * K);
    int lo = 0, hi = im.num_images - 1;                                   // the image: last n with roi_begin[n] <= r
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (im.roi_begin[mid] <= r) lo = mid; else hi = mid - 1;
    }
    const int n = lo, b0 = im.box_begin[n], nb = im.box_begin[n + 1] - b0;   // nb >= 1: the host checks it
    const int cnt = __ldg(counts + n);
    // picks out of range (inconsistent input) stay inside the image's boxes: the row is unspecified, the reads are not
    const int pos = min(max(__ldg(picks + r), 0), max(cnt - 1, 0));
    const int b = b0 + min(max(cnt > 0 ? __ldg(candidates + b0 + pos) : 0, 0), nb - 1);
    const float x1 = __ldg(boxes + 4 * b), y1 = __ldg(boxes + 4 * b + 1), x2 = __ldg(boxes + 4 * b + 2), y2 = __ldg(boxes + 4 * b + 3);
    // keypoint_rcnn.py:64-69: the person's keypoints when the map entry is >= 0, else -1 (weight 0)
    const int m = __ldg(box_to_gt + b);
    const int p = m >= 0 ? person_of(im, n, m, gt_inds) : -1;
    int kx = -1, ky = -1, v = -1;
    if (p >= 0) {
        const int* kp = keypoints + (size_t)p * 3 * K;
        kx = __ldg(kp + k); ky = __ldg(kp + K + k); v = __ldg(kp + 2 * K + k);
    }
    // keypoints_to_heatmap_labels (utils/keypoints.py:181-209), float32 throughout
    const float fHS = (float)HS, x = __int2float_rn(kx), y = __int2float_rn(ky);
    float fx = floorf(__fmul_rn(__fsub_rn(x, x1), __fdiv_rn(fHS, __fsub_rn(x2, x1))));
    float fy = floorf(__fmul_rn(__fsub_rn(y, y1), __fdiv_rn(fHS, __fsub_rn(y2, y1))));
    if (x == x2) fx = fHS - 1.f;                                          // on the right / bottom edge: the last cell
    if (y == y2) fy = fHS - 1.f;
    const bool valid = fx >= 0.f && fy >= 0.f && fx < fHS && fy < fHS && v > 0;
    const float lin = __fadd_rn(__fmul_rn(fy, fHS), fx);
    // lin * valid, then astype(int32): lin itself, 0 (from +-0), or INT_MIN (NaN from inf * 0 or NaN * 0)
    locations_out[i] = valid ? __float2int_rz(lin) : (isfinite(lin) ? 0 : INT_MIN);
    weights_out[i] = valid ? 1.f : 0.f;
    if (k == 0) {                                                         // keypoint_rcnn.py:78-81, float32 multiply
        const float s = im.im_scale[n];
        float* row = rois_out + 5 * (size_t)r;
        row[0] = im.batch_index[n];
        row[1] = __fmul_rn(x1, s); row[2] = __fmul_rn(y1, s); row[3] = __fmul_rn(x2, s); row[4] = __fmul_rn(y2, s);
    }
}

// the host tables shared by both launches; false for a bad table
bool kp_tables(KpImages& im, int num_images, const int* box_begin, const int* gt_begin, const int* person_begin) {
    if (!box_begin || !gt_begin || !person_begin || num_images < 1 || num_images > kKpMaxImages) return false;
    if (box_begin[0] != 0 || gt_begin[0] != 0 || person_begin[0] != 0) return false;
    im.num_images = num_images;
    for (int i = 0; i <= num_images; ++i) {
        if (i > 0 && (box_begin[i] < box_begin[i - 1] || gt_begin[i] < gt_begin[i - 1] || person_begin[i] < person_begin[i - 1]))
            return false;
        im.box_begin[i] = box_begin[i]; im.gt_begin[i] = gt_begin[i]; im.person_begin[i] = person_begin[i];
    }
    return box_begin[num_images] <= (1 << 29);                            // 4 * box index stays in int
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_keypoint_candidates(const float* boxes, const float* max_overlaps, const int* box_to_gt, int num_images, const int* box_begin,
                             const int* gt_inds, const int* gt_begin, const int* keypoints, const int* person_begin, int num_keypoints,
                             float fg_thresh, int* candidates_out, int* counts_out, b200_stream_t stream) {
    if (!boxes || !max_overlaps || !box_to_gt || !gt_inds || !keypoints || !candidates_out || !counts_out) return B200_ROI_EINVAL;
    if (num_keypoints < 1 || num_keypoints > kKpMaxKeypoints) return B200_ROI_EINVAL;
    KpImages im{};
    if (!kp_tables(im, num_images, box_begin, gt_begin, person_begin)) return B200_ROI_EINVAL;
    keypoint_candidates_kernel<<<num_images, kCandThreads, 0, stream>>>(im, boxes, max_overlaps, box_to_gt, gt_inds, keypoints,
                                                                         num_keypoints, fg_thresh, candidates_out, counts_out);
    return finish_launch(1);
}

int b200_keypoint_targets(const float* boxes, const int* box_to_gt, int num_images, const int* box_begin, const int* gt_inds,
                          const int* gt_begin, const int* keypoints, const int* person_begin, int num_keypoints, int heatmap_size,
                          const int* candidates, const int* counts, const int* picks, const int* roi_begin, const float* im_scales,
                          const float* batch_index, float* rois_out, int* locations_out, float* weights_out, b200_stream_t stream) {
    if (!boxes || !box_to_gt || !gt_inds || !keypoints || !candidates || !counts || !picks || !roi_begin || !im_scales || !batch_index ||
        !rois_out || !locations_out || !weights_out)
        return B200_ROI_EINVAL;
    if (num_keypoints < 1 || num_keypoints > kKpMaxKeypoints || heatmap_size < 1 || heatmap_size > kKpMaxHeatmap) return B200_ROI_EINVAL;
    KpImages im{};
    if (!kp_tables(im, num_images, box_begin, gt_begin, person_begin) || roi_begin[0] != 0) return B200_ROI_EINVAL;
    for (int i = 0; i < num_images; ++i) {
        const int nr = roi_begin[i + 1] - roi_begin[i];
        if (nr < 0 || nr > box_begin[i + 1] - box_begin[i]) return B200_ROI_EINVAL;   // never more RoIs than boxes
        im.roi_begin[i] = roi_begin[i];
        im.im_scale[i] = im_scales[i];
        im.batch_index[i] = batch_index[i];
    }
    im.roi_begin[num_images] = roi_begin[num_images];
    const int R = roi_begin[num_images];
    if ((long long)R * num_keypoints >= (1LL << 31)) return B200_ROI_EINVAL;
    const long long total = (long long)R * num_keypoints;
    keypoint_targets_kernel<<<(unsigned)max((total + kEmitThreads - 1) / kEmitThreads, 1LL), kEmitThreads, 0, stream>>>(
        im, boxes, box_to_gt, gt_inds, keypoints, num_keypoints, heatmap_size, candidates, counts, picks, R, rois_out, locations_out,
        weights_out);
    return finish_launch(1);
}

}  // extern "C"
