// targets.cu -- RoI label / regression-target generation on the device (SURVEY.md 8f N4).
//
// The reference does this on the host, per image, in numpy + Cython, before every training step:
//   lib/utils/cython_bbox.pyx:32-73          bbox_overlaps (IoU with the "+1" pixel convention, float32)
//   lib/datasets/json_dataset.py:429-490     proposals merged into the roidb: best ground-truth box per proposal
//   lib/datasets/json_dataset.py:514-531     class assignment (max_overlaps / max_classes)
//   lib/roi_data/fast_rcnn.py:129-200        _sample_rois: foreground / background index sets, labels, scaled rois
//   lib/roi_data/fast_rcnn.py:203-248        _compute_targets (utils/boxes.py:199-230) + _expand_bbox_targets
// Here the proposals never leave the GPU: four small kernels, every operation written with _rn intrinsics in the order (and
// the precision: see cython_iou in common.cuh) of the reference's compiled code; only logf differs between libraries (<= 1 ulp).
#include "common.cuh"

namespace b200 {

namespace {

__device__ __forceinline__ float iou_plus1(const float4 b, const float4 q, float qarea) {
    return cython_iou(b.x, b.y, b.z, b.w, q.x, q.y, q.z, q.w, qarea);
}
__device__ __forceinline__ float area_plus1(const float4 q) { return cython_area(q.x, q.y, q.z, q.w); }

__global__ void __launch_bounds__(256)
bbox_overlaps_kernel(const float4* __restrict__ boxes, int N, const float4* __restrict__ query, int K, float* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
    if (idx >= (long long)N * K) return;
    const int n = (int)(idx / K), k = (int)(idx - (long long)n * K);
    const float4 q = __ldg(query + k);
    out[idx] = iou_plus1(__ldg(boxes + n), q, area_plus1(q));
}

// The images of a minibatch are segments of a concatenation: image b owns rows off[b] .. off[b + 1] - 1 (ascending offsets,
// (N + 1) of them, in device memory).  The one-image entry points pass off = nullptr and their row count as n.
struct Segs {
    const int* off;
    int n;
};
__device__ __forceinline__ int seg_begin(Segs s, int b) { return s.off ? __ldg(s.off + b) : 0; }
__device__ __forceinline__ int seg_end(Segs s, int b) { return s.off ? __ldg(s.off + b + 1) : s.n; }
// the image of row r < seg_end(s, N - 1): the last b with off[b] <= r, which skips empty images
__device__ __forceinline__ int seg_of(Segs s, int N, int r) {
    if (!s.off) return 0;
    int lo = 0, hi = N - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(s.off + mid) <= r) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// add_proposals (json_dataset.py:417-425 + _merge_proposal_boxes_into_roidb's np.append): image b's merged rows are its
// ground truth, then its proposals (rois5 grouped by image, prop_off[b] .. prop_off[b + 1] - 1) times the float32 1 / im_scale
__global__ void __launch_bounds__(256)
roi_merge_kernel(const float* __restrict__ rois5, const int* __restrict__ prop_off, const float4* __restrict__ gt, Segs gts,
                 const float* __restrict__ im_scales, Segs rows, int N, int max_rows, float4* __restrict__ out) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    if (t >= max_rows || t >= seg_end(rows, N - 1)) return;
    const int b = seg_of(rows, N, t), local = t - seg_begin(rows, b);
    const int g0 = seg_begin(gts, b), G = seg_end(gts, b) - g0;
    if (local < G) { out[t] = __ldg(gt + g0 + local); return; }
    const float* r = rois5 + 5 * (size_t)(__ldg(prop_off + b) + local - G);
    const float inv = __fdiv_rn(1.f, __ldg(im_scales + b));
    out[t] = make_float4(__fmul_rn(__ldg(r + 1), inv), __fmul_rn(__ldg(r + 2), inv), __fmul_rn(__ldg(r + 3), inv), __fmul_rn(__ldg(r + 4), inv));
}

// best ground-truth box of the row's own image: first maximum (numpy argmax), overlap 0 -> no assignment (json_dataset.py:455-463);
// argmax is an index into the concatenated ground truth.  gt_rows_first: the image's first G rows are its ground truth and keep
// what _add_gt_annotations gave them (json_dataset.py:208-290): themselves, overlap 1 and their class, or -1 and class 0 (crowd).
__global__ void __launch_bounds__(256)
roi_assign_kernel(const float4* __restrict__ boxes, Segs rows, int N, int max_rows, const float4* __restrict__ gt,
                  const int* __restrict__ gt_classes, const int* __restrict__ is_crowd, Segs gts, int gt_rows_first,
                  float* __restrict__ max_overlaps, int* __restrict__ argmax, int* __restrict__ max_classes) {
    const int n = blockIdx.x * 256 + threadIdx.x;
    if (n >= max_rows || n >= seg_end(rows, N - 1)) return;
    const int b = seg_of(rows, N, n), local = n - seg_begin(rows, b);
    const int g0 = seg_begin(gts, b), G = seg_end(gts, b) - g0;
    if (gt_rows_first && local < G) {
        const bool crowd = is_crowd && __ldg(is_crowd + g0 + local) != 0;
        max_overlaps[n] = crowd ? -1.f : 1.f;
        argmax[n] = g0 + local;
        max_classes[n] = crowd ? 0 : __ldg(gt_classes + g0 + local);
        return;
    }
    const float4 q = __ldg(boxes + n);
    float best = 0.f;
    int arg = -1;
#pragma unroll 1                                                            // unrolled, ptxas spills around the division
    for (int j = 0; j < G; ++j) {
        const float4 g = __ldg(gt + g0 + j);
        const float o = iou_plus1(q, g, area_plus1(g));
        if (j == 0 || o > best) { best = o; arg = j; }                      // strict >: the first maximum wins
    }
    const bool hit = arg >= 0 && best > 0.f;
    max_overlaps[n] = hit ? best : 0.f;
    argmax[n] = hit ? g0 + arg : -1;
    max_classes[n] = hit ? __ldg(gt_classes + g0 + arg) : 0;
}

// A CTA per image: np.where(max_overlaps >= fg) / np.where((max_overlaps < bg_hi) & (max_overlaps >= bg_lo)) as ascending lists
// of the image's own row indices, written from the image's first row on; counts[2b], counts[2b + 1] = their lengths
__global__ void __launch_bounds__(1024)
roi_select_kernel(const float* __restrict__ max_overlaps, Segs rows, float fg_thresh, float bg_hi, float bg_lo,
                  int* __restrict__ fg_inds, int* __restrict__ bg_inds, int* __restrict__ counts) {
    __shared__ int s_wf[32], s_wb[32];
    __shared__ int s_basef, s_baseb;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int r0 = seg_begin(rows, blockIdx.x), N = seg_end(rows, blockIdx.x) - r0;
    max_overlaps += r0; fg_inds += r0; bg_inds += r0;
    if (t == 0) { s_basef = 0; s_baseb = 0; }
    __syncthreads();
    for (int n0 = 0; n0 < N; n0 += 1024) {
        const int n = n0 + t;
        const float v = n < N ? max_overlaps[n] : -1.f;
        const bool f = n < N && v >= fg_thresh, b = n < N && v < bg_hi && v >= bg_lo;
        const unsigned mf = __ballot_sync(0xffffffffu, f), mb = __ballot_sync(0xffffffffu, b);
        if (lane == 0) { s_wf[warp] = __popc(mf); s_wb[warp] = __popc(mb); }
        __syncthreads();
        int pf = s_basef, pb = s_baseb;
        for (int w = 0; w < warp; ++w) { pf += s_wf[w]; pb += s_wb[w]; }
        if (f) fg_inds[pf + __popc(mf & ((1u << lane) - 1u))] = n;
        if (b) bg_inds[pb + __popc(mb & ((1u << lane) - 1u))] = n;
        __syncthreads();
        if (t == 0) { for (int w = 0; w < 32; ++w) { s_basef += s_wf[w]; s_baseb += s_wb[w]; } }
        __syncthreads();
    }
    if (t == 0) { counts[2 * blockIdx.x] = s_basef; counts[2 * blockIdx.x + 1] = s_baseb; }
}

// The kept rows of a minibatch: image b's are kept.off[b] .. kept.off[b + 1] - 1, its first num_fg[b] foreground, scaled by
// im_scale[b] into batch slot batch_idx[b].  The one-image entry point passes null tables and its values by value.
struct Kept {
    Segs seg;
    const int* num_fg;
    const float* im_scale;
    const float* batch_idx;
    int num_fg1;
    float im_scale1, batch_idx1;
};

// _sample_rois tail + _compute_targets + _expand_bbox_targets for the kept rows (keep: merged rows, argmax: concatenated gt)
__global__ void __launch_bounds__(256)
fast_rcnn_targets_kernel(const float4* __restrict__ boxes, const float4* __restrict__ gt, const int* __restrict__ argmax,
                         const int* __restrict__ max_classes, const int* __restrict__ keep, Kept kept, int N, float wx, float wy,
                         float ww, float wh, int reg_classes, int cls_agnostic, int* __restrict__ labels, float* __restrict__ rois,
                         float* __restrict__ bbox_targets, float* __restrict__ inside, float* __restrict__ outside) {
    const int i = blockIdx.x;
    const int b = seg_of(kept.seg, N, i);
    const int n_fg = kept.num_fg ? __ldg(kept.num_fg + b) : kept.num_fg1;
    const float im_scale = kept.im_scale ? __ldg(kept.im_scale + b) : kept.im_scale1;
    const float batch_idx = kept.batch_idx ? __ldg(kept.batch_idx + b) : kept.batch_idx1;
    const int src = __ldg(keep + i);
    const float4 ex = __ldg(boxes + src);
    int label = i - seg_begin(kept.seg, b) < n_fg ? __ldg(max_classes + src) : 0;   // fast_rcnn.py:166: background rows get class 0
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    const int a = __ldg(argmax + src);
    if (a >= 0) {                                                         // utils/boxes.py:212-226, float32 like numpy
        const float4 g = __ldg(gt + a);
        const float ew = __fadd_rn(__fsub_rn(ex.z, ex.x), 1.f), eh = __fadd_rn(__fsub_rn(ex.w, ex.y), 1.f);
        const float ecx = __fadd_rn(ex.x, __fmul_rn(0.5f, ew)), ecy = __fadd_rn(ex.y, __fmul_rn(0.5f, eh));
        const float gw = __fadd_rn(__fsub_rn(g.z, g.x), 1.f), gh = __fadd_rn(__fsub_rn(g.w, g.y), 1.f);
        const float gcx = __fadd_rn(g.x, __fmul_rn(0.5f, gw)), gcy = __fadd_rn(g.y, __fmul_rn(0.5f, gh));
        t[0] = __fdiv_rn(__fmul_rn(wx, __fsub_rn(gcx, ecx)), ew);
        t[1] = __fdiv_rn(__fmul_rn(wy, __fsub_rn(gcy, ecy)), eh);
        t[2] = __fmul_rn(ww, logf(__fdiv_rn(gw, ew)));
        t[3] = __fmul_rn(wh, logf(__fdiv_rn(gh, eh)));
    }
    if (cls_agnostic && label > 1) label = 1;                             // fast_rcnn.py:212-213 clips the labels in place: the blob's too
    const int col_cls = label;
    if (threadIdx.x == 0) {
        labels[i] = label;
        rois[5 * i] = batch_idx;
        rois[5 * i + 1] = __fmul_rn(ex.x, im_scale); rois[5 * i + 2] = __fmul_rn(ex.y, im_scale);
        rois[5 * i + 3] = __fmul_rn(ex.z, im_scale); rois[5 * i + 4] = __fmul_rn(ex.w, im_scale);
    }
    const int cols = 4 * reg_classes;
    for (int c = threadIdx.x; c < cols; c += 256) {
        const bool on = col_cls > 0 && (c >> 2) == col_cls;
        const float v = on ? t[c & 3] : 0.f, w = on ? 1.f : 0.f;
        bbox_targets[(size_t)i * cols + c] = v;
        inside[(size_t)i * cols + c] = w;
        outside[(size_t)i * cols + c] = w;                                // fast_rcnn.py:181-182: inside > 0
    }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_bbox_overlaps(const float* boxes, int N, const float* query, int K, float* out, b200_stream_t stream) {
    if (N < 0 || K < 0) return B200_ROI_EINVAL;
    if ((long long)N * K > 0 && (!boxes || !query || !out)) return B200_ROI_EINVAL;
    const long long total = (long long)N * K;
    if (total == 0) return B200_ROI_OK;
    bbox_overlaps_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>((const float4*)boxes, N, (const float4*)query, K, out);
    return finish_launch(1);
}

int b200_roi_assign(const float* boxes, int N, const float* gt, const int* gt_classes, int G, float* max_overlaps, int* argmax,
                    int* max_classes, b200_stream_t stream) {
    if (N < 0 || G < 0) return B200_ROI_EINVAL;
    if (N > 0 && (!boxes || !max_overlaps || !argmax || !max_classes)) return B200_ROI_EINVAL;
    if (N > 0 && G > 0 && (!gt || !gt_classes)) return B200_ROI_EINVAL;
    if (N == 0) return B200_ROI_OK;
    roi_assign_kernel<<<(N + 255) / 256, 256, 0, stream>>>((const float4*)boxes, Segs{nullptr, N}, 1, N, (const float4*)gt, gt_classes,
                                                          nullptr, Segs{nullptr, G}, 0, max_overlaps, argmax, max_classes);
    return finish_launch(1);
}

int b200_roi_select(const float* max_overlaps, int N, float fg_thresh, float bg_hi, float bg_lo, int* fg_inds, int* bg_inds, int* counts,
                    b200_stream_t stream) {
    if (N < 0 || !counts) return B200_ROI_EINVAL;
    if (N > 0 && (!max_overlaps || !fg_inds || !bg_inds)) return B200_ROI_EINVAL;
    roi_select_kernel<<<1, 1024, 0, stream>>>(max_overlaps, Segs{nullptr, N}, fg_thresh, bg_hi, bg_lo, fg_inds, bg_inds, counts);
    return finish_launch(1);
}

int b200_fast_rcnn_targets(const float* boxes, const float* gt, const int* argmax, const int* max_classes, const int* keep, int n, int n_fg,
                           const float* weights4_host, int reg_classes, int cls_agnostic, float im_scale, float batch_idx, int* labels,
                           float* rois, float* bbox_targets, float* inside, float* outside, b200_stream_t stream) {
    if (n < 0 || n_fg < 0 || n_fg > n || reg_classes < 1 || !weights4_host) return B200_ROI_EINVAL;
    if (n > 0 && (!boxes || !argmax || !max_classes || !keep || !labels || !rois || !bbox_targets || !inside || !outside))
        return B200_ROI_EINVAL;
    if (n == 0) return B200_ROI_OK;
    const Kept kept{Segs{nullptr, n}, nullptr, nullptr, nullptr, n_fg, im_scale, batch_idx};
    fast_rcnn_targets_kernel<<<n, 256, 0, stream>>>((const float4*)boxes, (const float4*)gt, argmax, max_classes, keep, kept, 1,
                                                    weights4_host[0], weights4_host[1], weights4_host[2], weights4_host[3], reg_classes,
                                                    cls_agnostic, labels, rois, bbox_targets, inside, outside);
    return finish_launch(1);
}

int b200_roi_merge_proposals(const float* rois5, const int* prop_off, const float* gt, const int* gt_off, const float* im_scales, int N,
                             const int* box_off, int max_rows, float* boxes, b200_stream_t stream) {
    if (N < 1 || max_rows < 0 || !prop_off || !gt_off || !im_scales || !box_off) return B200_ROI_EINVAL;
    if (max_rows > 0 && !boxes) return B200_ROI_EINVAL;                  // rois5 may be null: no proposals
    if (max_rows == 0) return B200_ROI_OK;
    roi_merge_kernel<<<(max_rows + 255) / 256, 256, 0, stream>>>(rois5, prop_off, (const float4*)gt, Segs{gt_off, 0}, im_scales,
                                                                Segs{box_off, 0}, N, max_rows, (float4*)boxes);
    return finish_launch(1);
}

int b200_roi_assign_batched(const float* boxes, const int* box_off, int N, int max_rows, const float* gt, const int* gt_classes,
                            const int* is_crowd, const int* gt_off, int gt_rows_first, float* max_overlaps, int* argmax, int* max_classes,
                            b200_stream_t stream) {
    if (N < 1 || max_rows < 0 || !box_off || !gt_off) return B200_ROI_EINVAL;
    if (max_rows > 0 && (!boxes || !max_overlaps || !argmax || !max_classes)) return B200_ROI_EINVAL;
    if (max_rows == 0) return B200_ROI_OK;
    roi_assign_kernel<<<(max_rows + 255) / 256, 256, 0, stream>>>((const float4*)boxes, Segs{box_off, 0}, N, max_rows, (const float4*)gt,
                                                                 gt_classes, is_crowd, Segs{gt_off, 0}, gt_rows_first, max_overlaps,
                                                                 argmax, max_classes);
    return finish_launch(1);
}

int b200_roi_select_batched(const float* max_overlaps, const int* box_off, int N, float fg_thresh, float bg_hi, float bg_lo, int* fg_inds,
                            int* bg_inds, int* counts, b200_stream_t stream) {
    if (N < 1 || !box_off || !counts || !max_overlaps || !fg_inds || !bg_inds) return B200_ROI_EINVAL;
    roi_select_kernel<<<N, 1024, 0, stream>>>(max_overlaps, Segs{box_off, 0}, fg_thresh, bg_hi, bg_lo, fg_inds, bg_inds, counts);
    return finish_launch(1);
}

int b200_fast_rcnn_targets_batched(const float* boxes, const float* gt, const int* argmax, const int* max_classes, const int* keep,
                                   const int* keep_off, const int* num_fg, const float* im_scales, const float* batch_idx, int N, int n,
                                   const float* weights4_host, int reg_classes, int cls_agnostic, int* labels, float* rois,
                                   float* bbox_targets, float* inside, float* outside, b200_stream_t stream) {
    if (N < 1 || n < 0 || reg_classes < 1 || !weights4_host || !keep_off || !num_fg || !im_scales || !batch_idx) return B200_ROI_EINVAL;
    if (n > 0 && (!boxes || !argmax || !max_classes || !keep || !labels || !rois || !bbox_targets || !inside || !outside))
        return B200_ROI_EINVAL;
    if (n == 0) return B200_ROI_OK;
    const Kept kept{Segs{keep_off, 0}, num_fg, im_scales, batch_idx, 0, 0.f, 0.f};
    fast_rcnn_targets_kernel<<<n, 256, 0, stream>>>((const float4*)boxes, (const float4*)gt, argmax, max_classes, keep, kept, N,
                                                    weights4_host[0], weights4_host[1], weights4_host[2], weights4_host[3], reg_classes,
                                                    cls_agnostic, labels, rois, bbox_targets, inside, outside);
    return finish_launch(1);
}

}  // extern "C"
