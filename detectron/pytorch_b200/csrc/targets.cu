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

// best ground-truth box per box: first maximum (numpy argmax), overlap 0 -> no assignment (json_dataset.py:455-463)
__global__ void __launch_bounds__(256)
roi_assign_kernel(const float4* __restrict__ boxes, int N, const float4* __restrict__ gt, const int* __restrict__ gt_classes, int G,
                  float* __restrict__ max_overlaps, int* __restrict__ argmax, int* __restrict__ max_classes) {
    __shared__ float4 s_gt[256];
    __shared__ float s_area[256];
    const int n = blockIdx.x * 256 + threadIdx.x;
    const float4 b = n < N ? __ldg(boxes + n) : make_float4(0.f, 0.f, 0.f, 0.f);
    float best = 0.f;
    int arg = -1;
    bool first = true;
    for (int g0 = 0; g0 < G; g0 += 256) {
        __syncthreads();
        if (g0 + (int)threadIdx.x < G) {
            const float4 q = __ldg(gt + g0 + threadIdx.x);
            s_gt[threadIdx.x] = q; s_area[threadIdx.x] = area_plus1(q);
        }
        __syncthreads();
        const int m = min(256, G - g0);
        for (int j = 0; j < m; ++j) {
            const float o = iou_plus1(b, s_gt[j], s_area[j]);
            if (first || o > best) { best = o; arg = g0 + j; first = false; }      // strict >: the first maximum wins
        }
    }
    if (n >= N) return;
    const bool hit = arg >= 0 && best > 0.f;
    max_overlaps[n] = hit ? best : 0.f;
    argmax[n] = hit ? arg : -1;
    max_classes[n] = hit ? __ldg(gt_classes + arg) : 0;
}

// np.where(max_overlaps >= fg) / np.where((max_overlaps < bg_hi) & (max_overlaps >= bg_lo)): ascending index lists
__global__ void __launch_bounds__(1024)
roi_select_kernel(const float* __restrict__ max_overlaps, int N, float fg_thresh, float bg_hi, float bg_lo,
                  int* __restrict__ fg_inds, int* __restrict__ bg_inds, int* __restrict__ counts) {
    __shared__ int s_wf[32], s_wb[32];
    __shared__ int s_basef, s_baseb;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
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
    if (t == 0) { counts[0] = s_basef; counts[1] = s_baseb; }
}

// _sample_rois tail + _compute_targets + _expand_bbox_targets for the kept rows (the first n_fg are foreground)
__global__ void __launch_bounds__(256)
fast_rcnn_targets_kernel(const float4* __restrict__ boxes, const float4* __restrict__ gt, const int* __restrict__ argmax,
                         const int* __restrict__ max_classes, const int* __restrict__ keep, int n, int n_fg, float wx, float wy,
                         float ww, float wh, int reg_classes, int cls_agnostic, float im_scale, float batch_idx,
                         int* __restrict__ labels, float* __restrict__ rois, float* __restrict__ bbox_targets,
                         float* __restrict__ inside, float* __restrict__ outside) {
    const int i = blockIdx.x;
    if (i >= n) return;
    const int src = __ldg(keep + i);
    const float4 ex = __ldg(boxes + src);
    int label = i < n_fg ? __ldg(max_classes + src) : 0;                 // fast_rcnn.py:166: background rows get class 0
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
    roi_assign_kernel<<<(N + 255) / 256, 256, 0, stream>>>((const float4*)boxes, N, (const float4*)gt, gt_classes, G, max_overlaps, argmax,
                                                          max_classes);
    return finish_launch(1);
}

int b200_roi_select(const float* max_overlaps, int N, float fg_thresh, float bg_hi, float bg_lo, int* fg_inds, int* bg_inds, int* counts,
                    b200_stream_t stream) {
    if (N < 0 || !counts) return B200_ROI_EINVAL;
    if (N > 0 && (!max_overlaps || !fg_inds || !bg_inds)) return B200_ROI_EINVAL;
    roi_select_kernel<<<1, 1024, 0, stream>>>(max_overlaps, N, fg_thresh, bg_hi, bg_lo, fg_inds, bg_inds, counts);
    return finish_launch(1);
}

int b200_fast_rcnn_targets(const float* boxes, const float* gt, const int* argmax, const int* max_classes, const int* keep, int n, int n_fg,
                           const float* weights4_host, int reg_classes, int cls_agnostic, float im_scale, float batch_idx, int* labels,
                           float* rois, float* bbox_targets, float* inside, float* outside, b200_stream_t stream) {
    if (n < 0 || n_fg < 0 || n_fg > n || reg_classes < 1 || !weights4_host) return B200_ROI_EINVAL;
    if (n > 0 && (!boxes || !argmax || !max_classes || !keep || !labels || !rois || !bbox_targets || !inside || !outside))
        return B200_ROI_EINVAL;
    if (n == 0) return B200_ROI_OK;
    fast_rcnn_targets_kernel<<<n, 256, 0, stream>>>((const float4*)boxes, (const float4*)gt, argmax, max_classes, keep, n, n_fg,
                                                    weights4_host[0], weights4_host[1], weights4_host[2], weights4_host[3], reg_classes,
                                                    cls_agnostic, im_scale, batch_idx, labels, rois, bbox_targets, inside, outside);
    return finish_launch(1);
}

}  // extern "C"
