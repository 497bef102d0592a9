// proposals.cu -- RPN proposal decode for the GPU-resident proposal layer (SURVEY.md 8f N1).
//
// One thread per pre-NMS candidate (already selected and sorted by score on the device): rebuild its anchor from the
// (H, W, A)-ordered index, apply the predicted deltas, clip to the image, evaluate the min-size / centre filter and
// emit the (x1, y1, x2, y2, score) row b200_nms consumes.  Candidates the filter rejects become the degenerate box
// (0, 0, -1, -1): its IoU with anything is 0 (or 0/0), so it neither suppresses nor is suppressed, and the caller
// drops it by the `valid` flag after NMS -- the candidate list keeps its length and no stream synchronisation or
// compaction is needed between decode and NMS.
//
// The decode and clip are bbox_transform.cuh's, with weights (1, 1, 1, 1) (oracle/proposals.py, pinned by
// tests/golden/proposals.npz).
//
// Semantics: lib/modeling/generate_proposals.py:66-89 (anchor enumeration), :108-150 (order, decode, clip, filter),
// :171-182 (_filter_boxes); lib/utils/boxes.py:138-154 (clip_tiled_boxes), :157-196 (bbox_transform); lib/core/config.py:936.
#include "common.cuh"
#include "bbox_transform.cuh"

namespace b200 {

__global__ void __launch_bounds__(256)
proposal_decode_kernel(const float* __restrict__ deltas,        // (4A, H, W) of one image
                       const float* __restrict__ anchors,       // (A, 4) cell anchors
                       const long long* __restrict__ order,     // (k) candidate indices in (H, W, A) order, best first
                       const float* __restrict__ scores,        // (k) their scores
                       int k, int A, int H, int W, float feat_stride, float im_h, float im_w, float min_size,
                       float* __restrict__ dets,                // (k, 5)
                       int* __restrict__ valid) {               // (k)
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= k) return;
    const long long idx = order[t];
    const int a = (int)(idx % A);
    const int w = (int)((idx / A) % W);
    const int h = (int)(idx / ((long long)A * W));
    // anchor + shift in double, then float32 (the reference adds float64 arrays and casts: boxes.astype(float32))
    const double sx = (double)w * (double)feat_stride, sy = (double)h * (double)feat_stride;
    const float x1 = (float)((double)anchors[4 * a + 0] + sx), y1 = (float)((double)anchors[4 * a + 1] + sy);
    const float x2 = (float)((double)anchors[4 * a + 2] + sx), y2 = (float)((double)anchors[4 * a + 3] + sy);
    const size_t plane = (size_t)H * W, cell = (size_t)h * W + w;
    const float dx = deltas[(size_t)(4 * a + 0) * plane + cell], dy = deltas[(size_t)(4 * a + 1) * plane + cell];
    const float dw = deltas[(size_t)(4 * a + 2) * plane + cell], dh = deltas[(size_t)(4 * a + 3) * plane + cell];

    const float4 p = bbox_transform(x1, y1, x2, y2, dx, dy, dw, dh, 1.f, 1.f, 1.f, 1.f, 4.135166556742356);   // log(1000 / 16)

    // NaN survives the reference's np.minimum / np.maximum clip and fails _filter_boxes
    const bool finite_box = !(p.x != p.x || p.y != p.y || p.z != p.z || p.w != p.w);
    const float wmax = __fsub_rn(im_w, 1.f), hmax = __fsub_rn(im_h, 1.f);
    const float bx1 = clip_coord(p.x, wmax), by1 = clip_coord(p.y, hmax), bx2 = clip_coord(p.z, wmax), by2 = clip_coord(p.w, hmax);

    const float ws = __fadd_rn(__fsub_rn(bx2, bx1), 1.f), hs = __fadd_rn(__fsub_rn(by2, by1), 1.f);
    const float xc = __fadd_rn(bx1, __fmul_rn(ws, .5f)), yc = __fadd_rn(by1, __fmul_rn(hs, .5f));
    const bool ok = finite_box && ws >= min_size && hs >= min_size && xc < im_w && yc < im_h;
    float* d = dets + (size_t)t * 5;
    d[0] = ok ? bx1 : 0.f; d[1] = ok ? by1 : 0.f; d[2] = ok ? bx2 : -1.f; d[3] = ok ? by2 : -1.f; d[4] = scores[t];
    valid[t] = ok ? 1 : 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_proposal_decode(const float* deltas, const float* anchors, const long long* order, const float* scores, int k, int A, int H,
                         int W, float feat_stride, float im_h, float im_w, float min_size, float* dets, int* valid, b200_stream_t stream) {
    if (k < 0 || A <= 0 || H <= 0 || W <= 0) return B200_ROI_EINVAL;
    if (k > 0 && (!deltas || !anchors || !order || !scores || !dets || !valid)) return B200_ROI_EINVAL;
    if (k == 0) return B200_ROI_OK;
    proposal_decode_kernel<<<(k + 255) / 256, 256, 0, stream>>>(deltas, anchors, order, scores, k, A, H, W, feat_stride, im_h, im_w,
                                                               min_size, dets, valid);
    return finish_launch();
}

}  // extern "C"
