// detect_bbox.cu -- the box head's decode of one test-time transform (lib/core/test.py:127-189, 289-362).
//
// One thread per (row, class) writes pred_boxes[r, 4j:4j+4] of the (R, 4K) result:
//   * input box: the model's rois[r, 1:5] / im_scale (in float64, the reference's im_scale is a one-element list; rounded to
//     float32 by bbox_transform's astype), or the float32 proposal box as given;
//   * TEST.BBOX_REG: bbox_transform.cuh's decode by bbox_pred[r, 4j:4j+4] (or, class-agnostic, by the row's last 4 columns) with
//     MODEL.BBOX_REG_WEIGHTS and BBOX_XFORM_CLIP, then clip_tiled_boxes to this transform's image; without it the box itself;
//   * the transform's inverse in the same store: flip_boxes with this transform's image width, `(float32(W) - x) - 1`, then the
//     aspect-ratio inverse, `x * float32(1 / ar)`.  The reference evaluates those in the dtype of its boxes: float32 after the
//     decode, float64 for undecoded rois (rois / im_scale stays float64 without BBOX_REG), rounded to float32 at the end.
#include "common.cuh"
#include "bbox_transform.cuh"

namespace b200 {

template <typename T>
__device__ __forceinline__ void bbox_inverse(T& x1, T& x2, int flip_width, double ar_inv) {
    if (flip_width > 0) {
        const T w = (T)flip_width, a = w - x2 - (T)1, b = w - x1 - (T)1;
        x1 = a; x2 = b;
    }
    x1 = x1 * (T)ar_inv; x2 = x2 * (T)ar_inv;
}

__global__ void __launch_bounds__(256)
bbox_decode_kernel(const float* __restrict__ boxes, int box_stride, int box_col, double im_scale, const float* __restrict__ deltas,
                   int delta_stride, int agnostic, int R, int K, int bbox_reg, float wx, float wy, float ww, float wh, double xform_clip,
                   int im_h, int im_w, int flip_width, double ar_inv, float* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)R * K) return;
    const int r = (int)(t / K), j = (int)(t % K);
    const float* b = boxes + (size_t)r * box_stride + box_col;
    float4 o;
    if (bbox_reg) {
        float x1 = b[0], y1 = b[1], x2 = b[2], y2 = b[3];
        if (im_scale > 0.0) {
            x1 = (float)((double)x1 / im_scale); y1 = (float)((double)y1 / im_scale);
            x2 = (float)((double)x2 / im_scale); y2 = (float)((double)y2 / im_scale);
        }
        const float* d = deltas + (size_t)r * delta_stride + (agnostic ? delta_stride - 4 : 4 * j);
        o = bbox_transform(x1, y1, x2, y2, d[0], d[1], d[2], d[3], wx, wy, ww, wh, xform_clip);
        const float wmax = (float)(im_w - 1), hmax = (float)(im_h - 1);
        o.x = clip_coord(o.x, wmax); o.y = clip_coord(o.y, hmax); o.z = clip_coord(o.z, wmax); o.w = clip_coord(o.w, hmax);
        bbox_inverse<float>(o.x, o.z, flip_width, ar_inv);
    } else if (im_scale > 0.0) {
        double x1 = (double)b[0] / im_scale, x2 = (double)b[2] / im_scale;
        bbox_inverse<double>(x1, x2, flip_width, ar_inv);
        o = make_float4((float)x1, (float)((double)b[1] / im_scale), (float)x2, (float)((double)b[3] / im_scale));
    } else {
        o = make_float4(b[0], b[1], b[2], b[3]);
        bbox_inverse<float>(o.x, o.z, flip_width, ar_inv);
    }
    reinterpret_cast<float4*>(out)[t] = o;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_bbox_decode(const float* boxes, int box_stride, int box_col, double im_scale, const float* deltas, int delta_stride,
                     int agnostic, int num_rows, int num_classes, int bbox_reg, const float* weights, double xform_clip, int im_h,
                     int im_w, int flip_width, double ar_inv, float* pred_boxes, b200_stream_t stream) {
    if (num_rows < 0 || num_classes < 1 || box_col < 0 || box_stride < box_col + 4 || !(im_scale >= 0.0)) return B200_ROI_EINVAL;
    if (bbox_reg && (!weights || im_h < 1 || im_w < 1 || delta_stride < 4 || (!agnostic && delta_stride < 4 * num_classes)))
        return B200_ROI_EINVAL;
    if ((long long)num_rows * num_classes >= (1LL << 31)) return B200_ROI_EINVAL;
    if (num_rows == 0) return B200_ROI_OK;
    if (!boxes || !pred_boxes || (bbox_reg && !deltas) || reinterpret_cast<uintptr_t>(pred_boxes) % 16 != 0) return B200_ROI_EINVAL;
    const float w[4] = {bbox_reg ? weights[0] : 1.f, bbox_reg ? weights[1] : 1.f, bbox_reg ? weights[2] : 1.f, bbox_reg ? weights[3] : 1.f};
    const long long n = (long long)num_rows * num_classes;
    bbox_decode_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(boxes, box_stride, box_col, im_scale, deltas, delta_stride, agnostic != 0,
                                                                       num_rows, num_classes, bbox_reg != 0, w[0], w[1], w[2], w[3],
                                                                       xform_clip, im_h, im_w, flip_width, ar_inv, pred_boxes);
    return finish_launch();
}

}  // extern "C"
