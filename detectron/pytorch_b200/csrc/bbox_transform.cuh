// bbox_transform.cuh -- the box decode shared by the RPN proposal layer (proposals.cu) and the box head (detect_bbox.cu).
//
// lib/utils/boxes.py:157-196 (bbox_transform) and :138-154 (clip_tiled_boxes) as the reference's numpy lines evaluate under
// numpy >= 2 (oracle/proposals.py, pinned by tests/golden/proposals.npz and tests/golden/detect_bbox.npz): float32 for widths,
// centres, `d / w*` and `dx * w + ctr`; float64 for min(dw, BBOX_XFORM_CLIP) (an np.float64 scalar), exp, `exp * w` and
// `ctr -/+ 0.5 * pred_w (- 1)`, rounded to float32 once.
#pragma once

namespace b200 {

// (x1, y1, x2, y2) decoded by one set of deltas with weights (wx, wy, ww, wh) and the log-space clip `xform_clip`
__device__ __forceinline__ float4 bbox_transform(float x1, float y1, float x2, float y2, float dx, float dy, float dw, float dh, float wx,
                                                 float wy, float ww, float wh, double xform_clip) {
    dx = __fdiv_rn(dx, wx); dy = __fdiv_rn(dy, wy); dw = __fdiv_rn(dw, ww); dh = __fdiv_rn(dh, wh);
    const float widths = __fadd_rn(__fsub_rn(x2, x1), 1.f), heights = __fadd_rn(__fsub_rn(y2, y1), 1.f);
    const float ctr_x = __fadd_rn(x1, __fmul_rn(.5f, widths)), ctr_y = __fadd_rn(y1, __fmul_rn(.5f, heights));
    const float pcx = __fadd_rn(__fmul_rn(dx, widths), ctr_x), pcy = __fadd_rn(__fmul_rn(dy, heights), ctr_y);
    // np.minimum(d, clip): a NaN delta stays NaN (fmin would return the clip)
    const double dwc = (double)dw > xform_clip ? xform_clip : (double)dw, dhc = (double)dh > xform_clip ? xform_clip : (double)dh;
    const double pw = __dmul_rn(exp(dwc), (double)widths);
    const double ph = __dmul_rn(exp(dhc), (double)heights);
    const double hw = __dmul_rn(.5, pw), hh = __dmul_rn(.5, ph);
    return make_float4((float)__dsub_rn((double)pcx, hw), (float)__dsub_rn((double)pcy, hh),
                       (float)__dsub_rn(__dadd_rn((double)pcx, hw), 1.0), (float)__dsub_rn(__dadd_rn((double)pcy, hh), 1.0));
}

// np.maximum(np.minimum(v, hi), 0): NaN propagates, as it does through numpy (fminf / fmaxf alone would clip it)
__device__ __forceinline__ float clip_coord(float v, float hi) { return v != v ? v : fmaxf(fminf(v, hi), 0.f); }

}  // namespace b200
