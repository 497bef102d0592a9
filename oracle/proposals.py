"""numpy restatement of the reference's RPN proposal layer.  TEST INFRASTRUCTURE ONLY (SURVEY.md 8f N1).

Follows, step for step and in float32 like the reference (whose arrays come from `.cpu().numpy()` of fp32 tensors):

  * GenerateProposalsOp.forward / proposals_for_one_image   lib/modeling/generate_proposals.py:19-104, 106-168
  * _filter_boxes                                           lib/modeling/generate_proposals.py:171-182
  * bbox_transform (weights (1, 1, 1, 1))                   lib/utils/boxes.py:157-196
  * clip_tiled_boxes                                        lib/utils/boxes.py:138-154
  * BBOX_XFORM_CLIP = log(1000 / 16)                        lib/core/config.py:936

Two places where the reference is not a function of its inputs are made deterministic here and documented as such:
  * top-k: the reference orders the pre-NMS candidates with np.argpartition + np.argsort (unstable: equal scores come
    out in an unspecified order); this restatement uses a stable descending sort, i.e. ties keep ascending anchor
    index in (H, W, A) order and NaN scores come last -- the rule b200_topk_batched and the torch.sort fallback follow;
  * NMS: the reference calls utils.boxes.nms -> cython_nms.nms on the host (suppress when IoU >= thresh).  The device
    path uses the CUDA kernel's semantics (IoU > thresh, the SASS rounding recipe); `nms="cuda"` (default) selects
    oracle_nms_cuda, `nms="cython"` the restatement of the Cython routine, so both can be compared.
Pinning: the reference ships no golden outputs for this layer, so tests/golden/make_golden_proposals.py runs the
UNMODIFIED reference op (GenerateProposalsOp + utils.boxes + the reference's own Cython NMS, built from a patched copy
in a temp dir) on seeded inputs on the CPU and stores inputs and outputs in tests/golden/proposals.npz;
tests/test_oracle_proposals.py requires this restatement to reproduce them bit for bit (nms="cython"), and requires
the same result with the CUDA NMS semantics on those inputs.  See bbox_transform for the precision the reference's
lines actually evaluate in.
"""
import numpy as np

from . import cpu as O

BBOX_XFORM_CLIP = np.float64(np.log(1000.0 / 16.0))       # core/config.py:936 -- an np.float64 SCALAR, see bbox_transform


def shifted_anchors(anchors, height, width, feat_stride):
    """(H*W*A, 4) anchors in (H, W, A) order -- generate_proposals.py:66-89."""
    shift_x = np.arange(0, width) * feat_stride
    shift_y = np.arange(0, height) * feat_stride
    shift_x, shift_y = np.meshgrid(shift_x, shift_y, copy=False)
    shifts = np.vstack((shift_x.ravel(), shift_y.ravel(), shift_x.ravel(), shift_y.ravel())).transpose()
    A, K = anchors.shape[0], shifts.shape[0]
    return (np.asarray(anchors, dtype=np.float64)[np.newaxis, :, :] + shifts[:, np.newaxis, :]).reshape((K * A, 4))


def bbox_transform(boxes, deltas):
    """boxes (n, 4), deltas (n, 4) float32 -> decoded boxes (n, 4) float32 -- utils/boxes.py:157-196.

    Precision, as the reference's lines evaluate under numpy >= 2 (the only numpy the reference can be run with here;
    the golden vectors pin exactly this): widths / centres / dx * w + ctr are float32; `np.minimum(dw, cfg.BBOX_XFORM_CLIP)`
    promotes dw, dh to float64 because the clip constant is an np.float64 scalar, so exp, exp * width and the final
    `ctr -/+ 0.5 * pred_w (- 1)` run in float64 and are rounded to float32 once, on assignment into the float32 output.
    (Under numpy 1.x value-based casting the same lines stayed in float32; the two differ by <= 1 ulp.)"""
    boxes = boxes.astype(np.float32, copy=False)
    deltas = deltas.astype(np.float32, copy=False)
    one, half = np.float32(1.0), np.float32(0.5)
    widths = boxes[:, 2] - boxes[:, 0] + one
    heights = boxes[:, 3] - boxes[:, 1] + one
    ctr_x = boxes[:, 0] + half * widths
    ctr_y = boxes[:, 1] + half * heights
    dx, dy = deltas[:, 0], deltas[:, 1]
    dw = np.minimum(deltas[:, 2].astype(np.float64), BBOX_XFORM_CLIP)
    dh = np.minimum(deltas[:, 3].astype(np.float64), BBOX_XFORM_CLIP)
    pred_ctr_x = (dx * widths + ctr_x).astype(np.float64)            # float32 arithmetic, then widened
    pred_ctr_y = (dy * heights + ctr_y).astype(np.float64)
    pred_w = np.exp(dw) * widths.astype(np.float64)
    pred_h = np.exp(dh) * heights.astype(np.float64)
    out = np.zeros(deltas.shape, dtype=np.float32)
    out[:, 0] = pred_ctr_x - 0.5 * pred_w
    out[:, 1] = pred_ctr_y - 0.5 * pred_h
    out[:, 2] = pred_ctr_x + 0.5 * pred_w - 1
    out[:, 3] = pred_ctr_y + 0.5 * pred_h - 1
    return out


def clip_boxes(boxes, im_h, im_w):
    """utils/boxes.py:138-154 (float32 image size, as im_info holds it)."""
    wmax, hmax = np.float32(im_w) - np.float32(1), np.float32(im_h) - np.float32(1)
    boxes = boxes.copy()
    boxes[:, 0] = np.maximum(np.minimum(boxes[:, 0], wmax), 0)
    boxes[:, 1] = np.maximum(np.minimum(boxes[:, 1], hmax), 0)
    boxes[:, 2] = np.maximum(np.minimum(boxes[:, 2], wmax), 0)
    boxes[:, 3] = np.maximum(np.minimum(boxes[:, 3], hmax), 0)
    return boxes


def filter_boxes(boxes, min_size, im_info):
    """generate_proposals.py:171-182: both sides >= min_size * scale and centre inside the image."""
    min_size = np.float32(min_size) * np.float32(im_info[2])
    one = np.float32(1.0)
    ws = boxes[:, 2] - boxes[:, 0] + one
    hs = boxes[:, 3] - boxes[:, 1] + one
    x_ctr = boxes[:, 0] + ws / np.float32(2.0)
    y_ctr = boxes[:, 1] + hs / np.float32(2.0)
    return np.where((ws >= min_size) & (hs >= min_size) & (x_ctr < np.float32(im_info[1])) & (y_ctr < np.float32(im_info[0])))[0]


def proposals_for_one_image(im_info, anchors, feat_stride, bbox_deltas, scores, pre_nms_topN, post_nms_topN, nms_thresh,
                            min_size, nms="cuda"):
    """bbox_deltas (4A, H, W), scores (A, H, W) of ONE image -> (proposals (n, 4), scores (n, 1)) float32."""
    A, H, W = scores.shape
    all_anchors = shifted_anchors(anchors, H, W, feat_stride)
    deltas = np.ascontiguousarray(bbox_deltas, dtype=np.float32).transpose((1, 2, 0)).reshape((-1, 4))
    sc = np.ascontiguousarray(scores, dtype=np.float32).transpose((1, 2, 0)).reshape(-1)
    order = np.argsort(-sc, kind="stable")
    if 0 < pre_nms_topN < len(sc):
        order = order[:pre_nms_topN]
    proposals = bbox_transform(all_anchors[order, :], deltas[order, :])
    proposals = clip_boxes(proposals, im_info[0], im_info[1])
    sc = sc[order]
    keep = filter_boxes(proposals, min_size, im_info)
    proposals, sc = proposals[keep, :], sc[keep]
    if nms_thresh > 0 and len(sc):
        dets = np.hstack((proposals, sc[:, None])).astype(np.float32)
        k = O.nms_cuda(dets, nms_thresh) if nms == "cuda" else O.nms_cython(dets, nms_thresh)
        k = np.asarray(k, dtype=np.int64).reshape(-1)
        if post_nms_topN > 0:
            k = k[:post_nms_topN]
        proposals, sc = proposals[k, :], sc[k]
    return proposals, sc.reshape(-1, 1)


def generate_proposals(rpn_cls_prob, rpn_bbox_pred, im_info, anchors, feat_stride, pre_nms_topN, post_nms_topN, nms_thresh,
                       min_size, nms="cuda"):
    """The whole op: (N, A, H, W), (N, 4A, H, W), (N, 3) -> rois (R, 5) [batch, x1, y1, x2, y2], roi_probs (R, 1)."""
    rois = np.empty((0, 5), dtype=np.float32)
    probs = np.empty((0, 1), dtype=np.float32)
    for i in range(rpn_cls_prob.shape[0]):
        b, s = proposals_for_one_image(im_info[i], anchors, feat_stride, rpn_bbox_pred[i], rpn_cls_prob[i], pre_nms_topN,
                                       post_nms_topN, nms_thresh, min_size, nms=nms)
        rois = np.append(rois, np.hstack((np.full((b.shape[0], 1), i, dtype=np.float32), b)), axis=0)
        probs = np.append(probs, s, axis=0)
    return rois, probs
