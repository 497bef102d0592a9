"""numpy restatement of the box head's decode of one test-time transform and of the box combine.  TEST INFRASTRUCTURE ONLY.

  * im_detect_bbox's decode                lib/core/test.py:154-189
  * the flipped / aspect-ratio inverses    lib/core/test.py:289-362, lib/utils/boxes.py:252-265
  * SCORE_HEUR / COORD_HEUR                lib/core/test.py:262-284

Precision as the reference's lines evaluate under numpy >= 2 (pinned by tests/golden/detect_bbox.npz): the model's rois are
divided by the one-element list im_scale in float64; the deltas are divided by the weights in float32 and decoded by
oracle/proposals.bbox_transform, the proposal layer's decode with weights 1; the clip,
flip and aspect inverses run in the dtype of the boxes (float32 after a decode, float64 for undecoded rois), with the image
width and 1 / aspect_ratio as Python numbers (weak scalars).
"""
import numpy as np

from . import proposals as P


def decode(boxes, deltas, num_classes, im_h, im_w, im_scale=None, bbox_reg=True, weights=(10.0, 10.0, 5.0, 5.0), agnostic=False,
           flip_width=None, ar_inv=1.0):
    """pred_boxes (R, 4K) float32 of one transform: boxes the model's rois (R, 5) with im_scale, or float32 proposals (R, 4)."""
    K = int(num_classes)
    b = np.asarray(boxes)
    b = b[:, 1:5] / [im_scale] if im_scale is not None else b.astype(np.float32, copy=False)
    R = b.shape[0]
    if bbox_reg:
        d = np.asarray(deltas, dtype=np.float32)
        d = d[:, -4:] if agnostic else d
        k = d.shape[1] // 4
        # the reference's `deltas[:, i::4] / w*` (float32, Python-float weights), then proposals.bbox_transform's weight-1 decode
        d = d.reshape(R * k, 4) / np.array([float(w) for w in weights], dtype=np.float32)
        out = P.bbox_transform(np.repeat(b, k, axis=0), d).reshape(R, 4 * k)
        out[:, 0::4] = np.maximum(np.minimum(out[:, 0::4], im_w - 1), 0)
        out[:, 1::4] = np.maximum(np.minimum(out[:, 1::4], im_h - 1), 0)
        out[:, 2::4] = np.maximum(np.minimum(out[:, 2::4], im_w - 1), 0)
        out[:, 3::4] = np.maximum(np.minimum(out[:, 3::4], im_h - 1), 0)
        if agnostic:
            out = np.tile(out, (1, K))
    else:
        out = np.tile(b, (1, K))
    if flip_width is not None:
        f = out.copy()
        f[:, 0::4] = int(flip_width) - out[:, 2::4] - 1
        f[:, 2::4] = int(flip_width) - out[:, 0::4] - 1
        out = f
    if ar_inv != 1.0:
        out[:, 0::4] = float(ar_inv) * out[:, 0::4]
        out[:, 2::4] = float(ar_inv) * out[:, 2::4]
    return out.astype(np.float32, copy=False)


def combine(outs, heur, identity):
    """SCORE_HEUR / COORD_HEUR over the transforms' outputs (the identity's is `identity`)."""
    if heur == "ID":
        return identity
    if heur == "AVG":
        return np.mean(outs, axis=0)
    return np.vstack(outs)
