"""Host-array front door of the device NMS, shaped like the reference's `utils.boxes.nms`
(lib/utils/boxes.py:320-324: numpy (N, 5) [x1, y1, x2, y2, score] in any order -> kept indices).

`generate_proposals.py:161` and `core/test.py:764` call `box_utils.nms(dets, thresh)` with numpy arrays; re-pointing
that name at this function (`install_reference_aliases(nms=True)` or `utils.boxes.nms = nms`) moves the O(N^2) work to
the device while the callers stay unchanged.  Flavour note: this is the routine the reference calls there,
cython_nms.nms (lib/utils/cython_nms.pyx:37-87): both box areas rounded on their own, IoU = inter / ((area_i + area_j) -
inter) in float32, suppress when IoU >= float32(thresh).  It runs as one problem of `b200_nms_batched_cython`.  The
proposal layer of this package (modeling/generate_proposals.py) and `nms_gpu` keep the reference CUDA kernel's fused
area and `IoU > thresh` instead (lib/model/nms/src/nms_cuda_kernel.cu:31-39); the two differ on pairs whose IoU lies
within about one ulp of the threshold, for example integer boxes whose IoU is exactly 0.5 or 7/10.

Tied scores: the reference orders by `scores.argsort()[::-1]`, which is not stable, so among boxes with equal scores its
order is arbitrary; here they go lower index first.  The results differ only where tied boxes overlap each other.
"""
import numpy as np
import torch

from .. import ops


def nms(dets, thresh):
    """Classic greedy NMS.  Returns the kept row indices in ascending order, like cython_nms.nms
    (`np.where(suppressed == 0)[0]`, lib/utils/cython_nms.pyx:87).  Up to ~13 800 rows (b200_nms_batched_cython)."""
    if dets.shape[0] == 0:
        return []
    dets = np.ascontiguousarray(dets, dtype=np.float32)
    order = np.argsort(-dets[:, 4], kind="stable")                  # the batched NMS expects score-sorted rows
    keep, num = ops.nms_batched_raw(torch.from_numpy(dets[order]).cuda(), [dets.shape[0]], float(thresh), cython=True)
    return np.sort(order[keep[:int(num[0])].cpu().numpy()]).astype(np.int64)


def flip_boxes(boxes, im_width):
    """lib/utils/boxes.py:252-257: boxes (R, 4k) mirrored in an image of width im_width (x -> im_width - x - 1), host numpy."""
    boxes_flipped = boxes.copy()
    boxes_flipped[:, 0::4] = im_width - boxes[:, 2::4] - 1
    boxes_flipped[:, 2::4] = im_width - boxes[:, 0::4] - 1
    return boxes_flipped


def aspect_ratio(boxes, aspect_ratio):
    """lib/utils/boxes.py:260-265: the x coordinates of boxes (R, 4k) scaled by aspect_ratio, host numpy."""
    boxes_ar = boxes.copy()
    boxes_ar[:, 0::4] = aspect_ratio * boxes[:, 0::4]
    boxes_ar[:, 2::4] = aspect_ratio * boxes[:, 2::4]
    return boxes_ar
