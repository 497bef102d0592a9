"""Fast R-CNN box-head losses on device or host target blobs (lib/modeling/fast_rcnn_heads.py:50-68).

The reference converts the host blobs with `torch.from_numpy(label_int32.astype('int64'))` and copies them to the GPU; with the
targets built on the device (roi_data/fast_rcnn.py, the training branch of collect_and_distribute_fpn_rpn_proposals.py) they are
already CUDA tensors, which `.astype` cannot take.  Same math (cross entropy averaged over the RoIs, net_utils.smooth_l1_loss with
beta = 1 divided by R, the class accuracy of the argmax) in one launch forward and one backward (csrc/losses.cu).
"""
from .. import ops


def fast_rcnn_losses(cls_score, bbox_pred, label_int32, bbox_targets, bbox_inside_weights, bbox_outside_weights):
    """cls_score (R, C) and bbox_pred (R, 4 C') float32 CUDA; label_int32 (R,) int32 / int64 and the (R, 4 C') target and weight
    blobs as CUDA tensors or numpy arrays.  Returns (loss_cls, loss_bbox, accuracy_cls), 0-d CUDA tensors; accuracy_cls has no
    gradient.  Numpy labels outside [0, C) raise ValueError; on the device such a label gives a NaN loss_cls."""
    return ops.fast_rcnn_losses(cls_score, bbox_pred, label_int32, bbox_targets, bbox_inside_weights, bbox_outside_weights)
