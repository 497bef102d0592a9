"""Mask R-CNN mask loss on a device target blob (lib/modeling/mask_rcnn_heads.py:90-99).

The reference converts the host int32 blob with `.astype('float32')` and copies it to the GPU; with the targets built on the
device (roi_data/mask_rcnn.py) `masks_int32` is already a CUDA int32 tensor, which `.astype` cannot take.  Same math:
per-element BCE-with-logits summed over the elements whose target is not -1, divided by their count, times
MRCNN.WEIGHT_LOSS_MASK.
"""
import torch
import torch.nn.functional as F


def mask_rcnn_losses(masks_pred, masks_int32, weight_loss_mask=None, cfg=None):
    """masks_pred (R, C, M, M) logits; masks_int32 (R, C * M * M) int32 in {1, 0, -1} (-1: ignore), a tensor or a numpy array.
    weight_loss_mask: the loss weight, else cfg.MRCNN.WEIGHT_LOSS_MASK, else 1.0."""
    if weight_loss_mask is None:
        weight_loss_mask = float(cfg.MRCNN.WEIGHT_LOSS_MASK) if cfg is not None else 1.0
    n_rois = masks_pred.size(0)
    masks_gt = torch.as_tensor(masks_int32).to(device=masks_pred.device, dtype=torch.float32)
    weight = (masks_gt > -1).float()
    loss = F.binary_cross_entropy_with_logits(masks_pred.view(n_rois, -1), masks_gt, weight, reduction="sum")
    loss = loss / weight.sum()
    return loss * weight_loss_mask
