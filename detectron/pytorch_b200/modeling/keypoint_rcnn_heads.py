"""Keypoint R-CNN keypoint loss on device or host target blobs (lib/modeling/keypoint_rcnn_heads.py:91-122).

The reference converts the host blobs with `torch.from_numpy(...astype('int64'))` and copies them to the GPU; with the targets
built on the device (roi_data/keypoint_rcnn.py) they are already CUDA tensors, and the normalizer is a 0-d CUDA tensor whose
`.item()` would stall the step.  Same math: cross entropy over the HEATMAP_SIZE^2 locations, summed with the weights,
divided by their sum, times KRCNN.LOSS_WEIGHT, times the normalizer when the loss is not normalised by the visible
keypoints.  A target whose weight is 0 is set to 0 first: its product with the weight is unchanged, and a location of INT_MIN
(the reference's label of a keypoint against a zero-width box) would otherwise be an out-of-range class.
"""
import torch
import torch.nn.functional as F


def keypoint_losses(kps_pred, keypoint_locations_int32, keypoint_weights, keypoint_loss_normalizer=None, cfg=None, heatmap_size=None,
                    loss_weight=None, normalize_by_visible_keypoints=None):
    """kps_pred (R, K, HS, HS) logits; keypoint_locations_int32 / keypoint_weights (R * K,) tensors or numpy arrays, on any
    device; keypoint_loss_normalizer: a tensor or a numpy scalar.  heatmap_size, loss_weight (default 1.0) and
    normalize_by_visible_keypoints come from cfg.KRCNN when not given; without cfg the normalizer is applied exactly when it
    is passed."""
    if cfg is not None:
        heatmap_size = cfg.KRCNN.HEATMAP_SIZE if heatmap_size is None else heatmap_size
        loss_weight = cfg.KRCNN.LOSS_WEIGHT if loss_weight is None else loss_weight
        if normalize_by_visible_keypoints is None:
            normalize_by_visible_keypoints = cfg.KRCNN.NORMALIZE_BY_VISIBLE_KEYPOINTS
    if heatmap_size is None:
        heatmap_size = kps_pred.size(-1)
    if normalize_by_visible_keypoints is None:
        normalize_by_visible_keypoints = keypoint_loss_normalizer is None
    dev = kps_pred.device
    weights = torch.as_tensor(keypoint_weights).to(device=dev, dtype=torch.float32).reshape(-1)
    target = torch.as_tensor(keypoint_locations_int32).to(device=dev).reshape(-1).long()
    target = torch.where(weights > 0, target, torch.zeros_like(target))
    loss = F.cross_entropy(kps_pred.reshape(-1, int(heatmap_size) ** 2), target, reduction="none")
    loss = torch.sum(loss * weights) / torch.sum(weights)
    loss = loss * (1.0 if loss_weight is None else float(loss_weight))
    if not normalize_by_visible_keypoints:
        loss = loss * torch.as_tensor(keypoint_loss_normalizer).to(device=dev, dtype=loss.dtype)
    return loss
