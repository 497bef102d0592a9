"""The training labels of the RPN proposals for single-scale (C4) models, on the device -- `GenerateProposalLabelsOp`,
lib/modeling/generate_proposal_labels.py (reference, numpy on the host).

The reference calls json_dataset.add_proposals(roidb, rpn_rois, im_scales, crowd_thresh=0) (the proposals, scaled back by the
float32 1. / im_scale, are merged into every roidb entry behind its ground-truth boxes and take their best ground-truth box;
no crowd filtering) and roi_data.fast_rcnn.add_fast_rcnn_blobs (_sample_rois per image, concatenated; the mask and keypoint
blobs with MODEL.MASK_ON / MODEL.KEYPOINTS_ON).  Here roi_data/fast_rcnn.add_fast_rcnn_blobs does the same for the whole
minibatch at once, with one host read of the per-image counts for the sampling; the random draws are inputs (`choices`).  The
caller's roidb is not modified (the reference appends the proposals to it; nothing reads that afterwards).
"""
import numpy as np
import torch
from torch import nn

from detectron.pytorch_b200.roi_data import fast_rcnn as FR


class GenerateProposalLabelsOp(nn.Module):
    def __init__(self, cfg=None, train=None):
        """`cfg`: the reference's config object, read at call time (TRAIN.*, MODEL.*, MRCNN.*, KRCNN.*, see
        roi_data.fast_rcnn.train_keys); otherwise `train`, a dict of those keys (as CollectAndDistributeFpnRpnProposalsOp's)."""
        super().__init__()
        self._cfg = cfg
        self._train = None if train is None else dict(train)

    def forward(self, rpn_rois, roidb, im_info, choices=None, train=None):
        """rpn_rois: (R, 5) [batch index, x1, y1, x2, y2], numpy (as the reference passes it) or a CUDA tensor
        (GenerateProposalsOp with return_tensors=True); roidb: one entry per image with the ground truth ('boxes' (G, 4)
        unscaled, 'gt_classes' (G,), 'is_crowd' (G,) where crowd objects exist, 'segms' with MASK_ON, 'gt_keypoints' with
        KEYPOINTS_ON); im_info: (N, 3) [height, width, scale]; choices: per image (fg_choice, bg_choice) or, with keypoints,
        (fg_choice, bg_choice, keypoint_choice): the np.random.choice positions, or None (device randperm).  Returns
        get_fast_rcnn_blob_names() with FPN off as CUDA tensors: rois, labels_int32, bbox_targets, bbox_inside_weights,
        bbox_outside_weights (+ mask_rois, roi_has_mask_int32, masks_int32; + keypoint_rois, keypoint_locations_int32,
        keypoint_weights, keypoint_loss_normalizer)."""
        t = train if train is not None else self._train
        if t is None:
            if self._cfg is None:
                raise ValueError("GenerateProposalLabelsOp needs `train=` (or cfg=) for the TRAIN.* / MODEL.* keys")
            t = FR.train_keys(self._cfg)
        t = dict(t)
        if torch.is_tensor(rpn_rois):
            if not rpn_rois.is_cuda:
                raise NotImplementedError("rpn_rois must be numpy or a CUDA tensor (the labels are computed on the device)")
            rois = rpn_rois
        else:
            rois = torch.from_numpy(np.ascontiguousarray(rpn_rois, dtype=np.float32)).cuda()
        scales = torch.as_tensor(im_info, dtype=torch.float32)[:, 2].cpu()
        blobs = FR.add_fast_rcnn_blobs(rois, roidb, [float(s) for s in scales], t, choices)
        names = FR.get_fast_rcnn_blob_names(True, MASK_ON=t.get("MASK_ON", False), KEYPOINTS_ON=t.get("KEYPOINTS_ON", False))
        return {k: blobs[k] for k in names}
