"""Merge the per-level RPN proposals and hand them out to the RoI levels, on tensors (any device) -- the inference
path of `CollectAndDistributeFpnRpnProposalsOp`, lib/modeling/collect_and_distribute_fpn_rpn_proposals.py:10-119
(reference, numpy on the host).  Together with modeling/generate_proposals.py (device proposals) and
roi_align_fpn.RoIAlignFPNFunction (per-level RoIAlign written in restored order) the RoIs no longer leave the GPU
between the RPN heads and the box head; the only host read is the four per-level counts the launches need.

  collect     :72-87    concatenate the levels, keep the `post_nms_topN` best by score
  distribute  :90-119   level of every RoI (utils.fpn.map_rois_to_fpn_levels), per-level RoI blobs in ascending
                        original index, and `rois_idx_restore_int32` = the inverse of that regrouping

Equal scores: the reference's np.argsort(-scores) leaves their order unspecified; here the sort is stable (ties keep
concatenation order).

Training branch (:49-63).  The reference "reuses the data loader code": json_dataset.add_proposals (proposals / im_scale are
merged into every roidb entry behind its ground-truth boxes, best-gt assignment through cython_bbox.bbox_overlaps,
crowd_thresh = 0 so nothing is filtered) and roi_data.fast_rcnn.add_fast_rcnn_blobs (_sample_rois per image, concatenation,
_add_multilevel_rois).  Here the same blobs are produced on the device with roi_data/fast_rcnn.py (SURVEY.md 8f N4); the
random draws are inputs (`choices`), see there.  One batched sampler
(fast_rcnn.add_fast_rcnn_blobs, shared with modeling/generate_proposal_labels.py) labels every image of the minibatch with a
single host read.  With MODEL.MASK_ON the mask blobs (mask_rois, roi_has_mask_int32,
masks_int32 and the mask_rois FPN blobs) come from roi_data/mask_rcnn.py, and with MODEL.KEYPOINTS_ON the keypoint blobs
(keypoint_rois, keypoint_locations_int32, keypoint_weights, keypoint_loss_normalizer and the keypoint_rois FPN blobs) from
roi_data/keypoint_rcnn.py, on the device too.  Every blob sees the reference's merged roidb (fast_rcnn.roidb_assignment): a
proposal takes its best ground-truth box, crowd objects included; a ground-truth row maps to itself with overlap 1 and its own
class, or overlap -1 and class 0 when the entry's 'is_crowd' marks it, so that no crowd row is ever sampled.
"""
import torch
from torch import nn

from detectron.pytorch_b200.utils.fpn import map_rois_to_fpn_levels


def collect(roi_inputs, score_inputs, post_nms_topN):
    """roi_inputs: list of (R_l, 5) tensors, score_inputs: list of (R_l, 1) or (R_l,) tensors -> (min(R, topN), 5)."""
    rois = torch.cat([r.reshape(-1, 5) for r in roi_inputs], dim=0)
    scores = torch.cat([s.reshape(-1) for s in score_inputs], dim=0)
    order = torch.sort(scores, descending=True, stable=True).indices
    if post_nms_topN >= 0:
        order = order[:int(post_nms_topN)]
    return rois[order]


def distribute(rois, lvl_min, lvl_max, canonical_scale=224, canonical_level=4):
    """rois (R, 5) -> dict with 'rois', 'rois_fpn<lvl>' for lvl_min..lvl_max and 'rois_idx_restore_int32', exactly the
    blobs of the reference's inference path; plus 'counts' (python ints per level, one small host read)."""
    lvls = map_rois_to_fpn_levels(rois[:, 1:5], lvl_min, lvl_max, canonical_scale, canonical_level)
    order = torch.sort(lvls, stable=True).indices                      # level by level, ascending original index inside
    restore = torch.empty_like(order)
    restore[order] = torch.arange(order.numel(), device=order.device)
    counts = torch.bincount((lvls - lvl_min).long(), minlength=lvl_max - lvl_min + 1).tolist()
    out = {"rois": rois, "counts": counts}
    grouped = rois[order]
    start = 0
    for lvl, n in zip(range(lvl_min, lvl_max + 1), counts):
        out["rois_fpn%d" % lvl] = grouped[start:start + n]
        start += n
    out["rois_idx_restore_int32"] = restore.to(torch.int32)
    return out


class CollectAndDistributeFpnRpnProposalsOp(nn.Module):
    def __init__(self, rpn_min_level=2, rpn_max_level=6, roi_min_level=2, roi_max_level=5, post_nms_topN=None,
                 collect_scale=1, canonical_scale=224, canonical_level=4, cfg=None):
        """`cfg`: the reference's config object (FPN.RPN_*_LEVEL, FPN.ROI_*_LEVEL, FPN.RPN_COLLECT_SCALE,
        FPN.ROI_CANONICAL_*, TRAIN/TEST.RPN_POST_NMS_TOP_N are then read at call time); otherwise the keyword values
        (defaults = lib/core/config.py:700-723; post_nms_topN defaults to the TEST value 1000)."""
        super().__init__()
        self._cfg = cfg
        self._p = dict(rpn_min=rpn_min_level, rpn_max=rpn_max_level, roi_min=roi_min_level, roi_max=roi_max_level,
                       topn=1000 if post_nms_topN is None else post_nms_topN, scale=collect_scale, s0=canonical_scale,
                       k0=canonical_level)

    def _params(self):
        if self._cfg is None:
            return dict(self._p)
        c = self._cfg
        key = 'TRAIN' if self.training else 'TEST'
        return dict(rpn_min=c.FPN.RPN_MIN_LEVEL, rpn_max=c.FPN.RPN_MAX_LEVEL, roi_min=c.FPN.ROI_MIN_LEVEL,
                    roi_max=c.FPN.ROI_MAX_LEVEL, topn=c[key].RPN_POST_NMS_TOP_N, scale=c.FPN.RPN_COLLECT_SCALE,
                    s0=c.FPN.ROI_CANONICAL_SCALE, k0=c.FPN.ROI_CANONICAL_LEVEL)

    def forward(self, inputs, roidb=None, im_info=None, choices=None, train=None):
        """inputs: [rpn_rois_fpn<min> .. rpn_rois_fpn<max>, rpn_roi_probs_fpn<min> .. rpn_roi_probs_fpn<max>] tensors.
        Training (module in training mode): roidb = one dict per image with the ground truth ('boxes' (G, 4) unscaled,
        'gt_classes' (G,), 'is_crowd' (G,) where crowd objects exist; numpy or tensors), im_info = (N, 3) [height, width,
        scale]; `train` = the TRAIN / MODEL keys (dict, or taken from `cfg`): BATCH_SIZE_PER_IM, FG_FRACTION, FG_THRESH,
        BG_THRESH_HI, BG_THRESH_LO, NUM_CLASSES, BBOX_REG_WEIGHTS, CLS_AGNOSTIC_BBOX_REG, and for Mask R-CNN MASK_ON,
        MRCNN_RESOLUTION (default 14), CLS_SPECIFIC_MASK (default True), with the roidb entries' 'segms'; for Keypoint R-CNN
        KEYPOINTS_ON, HEATMAP_SIZE, NUM_KEYPOINTS, IMS_PER_BATCH (default 2), MIN_KEYPOINT_COUNT (default 20), with the roidb
        entries' 'gt_keypoints' (G, 3, K); choices = per image (fg_choice, bg_choice) or, with keypoints,
        (fg_choice, bg_choice, keypoint_choice), or None (device randperm)."""
        p = self._params()
        n = p["rpn_max"] - p["rpn_min"] + 1
        topn = int(p["topn"] * p["scale"] + 0.5)
        rois = collect(inputs[:n], inputs[n:], topn)
        if not self.training:
            return distribute(rois, p["roi_min"], p["roi_max"], p["s0"], p["k0"])
        if not rois.is_cuda:
            raise NotImplementedError("the training branch runs on CUDA tensors (labels / targets are computed on the device)")
        from detectron.pytorch_b200.roi_data import fast_rcnn as FR
        t = dict(train) if train is not None else None
        if t is None:
            if self._cfg is None:
                raise ValueError("training needs `train=` (or cfg=) for the TRAIN.* / MODEL.* keys")
            t = FR.train_keys(self._cfg)
        scales = torch.as_tensor(im_info, dtype=torch.float32)[:, 2].cpu()
        blobs = FR.add_fast_rcnn_blobs(rois, roidb, [float(s) for s in scales], t, choices)
        mask_on = bool(t.get("MASK_ON", False))
        kp_on = bool(t.get("KEYPOINTS_ON", False))
        # roi_data/fast_rcnn.py:251-283 (_add_multilevel_rois): the sampled rois go to their FPN levels
        d = distribute(blobs["rois"], p["roi_min"], p["roi_max"], p["s0"], p["k0"])
        for k, v in d.items():
            if k != "rois":
                blobs[k] = v
        if mask_on:
            # fast_rcnn.py:275-276: mask_rois to their FPN levels
            d = distribute(blobs["mask_rois"], p["roi_min"], p["roi_max"], p["s0"], p["k0"])
            for k, v in d.items():
                if k not in ("rois", "counts"):
                    blobs["mask_" + k] = v
        if kp_on:
            # fast_rcnn.py:277-278: keypoint_rois to their FPN levels
            d = distribute(blobs["keypoint_rois"], p["roi_min"], p["roi_max"], p["s0"], p["k0"])
            for k, v in d.items():
                if k not in ("rois", "counts"):
                    blobs["keypoint_" + k] = v
        return blobs
