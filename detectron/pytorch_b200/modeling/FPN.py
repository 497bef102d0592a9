"""FPN RPN losses (lib/modeling/FPN.py:422-466): every level of a step in one launch forward and one backward (ops.rpn_losses).

The sigmoid cls loss of each level is divided by TRAIN.RPN_BATCH_SIZE_PER_IM * TRAIN.IMS_PER_BATCH, the softmax one by its
number of labels other than -1; the box loss by N.  Configuration as in rpn_heads.py.
"""
from .. import ops
from .rpn_heads import _params


def fpn_rpn_losses(cfg=None, rpn_min_level=None, rpn_max_level=None, cls_activation=None, rpn_batch_size_per_im=None, ims_per_batch=None,
                   fpn_on=None, **kwargs):
    """kwargs: rpn_cls_logits_fpn<l>, rpn_bbox_pred_fpn<l> and the four rpn_*_wide_fpn<l> blobs for every level l from
    RPN_MIN_LEVEL to RPN_MAX_LEVEL (other keys are ignored, as the reference ignores them).  Returns (losses_cls, losses_bbox):
    per-level lists of 0-d CUDA tensors, views of one (L, 2) result."""
    conf = {k: v for k, v in dict(rpn_min_level=rpn_min_level, rpn_max_level=rpn_max_level, cls_activation=cls_activation,
                                  rpn_batch_size_per_im=rpn_batch_size_per_im, ims_per_batch=ims_per_batch).items() if v is not None}
    p = _params(cfg, conf)
    levels = []
    for lvl in range(p["rpn_min_level"], p["rpn_max_level"] + 1):
        s = str(lvl)
        names = ["rpn_cls_logits_fpn" + s, "rpn_bbox_pred_fpn" + s] + [k + "_fpn" + s for k in (
            "rpn_labels_int32_wide", "rpn_bbox_targets_wide", "rpn_bbox_inside_weights_wide", "rpn_bbox_outside_weights_wide")]
        missing = [k for k in names if k not in kwargs]
        if missing:
            raise ValueError("fpn_rpn_losses: missing %s" % missing)
        levels.append(tuple(kwargs[k] for k in names))
    softmax = p["cls_activation"] == "softmax"
    divisor = 0.0 if softmax else float(p["rpn_batch_size_per_im"] * p["ims_per_batch"])
    losses = ops.rpn_losses(levels, softmax=softmax, fixed_divisor=divisor)
    cls, bbox = losses.unbind(1)
    return list(cls.unbind(0)), list(bbox.unbind(0))
