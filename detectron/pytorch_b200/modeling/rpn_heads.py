"""Single-scale RPN losses (lib/modeling/rpn_heads.py:29-34, 130-161) in one launch forward and one backward.

The reference narrows the four "wide" target blobs to the prediction's h x w and runs net_utils.smooth_l1_loss (about a dozen
elementwise ops) plus the BCE or cross entropy, a weight mask and a sum.  Here csrc/losses.cu reads the [:h, :w] window of each wide
blob in place and evaluates every element with the same float32 operations (ops.rpn_losses).

Configuration: pass the reference's `cfg` (read at call time: RPN.CLS_ACTIVATION, FPN.FPN_ON, FPN.RPN_MIN_LEVEL / RPN_MAX_LEVEL,
TRAIN.RPN_BATCH_SIZE_PER_IM, TRAIN.IMS_PER_BATCH) or the same values as keywords (see `_DEFAULTS`, the reference's config
defaults).
"""
from .. import ops

_DEFAULTS = dict(cls_activation="sigmoid", fpn_on=False, rpn_min_level=2, rpn_max_level=6, rpn_batch_size_per_im=256, ims_per_batch=2)


def _params(cfg, kw):
    p = dict(_DEFAULTS)
    if cfg is not None:
        p.update(cls_activation=cfg.RPN.CLS_ACTIVATION, fpn_on=bool(cfg.FPN.FPN_ON), rpn_min_level=cfg.FPN.RPN_MIN_LEVEL,
                 rpn_max_level=cfg.FPN.RPN_MAX_LEVEL, rpn_batch_size_per_im=cfg.TRAIN.RPN_BATCH_SIZE_PER_IM,
                 ims_per_batch=cfg.TRAIN.IMS_PER_BATCH)
    unknown = set(kw) - set(_DEFAULTS)
    if unknown:
        raise TypeError("unknown RPN loss parameters: %s" % sorted(unknown))
    p.update(kw)
    if p["cls_activation"] not in ("sigmoid", "softmax"):
        raise ValueError("RPN.CLS_ACTIVATION must be 'sigmoid' or 'softmax', got %r" % (p["cls_activation"],))
    return p


def _split_params(kwargs):
    conf = {k: kwargs.pop(k) for k in list(kwargs) if k in _DEFAULTS}
    return kwargs.pop("cfg", None), conf


def generic_rpn_losses(*inputs, **kwargs):
    """FPN.fpn_rpn_losses when FPN.FPN_ON (keyword `fpn_on`), else single_scale_rpn_losses."""
    cfg, conf = _split_params(kwargs)
    if _params(cfg, conf)["fpn_on"]:
        from . import FPN
        return FPN.fpn_rpn_losses(*inputs, cfg=cfg, **conf, **kwargs)
    return single_scale_rpn_losses(*inputs, cfg=cfg, **conf, **kwargs)


def single_scale_rpn_losses(rpn_cls_logits, rpn_bbox_pred, rpn_labels_int32_wide, rpn_bbox_targets_wide, rpn_bbox_inside_weights_wide,
                            rpn_bbox_outside_weights_wide, cfg=None, **kw):
    """(loss_rpn_cls, loss_rpn_bbox), 0-d CUDA tensors.  rpn_cls_logits (N, A, h, w) (sigmoid) or (N, 2A, h, w) (softmax) and
    rpn_bbox_pred (N, 4A, h', w') float32 CUDA; the wide blobs (N, A, >= h, >= w) int32 and (N, 4A, >= h', >= w') float32.  The
    cls loss is divided by the number of labels >= 0 (the ignored label is -1), the box loss by N."""
    p = _params(cfg, kw)
    losses = ops.rpn_losses([(rpn_cls_logits, rpn_bbox_pred, rpn_labels_int32_wide, rpn_bbox_targets_wide, rpn_bbox_inside_weights_wide,
                              rpn_bbox_outside_weights_wide)], softmax=p["cls_activation"] == "softmax")
    loss_cls, loss_bbox = losses[0].unbind(0)
    return loss_cls, loss_bbox
