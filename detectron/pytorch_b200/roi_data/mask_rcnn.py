"""Mask R-CNN training mask targets on the device (SURVEY.md 8f N4): add_mask_rcnn_blobs, lib/roi_data/mask_rcnn.py:34-122.

The reference runs one Python iteration per fg RoI, rasterising the best-matching object's polygons with pycocotools, and
hands the model an (n_fg, NUM_CLASSES * M * M) int32 host blob (32.5 MB per image at M = 28, 81 classes, 128 fg RoIs).  Here
every image of a step goes through one b200_mask_targets call (csrc/mask_targets.cu, 2 launches); the polygons are packed
on the host (ops.pack_polygons) and uploaded once, and the blobs come out as CUDA tensors.

Kept from the reference:
  * only objects with gt_classes > 0 and is_crowd == 0 have masks; an fg RoI matched to a crowd box still takes the best
    non-crowd polygon box by IoU (first maximum; zero IoU everywhere picks the first object);
  * mask_rois are the fg rows of `rois` (the same float32 arithmetic: unscaled box * im_scale, batch index in column 0);
  * an image without fg RoIs contributes its first bg RoI with an all -1 mask, class 0, and roi_has_mask_int32[0] = 1;
  * ValueError where the reference throws: no RoI at all, or fg RoIs but no non-crowd polygon (np.argmax of an empty row).
Configuration (MRCNN.RESOLUTION, MRCNN.CLS_SPECIFIC_MASK, MODEL.NUM_CLASSES) is read from `cfg` at call time, or from
keywords with the reference's defaults (14, True).
"""
import numpy as np
import torch

from .. import ops


def _config(cfg, resolution, cls_specific_mask, num_classes):
    if cfg is not None:
        return int(cfg.MRCNN.RESOLUTION), bool(cfg.MRCNN.CLS_SPECIFIC_MASK), int(cfg.MODEL.NUM_CLASSES)
    if cls_specific_mask and num_classes is None:
        raise ValueError("class-specific mask targets need num_classes (or cfg=)")
    return int(resolution), bool(cls_specific_mask), int(num_classes or 0)


def mask_polygons(entry):
    """The polygons of the roidb entry's objects that get masks (gt_classes > 0, is_crowd == 0), in roidb order."""
    cls = np.asarray(entry["gt_classes"]).reshape(-1)
    crowd = np.asarray(entry["is_crowd"]).reshape(-1) if "is_crowd" in entry else np.zeros(cls.shape, bool)
    inds = np.where((cls > 0) & (crowd == 0))[0]
    return [entry["segms"][i] for i in inds]


def mask_rcnn_blobs(labels, rois, boxes, num_fg, roidb, resolution=14, cls_specific_mask=True, num_classes=None):
    """The mask blobs of N images in one device call.  Per image n: labels[n] int32 (n_i,) and rois[n] float32 (n_i, 5) are the
    Fast R-CNN blobs, boxes[n] float32 (n_i, 4) the unscaled sampled boxes, all CUDA, with the num_fg[n] (host int) fg rows
    first, as _sample_rois orders them.  Returns dict(mask_rois, roi_has_mask_int32, masks_int32), concatenated over images."""
    M, K = int(resolution), (int(num_classes) if cls_specific_mask else 0)
    sel_boxes, sel_cls, roi_image, mask_rois, has_mask, polys = [], [], [], [], [], []
    for n, (lab, r, b, nf, entry) in enumerate(zip(labels, rois, boxes, num_fg, roidb)):
        nf = int(nf)
        if lab.numel() == 0:
            raise ValueError("image %d has no RoI at all (the reference indexes an empty bg list)" % n)
        obj = mask_polygons(entry)
        if nf > 0 and not obj:
            raise ValueError("image %d has fg RoIs but no non-crowd polygon (the reference's argmax of an empty row)" % n)
        h = (lab > 0).to(torch.int32)
        if nf > 0:
            sel_boxes.append(b[:nf]); sel_cls.append(lab[:nf].to(torch.int32)); mask_rois.append(r[:nf])
        else:                                       # the first bg RoI, class 0: an all -1 row (mask_rcnn.py:77-92)
            sel_boxes.append(b[:1]); sel_cls.append(torch.zeros((1,), dtype=torch.int32, device=lab.device)); mask_rois.append(r[:1])
            h[0] = 1
        roi_image += [n] * max(nf, 1)
        has_mask.append(h)
        polys.append(obj)
    masks = ops.mask_targets_raw(torch.cat(sel_boxes).contiguous(), roi_image, torch.cat(sel_cls), ops.pack_polygons(polys), M, K)
    return dict(mask_rois=torch.cat(mask_rois), roi_has_mask_int32=torch.cat(has_mask), masks_int32=masks)


def add_mask_rcnn_blobs(blobs, sampled_boxes, roidb, im_scale, batch_idx, cfg=None, resolution=14, cls_specific_mask=True,
                        num_classes=None):
    """The reference's signature for one image: blobs['labels_int32'] (CUDA int32), sampled_boxes (n, 4) unscaled float32 CUDA,
    roidb = the image's entry ('gt_classes', 'is_crowd', 'segms').  Adds 'mask_rois' (k, 5) float32, 'roi_has_mask_int32' (n,)
    and 'masks_int32' (k, NUM_CLASSES * M * M or M * M) int32, all CUDA.  One host read: the fg indices."""
    M, cls_specific, K = _config(cfg, resolution, cls_specific_mask, num_classes)
    labels = blobs["labels_int32"]
    if not torch.is_tensor(labels) or not labels.is_cuda or not torch.is_tensor(sampled_boxes) or not sampled_boxes.is_cuda:
        raise NotImplementedError("add_mask_rcnn_blobs runs on CUDA tensors (the targets are rasterised on the device)")
    labels = labels.reshape(-1).to(torch.int32)
    boxes = sampled_boxes.reshape(-1, 4).to(torch.float32)
    fg = torch.nonzero(labels > 0).reshape(-1)
    order = fg if fg.numel() else torch.nonzero(labels == 0).reshape(-1)[:1]
    if order.numel() == 0:
        raise ValueError("no RoI at all (the reference indexes an empty bg list)")
    sel = boxes[order]
    rois = torch.cat([torch.full((sel.size(0), 1), float(batch_idx), dtype=torch.float32, device=sel.device),
                      sel * float(np.float32(im_scale))], dim=1)
    out = mask_rcnn_blobs([labels[order]], [rois], [sel], [fg.numel()], [roidb], M, cls_specific, K)
    has = (labels > 0).to(torch.int32)
    if fg.numel() == 0:
        has[0] = 1
    blobs["mask_rois"] = out["mask_rois"][:max(fg.numel(), 1)]
    blobs["roi_has_mask_int32"] = has
    blobs["masks_int32"] = out["masks_int32"]
