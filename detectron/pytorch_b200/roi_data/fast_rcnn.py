"""RoI labels and box-regression targets on the device (SURVEY.md 8f N4).

Mirrors, for proposals that already live on the GPU, what the reference does per image on the host:
  * `bbox_overlaps`          lib/utils/cython_bbox.pyx:32-73
  * `assign_rois`            lib/datasets/json_dataset.py:429-490 (_merge_proposal_boxes_into_roidb) + :514-531
  * `roidb_assignment`       the same for a merged roidb entry, its ground-truth rows as :208-290 (_add_gt_annotations) left them
  * `sample_rois`            lib/roi_data/fast_rcnn.py:129-200 (_sample_rois), :203-248 (_compute_targets, _expand_bbox_targets)
Mask targets are in roi_data/mask_rcnn.py (device polygon rasteriser), keypoint targets in roi_data/keypoint_rcnn.py.

The random choice of the reference (`npr.choice(inds, size, replace=False)` = a permutation prefix) is an INPUT here: pass
the positions it picked (`fg_choice`, `bg_choice`, e.g. from the same numpy RandomState) for a bit-identical minibatch, or
leave them None for a torch.randperm draw on the device.
"""
import ctypes

import torch

from ..ops import _host_array, _launch, _need_cuda_f32, _ptr


def _boxes4(t, name):
    _need_cuda_f32(t, name)
    if t.dim() != 2 or t.size(1) != 4:
        raise ValueError("%s must be (N, 4) = [x1, y1, x2, y2], got %s" % (name, tuple(t.shape)))
    return t.contiguous()


def bbox_overlaps(boxes, query_boxes):
    """(N, K) float32 IoU, +1 pixel convention -- utils.cython_bbox.bbox_overlaps on CUDA tensors."""
    boxes = _boxes4(boxes, "boxes"); query_boxes = _boxes4(query_boxes, "query_boxes")
    N, K = boxes.size(0), query_boxes.size(0)
    out = torch.empty((N, K), dtype=torch.float32, device=boxes.device)
    _launch("b200_bbox_overlaps", boxes.device, boxes.data_ptr(), N, query_boxes.data_ptr(), K, out.data_ptr())
    return out


def assign_rois(boxes, gt_boxes, gt_classes):
    """Best ground-truth box per box: (max_overlaps float32, box_to_gt_ind int32 (-1: none), max_classes int32 (0: none))."""
    boxes = _boxes4(boxes, "boxes")
    N = boxes.size(0)
    G = int(gt_boxes.size(0)) if gt_boxes is not None else 0
    dev = boxes.device
    max_overlaps = torch.empty((N,), dtype=torch.float32, device=dev)
    argmax = torch.empty((N,), dtype=torch.int32, device=dev)
    max_classes = torch.empty((N,), dtype=torch.int32, device=dev)
    if G:
        gt_boxes = _boxes4(gt_boxes, "gt_boxes")
        gt_classes = gt_classes.to(device=dev, dtype=torch.int32).contiguous()
    _launch("b200_roi_assign", dev, boxes.data_ptr(), N, gt_boxes.data_ptr() if G else None, gt_classes.data_ptr() if G else None, G,
            max_overlaps.data_ptr(), argmax.data_ptr(), max_classes.data_ptr())
    return max_overlaps, argmax, max_classes


def roidb_assignment(boxes, gt_boxes, gt_classes, is_crowd=None):
    """assign_rois for the rows of a merged roidb entry, its G ground-truth boxes first: a ground-truth row keeps what
    _add_gt_annotations gave it -- itself, overlap 1 with its own class, or overlap -1 and class 0 when it is a crowd object
    (is_crowd: (G,) flags, host or device; None: no crowd) -- so that no crowd row is ever sampled and each of several
    identical boxes keeps its own class.  Proposal rows keep the IoU assignment, crowd objects included."""
    max_overlaps, argmax, max_classes = assign_rois(boxes, gt_boxes, gt_classes)
    G = int(gt_boxes.size(0)) if gt_boxes is not None else 0
    if G:
        dev = max_overlaps.device
        gcls = gt_classes.to(device=dev, dtype=torch.int32).reshape(-1)
        crowd = torch.zeros(G, dtype=torch.bool, device=dev) if is_crowd is None else torch.as_tensor(is_crowd).to(dev).reshape(-1) != 0
        if crowd.numel() != G:
            raise ValueError("is_crowd has %d flags for %d ground-truth boxes" % (crowd.numel(), G))
        max_overlaps[:G] = torch.where(crowd, -1.0, 1.0)
        max_classes[:G] = torch.where(crowd, 0, gcls)
        argmax[:G] = torch.arange(G, dtype=torch.int32, device=dev)
    return max_overlaps, argmax, max_classes


def select_fg_bg(max_overlaps, fg_thresh, bg_thresh_hi, bg_thresh_lo):
    """np.where(max_overlaps >= fg) and np.where((max_overlaps < hi) & (max_overlaps >= lo)) as ascending int32 index tensors
    (one host read of the two counts)."""
    max_overlaps = max_overlaps.contiguous()
    N = max_overlaps.numel()
    dev = max_overlaps.device
    fg = torch.empty((N,), dtype=torch.int32, device=dev)
    bg = torch.empty((N,), dtype=torch.int32, device=dev)
    counts = torch.empty((2,), dtype=torch.int32, device=dev)
    _launch("b200_roi_select", dev, max_overlaps.data_ptr(), N, float(fg_thresh), float(bg_thresh_hi), float(bg_thresh_lo), fg.data_ptr(),
            bg.data_ptr(), counts.data_ptr())
    nf, nb = counts.tolist()
    return fg[:nf], bg[:nb]


def sample_rois(boxes, gt_boxes, gt_classes, im_scale, batch_idx, num_classes, batch_size_per_im=512, fg_fraction=0.25,
                fg_thresh=0.5, bg_thresh_hi=0.5, bg_thresh_lo=0.0, bbox_reg_weights=(10.0, 10.0, 5.0, 5.0),
                cls_agnostic_bbox_reg=False, fg_choice=None, bg_choice=None, assignment=None, is_crowd=None):
    """_sample_rois for one image.  `boxes`: the roidb's boxes (ground truth first, then proposals; unscaled image
    coordinates); is_crowd: the roidb's crowd flags of the ground-truth rows.  Returns the reference's blob dict with CUDA
    tensors: labels_int32, rois, bbox_targets, bbox_inside_weights, bbox_outside_weights (+ keep_inds, the rows of `boxes`
    that were sampled).  assignment: (max_overlaps, box_to_gt_ind, max_classes) when the caller already has them
    (roidb_assignment)."""
    return _sample_rois(boxes, gt_boxes, gt_classes, im_scale, batch_idx, num_classes, batch_size_per_im, fg_fraction, fg_thresh,
                        bg_thresh_hi, bg_thresh_lo, bbox_reg_weights, cls_agnostic_bbox_reg, fg_choice, bg_choice, assignment, is_crowd)[0]


def _sample_rois(boxes, gt_boxes, gt_classes, im_scale, batch_idx, num_classes, batch_size_per_im, fg_fraction, fg_thresh, bg_thresh_hi,
                 bg_thresh_lo, bbox_reg_weights, cls_agnostic_bbox_reg, fg_choice, bg_choice, assignment, is_crowd=None):
    """sample_rois' blobs and the number of fg rows (a host int; they come first)."""
    boxes = _boxes4(boxes, "boxes")
    dev = boxes.device
    if assignment is None:
        assignment = roidb_assignment(boxes, gt_boxes, gt_classes, is_crowd)
    max_overlaps, argmax, max_classes = assignment
    rois_per_image = int(batch_size_per_im)
    fg_rois_per_image = int(round(fg_fraction * rois_per_image))
    fg_inds, bg_inds = select_fg_bg(max_overlaps, fg_thresh, bg_thresh_hi, bg_thresh_lo)

    def pick(inds, size, choice):
        if inds.numel() == 0:
            return inds
        if choice is None:
            choice = torch.randperm(inds.numel(), device=dev)[:size]
        else:
            choice = torch.as_tensor(choice, device=dev, dtype=torch.long)
            if choice.numel() != size:
                raise ValueError("choice has %d entries, the minibatch takes %d" % (choice.numel(), size))
        return inds[choice.long()]

    n_fg = min(fg_rois_per_image, fg_inds.numel())
    fg_keep = pick(fg_inds, n_fg, fg_choice)
    n_bg = min(rois_per_image - n_fg, bg_inds.numel())
    bg_keep = pick(bg_inds, n_bg, bg_choice)
    keep = torch.cat([fg_keep, bg_keep]).to(torch.int32).contiguous()
    n = keep.numel()
    reg_classes = 2 if cls_agnostic_bbox_reg else int(num_classes)
    labels = torch.empty((n,), dtype=torch.int32, device=dev)
    rois = torch.empty((n, 5), dtype=torch.float32, device=dev)
    targets = torch.empty((n, 4 * reg_classes), dtype=torch.float32, device=dev)
    inside = torch.empty_like(targets)
    outside = torch.empty_like(targets)
    if len(bbox_reg_weights) != 4:
        raise ValueError("bbox_reg_weights must be 4 values (wx, wy, ww, wh), got %d" % len(bbox_reg_weights))
    w = _host_array(ctypes.c_float, [float(v) for v in bbox_reg_weights])
    G = int(gt_boxes.size(0)) if gt_boxes is not None else 0
    gt = _boxes4(gt_boxes, "gt_boxes") if G else None
    _launch("b200_fast_rcnn_targets", dev, boxes.data_ptr(), _ptr(gt), argmax.data_ptr(), max_classes.data_ptr(), keep.data_ptr(), n, n_fg,
            w, reg_classes, 1 if cls_agnostic_bbox_reg else 0, float(im_scale), float(batch_idx), labels.data_ptr(), rois.data_ptr(),
            targets.data_ptr(), inside.data_ptr(), outside.data_ptr())
    return dict(labels_int32=labels, rois=rois, bbox_targets=targets, bbox_inside_weights=inside, bbox_outside_weights=outside,
                keep_inds=keep), n_fg
