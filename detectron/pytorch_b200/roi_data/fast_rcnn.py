"""RoI labels and box-regression targets on the device (SURVEY.md 8f N4).

Mirrors, for proposals that already live on the GPU, what the reference does per image on the host:
  * `bbox_overlaps`          lib/utils/cython_bbox.pyx:32-73
  * `assign_rois`            lib/datasets/json_dataset.py:429-490 (_merge_proposal_boxes_into_roidb) + :514-531
  * `roidb_assignment`       the same for a merged roidb entry, its ground-truth rows as :208-290 (_add_gt_annotations) left them
  * `sample_rois`            lib/roi_data/fast_rcnn.py:129-200 (_sample_rois), :203-248 (_compute_targets, _expand_bbox_targets)
  * `sample_rois_batched`    the same for every image of a minibatch at once (one read of the per-image counts)
  * `add_fast_rcnn_blobs`    lib/roi_data/fast_rcnn.py:105-126 with json_dataset.add_proposals(crowd_thresh=0) before it, from the
                             RPN proposals of a minibatch; FPN's _add_multilevel_rois is left to the caller
  * `get_fast_rcnn_blob_names`  lib/roi_data/fast_rcnn.py:36-102
Mask targets are in roi_data/mask_rcnn.py (device polygon rasteriser), keypoint targets in roi_data/keypoint_rcnn.py.

The random choice of the reference (`npr.choice(inds, size, replace=False)` = a permutation prefix) is an INPUT here: pass
the positions it picked (`fg_choice`, `bg_choice`, e.g. from the same numpy RandomState) for a bit-identical minibatch, or
leave them None for a torch.randperm draw on the device.
"""
import ctypes

import numpy as np
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


def sample_rois_batched(boxes, box_off, gt_boxes, gt_classes, gt_off, im_scales, num_classes, batch_size_per_im=512, fg_fraction=0.25,
                        fg_thresh=0.5, bg_thresh_hi=0.5, bg_thresh_lo=0.0, bbox_reg_weights=(10.0, 10.0, 5.0, 5.0),
                        cls_agnostic_bbox_reg=False, choices=None, is_crowd=None, batch_idx=None):
    """_sample_rois for the N images of a minibatch, given in CSR form on the device: `boxes` (T, 4) the merged roidb rows of
    every image (its ground truth first, then its proposals, unscaled), image b's being box_off[b] .. box_off[b + 1] - 1
    (int32 (N + 1,); T may exceed box_off[N]); `gt_boxes` (G, 4), `gt_classes` (G,) int32 and `is_crowd` (G,) int32 (None: no
    crowd) the concatenated ground truth, image b's in rows gt_off[b] .. gt_off[b + 1] - 1; im_scales (N,) float32 and
    batch_idx (N,) float32 (None: 0 .. N - 1).  choices: per image (fg_choice, bg_choice), each the npr.choice positions or
    None (torch.randperm on the device, drawn in sample_rois' order); None: every draw on the device.

    Returns (blobs, info).  blobs: labels_int32, rois, bbox_targets, bbox_inside_weights, bbox_outside_weights, each image's fg
    rows then its bg rows, images in order, as np.concatenate of the per-image blobs gives; keep_inds: the merged rows taken.
    info: num_fg (per image), keep_begin / box_begin (host (N + 1,) offsets of each image's kept / merged rows), keep_inds (per
    image, its own row indices), assignment (max_overlaps, box_to_gt_ind (into the concatenated ground truth), max_classes).
    The only host read is one copy of the per-image counts and box offsets."""
    boxes = _boxes4(boxes, "boxes")
    dev = boxes.device
    N = box_off.numel() - 1
    if N < 1:
        raise ValueError("a minibatch has at least one image")
    T = max(boxes.size(0), 1)
    G = int(gt_boxes.size(0)) if gt_boxes is not None else 0
    gt = _boxes4(gt_boxes, "gt_boxes") if G else None
    box_off = box_off.to(device=dev, dtype=torch.int32).contiguous()
    gt_off = gt_off.to(device=dev, dtype=torch.int32).contiguous()
    gcls = gt_classes.to(device=dev, dtype=torch.int32).contiguous() if G else None
    crowd = is_crowd.to(device=dev, dtype=torch.int32).contiguous() if G and is_crowd is not None else None
    max_overlaps = torch.empty((T,), dtype=torch.float32, device=dev)
    argmax = torch.empty((T,), dtype=torch.int32, device=dev)
    max_classes = torch.empty((T,), dtype=torch.int32, device=dev)
    _launch("b200_roi_assign_batched", dev, _ptr(boxes), box_off.data_ptr(), N, boxes.size(0), _ptr(gt), _ptr(gcls), _ptr(crowd),
            gt_off.data_ptr(), 1, max_overlaps.data_ptr(), argmax.data_ptr(), max_classes.data_ptr())
    fg = torch.empty((T,), dtype=torch.int32, device=dev)
    bg = torch.empty((T,), dtype=torch.int32, device=dev)
    table = torch.empty((3 * N + 1,), dtype=torch.int32, device=dev)        # (N, 2) fg / bg counts, then the box offsets
    _launch("b200_roi_select_batched", dev, max_overlaps.data_ptr(), box_off.data_ptr(), N, float(fg_thresh), float(bg_thresh_hi),
            float(bg_thresh_lo), fg.data_ptr(), bg.data_ptr(), table.data_ptr())
    table[2 * N:].copy_(box_off)
    host = table.cpu().numpy()                                               # the one read
    counts, box_begin = host[:2 * N].reshape(N, 2), host[2 * N:].astype(np.int64)

    # npr.choice per image (fast_rcnn.py:143-157): positions into its fg list, then into its bg list
    rois_per_image = int(batch_size_per_im)
    fg_rois_per_image = int(round(fg_fraction * rois_per_image))
    num_fg, num_bg, parts, host_pos = [], [], [], []
    for b in range(N):
        nf = min(fg_rois_per_image, int(counts[b, 0]))
        nb = min(rois_per_image - nf, int(counts[b, 1]))
        ch = tuple(choices[b]) if choices is not None else (None, None)
        for total, size, choice in ((int(counts[b, 0]), nf, ch[0]), (int(counts[b, 1]), nb, ch[1])):
            if total == 0:
                continue
            if choice is None:
                parts.append(torch.randperm(total, device=dev)[:size])
                continue
            choice = np.asarray(choice, dtype=np.int64).reshape(-1)
            if choice.size != size:
                raise ValueError("choice has %d entries, the minibatch takes %d" % (choice.size, size))
            if size and (choice.min() < 0 or choice.max() >= total):
                raise ValueError("choice positions must lie in [0, %d)" % total)
            parts.append((sum(len(q) for q in host_pos), size))
            host_pos.append(choice)
        num_fg.append(nf); num_bg.append(nb)
    kept = np.asarray(num_fg) + np.asarray(num_bg)
    keep_begin = np.concatenate([[0], np.cumsum(kept)]).astype(np.int64)
    n = int(keep_begin[-1])
    image = np.repeat(np.arange(N), kept)
    is_fg = np.concatenate([np.arange(k) < f for k, f in zip(kept, num_fg)]) if n else np.zeros(0, bool)
    pos_host = np.concatenate(host_pos) if host_pos else np.zeros(0, np.int64)
    up = torch.from_numpy(np.concatenate([keep_begin, num_fg, image, is_fg, pos_host]).astype(np.int32)).to(dev)   # one upload
    keep_off_d, num_fg_d = up[:N + 1], up[N + 1:2 * N + 1]
    image_d, is_fg_d, pos_d = up[2 * N + 1:2 * N + 1 + n], up[2 * N + 1 + n:2 * N + 1 + 2 * n], up[2 * N + 1 + 2 * n:]
    if any(torch.is_tensor(p) for p in parts):
        pos = torch.cat([p if torch.is_tensor(p) else pos_d[p[0]:p[0] + p[1]] for p in parts])
    else:
        pos = pos_d
    base = box_off.long()[image_d.long()]
    idx = base + pos.long()
    keep = (torch.where(is_fg_d != 0, fg.long()[idx], bg.long()[idx]) + base).to(torch.int32).contiguous()

    reg_classes = 2 if cls_agnostic_bbox_reg else int(num_classes)
    labels = torch.empty((n,), dtype=torch.int32, device=dev)
    rois = torch.empty((n, 5), dtype=torch.float32, device=dev)
    targets = torch.empty((n, 4 * reg_classes), dtype=torch.float32, device=dev)
    inside = torch.empty_like(targets)
    outside = torch.empty_like(targets)
    if len(bbox_reg_weights) != 4:
        raise ValueError("bbox_reg_weights must be 4 values (wx, wy, ww, wh), got %d" % len(bbox_reg_weights))
    w = _host_array(ctypes.c_float, [float(v) for v in bbox_reg_weights])
    im_scales = im_scales.to(device=dev, dtype=torch.float32).contiguous()
    batch_idx = (torch.arange(N, dtype=torch.float32, device=dev) if batch_idx is None
                 else batch_idx.to(device=dev, dtype=torch.float32).contiguous())
    _launch("b200_fast_rcnn_targets_batched", dev, boxes.data_ptr(), _ptr(gt), argmax.data_ptr(), max_classes.data_ptr(), keep.data_ptr(),
            keep_off_d.data_ptr(), num_fg_d.data_ptr(), im_scales.data_ptr(), batch_idx.data_ptr(), N, n, w, reg_classes,
            1 if cls_agnostic_bbox_reg else 0, labels.data_ptr(), rois.data_ptr(), targets.data_ptr(), inside.data_ptr(),
            outside.data_ptr())
    local = keep - base.to(torch.int32)
    blobs = dict(labels_int32=labels, rois=rois, bbox_targets=targets, bbox_inside_weights=inside, bbox_outside_weights=outside,
                 keep_inds=keep)
    info = dict(num_fg=num_fg, keep_begin=keep_begin, box_begin=box_begin,
                keep_inds=[local[keep_begin[b]:keep_begin[b + 1]] for b in range(N)],
                assignment=(max_overlaps, argmax, max_classes))
    return blobs, info


def train_keys(cfg):
    """The TRAIN.* / MODEL.* keys that add_fast_rcnn_blobs reads, from the reference's config object."""
    c = cfg
    t = dict(BATCH_SIZE_PER_IM=c.TRAIN.BATCH_SIZE_PER_IM, FG_FRACTION=c.TRAIN.FG_FRACTION, FG_THRESH=c.TRAIN.FG_THRESH,
             BG_THRESH_HI=c.TRAIN.BG_THRESH_HI, BG_THRESH_LO=c.TRAIN.BG_THRESH_LO, NUM_CLASSES=c.MODEL.NUM_CLASSES,
             BBOX_REG_WEIGHTS=c.MODEL.BBOX_REG_WEIGHTS, CLS_AGNOSTIC_BBOX_REG=c.MODEL.CLS_AGNOSTIC_BBOX_REG)
    if getattr(c.MODEL, "MASK_ON", False):
        t.update(MASK_ON=True, MRCNN_RESOLUTION=c.MRCNN.RESOLUTION, CLS_SPECIFIC_MASK=c.MRCNN.CLS_SPECIFIC_MASK)
    if getattr(c.MODEL, "KEYPOINTS_ON", False):
        t.update(KEYPOINTS_ON=True, HEATMAP_SIZE=c.KRCNN.HEATMAP_SIZE, NUM_KEYPOINTS=c.KRCNN.NUM_KEYPOINTS,
                 IMS_PER_BATCH=c.TRAIN.IMS_PER_BATCH, MIN_KEYPOINT_COUNT=c.KRCNN.MIN_KEYPOINT_COUNT_FOR_VALID_MINIBATCH)
    return t


def get_fast_rcnn_blob_names(is_training=True, cfg=None, **kw):
    """The blob names of lib/roi_data/fast_rcnn.py:36-102, in its order.  The switches come from `cfg` (MODEL.MASK_ON,
    MODEL.KEYPOINTS_ON, FPN.FPN_ON, FPN.MULTILEVEL_ROIS, FPN.ROI_MIN_LEVEL, FPN.ROI_MAX_LEVEL) or from keywords of those names
    (defaults: all off, levels 2 .. 5)."""
    if cfg is not None:
        kw = dict(MASK_ON=cfg.MODEL.MASK_ON, KEYPOINTS_ON=cfg.MODEL.KEYPOINTS_ON, FPN_ON=cfg.FPN.FPN_ON,
                  MULTILEVEL_ROIS=cfg.FPN.MULTILEVEL_ROIS, ROI_MIN_LEVEL=cfg.FPN.ROI_MIN_LEVEL, ROI_MAX_LEVEL=cfg.FPN.ROI_MAX_LEVEL)
    mask, kp = kw.get("MASK_ON", False), kw.get("KEYPOINTS_ON", False)
    names = ["rois"]
    if is_training:
        names += ["labels_int32", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights"]
        if mask:
            names += ["mask_rois", "roi_has_mask_int32", "masks_int32"]
        if kp:
            names += ["keypoint_rois", "keypoint_locations_int32", "keypoint_weights", "keypoint_loss_normalizer"]
    if kw.get("FPN_ON", False) and kw.get("MULTILEVEL_ROIS", False):
        levels = range(kw.get("ROI_MIN_LEVEL", 2), kw.get("ROI_MAX_LEVEL", 5) + 1)
        names += ["rois_fpn%d" % l for l in levels] + ["rois_idx_restore_int32"]
        if is_training and mask:
            names += ["mask_rois_fpn%d" % l for l in levels] + ["mask_rois_idx_restore_int32"]
        if is_training and kp:
            names += ["keypoint_rois_fpn%d" % l for l in levels] + ["keypoint_rois_idx_restore_int32"]
    return names


def _host(x):
    return x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def add_fast_rcnn_blobs(rpn_rois, roidb, im_scales, train, choices=None):
    """json_dataset.add_proposals(roidb, rpn_rois, im_scales, crowd_thresh=0) and roi_data.fast_rcnn.add_fast_rcnn_blobs for a
    minibatch, on the device, without FPN's multi-level RoIs.  rpn_rois: (R, 5) [batch index, x1, y1, x2, y2] at the network's
    scale, CUDA; roidb: per image its ground truth ('boxes' (G, 4) unscaled, 'gt_classes' (G,), 'is_crowd' (G,) where crowd
    objects exist, 'segms' with MASK_ON, 'gt_keypoints' with KEYPOINTS_ON; host arrays, not modified); im_scales: N host
    floats; train: the keys of train_keys(); choices: per image (fg_choice, bg_choice) or, with keypoints, (fg_choice,
    bg_choice, keypoint_choice), or None (device randperm).  Each image's proposals keep their rpn_rois order (a stable sort
    on the batch index groups them).  Host reads: one for sampling, and those of the mask and keypoint steps."""
    dev = rpn_rois.device
    N = len(roidb)
    gts, classes, crowds, gt_rows = [], [], [], []
    for e in roidb:                                                   # the ground-truth rows that bbox_overlaps sees: class > 0
        cls = _host(e["gt_classes"]).reshape(-1)
        rows = np.where(cls > 0)[0]
        gts.append(_host(e["boxes"]).astype(np.float32).reshape(-1, 4)[rows])
        classes.append(cls[rows])
        crowds.append(_host(e["is_crowd"]).reshape(-1)[rows] != 0 if "is_crowd" in e else np.zeros(rows.size, bool))
        gt_rows.append(rows)
    sizes = [g.shape[0] for g in gts]
    G = int(sum(sizes))
    gt_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    scales = np.asarray([float(s) for s in im_scales], np.float32)
    fl = torch.from_numpy(np.concatenate([np.concatenate(gts).reshape(-1), scales])).to(dev)
    it = torch.from_numpy(np.concatenate([np.concatenate(classes), np.concatenate(crowds), gt_off, np.concatenate(gt_rows)])
                          .astype(np.int32)).to(dev)
    gt, scales_d = fl[:4 * G].view(G, 4), fl[4 * G:]
    gcls, crowd, gt_off_d, gt_rows_d = it[:G], it[G:2 * G], it[2 * G:2 * G + N + 1], it[2 * G + N + 1:]

    rois = rpn_rois.to(torch.float32).reshape(-1, 5)
    rois = rois[torch.sort(rois[:, 0], stable=True).indices].contiguous()
    prop_off = torch.searchsorted(rois[:, 0].contiguous(), torch.arange(N + 1, dtype=torch.float32, device=dev)).to(torch.int32)
    box_off = gt_off_d + (prop_off - prop_off[:1])
    T = G + rois.size(0)
    boxes = torch.empty((T, 4), dtype=torch.float32, device=dev)
    _launch("b200_roi_merge_proposals", dev, _ptr(rois), prop_off.data_ptr(), _ptr(gt), gt_off_d.data_ptr(), scales_d.data_ptr(), N,
            box_off.data_ptr(), T, _ptr(boxes))
    t = train
    blobs, info = sample_rois_batched(boxes, box_off, gt, gcls, gt_off_d, scales_d, t["NUM_CLASSES"], t["BATCH_SIZE_PER_IM"],
                                      t["FG_FRACTION"], t["FG_THRESH"], t["BG_THRESH_HI"], t["BG_THRESH_LO"], t["BBOX_REG_WEIGHTS"],
                                      t["CLS_AGNOSTIC_BBOX_REG"], choices=choices, is_crowd=crowd)
    keep = blobs.pop("keep_inds")
    if t.get("MASK_ON", False):
        # roi_data/mask_rcnn.py:34-122 per image, concatenated
        from detectron.pytorch_b200.roi_data import mask_rcnn as MR
        kb = info["keep_begin"]
        per = [slice(int(kb[b]), int(kb[b + 1])) for b in range(N)]
        sampled = boxes[keep.long()]
        blobs.update(MR.mask_rcnn_blobs([blobs["labels_int32"][s] for s in per], [blobs["rois"][s] for s in per], [sampled[s] for s in per],
                                        info["num_fg"], roidb, t.get("MRCNN_RESOLUTION", 14), t.get("CLS_SPECIFIC_MASK", True),
                                        t["NUM_CLASSES"]))
    if t.get("KEYPOINTS_ON", False):
        # roi_data/keypoint_rcnn.py:33-96 for every image in one device call, then fast_rcnn.py:120-124
        from detectron.pytorch_b200.roi_data import keypoint_rcnn as KR
        box_begin = info["box_begin"]
        rows = int(box_begin[-1])
        mo, am = info["assignment"][0][:rows], info["assignment"][1][:rows]
        # add_keypoint_rcnn_blobs reads box_to_gt_ind_map as roidb rows: the assigned gt's row in its own entry
        kp_map = torch.where(am >= 0, gt_rows_d[am.clamp(min=0).long()], am) if G else am
        kp_choices = [tuple(c)[2] if len(tuple(c)) > 2 else None for c in choices] if choices is not None else None
        kb = KR.keypoint_rcnn_blobs(boxes[:rows], box_begin, mo, kp_map, roidb, [float(s) for s in scales],
                                    int(round(t["FG_FRACTION"] * int(t["BATCH_SIZE_PER_IM"]))), t["HEATMAP_SIZE"], t["NUM_KEYPOINTS"],
                                    t["FG_THRESH"], choices=kp_choices)
        KR.finalize_keypoint_minibatch(kb, True, ims_per_batch=t.get("IMS_PER_BATCH", 2), batch_size_per_im=t["BATCH_SIZE_PER_IM"],
                                       fg_fraction=t["FG_FRACTION"], num_keypoints=t["NUM_KEYPOINTS"],
                                       min_count=t.get("MIN_KEYPOINT_COUNT", 20))
        blobs.update(kb)
    return blobs
