"""TEST INFRASTRUCTURE (CPU oracle, never imported by the product): numpy restatement of the reference's RoI label /
target generation for one image.

  bbox_overlaps     lib/utils/cython_bbox.pyx:32-73 (float32 arithmetic, +1 pixel convention)
  assign_rois       lib/datasets/json_dataset.py:429-490, :514-531 (ground-truth rows: :208-290, _add_gt_annotations)
  sample_rois       lib/roi_data/fast_rcnn.py:129-200, :203-248; lib/utils/boxes.py:199-230

Pinned by tests/golden/targets.npz, produced by the UNMODIFIED reference functions (tests/golden/make_golden_targets.py).
"""
import numpy as np

f32 = np.float32


def bbox_overlaps(boxes, query):
    """The generated C adds the literal 1.0 as a double: widths / heights, their products and the union are double expressions
    rounded to float32 once, on assignment to the float variables box_area, iw, ih, ua; iw * ih and the quotient are float32."""
    boxes = np.asarray(boxes, f32); query = np.asarray(query, f32)
    N, K = boxes.shape[0], query.shape[0]
    out = np.zeros((N, K), f32)
    if N == 0 or K == 0:
        return out
    f64 = np.float64
    qarea = (((query[:, 2] - query[:, 0]).astype(f64) + 1.0) * ((query[:, 3] - query[:, 1]).astype(f64) + 1.0)).astype(f32)
    barea = ((boxes[:, 2] - boxes[:, 0]).astype(f64) + 1.0) * ((boxes[:, 3] - boxes[:, 1]).astype(f64) + 1.0)          # stays double
    iw = ((np.minimum(boxes[:, None, 2], query[None, :, 2]) - np.maximum(boxes[:, None, 0], query[None, :, 0])).astype(f64) + 1.0).astype(f32)
    ih = ((np.minimum(boxes[:, None, 3], query[None, :, 3]) - np.maximum(boxes[:, None, 1], query[None, :, 1])).astype(f64) + 1.0).astype(f32)
    ok = (iw > 0) & (ih > 0)
    inter = (iw * ih).astype(f32)
    ua = ((barea[:, None] + qarea[None, :].astype(f64)) - inter.astype(f64)).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        out[ok] = (inter / ua).astype(f32)[ok]
    return out


def assign_rois(boxes, gt_boxes, gt_classes, is_crowd=None):
    """max_overlaps, box_to_gt_ind_map, max_classes of a merged roidb entry.  `boxes`: its rows, the G ground-truth boxes first.
    A ground-truth row keeps what _add_gt_annotations gave it: itself, overlap 1 with its own class, or overlap -1 (class 0)
    when it is a crowd object.  A proposal row takes the first maximum of its IoU with every ground-truth box, crowd
    objects included (0: none)."""
    boxes = np.asarray(boxes, f32)
    N, G = boxes.shape[0], len(gt_boxes)
    max_overlaps = np.zeros((N,), f32); argmax = -np.ones((N,), np.int32); max_classes = np.zeros((N,), np.int32)
    if G:
        ov = bbox_overlaps(boxes, gt_boxes)
        am = ov.argmax(axis=1); mx = ov.max(axis=1)
        hit = mx > 0
        max_overlaps[hit] = mx[hit]; argmax[hit] = am[hit]; max_classes[hit] = np.asarray(gt_classes)[am[hit]]
        crowd = np.zeros(G, bool) if is_crowd is None else np.asarray(is_crowd).reshape(-1) != 0
        max_overlaps[:G] = np.where(crowd, f32(-1), f32(1))
        argmax[:G] = np.arange(G)
        max_classes[:G] = np.where(crowd, 0, np.asarray(gt_classes).reshape(-1))
    return max_overlaps, argmax, max_classes


def bbox_transform_inv(ex, gt, weights):
    ex = np.asarray(ex, f32); gt = np.asarray(gt, f32)
    one, half = f32(1), f32(0.5)
    ew = ex[:, 2] - ex[:, 0] + one; eh = ex[:, 3] - ex[:, 1] + one
    ecx = ex[:, 0] + half * ew; ecy = ex[:, 1] + half * eh
    gw = gt[:, 2] - gt[:, 0] + one; gh = gt[:, 3] - gt[:, 1] + one
    gcx = gt[:, 0] + half * gw; gcy = gt[:, 1] + half * gh
    wx, wy, ww, wh = [f32(w) for w in weights]
    return np.stack([wx * (gcx - ecx) / ew, wy * (gcy - ecy) / eh, ww * np.log(gw / ew), wh * np.log(gh / eh)], axis=1).astype(f32)


def sample_rois(boxes, gt_boxes, gt_classes, im_scale, batch_idx, num_classes, fg_choice, bg_choice, batch_size_per_im=512,
                fg_fraction=0.25, fg_thresh=0.5, bg_thresh_hi=0.5, bg_thresh_lo=0.0, bbox_reg_weights=(10.0, 10.0, 5.0, 5.0),
                cls_agnostic_bbox_reg=False, is_crowd=None):
    boxes = np.asarray(boxes, f32)
    max_overlaps, argmax, max_classes = assign_rois(boxes, gt_boxes, gt_classes, is_crowd)
    fg_inds = np.where(max_overlaps >= f32(fg_thresh))[0]
    bg_inds = np.where((max_overlaps < f32(bg_thresh_hi)) & (max_overlaps >= f32(bg_thresh_lo)))[0]
    fg_per_image = int(np.round(fg_fraction * batch_size_per_im))
    n_fg = min(fg_per_image, fg_inds.size)
    n_bg = min(batch_size_per_im - n_fg, bg_inds.size)
    fg_keep = fg_inds[np.asarray(fg_choice, np.int64)] if fg_inds.size else fg_inds
    bg_keep = bg_inds[np.asarray(bg_choice, np.int64)] if bg_inds.size else bg_inds
    assert fg_keep.size == n_fg and bg_keep.size == n_bg
    keep = np.append(fg_keep, bg_keep).astype(np.int64)
    labels = max_classes[keep].copy(); labels[n_fg:] = 0
    sampled = boxes[keep]
    t = np.zeros((keep.size, 4), f32)
    has = argmax[keep] >= 0
    if has.any():
        t[has] = bbox_transform_inv(sampled[has], np.asarray(gt_boxes, f32)[argmax[keep][has]], bbox_reg_weights)
    reg_classes = 2 if cls_agnostic_bbox_reg else num_classes
    if cls_agnostic_bbox_reg:
        labels = np.minimum(labels, 1)          # fast_rcnn.py:212-213 clips `labels` IN PLACE: the returned labels_int32 are clipped too
    col = labels
    targets = np.zeros((keep.size, 4 * reg_classes), f32); inside = np.zeros_like(targets)
    for i in np.where(col > 0)[0]:
        targets[i, 4 * col[i]:4 * col[i] + 4] = t[i]; inside[i, 4 * col[i]:4 * col[i] + 4] = 1
    rois = np.hstack([np.full((keep.size, 1), batch_idx, f32), (sampled * f32(im_scale)).astype(f32)]).astype(f32)
    return dict(labels_int32=labels.astype(np.int32), rois=rois, bbox_targets=targets, bbox_inside_weights=inside,
                bbox_outside_weights=(inside > 0).astype(f32), keep_inds=keep.astype(np.int32))
