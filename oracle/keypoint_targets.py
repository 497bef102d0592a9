"""TEST INFRASTRUCTURE (CPU oracle, never imported by the product): the Keypoint R-CNN training targets
(lib/roi_data/keypoint_rcnn.py:33-96 with lib/utils/keypoints.py:160-211), restated in numpy with the dtypes numpy 2 gives
the reference's expressions:

  candidates   max_overlaps (float32) >= FG_THRESH, and some keypoint with v > 0 of person gt_inds[box_to_gt_ind_map] (numpy
               indexing: -1 is the last person) inside the box, ends included -- int32 against float32, compared in float64
  draw         the first min(fg_rois_per_image, #candidates) in ascending order, or the caller's np.random.choice positions
               when there are more candidates
  labels       per (RoI, keypoint), float32: x = float32(kx), s = HS / (x2 - x1), floor((x - x1) * s), HS - 1 when x == x2
               (decided before the transform; the same for y); valid = 0 <= x, y < HS and v > 0; lin = y * HS + x; the
               heat is lin * valid (float64, stored as float32: NaN where lin is not finite and valid is 0), then
               astype(int32) -- x86 gives INT_MIN for NaN and +-inf
  rois         float32 box * float32(im_scale), the batch index in front
  normalizer   float32(sum of the weights) / float32(IMS_PER_BATCH * BATCH_SIZE_PER_IM * FG_FRACTION * NUM_KEYPOINTS)

Pinned by tests/golden/keypoint_targets.npz, produced by the UNMODIFIED reference functions (tests/golden/
make_golden_keypoint_targets.py).
"""
import numpy as np

f32 = np.float32
INT_MIN = -2 ** 31


def to_int32(a):
    """numpy's float -> int32 astype on x86: truncation for finite values in range, INT_MIN for NaN and +-inf."""
    a = np.asarray(a, np.float64)
    out = np.full(a.shape, INT_MIN, np.int64)
    ok = np.isfinite(a)
    out[ok] = np.trunc(a[ok])
    return out.astype(np.int32)


def within_box(points, boxes):
    """points (R, 2, K) int32, boxes (R, 4) float32 -> (R, K) bool, compared in float64."""
    p = points.astype(np.float64)
    b = boxes.astype(np.float64)
    return ((p[:, 0, :] >= b[:, 0:1]) & (p[:, 0, :] <= b[:, 2:3]) & (p[:, 1, :] >= b[:, 1:2]) & (p[:, 1, :] <= b[:, 3:4]))


def candidates(boxes, max_overlaps, box_to_gt_ind_map, gt_inds, gt_keypoints, fg_thresh):
    """np.where of the keypoint fg condition: ascending indices into `boxes`."""
    boxes = np.asarray(boxes, f32).reshape(-1, 4)
    if boxes.shape[0] == 0:
        return np.zeros((0,), np.int64)
    ind_kp = np.asarray(gt_inds)[np.asarray(box_to_gt_ind_map)]
    kp = np.asarray(gt_keypoints)[ind_kp]
    vis = kp[:, 2, :] > 0
    ok = (np.asarray(max_overlaps, f32) >= f32(fg_thresh)) & (vis & within_box(kp[:, :2, :], boxes)).any(axis=1)
    return np.where(ok)[0]


def heatmap_labels(keypoints, rois, HS):
    """keypoints (R, 3, K) int32, rois (R, >=4) float32 -> (heats int32 (R, K), weights float32 (R, K))."""
    rois = np.asarray(rois, f32)
    keypoints = np.asarray(keypoints)
    R, K = keypoints.shape[0], keypoints.shape[2]
    heats = np.zeros((R, K), f32)
    weights = np.zeros((R, K), f32)
    hs = f32(HS)
    x1, y1, x2, y2 = rois[:, 0], rois[:, 1], rois[:, 2], rois[:, 3]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        sx = (hs / (x2 - x1)).astype(f32)
        sy = (hs / (y2 - y1)).astype(f32)
        for k in range(K):
            x = keypoints[:, 0, k].astype(f32)
            y = keypoints[:, 1, k].astype(f32)
            xb, yb = x == x2, y == y2
            fx = np.floor(((x - x1).astype(f32) * sx).astype(f32))
            fy = np.floor(((y - y1).astype(f32) * sy).astype(f32))
            fx[xb] = hs - 1
            fy[yb] = hs - 1
            valid = (fx >= 0) & (fy >= 0) & (fx < hs) & (fy < hs) & (keypoints[:, 2, k] > 0)
            lin = ((fy * hs).astype(f32) + fx).astype(f32)
            heats[:, k] = (lin.astype(np.float64) * valid.astype(np.int32)).astype(f32)
            weights[:, k] = valid
    return to_int32(heats), weights


def add_keypoint_rcnn_blobs(blobs, roidb, fg_rois_per_image, im_scale, batch_idx, HS, fg_thresh, choice=None):
    """One image.  roidb: the merged entry (boxes float32, max_overlaps, box_to_gt_ind_map, gt_classes, gt_keypoints).
    choice: the np.random.choice positions, used when there are more candidates than fg_rois_per_image."""
    gt_inds = np.where(np.asarray(roidb["gt_classes"]) > 0)[0]
    boxes = np.asarray(roidb["boxes"], f32).reshape(-1, 4)
    cand = candidates(boxes, roidb["max_overlaps"], roidb["box_to_gt_ind_map"], gt_inds, roidb["gt_keypoints"], fg_thresh)
    n = min(int(fg_rois_per_image), cand.size)
    if cand.size > n:
        cand = cand[np.asarray(choice, np.int64)]
    gt_kp = np.asarray(roidb["gt_keypoints"])
    sampled = boxes[cand].copy()
    m = np.asarray(roidb["box_to_gt_ind_map"])[cand]
    kps = -np.ones((cand.size, 3, gt_kp.shape[2]), gt_kp.dtype)
    for i, ind in enumerate(m):
        if ind >= 0:
            kps[i] = gt_kp[gt_inds[ind]]
    heats, weights = heatmap_labels(kps, sampled, HS)
    rois = np.hstack([np.full((cand.size, 1), f32(batch_idx), f32), (sampled * f32(im_scale)).astype(f32)]).astype(f32)
    blobs["keypoint_rois"] = rois
    blobs["keypoint_locations_int32"] = heats.reshape(-1)
    blobs["keypoint_weights"] = weights.reshape(-1)
    return cand


def finalize_keypoint_minibatch(blobs, valid, ims_per_batch, batch_size_per_im, fg_fraction, num_keypoints, min_count=20):
    w = blobs["keypoint_weights"]
    s = np.sum(w, dtype=f32)
    valid = valid and len(w) > 0 and s > min_count
    blobs["keypoint_loss_normalizer"] = np.array(f32(s) / f32(ims_per_batch * batch_size_per_im * fg_fraction * num_keypoints), f32)
    return valid
