"""TEST INFRASTRUCTURE: numpy restatement of the reference's test-time detection post-processing,
box_results_with_nms_and_limit (lib/core/test.py:732-790), and of the routines it calls.  Nothing under detectron/ imports
this module.

  * nms: cython_nms.nms (lib/utils/cython_nms.pyx:37-87).  float32 throughout, every operation rounded on its own: the box
    areas (x2 - x1 + 1) * (y2 - y1 + 1) are numpy float32 products, IoU = inter / ((area_i + area_j) - inter), and a box is
    suppressed when IoU >= float32(thresh) (the .pyx declares thresh np.float32_t).  The reference orders the boxes by
    scores.argsort()[::-1], which is not stable; here tied scores go lower index first, like the device.  The two agree
    whenever no two boxes with equal scores overlap.
  * soft_nms: cython_nms.soft_nms (lib/utils/cython_nms.pyx:98-203).  The C that Cython generates adds the literal 1.0 in
    double, so a box's area is a double product rounded to float once, and the union is formed in double and rounded once;
    the intersection iw * ih, the IoU and the score product are float32.  The decays of one step are independent per
    box; the drops are then applied in the reference's order (a dropped box is overwritten by the current last one, which
    is examined in place).
  * box_voting: lib/utils/boxes.py:268-317 with cython_bbox.bbox_overlaps (lib/utils/cython_bbox.pyx:32-73, same
    double-then-float arithmetic), votes selected with IoU >= float32(thresh) like numpy 2 compares, the weighted average
    and the score methods in float64 (the reference averages in float32).
  * the per-image limit: keep the detections whose score is >= the DETECTIONS_PER_IM-th best over all classes.
"""
import numpy as np

f32 = np.float32
METHODS = {"hard": 0, "linear": 1, "gaussian": 2}


def nms_iou(a, b):
    """Cython-NMS IoU of box a (the higher-scoring one) with box b, float32, as cython_nms.nms computes it.  a, b: (..., 4),
    broadcast against each other."""
    a = np.asarray(a, f32)
    b = np.asarray(b, f32)
    area_a = (a[..., 2] - a[..., 0] + f32(1)) * (a[..., 3] - a[..., 1] + f32(1))
    area_b = (b[..., 2] - b[..., 0] + f32(1)) * (b[..., 3] - b[..., 1] + f32(1))
    w = np.maximum(f32(0), np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]) + f32(1))
    h = np.maximum(f32(0), np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]) + f32(1))
    inter = w * h
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter / ((area_a + area_b) - inter)


def score_order(scores):
    """Descending score, ties lower index first (the device's rule)."""
    return np.argsort(-np.asarray(scores, f32), kind="stable")


def nms(dets, thresh):
    """cython_nms.nms: kept row indices, ascending."""
    dets = np.asarray(dets, f32)
    n = dets.shape[0]
    if n == 0:
        return np.zeros((0,), np.int64)
    t = f32(thresh)
    order = score_order(dets[:, 4])
    suppressed = np.zeros(n, bool)
    for _i in range(n):
        i = order[_i]
        if suppressed[i]:
            continue
        rest = order[_i + 1:]
        rest = rest[~suppressed[rest]]
        if len(rest):
            suppressed[rest[nms_iou(dets[i, :4], dets[rest, :4]) >= t]] = True
    return np.nonzero(~suppressed)[0].astype(np.int64)


def _area_f(x1, y1, x2, y2):
    """float((x2 - x1) + 1.0) * ((y2 - y1) + 1.0)) with the differences in float32 and the rest in double."""
    return (((x2 - x1).astype(np.float64) + 1.0) * ((y2 - y1).astype(np.float64) + 1.0)).astype(f32)


def soft_nms(dets, sigma=0.5, overlap_thresh=0.3, score_thresh=0.001, method="linear"):
    """cython_nms.soft_nms through utils.boxes.soft_nms: (surviving rows with decayed scores, their original indices)."""
    boxes = np.array(dets, dtype=f32).reshape(-1, 5)
    if boxes.shape[0] == 0:
        return boxes, np.zeros((0,), np.int64)
    sigma, Nt, threshold, m = f32(sigma), f32(overlap_thresh), f32(score_thresh), METHODS[method]
    N = boxes.shape[0]
    inds = np.arange(N)
    i = 0
    while i < N:
        maxpos = i + int(np.argmax(boxes[i:N, 4]))                        # first maximum, like `maxscore < score`
        boxes[[i, maxpos]] = boxes[[maxpos, i]]
        inds[[i, maxpos]] = inds[[maxpos, i]]
        tx1, ty1, tx2, ty2 = boxes[i, :4]
        b = boxes[i + 1:N]
        iw = ((np.minimum(tx2, b[:, 2]) - np.maximum(tx1, b[:, 0])).astype(np.float64) + 1.0).astype(f32)
        ih = ((np.minimum(ty2, b[:, 3]) - np.maximum(ty1, b[:, 1])).astype(np.float64) + 1.0).astype(f32)
        hit = (iw > 0) & (ih > 0)
        inter = iw * ih
        area = _area_f(b[:, 0], b[:, 1], b[:, 2], b[:, 3])
        t_area = (float(tx2 - tx1) + 1.0) * (float(ty2 - ty1) + 1.0)
        ua = ((t_area + area.astype(np.float64)) - inter.astype(np.float64)).astype(f32)
        with np.errstate(divide="ignore", invalid="ignore"):
            ov = inter / ua
        if m == 1:
            weight = np.where(ov > Nt, (1.0 - ov.astype(np.float64)).astype(f32), f32(1))
        elif m == 2:
            weight = np.exp((-(ov * ov) / sigma).astype(np.float64)).astype(f32)
        else:
            weight = np.where(ov > Nt, f32(0), f32(1))
        new = np.where(hit, weight * b[:, 4], b[:, 4]).astype(f32)
        boxes[i + 1:N, 4] = new
        drop = np.zeros(N, bool)
        drop[i + 1:N] = hit & (new < threshold)
        pos = i + 1
        while pos < N:                                                    # the reference's order of the drops
            if drop[pos]:
                boxes[pos] = boxes[N - 1]; inds[pos] = inds[N - 1]; drop[pos] = drop[N - 1]
                N -= 1
            else:
                pos += 1
        i += 1
    return boxes[:N], inds[:N].astype(np.int64)


def overlaps(b, q):
    """cython_bbox.bbox_overlaps of box b (a "boxes" row) with box q (a "query_boxes" row), float32; (..., 4) arrays,
    broadcast.  The +1 and the union are formed in double and rounded to float where the .pyx assigns to a float."""
    b = np.asarray(b, f32)
    q = np.asarray(q, f32)
    q_area = _area_f(q[..., 0], q[..., 1], q[..., 2], q[..., 3])
    iw = ((np.minimum(b[..., 2], q[..., 2]) - np.maximum(b[..., 0], q[..., 0])).astype(np.float64) + 1.0).astype(f32)
    ih = ((np.minimum(b[..., 3], q[..., 3]) - np.maximum(b[..., 1], q[..., 1])).astype(np.float64) + 1.0).astype(f32)
    b_area = ((b[..., 2] - b[..., 0]).astype(np.float64) + 1.0) * ((b[..., 3] - b[..., 1]).astype(np.float64) + 1.0)
    inter = iw * ih
    ua = ((b_area + q_area.astype(np.float64)) - inter.astype(np.float64)).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ov = inter / ua
    return np.where((iw > 0) & (ih > 0), ov, f32(0)).astype(f32)


def bbox_overlaps(boxes, query):
    """cython_bbox.bbox_overlaps: (N, K) float32."""
    return overlaps(np.asarray(boxes, f32).reshape(-1, 4)[:, None, :], np.asarray(query, f32).reshape(-1, 4)[None, :, :])


def box_voting(top_dets, all_dets, thresh, scoring_method="ID", beta=1.0):
    """utils.boxes.box_voting in float64: returns float64 (n, 5)."""
    top = np.asarray(top_dets, f32).reshape(-1, 5)
    alld = np.asarray(all_dets, f32).reshape(-1, 5)
    out = top.astype(np.float64)
    ov = bbox_overlaps(top[:, :4], alld[:, :4])
    for k in range(top.shape[0]):
        sel = np.nonzero(ov[k] >= f32(thresh))[0]
        ws = alld[sel, 4].astype(np.float64)
        out[k, :4] = (alld[sel, :4].astype(np.float64) * ws[:, None]).sum(0) / ws.sum()
        if scoring_method == "ID":
            pass
        elif scoring_method == "TEMP_AVG":
            P = np.vstack((ws, 1.0 - ws))
            X = np.exp(np.log(P / P.max(axis=0)) / beta)
            out[k, 4] = (X / X.sum(axis=0))[0].mean()
        elif scoring_method == "AVG":
            out[k, 4] = ws.mean()
        elif scoring_method == "IOU_AVG":
            w = ov[k, sel].astype(np.float64)
            out[k, 4] = (ws * w).sum() / w.sum()
        elif scoring_method == "GENERALIZED_AVG":
            out[k, 4] = np.mean(ws ** beta) ** (1.0 / beta)
        elif scoring_method == "QUASI_SUM":
            out[k, 4] = ws.sum() / float(len(ws)) ** beta
        else:
            raise NotImplementedError(scoring_method)
    return out


def box_results_with_nms_and_limit(scores, boxes, num_classes, score_thresh=0.05, nms_thresh=0.5, detections_per_im=100,
                                   soft_nms_enabled=False, soft_sigma=0.5, soft_method="linear", bbox_vote=False, vote_th=0.8,
                                   vote_scoring="ID"):
    """lib/core/test.py:732-790 -> cls_boxes, a list of num_classes arrays (n_j, 5) (index 0 empty).  With voting the
    arrays are float64 (see box_voting), else float32 like the reference's."""
    scores = np.asarray(scores, f32)
    boxes = np.asarray(boxes, f32)
    cls_boxes = [np.zeros((0, 5), f32) for _ in range(num_classes)]
    for j in range(1, num_classes):
        inds = np.nonzero(scores[:, j] > f32(score_thresh))[0]
        dets_j = np.hstack((boxes[inds, 4 * j:4 * j + 4], scores[inds, j][:, None])).astype(f32)
        if soft_nms_enabled:
            nms_dets, _ = soft_nms(dets_j, soft_sigma, nms_thresh, 0.0001, soft_method)
        else:
            nms_dets = dets_j[nms(dets_j, nms_thresh)]
        if bbox_vote:
            nms_dets = box_voting(nms_dets, dets_j, vote_th, vote_scoring)
        cls_boxes[j] = nms_dets
    return limit_per_image(cls_boxes, detections_per_im)


def limit_per_image(cls_boxes, detections_per_im):
    """Keep, over all classes, the detections scoring >= the detections_per_im-th best score (all of them when there are
    fewer, or when detections_per_im <= 0)."""
    cls_boxes = list(cls_boxes)
    if detections_per_im > 0:
        image_scores = np.hstack([c[:, -1] for c in cls_boxes[1:]]) if len(cls_boxes) > 1 else np.zeros((0,))
        if len(image_scores) > detections_per_im:
            image_thresh = np.sort(image_scores)[-detections_per_im]
            cls_boxes[1:] = [c[c[:, -1] >= image_thresh] for c in cls_boxes[1:]]
    return cls_boxes
