"""Test-time post-processing of the detection head on the device (SURVEY.md 8f N3).

Mirrors `box_results_with_nms_and_limit(scores, boxes)` of lib/core/test.py:732-790 (reference): per class j >= 1 keep the
detections with score > SCORE_THRESH, run NMS (or soft-NMS), optionally refine the kept boxes by box voting, then limit
the image to DETECTIONS_PER_IM detections over all classes.  The reference loops over the (80) classes on the host and
calls the Cython NMS once per class; here the per-class problems of an image go through ONE batched launch pair
(`b200_nms_batched`; soft-NMS: one warp per class in `b200_soft_nms_batched`; voting: `b200_box_voting_batched`), with one
host read of the kept counts.

Configuration: pass the reference's `cfg` object (read at call time like the reference: cfg.MODEL.NUM_CLASSES,
cfg.TEST.SCORE_THRESH / NMS / SOFT_NMS.* / BBOX_VOTE.* / DETECTIONS_PER_IM) or the same values as keyword arguments.
Inputs and outputs are numpy arrays like the reference's; CUDA tensors are accepted and skip the upload.

Flavour note: classic NMS is the Cython routine the reference calls here, cython_nms.nms (lib/utils/cython_nms.pyx:37-87):
`b200_nms_batched_cython` rounds both box areas on their own, forms IoU = inter / ((area_i + area_j) - inter) in float32
and suppresses when IoU >= float32(NMS).  (The proposal layer keeps the reference CUDA kernel's fused area and `>`; the
two differ on pairs whose IoU lies within about one ulp of the threshold.)  Tie rule: each class's candidates are sorted
by descending score, stably, so among equal scores the lower detection index comes first and suppresses the other.  The
reference sorts with `scores.argsort()[::-1]`, which is not stable, so where two overlapping boxes of one class tie its
result is arbitrary; elsewhere the order of tied boxes does not change the result.
Soft-NMS follows lib/utils/cython_nms.pyx:98-203 step for step (same greedy order, same drop rule, and the arithmetic of
the C that Cython generates from it: the literal 1.0 makes box areas and the union double expressions, rounded to float
once).

`segm_results(cls_boxes, masks, ref_boxes, im_h, im_w)` is the Mask R-CNN step after it (lib/core/test.py:793-847): every
detection's mask is pasted into the image and run-length encoded on the device in two launches per image, with one host
read of the per-detection sizes; the result is the reference's list of COCO RLE dicts.

`keypoint_results(cls_boxes, pred_heatmaps, ref_boxes)` is the Keypoint R-CNN step (lib/core/test.py:850-866): every
detection's 17 heatmaps are resized, searched for their maximum and soft-maxed on the device in one launch (plus one for
the optional OKS NMS), with one host read of the (R, 4, 17) result; the result is the reference's cls_keyps.

`get_blobs(im, rois, target_scale, target_max_size)` is _get_blobs with _get_rois_blob (lib/core/test.py:869-929): the `data` blob
is built on the device from the uint8 image (utils/blob.py).
"""
import numpy as np
import torch

from .. import ops

_SOFT_METHODS = {"hard": 0, "linear": 1, "gaussian": 2}
_VOTE_SCORING = {"ID": 0, "AVG": 1, "IOU_AVG": 2, "TEMP_AVG": 3, "GENERALIZED_AVG": 4, "QUASI_SUM": 5}


def _params(cfg, kw):
    if cfg is not None:
        t = cfg.TEST
        p = dict(num_classes=cfg.MODEL.NUM_CLASSES, score_thresh=t.SCORE_THRESH, nms=t.NMS, detections_per_im=t.DETECTIONS_PER_IM,
                 soft_nms=t.SOFT_NMS.ENABLED, soft_sigma=t.SOFT_NMS.SIGMA, soft_method=t.SOFT_NMS.METHOD,
                 bbox_vote=t.BBOX_VOTE.ENABLED, vote_th=t.BBOX_VOTE.VOTE_TH, vote_scoring=t.BBOX_VOTE.SCORING_METHOD)
    else:
        p = dict(num_classes=None, score_thresh=0.05, nms=0.5, detections_per_im=100, soft_nms=False, soft_sigma=0.5,
                 soft_method="linear", bbox_vote=False, vote_th=0.8, vote_scoring="ID")       # lib/core/config.py:262-330
    p.update(kw)
    return p


def box_results_with_nms_and_limit(scores, boxes, cfg=None, **kw):
    """scores (R, K), boxes (R, 4K) -> (scores (D,), boxes (D, 4), cls_boxes list of K arrays (n_j, 5)), like the reference."""
    p = _params(cfg, kw)
    dev = torch.device("cuda", torch.cuda.current_device())
    S = scores if torch.is_tensor(scores) else torch.from_numpy(np.ascontiguousarray(scores, dtype=np.float32))
    B = boxes if torch.is_tensor(boxes) else torch.from_numpy(np.ascontiguousarray(boxes, dtype=np.float32))
    S = S.to(dev, dtype=torch.float32); B = B.to(dev, dtype=torch.float32)
    K = int(p["num_classes"] or S.size(1))
    cls_boxes = [[] for _ in range(K)]
    # candidates of every class, in the reference's order (ascending detection index), one host read for the counts
    mask = S[:, 1:K] > float(p["score_thresh"])                       # (R, K-1)
    counts = mask.sum(dim=0).cpu().numpy().astype(np.int64)            # per class
    cls_idx, det_idx = torch.nonzero(mask.t(), as_tuple=True)          # grouped by class, ascending detection index inside
    j_of = cls_idx + 1
    sc = S[det_idx, j_of]
    bx = B.view(B.size(0), -1, 4)[det_idx, j_of]
    dets = torch.cat([bx, sc[:, None]], dim=1).contiguous()            # (sum counts, 5), class-major
    offs = np.concatenate([[0], np.cumsum(counts)])
    live = [j for j in range(K - 1) if counts[j] > 0]
    kept = {}
    if live:
        if p["soft_nms"]:
            out, inds, n_out = ops.soft_nms_batched(dets, [int(c) for c in counts], sigma=float(p["soft_sigma"]), overlap_thresh=float(p["nms"]),
                                                    score_thresh=0.0001, method=_SOFT_METHODS.get(p["soft_method"], 0))
            n_out = n_out.cpu().numpy()
            for j in live:
                kept[j] = out[offs[j]:offs[j] + int(n_out[j])]
        else:
            # score-sorted copies per class (stable), batched NMS, back to ascending original order like cython_nms.nms
            order = torch.empty_like(det_idx)
            for j in live:                                             # tiny per-class sorts; keys are (class, -score)
                seg = slice(int(offs[j]), int(offs[j + 1]))
                order[seg] = torch.sort(sc[seg], descending=True, stable=True)[1] + int(offs[j])
            sorted_dets = dets[order]
            keep, num = ops.nms_batched_chunked(sorted_dets, [int(c) for c in counts], float(p["nms"]), cython=True)
            num = num.cpu().numpy()
            for j in live:
                k = keep[offs[j]:offs[j] + int(num[j])].long() + int(offs[j])      # positions in the sorted copy
                orig = torch.sort(order[k])[0]                                       # ascending original index
                kept[j] = dets[orig]
        if p["bbox_vote"]:
            top_counts = [int(kept[j].size(0)) if j in kept else 0 for j in range(K - 1)]
            top = torch.cat([kept[j] for j in live], dim=0) if live else dets[:0]
            voted = ops.box_voting_batched(top, top_counts, dets, [int(c) for c in counts], float(p["vote_th"]),
                                           _VOTE_SCORING[p["vote_scoring"]], 1.0)
            o = 0
            for j in live:
                kept[j] = voted[o:o + top_counts[j]]; o += top_counts[j]
    for j in range(1, K):
        cls_boxes[j] = kept[j - 1].cpu().numpy() if (j - 1) in kept else np.zeros((0, 5), dtype=np.float32)
    # limit to max_per_image detections over all classes (host, like the reference: a sort of <= a few thousand scores)
    dpi = int(p["detections_per_im"])
    if dpi > 0:
        image_scores = np.hstack([cls_boxes[j][:, -1] for j in range(1, K)]) if K > 1 else np.zeros((0,), np.float32)
        if len(image_scores) > dpi:
            image_thresh = np.sort(image_scores)[-dpi]
            for j in range(1, K):
                keep = np.where(cls_boxes[j][:, -1] >= image_thresh)[0]
                cls_boxes[j] = cls_boxes[j][keep, :]
    im_results = np.vstack([cls_boxes[j] for j in range(1, K)]) if K > 1 else np.zeros((0, 5), np.float32)
    return im_results[:, -1], im_results[:, :-1], cls_boxes


def _segm_params(cfg, kw):
    if cfg is not None:
        p = dict(num_classes=cfg.MODEL.NUM_CLASSES, resolution=cfg.MRCNN.RESOLUTION, cls_specific_mask=cfg.MRCNN.CLS_SPECIFIC_MASK,
                 thresh_binarize=cfg.MRCNN.THRESH_BINARIZE)
    else:
        p = dict(num_classes=None, resolution=14, cls_specific_mask=True, thresh_binarize=0.5)       # lib/core/config.py:741-776
    p.update(kw)
    return p


def segm_results(cls_boxes, masks, ref_boxes, im_h, im_w, cfg=None, **kw):
    """cls_segms of lib/core/test.py:793-847: a list over classes of lists of COCO RLEs {'size': [im_h, im_w], 'counts': str},
    one per row of cls_boxes[j] (j >= 1), in the reference's order.  The masks are pasted and run-length encoded on the device
    (ops.segm_rle_raw: cv2's IPP-off resize arithmetic; pycocotools is not needed); the host only slices one string buffer.

    masks: the mask head's output, a numpy array (R, Kc, M, M) like the reference's or a float32 CUDA tensor (R, Kc * M * M) /
    (R, Kc, M, M), which skips the device-to-host copy; Kc is the number of classes for class-specific masks, else 1.
    ref_boxes: (R, 4) detections, numpy or CUDA, in the class-major order of cls_boxes.  Configuration: the reference's
    `cfg` (MODEL.NUM_CLASSES, MRCNN.RESOLUTION / CLS_SPECIFIC_MASK / THRESH_BINARIZE) or keyword arguments num_classes,
    resolution, cls_specific_mask, thresh_binarize."""
    p = _segm_params(cfg, kw)
    K = int(p["num_classes"] or len(cls_boxes))
    M = int(p["resolution"])
    im_h, im_w = int(im_h), int(im_w)
    n_per_class = [len(cls_boxes[j]) for j in range(1, K)]
    D = sum(n_per_class)
    if int(masks.shape[0]) != D:
        raise ValueError("segm_results: %d masks for %d detections" % (int(masks.shape[0]), D))
    cls_segms = [[] for _ in range(K)]
    if D == 0:
        return cls_segms
    dev = masks.device if torch.is_tensor(masks) and masks.is_cuda else torch.device("cuda", torch.cuda.current_device())
    mk = masks if torch.is_tensor(masks) else torch.from_numpy(np.ascontiguousarray(masks, dtype=np.float32))
    mk = mk.to(dev, dtype=torch.float32).reshape(D, -1, M, M)
    bx = ref_boxes if torch.is_tensor(ref_boxes) else torch.from_numpy(np.ascontiguousarray(ref_boxes, dtype=np.float32))
    bx = bx.to(dev, dtype=torch.float32)[:, :4]
    cls_of = np.repeat(np.arange(1, K, dtype=np.int32), n_per_class)
    if p["cls_specific_mask"]:
        if mk.size(1) < K:
            raise ValueError("segm_results: class-specific masks need %d channels, got %d" % (K, mk.size(1)))
        mask_class = torch.from_numpy(cls_of).to(dev)
    else:
        mask_class = torch.zeros((D,), dtype=torch.int32, device=dev)
    _, _, strings, string_offs = ops.segm_rle_raw(mk, mask_class, bx, im_h, im_w, float(p["thresh_binarize"]))
    buf = strings.cpu().numpy().tobytes()
    offs = string_offs.cpu().numpy()
    d = 0
    for j in range(1, K):
        segms = []
        for _ in range(n_per_class[j - 1]):
            segms.append({"size": [im_h, im_w], "counts": buf[offs[d]:offs[d + 1]].decode("ascii")})
            d += 1
        cls_segms[j] = segms
    return cls_segms


PERSON_CLASS_INDEX = 1          # lib/utils/keypoints.py:66-68


def _keypoint_params(cfg, kw):
    if cfg is not None:
        p = dict(num_classes=cfg.MODEL.NUM_CLASSES, num_keypoints=cfg.KRCNN.NUM_KEYPOINTS, inference_min_size=cfg.KRCNN.INFERENCE_MIN_SIZE,
                 nms_oks=cfg.KRCNN.NMS_OKS)
    else:
        p = dict(num_classes=None, num_keypoints=17, inference_min_size=0, nms_oks=False)        # lib/core/config.py:782-870
    p.update(kw)
    return p


def keypoint_results(cls_boxes, pred_heatmaps, ref_boxes, cfg=None, **kw):
    """cls_keyps of lib/core/test.py:850-866: a list over classes, empty except at the person class (index 1), which holds
    one float32 (4, K) array of (x, y, logit, prob) rows per detection, in the order of ref_boxes.  With NMS_OKS the OKS
    NMS (threshold 0.3) drops detections and cls_boxes[1] is filtered in place, like the reference.

    pred_heatmaps: the keypoint head's logits, a numpy array (R, K, M, M) like the reference's or a float32 CUDA tensor,
    which skips the device-to-host copy.  ref_boxes: (R, >=4) detections, numpy or CUDA.  The keypoints are extracted on
    the device in one launch (ops.heatmaps_to_keypoints_raw: cv2's float32 INTER_CUBIC arithmetic), plus one for the OKS
    NMS; the host reads the (R, 4, K) result once (and, with NMS_OKS, the kept indices).  Configuration: the reference's
    `cfg` (MODEL.NUM_CLASSES, KRCNN.NUM_KEYPOINTS / INFERENCE_MIN_SIZE / NMS_OKS) or keyword arguments num_classes,
    num_keypoints, inference_min_size, nms_oks."""
    p = _keypoint_params(cfg, kw)
    num_classes = int(p["num_classes"] or len(cls_boxes))
    cls_keyps = [[] for _ in range(num_classes)]
    D = int(pred_heatmaps.shape[0])
    if len(pred_heatmaps.shape) != 4 or int(pred_heatmaps.shape[1]) != int(p["num_keypoints"]):
        raise ValueError("keypoint_results: heatmaps must be (R, %d, M, M), got %s" % (int(p["num_keypoints"]), tuple(pred_heatmaps.shape)))
    if int(ref_boxes.shape[0]) != D:
        raise ValueError("keypoint_results: %d heatmaps for %d boxes" % (D, int(ref_boxes.shape[0])))
    if D == 0:
        return cls_keyps
    dev = next((x.device for x in (pred_heatmaps, ref_boxes) if torch.is_tensor(x) and x.is_cuda),
               torch.device("cuda", torch.cuda.current_device()))
    maps = pred_heatmaps if torch.is_tensor(pred_heatmaps) else torch.from_numpy(np.ascontiguousarray(pred_heatmaps, dtype=np.float32))
    rois = ref_boxes if torch.is_tensor(ref_boxes) else torch.from_numpy(np.ascontiguousarray(ref_boxes, dtype=np.float32))
    maps = maps.to(dev, dtype=torch.float32)
    rois = rois.to(dev, dtype=torch.float32)
    xy = ops.heatmaps_to_keypoints_raw(maps, rois, int(p["inference_min_size"]))
    if p["nms_oks"]:
        keep_dev, num_keep = ops.nms_oks_raw(xy, rois, 0.3)
    xy_preds = xy.cpu().numpy()
    if p["nms_oks"]:
        keep = keep_dev[:int(num_keep.item())].cpu().tolist()
        xy_preds = xy_preds[keep]
        cls_boxes[PERSON_CLASS_INDEX] = cls_boxes[PERSON_CLASS_INDEX][keep, :]
    cls_keyps[PERSON_CLASS_INDEX] = [xy_preds[i] for i in range(xy_preds.shape[0])]
    return cls_keyps


def get_blobs(im, rois, target_scale, target_max_size, cfg=None, **kw):
    """_get_blobs with _get_rois_blob (lib/core/test.py:869-929): blobs['data'] is the device image blob (utils/blob.py),
    blobs['im_info'] the float32 (1, 3) numpy (Hp, Wp, im_scale); with rois (R, 4) in image coordinates, blobs['rois'] is
    the float32 (R, 5) [0, x1, y1, x2, y2] projection, multiplied in float64 like _project_im_rois.  Returns (blobs, im_scale)."""
    from ..utils import blob as blob_utils
    blobs = {}
    blobs["data"], im_scale, blobs["im_info"] = blob_utils.get_image_blob(im, target_scale, target_max_size, cfg, **kw)
    if rois is not None:
        r = np.asarray(rois).astype(np.float64, copy=False) * im_scale
        levels = np.zeros((r.shape[0], 1), dtype=np.int64)
        blobs["rois"] = np.hstack((levels, r)).astype(np.float32, copy=False)
    return blobs, im_scale
