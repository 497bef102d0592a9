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

`im_detect_mask_aug` / `im_detect_keypoints_aug` (lib/core/test.py:365-729) run the heads over the test-time transforms in the
reference's order, build every transform's blob on the device and fold each head output into one running CUDA accumulator
(ops.tta_combine_raw); the combined masks / heatmaps are CUDA tensors for segm_results / keypoint_results.

`im_detect_bbox` / `im_detect_bbox_aug` (lib/core/test.py:127-362) decode the box head on the device, one launch per transform with
the transform's inverse in the same store (ops.bbox_decode_raw), and combine the transforms there; scores and boxes are CUDA tensors
for box_results_with_nms_and_limit.
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


def get_blobs(im, rois, target_scale, target_max_size, cfg=None, _hflip=False, **kw):
    """_get_blobs with _get_rois_blob (lib/core/test.py:869-929): blobs['data'] is the device image blob (utils/blob.py),
    blobs['im_info'] the float32 (1, 3) numpy (Hp, Wp, im_scale); with rois (R, 4) in image coordinates, blobs['rois'] is
    the float32 (R, 5) [0, x1, y1, x2, y2] projection, multiplied in float64 like _project_im_rois.  Returns (blobs, im_scale).
    _hflip: the blobs of im[:, ::-1, :] (the rois are taken as given)."""
    from ..utils import blob as blob_utils
    blobs = {}
    blobs["data"], im_scale, blobs["im_info"] = blob_utils.get_image_blob(im, target_scale, target_max_size, cfg, _hflip=_hflip, **kw)
    if rois is not None:
        blobs["rois"] = _get_rois_blob(rois, im_scale)
    return blobs, im_scale


# ------------------------------------------------------------------------------------------------
# Test-time augmentation of the mask and keypoint heads (lib/core/test.py:365-729)
# ------------------------------------------------------------------------------------------------
_MASK_HEURS = ("SOFT_AVG", "SOFT_MAX", "LOGIT_AVG")
_KPS_HEURS = ("HM_AVG", "HM_MAX")


def _aug_params(cfg, kw):
    """The configuration the mask / keypoint test-time functions read (flat keys; `mask_aug` / `kps_aug` hold TEST.MASK_AUG /
    TEST.KPS_AUG as dicts of lower-case keys).  From the reference's `cfg` at call time, else the reference's defaults
    (lib/core/config.py), then the keyword arguments.  Blob keys (pixel_means, fpn_on, coarsest_stride) go to utils/blob.py."""
    def aug(a):
        return dict(heur=a.HEUR, h_flip=a.H_FLIP, scales=tuple(a.SCALES), max_size=a.MAX_SIZE, scale_h_flip=a.SCALE_H_FLIP,
                    scale_size_dep=a.SCALE_SIZE_DEP, area_th=a.AREA_TH, aspect_ratios=tuple(a.ASPECT_RATIOS),
                    aspect_ratio_h_flip=a.ASPECT_RATIO_H_FLIP)
    def bbox_aug(a):
        return dict(score_heur=a.SCORE_HEUR, coord_heur=a.COORD_HEUR, h_flip=a.H_FLIP, scales=tuple(a.SCALES), max_size=a.MAX_SIZE,
                    scale_h_flip=a.SCALE_H_FLIP, scale_size_dep=a.SCALE_SIZE_DEP, aspect_ratios=tuple(a.ASPECT_RATIOS),
                    aspect_ratio_h_flip=a.ASPECT_RATIO_H_FLIP)
    if cfg is not None:
        p = dict(num_classes=cfg.MODEL.NUM_CLASSES, resolution=cfg.MRCNN.RESOLUTION, cls_specific_mask=cfg.MRCNN.CLS_SPECIFIC_MASK,
                 num_keypoints=cfg.KRCNN.NUM_KEYPOINTS, heatmap_size=cfg.KRCNN.HEATMAP_SIZE, test_scale=cfg.TEST.SCALE,
                 test_max_size=cfg.TEST.MAX_SIZE, multilevel_rois=cfg.FPN.MULTILEVEL_ROIS, roi_min_level=cfg.FPN.ROI_MIN_LEVEL,
                 roi_max_level=cfg.FPN.ROI_MAX_LEVEL, roi_canonical_scale=cfg.FPN.ROI_CANONICAL_SCALE,
                 roi_canonical_level=cfg.FPN.ROI_CANONICAL_LEVEL, mask_aug=aug(cfg.TEST.MASK_AUG), kps_aug=aug(cfg.TEST.KPS_AUG),
                 faster_rcnn=bool(cfg.MODEL.FASTER_RCNN), dedup_boxes=cfg.DEDUP_BOXES, bbox_reg=bool(cfg.TEST.BBOX_REG),
                 cls_agnostic_bbox_reg=bool(cfg.MODEL.CLS_AGNOSTIC_BBOX_REG), bbox_reg_weights=tuple(cfg.MODEL.BBOX_REG_WEIGHTS),
                 bbox_xform_clip=float(cfg.BBOX_XFORM_CLIP),
                 bbox_normalize_targets_precomputed=bool(cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED),
                 bbox_aug=bbox_aug(cfg.TEST.BBOX_AUG),
                 blob=dict(pixel_means=cfg.PIXEL_MEANS, fpn_on=bool(cfg.FPN.FPN_ON), coarsest_stride=int(cfg.FPN.COARSEST_STRIDE)))
    else:
        from ..utils.blob import blob_params
        defaults = dict(heur=None, h_flip=False, scales=(), max_size=4000, scale_h_flip=False, scale_size_dep=False, area_th=180 ** 2,
                        aspect_ratios=(), aspect_ratio_h_flip=False)             # lib/core/config.py:249-354
        p = dict(num_classes=None, resolution=14, cls_specific_mask=True, num_keypoints=17, heatmap_size=56, test_scale=600,
                 test_max_size=1000, multilevel_rois=False, roi_min_level=2, roi_max_level=5, roi_canonical_scale=224,
                 roi_canonical_level=4, mask_aug=dict(defaults, heur="SOFT_AVG"), kps_aug=dict(defaults, heur="HM_AVG"),
                 faster_rcnn=False, dedup_boxes=1. / 16., bbox_reg=True, cls_agnostic_bbox_reg=False,
                 bbox_reg_weights=(10., 10., 5., 5.), bbox_xform_clip=float(np.log(1000. / 16.)),
                 bbox_normalize_targets_precomputed=False,                       # lib/core/config.py:96, 196, 408-430, 931-936
                 bbox_aug=dict(defaults, score_heur="UNION", coord_heur="UNION"),
                 blob=blob_params())
        del p["bbox_aug"]["heur"], p["bbox_aug"]["area_th"]
    for key in ("mask_aug", "kps_aug", "bbox_aug", "blob"):
        p[key] = dict(p[key], **kw.pop(key, {}))
    for key in ("pixel_means", "fpn_on", "coarsest_stride"):
        if key in kw:
            p["blob"][key] = kw.pop(key)
    unknown = set(kw) - set(p)
    if unknown:
        raise TypeError("unexpected configuration keywords %s" % sorted(unknown))
    p.update(kw)
    return p


def _get_rois_blob(im_rois, im_scale):
    """lib/core/test.py:869-898: (R, 5) float32 [0, x1, y1, x2, y2], the boxes multiplied by im_scale in float64."""
    rois = np.asarray(im_rois).astype(np.float64, copy=False) * im_scale
    levels = np.zeros((rois.shape[0], 1), dtype=np.int64)
    return np.hstack((levels, rois)).astype(np.float32, copy=False)


def _add_multilevel_rois_for_test(blobs, name, p):
    """lib/core/test.py:901-920 with lib/utils/fpn.py: blobs[name + '_fpn<l>'] the rows of blobs[name] whose FPN level is l
    (numpy's float32 Eqn. (1) of the FPN paper, as the reference evaluates it) and blobs[name + '_idx_restore_int32'] the
    permutation back to the original order.  Host numpy: these are a few hundred rows, and the RoI transform reads them there."""
    lvl_min, lvl_max = int(p["roi_min_level"]), int(p["roi_max_level"])
    rois = blobs[name]
    boxes = rois[:, 1:5]
    areas = (boxes[:, 2] - boxes[:, 0] + 1) * (boxes[:, 3] - boxes[:, 1] + 1)
    areas[areas < 0] = 0
    s = np.sqrt(areas)
    lvls = np.clip(np.floor(p["roi_canonical_level"] + np.log2(s / p["roi_canonical_scale"] + 1e-6)), lvl_min, lvl_max)
    idx_order = np.empty((0,))
    for lvl in range(lvl_min, lvl_max + 1):
        idx_lvl = np.where(lvls == lvl)[0]
        blobs[name + "_fpn" + str(lvl)] = rois[idx_lvl, :]
        idx_order = np.concatenate((idx_order, idx_lvl))
    blobs[name + "_idx_restore_int32"] = np.argsort(idx_order).astype(np.int32, copy=False)


class _RunningCombine:
    """The reference's list of per-transform head outputs and its np.mean / np.amax (or logit mean) over them, kept as one
    running (R, C, M, M) CUDA accumulator that each transform is folded into as it arrives (ops.tta_combine_raw): a transform is
    read once, mirrored and channel-permuted in that read when it came from a flipped image.  `include` (R,) bool selects the
    rows a transform takes part in (combine_heatmaps_size_dep); every row must be included at least once."""

    def __init__(self, heur):
        self.heur = ops.TTA_HEURISTICS[heur]
        self.acc = None
        self.count = None

    def add(self, out, hflip=False, perm=None, include=None):
        if self.acc is None:
            self.acc = torch.empty(out.shape, dtype=torch.float32, device=out.device)
            self.count = np.zeros((out.shape[0],), dtype=np.int64)
        if self.acc.numel() == 0:
            return
        row_op, op = None, ops.TTA_FOLD if self.count.any() else ops.TTA_START
        if include is not None:
            include = np.asarray(include, dtype=bool)
            ops_host = np.where(include, np.where(self.count == 0, ops.TTA_START, ops.TTA_FOLD), ops.TTA_SKIP).astype(np.uint8)
            row_op = torch.from_numpy(ops_host).to(out.device)
            self.count += include
        else:
            if self.count.any() and not self.count.all():
                raise ValueError("a transform for every row after one for some rows")
            self.count += 1
        ops.tta_combine_raw(out, self.acc, self.heur, op=op, hflip=hflip, channel_perm=perm, row_op=row_op)

    def result(self):
        if self.acc.numel() == 0:
            return self.acc
        if (self.count < 1).any():
            raise ValueError("every row needs at least one transform")
        if (self.count == self.count[0]).all():
            return ops.tta_finish_raw(self.acc, self.heur, count=int(self.count[0]))
        return ops.tta_finish_raw(self.acc, self.heur, row_count=torch.from_numpy(self.count.astype(np.int32)))


def _conv_body(model, im, target_scale, target_max_size, hflip, p):
    """im_conv_body_only on the image, or on im[:, ::-1, :] when hflip (the blob kernel's flip flag reads it mirrored)."""
    from ..utils import blob as blob_utils
    h, w = int(im.shape[0]), int(im.shape[1])
    im_scale = blob_utils.get_target_scale(min(h, w), max(h, w), target_scale, target_max_size)
    bp = p["blob"]
    data, _ = ops.image_blob_raw([im], [im_scale], [hflip], bp["pixel_means"], bp["coarsest_stride"] if bp["fpn_on"] else None)
    blob_conv = model.module.convbody_net(data=data)
    return blob_conv, im_scale


def im_conv_body_only(model, im, target_scale, target_max_size, cfg=None, **kw):
    """lib/core/test.py:117-129: the backbone on the device blob of im (uint8 (H, W, 3), host or CUDA).  Returns (blob_conv, im_scale)."""
    return _conv_body(model, im, target_scale, target_max_size, False, _aug_params(cfg, kw))


def _head_inputs(name, boxes, im_scale, p):
    inputs = {name: _get_rois_blob(boxes, im_scale)}
    if p["multilevel_rois"]:
        _add_multilevel_rois_for_test(inputs, name, p)
    return inputs


def _detect_mask(model, im_scale, boxes, blob_conv, p):
    M = int(p["resolution"])
    if boxes.shape[0] == 0:
        return torch.zeros((0, M, M), dtype=torch.float32, device=torch.device("cuda", torch.cuda.current_device()))
    pred_masks = model.module.mask_net(blob_conv, _head_inputs("mask_rois", boxes, im_scale, p))
    return pred_masks.detach().to(torch.float32).reshape(boxes.shape[0], -1, M, M)


def _detect_keypoints(model, im_scale, boxes, blob_conv, p):
    M = int(p["heatmap_size"])
    if boxes.shape[0] == 0:
        return torch.zeros((0, int(p["num_keypoints"]), M, M), dtype=torch.float32, device=torch.device("cuda", torch.cuda.current_device()))
    pred_heatmaps = model.module.keypoint_net(blob_conv, _head_inputs("keypoint_rois", boxes, im_scale, p))
    return pred_heatmaps.detach().to(torch.float32).reshape(boxes.shape[0], -1, M, M)


def _transform(out, hflip, perm):
    """A flipped transform's output as the reference returns it (masks[..., ::-1] / flip_heatmaps), in one copy kernel."""
    if not hflip:
        return out
    return ops.tta_combine_raw(out, torch.empty(out.shape, dtype=torch.float32, device=out.device), ops.TTA_HEURISTICS["HM_MAX"],
                               op=ops.TTA_START, hflip=True, channel_perm=perm)


def _flip_perm(kind, J):
    if kind == "mask":
        return None
    from ..utils.keypoints import flip_permutation
    return flip_permutation(J)


def _detect(kind, model, im_scale, boxes, blob_conv, p):
    return (_detect_mask if kind == "mask" else _detect_keypoints)(model, im_scale, boxes, blob_conv, p)


def _hflip_raw(kind, model, im, target_scale, target_max_size, boxes, p):
    """im_detect_<kind>_hflip without the final inversion: the head output on the flipped image (the caller mirrors it)."""
    from ..utils.boxes import flip_boxes
    boxes_hf = flip_boxes(boxes, int(im.shape[1]))
    blob_conv, im_scale = _conv_body(model, im, target_scale, target_max_size, True, p)
    return _detect(kind, model, im_scale, boxes_hf, blob_conv, p)


def _scale_raw(kind, model, im, target_scale, target_max_size, boxes, hflip, p):
    if hflip:
        return _hflip_raw(kind, model, im, target_scale, target_max_size, boxes, p)
    blob_conv, im_scale = _conv_body(model, im, target_scale, target_max_size, False, p)
    return _detect(kind, model, im_scale, boxes, blob_conv, p)


def _aspect_ratio_raw(kind, model, im, aspect_ratio, boxes, hflip, p):
    from ..utils.boxes import aspect_ratio as boxes_aspect_ratio
    from ..utils.image import aspect_ratio_rel
    im_ar = aspect_ratio_rel(im, aspect_ratio)
    boxes_ar = boxes_aspect_ratio(boxes, aspect_ratio)
    return _scale_raw(kind, model, im_ar, p["test_scale"], p["test_max_size"], boxes_ar, hflip, p)


def _size_dep_include(boxes, ds_t, us_t, area_th):
    """combine_heatmaps_size_dep's selection: a downscaled transform is left out for small and medium objects (area < AREA_TH),
    an upscaled one for large objects.  Areas are the reference's float32 `+ 1` box areas."""
    b = np.asarray(boxes)
    areas = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
    sm_objs = areas < area_th
    l_objs = areas >= area_th
    return ~((sm_objs & bool(ds_t)) | (l_objs & bool(us_t)))


def _aug(kind, model, im, boxes, im_scale, blob_conv, p):
    """The transform loop of im_detect_mask_aug / im_detect_keypoints_aug, in the reference's order, folding each output into
    the running combine as it arrives."""
    a = p["mask_aug" if kind == "mask" else "kps_aug"]
    if kind == "mask":
        assert not a["scale_size_dep"], 'Size dependent scaling not implemented'
    if a["heur"] not in (_MASK_HEURS if kind == "mask" else _KPS_HEURS):
        raise NotImplementedError('Heuristic {} not supported'.format(a["heur"]))
    size_dep = kind == "keypoints" and a["scale_size_dep"]
    comb = _RunningCombine(a["heur"])
    perm = [None]

    def add(out, hflip=False, ds_t=False, us_t=False):
        if hflip and perm[0] is None and kind != "mask":
            perm[0] = _flip_perm(kind, out.shape[1])
        comb.add(out, hflip=hflip, perm=perm[0] if hflip else None,
                 include=_size_dep_include(boxes, ds_t, us_t, a["area_th"]) if size_dep else None)

    add(_detect(kind, model, im_scale, boxes, blob_conv, p))
    if a["h_flip"]:
        add(_hflip_raw(kind, model, im, p["test_scale"], p["test_max_size"], boxes, p), hflip=True)
    for scale in a["scales"]:
        ds_scl, us_scl = scale < p["test_scale"], scale > p["test_scale"]
        add(_scale_raw(kind, model, im, scale, a["max_size"], boxes, False, p), ds_t=ds_scl, us_t=us_scl)
        if a["scale_h_flip"]:
            add(_scale_raw(kind, model, im, scale, a["max_size"], boxes, True, p), hflip=True, ds_t=ds_scl, us_t=us_scl)
    for aspect_ratio in a["aspect_ratios"]:
        add(_aspect_ratio_raw(kind, model, im, aspect_ratio, boxes, False, p))
        if a["aspect_ratio_h_flip"]:
            add(_aspect_ratio_raw(kind, model, im, aspect_ratio, boxes, True, p), hflip=True)
    return comb.result()


def im_detect_mask(model, im_scale, boxes, blob_conv, cfg=None, **kw):
    """lib/core/test.py:365-401: the mask head on boxes (R, 4) projected by im_scale (host rois / FPN blobs, like the reference).
    Returns the soft masks as a float32 CUDA tensor (R, Kc, M, M), which segm_results takes without a copy to the host."""
    return _detect_mask(model, im_scale, boxes, blob_conv, _aug_params(cfg, kw))


def im_detect_mask_aug(model, im, boxes, im_scale, blob_conv, cfg=None, **kw):
    """lib/core/test.py:404-475: the soft masks combined over TEST.MASK_AUG's transforms (identity, H_FLIP, SCALES with
    SCALE_H_FLIP, ASPECT_RATIOS with ASPECT_RATIO_H_FLIP) by HEUR, the model called in the reference's order.  The
    transforms are combined on the device as they arrive.  Returns a float32 CUDA tensor (R, Kc, M, M).  An unknown HEUR
    raises NotImplementedError before the first transform runs (the reference raises after the last)."""
    return _aug("mask", model, im, boxes, im_scale, blob_conv, _aug_params(cfg, kw))


def im_detect_mask_hflip(model, im, target_scale, target_max_size, boxes, cfg=None, **kw):
    """lib/core/test.py:478-492: masks of the flipped image, mirrored back.  float32 CUDA (R, Kc, M, M)."""
    return _transform(_hflip_raw("mask", model, im, target_scale, target_max_size, boxes, _aug_params(cfg, kw)), True, None)


def im_detect_mask_scale(model, im, target_scale, target_max_size, boxes, hflip=False, cfg=None, **kw):
    """lib/core/test.py:495-505."""
    return _transform(_scale_raw("mask", model, im, target_scale, target_max_size, boxes, hflip, _aug_params(cfg, kw)), hflip, None)


def im_detect_mask_aspect_ratio(model, im, aspect_ratio, boxes, hflip=False, cfg=None, **kw):
    """lib/core/test.py:508-526: the image resized by utils/image.py aspect_ratio_rel on the device."""
    return _transform(_aspect_ratio_raw("mask", model, im, aspect_ratio, boxes, hflip, _aug_params(cfg, kw)), hflip, None)


def im_detect_keypoints(model, im_scale, boxes, blob_conv, cfg=None, **kw):
    """lib/core/test.py:529-563: the keypoint head's logits as a float32 CUDA tensor (R, J, M, M), which keypoint_results takes
    without a copy to the host."""
    return _detect_keypoints(model, im_scale, boxes, blob_conv, _aug_params(cfg, kw))


def im_detect_keypoints_aug(model, im, boxes, im_scale, blob_conv, cfg=None, **kw):
    """lib/core/test.py:566-647: the heatmaps combined over TEST.KPS_AUG's transforms by HEUR (HM_AVG / HM_MAX), with
    SCALE_SIZE_DEP's per-object selection, on the device.  Returns a float32 CUDA tensor (R, J, M, M).

    With SCALE_SIZE_DEP the reference's combine_heatmaps_size_dep fails under this version of its utils.boxes.boxes_area,
    which returns (areas, negative indices); here the areas are used, as the selection intends."""
    return _aug("keypoints", model, im, boxes, im_scale, blob_conv, _aug_params(cfg, kw))


def im_detect_keypoints_hflip(model, im, target_scale, target_max_size, boxes, cfg=None, **kw):
    """lib/core/test.py:650-664: heatmaps of the flipped image, inverted by flip_heatmaps (one copy kernel)."""
    p = _aug_params(cfg, kw)
    out = _hflip_raw("keypoints", model, im, target_scale, target_max_size, boxes, p)
    return _transform(out, True, _flip_perm("keypoints", out.shape[1]))


def im_detect_keypoints_scale(model, im, target_scale, target_max_size, boxes, hflip=False, cfg=None, **kw):
    """lib/core/test.py:667-677."""
    out = _scale_raw("keypoints", model, im, target_scale, target_max_size, boxes, hflip, _aug_params(cfg, kw))
    return _transform(out, hflip, _flip_perm("keypoints", out.shape[1]) if hflip else None)


def im_detect_keypoints_aspect_ratio(model, im, aspect_ratio, boxes, hflip=False, cfg=None, **kw):
    """lib/core/test.py:680-697."""
    out = _aspect_ratio_raw("keypoints", model, im, aspect_ratio, boxes, hflip, _aug_params(cfg, kw))
    return _transform(out, hflip, _flip_perm("keypoints", out.shape[1]) if hflip else None)


def combine_heatmaps_size_dep(hms_ts, ds_ts, us_ts, boxes, heur, cfg=None, **kw):
    """lib/core/test.py:700-729: per object, the heatmaps of the transforms it keeps (no downscaled ones for objects with
    area < KPS_AUG.AREA_TH, no upscaled ones for the others) combined by heur ('HM_AVG' / 'HM_MAX', or np.mean / np.amax).
    hms_ts: (R, J, M, M) float32 CUDA tensors (or numpy).  Returns a float32 CUDA tensor."""
    assert len(hms_ts) == len(ds_ts) and len(ds_ts) == len(us_ts), \
        'All sets of hms must be tagged with downscaling and upscaling flags'
    p = _aug_params(cfg, kw)
    heur = {np.mean: "HM_AVG", np.amax: "HM_MAX", np.max: "HM_MAX"}.get(heur, heur)
    if heur not in _KPS_HEURS:
        raise NotImplementedError('Heuristic {} not supported'.format(heur))
    comb = _RunningCombine(heur)
    dev = torch.device("cuda", torch.cuda.current_device())
    for hms_t, ds_t, us_t in zip(hms_ts, ds_ts, us_ts):
        t = hms_t if torch.is_tensor(hms_t) else torch.from_numpy(np.ascontiguousarray(hms_t, dtype=np.float32))
        comb.add(t.to(dev, dtype=torch.float32), include=_size_dep_include(boxes, ds_t, us_t, p["kps_aug"]["area_th"]))
    return comb.result()


# ------------------------------------------------------------------------------------------------
# The box head and its test-time augmentation (lib/core/test.py:127-362)
# ------------------------------------------------------------------------------------------------
_BBOX_HEURS = ("ID", "AVG", "UNION")


def _head_rows(t):
    """The reference's `.squeeze()` then `.reshape([-1, shape[-1]])` (one proposal gives a 1-D squeeze), on the device."""
    t = t.detach() if torch.is_tensor(t) else torch.from_numpy(np.ascontiguousarray(t))
    t = t.to(torch.device("cuda", torch.cuda.current_device()) if not t.is_cuda else t.device, dtype=torch.float32).squeeze()
    return t.reshape(-1, t.shape[-1])


def _detect_bbox(model, im, target_scale, target_max_size, boxes, hflip, ar_inv, p):
    """im_detect_bbox on im (im[:, ::-1, :] when hflip, read mirrored by the blob kernel), with the transform's inverse
    (flip_boxes with im's width when hflip, then x * float32(ar_inv)) applied in the decode's store.  boxes: the proposals the
    model sees (already flipped / aspect-scaled), or None with FASTER_RCNN.  Returns (scores, pred_boxes, im_scale, blob_conv)."""
    if p["bbox_reg"] and p["bbox_normalize_targets_precomputed"]:
        # the reference's `box_deltas.view(-1, 4)` on a numpy array raises too (lib/core/test.py:172-175)
        raise NotImplementedError("TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED is not supported at test time")
    inputs, im_scale = get_blobs(im, boxes, target_scale, target_max_size, _hflip=hflip, **p["blob"])
    dedup = p["dedup_boxes"] > 0 and not p["faster_rcnn"]
    if dedup:
        v = np.array([1, 1e3, 1e6, 1e9, 1e12])
        hashes = np.round(inputs["rois"] * p["dedup_boxes"]).dot(v)
        _, index, inv_index = np.unique(hashes, return_index=True, return_inverse=True)
        inputs["rois"] = inputs["rois"][index, :]
        boxes = boxes[index, :]
    if p["multilevel_rois"] and not p["faster_rcnn"]:
        _add_multilevel_rois_for_test(inputs, "rois", p)
    inputs["data"] = [inputs["data"]]
    inputs["im_info"] = [torch.from_numpy(inputs["im_info"])]
    return_dict = model(**inputs)

    scores = _head_rows(return_dict["cls_score"])
    K = int(scores.shape[1])
    if p["faster_rcnn"]:
        rois, scale = return_dict["rois"], im_scale
        rois = rois.detach() if torch.is_tensor(rois) else torch.from_numpy(np.ascontiguousarray(rois))
    else:
        rois, scale = torch.from_numpy(np.ascontiguousarray(boxes, dtype=np.float32)), None
    rois = rois.to(scores.device, dtype=torch.float32)
    deltas = _head_rows(return_dict["bbox_pred"]) if p["bbox_reg"] else None
    pred_boxes = ops.bbox_decode_raw(rois, deltas, K, int(im.shape[0]), int(im.shape[1]), im_scale=scale, bbox_reg=p["bbox_reg"],
                                     weights=p["bbox_reg_weights"], xform_clip=p["bbox_xform_clip"],
                                     agnostic=p["cls_agnostic_bbox_reg"], flip_width=int(im.shape[1]) if hflip else None, ar_inv=ar_inv)
    if dedup:
        inv = torch.from_numpy(np.asarray(inv_index, dtype=np.int64).reshape(-1)).to(scores.device)
        scores, pred_boxes = scores[inv], pred_boxes[inv]
    return scores, pred_boxes, im_scale, return_dict["blob_conv"]


def im_detect_bbox(model, im, target_scale, target_max_size, boxes=None, cfg=None, **kw):
    """lib/core/test.py:127-189: the model on the device blob of im (with the proposals `boxes` (R, 4) unless FASTER_RCNN),
    the deltas decoded and clipped on the device (ops.bbox_decode_raw).  Returns (scores float32 CUDA (R, K), pred_boxes float32
    CUDA (R, 4K), im_scale, blob_conv); box_results_with_nms_and_limit takes both tensors as they are.  The host keeps only the
    small arrays the reference builds there: im_info, the rois / FPN level blobs and the DEDUP_BOXES hashes.
    TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED raises NotImplementedError (the reference's own line fails on its numpy deltas)."""
    return _detect_bbox(model, im, target_scale, target_max_size, boxes, False, 1.0, _aug_params(cfg, kw))


def _bbox_hflip(model, im, target_scale, target_max_size, box_proposals, ar_inv, p):
    from ..utils.boxes import flip_boxes
    box_proposals_hf = None if p["faster_rcnn"] else flip_boxes(box_proposals, int(im.shape[1]))
    scores_hf, boxes_inv, im_scale, _ = _detect_bbox(model, im, target_scale, target_max_size, box_proposals_hf, True, ar_inv, p)
    return scores_hf, boxes_inv, im_scale


def im_detect_bbox_hflip(model, im, target_scale, target_max_size, box_proposals=None, cfg=None, **kw):
    """lib/core/test.py:289-310: detections on the flipped image (the blob kernel reads im mirrored), flipped back in the decode.
    Returns (scores, boxes, im_scale), CUDA like im_detect_bbox."""
    return _bbox_hflip(model, im, target_scale, target_max_size, box_proposals, 1.0, _aug_params(cfg, kw))


def _bbox_scale(model, im, target_scale, target_max_size, box_proposals, hflip, p):
    if hflip:
        return _bbox_hflip(model, im, target_scale, target_max_size, box_proposals, 1.0, p)[:2]
    return _detect_bbox(model, im, target_scale, target_max_size, box_proposals, False, 1.0, p)[:2]


def im_detect_bbox_scale(model, im, target_scale, target_max_size, box_proposals=None, hflip=False, cfg=None, **kw):
    """lib/core/test.py:313-326.  Returns (scores, boxes), CUDA."""
    return _bbox_scale(model, im, target_scale, target_max_size, box_proposals, hflip, _aug_params(cfg, kw))


def _bbox_aspect_ratio(model, im, aspect_ratio, box_proposals, hflip, p):
    from ..utils.boxes import aspect_ratio as boxes_aspect_ratio
    from ..utils.image import aspect_ratio_rel
    im_ar = aspect_ratio_rel(im, aspect_ratio)
    box_proposals_ar = None if p["faster_rcnn"] else boxes_aspect_ratio(box_proposals, aspect_ratio)
    ar_inv = 1.0 / aspect_ratio
    if hflip:
        return _bbox_hflip(model, im_ar, p["test_scale"], p["test_max_size"], box_proposals_ar, ar_inv, p)[:2]
    return _detect_bbox(model, im_ar, p["test_scale"], p["test_max_size"], box_proposals_ar, False, ar_inv, p)[:2]


def im_detect_bbox_aspect_ratio(model, im, aspect_ratio, box_proposals=None, hflip=False, cfg=None, **kw):
    """lib/core/test.py:329-362: detections on the image resized by utils/image.py aspect_ratio_rel on the device, the boxes
    mapped back (`x * float32(1 / aspect_ratio)`) in the decode.  Returns (scores, boxes), CUDA."""
    return _bbox_aspect_ratio(model, im, aspect_ratio, box_proposals, hflip, _aug_params(cfg, kw))


class _BoxCombine:
    """One of SCORE_HEUR / COORD_HEUR over the transforms, as they arrive: UNION concatenates on the device, AVG folds each
    (R, C) output into _RunningCombine as an (R, C, 1, 1) view (np.mean over the stacked float32 outputs, bit for bit), ID keeps
    the identity transform's output."""

    def __init__(self, heur):
        self.heur, self.parts = heur, []
        self.mean = _RunningCombine("SOFT_AVG") if heur == "AVG" else None

    def add(self, out, identity):
        if self.heur == "UNION" or (self.heur == "ID" and identity):
            self.parts.append(out)
        elif self.heur == "AVG":
            self.mean.add(out.reshape(out.shape[0], out.shape[1], 1, 1))

    def result(self):
        if self.heur == "AVG":
            out = self.mean.result()
            return out.reshape(out.shape[0], out.shape[1])
        return self.parts[0] if len(self.parts) == 1 else torch.cat(self.parts, dim=0)


def im_detect_bbox_aug(model, im, box_proposals=None, cfg=None, **kw):
    """lib/core/test.py:192-286: scores and boxes over TEST.BBOX_AUG's transforms (H_FLIP, SCALES with SCALE_H_FLIP,
    ASPECT_RATIOS with ASPECT_RATIO_H_FLIP, then the identity last), the model called in the reference's order, every head
    output decoded and combined on the device (SCORE_HEUR / COORD_HEUR: UNION concatenates, AVG averages as np.mean does, ID
    takes the identity's).  Returns (scores float32 CUDA, boxes float32 CUDA, im_scale, blob_conv) of the identity transform.
    An unknown heuristic raises NotImplementedError before the first model call (the reference raises after the last)."""
    p = _aug_params(cfg, kw)
    a = p["bbox_aug"]
    assert not a["scale_size_dep"], 'Size dependent scaling not implemented'
    assert not a["score_heur"] == 'UNION' or a["coord_heur"] == 'UNION', \
        'Coord heuristic must be union whenever score heuristic is union'
    assert not a["coord_heur"] == 'UNION' or a["score_heur"] == 'UNION', \
        'Score heuristic must be union whenever coord heuristic is union'
    assert not p["faster_rcnn"] or a["score_heur"] == 'UNION', \
        'Union heuristic must be used to combine Faster RCNN predictions'
    if a["score_heur"] not in _BBOX_HEURS:
        raise NotImplementedError('Score heur {} not supported'.format(a["score_heur"]))
    if a["coord_heur"] not in _BBOX_HEURS:
        raise NotImplementedError('Coord heur {} not supported'.format(a["coord_heur"]))
    scores_c, boxes_c = _BoxCombine(a["score_heur"]), _BoxCombine(a["coord_heur"])

    def add_preds_t(scores_t, boxes_t, identity=False):
        scores_c.add(scores_t, identity)
        boxes_c.add(boxes_t, identity)

    if a["h_flip"]:
        add_preds_t(*_bbox_hflip(model, im, p["test_scale"], p["test_max_size"], box_proposals, 1.0, p)[:2])
    for scale in a["scales"]:
        add_preds_t(*_bbox_scale(model, im, scale, a["max_size"], box_proposals, False, p))
        if a["scale_h_flip"]:
            add_preds_t(*_bbox_scale(model, im, scale, a["max_size"], box_proposals, True, p))
    for aspect_ratio in a["aspect_ratios"]:
        add_preds_t(*_bbox_aspect_ratio(model, im, aspect_ratio, box_proposals, False, p))
        if a["aspect_ratio_h_flip"]:
            add_preds_t(*_bbox_aspect_ratio(model, im, aspect_ratio, box_proposals, True, p))
    # the identity transform last, so that its blob_conv / im_scale are returned (postcondition of im_detect_bbox)
    scores_i, boxes_i, im_scale_i, blob_conv_i = _detect_bbox(model, im, p["test_scale"], p["test_max_size"], box_proposals, False, 1.0, p)
    add_preds_t(scores_i, boxes_i, identity=True)
    return scores_c.result(), boxes_c.result(), im_scale_i, blob_conv_i
