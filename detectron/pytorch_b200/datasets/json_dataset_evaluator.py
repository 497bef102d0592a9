"""The reference's COCO evaluators (lib/datasets/json_dataset_evaluator.py:38-233, 320-430) with COCOeval on the device, and its
proposal recall (:236-317, evaluate_box_proposals) with the greedy matching on the device (csrc/box_proposals.cu).

evaluate_boxes / evaluate_masks / evaluate_keypoints take the reference's arguments and return an object shaped like
pycocotools' COCOeval after accumulate() and summarize() (datasets/coco_eval.py): `.params`, `.eval`, `.stats`,
`.summarize()`.  They log the reference's per-category AP lines and pickle the result to its file names in output_dir.

The results are not written to JSON and read back: the evaluator works on the float64 values the reference's writers put in
that file (json round-trips float64 exactly).  The conversion is the writers', step for step:
  * boxes: float64 of the float32 all_boxes, xyxy_to_xywh with the + 1, score = the box's last column;
  * masks: the compressed COCO strings of all_segms, the box score;
  * keypoints: float64 of x and y of cls_keyps (v = 1), score = the box score (KEYPOINT_CONFIDENCE 'bbox') or the mean of
    row 2 ('logit') / row 3 ('prob') over the keypoints, summed in order in float64 -- the reference's `kps_score = 0;
    kps_score += ...` under numpy 1's promotion of a Python int plus a float32 scalar.
`use_salt` / `cleanup` are accepted for the reference's signature; there is no results file to salt or remove.
"""
import json
import logging
import operator
import os
import pickle
from collections import OrderedDict

import numpy as np

from . import coco_eval

logger = logging.getLogger(__name__)


class JsonDataset:
    """The parts of the reference's JsonDataset the evaluators read: name, classes, category_to_id_map and COCO, whose
    `dataset` is the annotation-file dict and getImgIds() its image ids; devkit_path is a PASCAL VOC dataset's devkit directory
    (the reference's catalog entry DEVKIT_DIR)."""

    class _Coco:
        def __init__(self, dataset):
            self.dataset = dataset

        def getImgIds(self):
            return [img["id"] for img in self.dataset.get("images", [])]

        def getCatIds(self):
            return [c["id"] for c in self.dataset.get("categories", [])]

    def __init__(self, name, dataset, devkit_path=None):
        self.name = name
        self.devkit_path = devkit_path
        self.COCO = JsonDataset._Coco(dataset)
        category_ids = sorted(self.COCO.getCatIds())
        names = {c["id"]: c["name"] for c in dataset.get("categories", [])}
        categories = [names[i] for i in category_ids]
        self.category_to_id_map = dict(zip(categories, category_ids))     # json_dataset.py:69-80
        self.classes = ["__background__"] + categories
        self.num_classes = len(self.classes)
        self.json_category_id_to_contiguous_id = {v: i + 1 for i, v in enumerate(category_ids)}
        self.contiguous_category_id_to_json_id = {v: k for k, v in self.json_category_id_to_contiguous_id.items()}


def load_json_dataset(name, annotation_file_or_dict, devkit_path=None):
    """A JsonDataset from a COCO annotation file (path) or its already-loaded dict, without pycocotools.  devkit_path: the
    VOCdevkit directory that voc_dataset_evaluator reads a `voc_*` dataset's image set and annotations from."""
    if isinstance(annotation_file_or_dict, dict):
        return JsonDataset(name, annotation_file_or_dict, devkit_path)
    with open(annotation_file_or_dict) as f:
        return JsonDataset(name, json.load(f), devkit_path)


def _image_ids(json_dataset):
    ids = json_dataset.COCO.getImgIds()
    ids.sort()
    return ids


def _classes(json_dataset, n):
    """(cls_ind, cat_id) in the writers' order: classes after __background__, stopping at the length of the per-class list."""
    for cls_ind, cls in enumerate(json_dataset.classes):
        if cls == "__background__":
            continue
        if cls_ind >= n:
            break
        yield cls_ind, json_dataset.category_to_id_map[cls]


def _empty(dets):
    return isinstance(dets, list) and len(dets) == 0


def _box_results(json_dataset, all_boxes):
    image_ids = _image_ids(json_dataset)
    img, cat, score, box = [], [], [], []
    for cls_ind, cat_id in _classes(json_dataset, len(all_boxes)):
        assert len(all_boxes[cls_ind]) == len(image_ids)
        for i, image_id in enumerate(image_ids):
            dets = all_boxes[cls_ind][i]
            if _empty(dets):
                continue
            dets = np.asarray(dets).astype(np.float64)
            xy = dets[:, 0:4]
            box.append(np.hstack((xy[:, 0:2], xy[:, 2:4] - xy[:, 0:2] + 1)))      # utils/boxes.py xyxy_to_xywh
            score.append(dets[:, -1]); img.append(np.full(len(dets), image_id)); cat.append(np.full(len(dets), cat_id))
    cat_ = lambda xs, w: np.concatenate(xs) if xs else np.zeros((0,) + w)  # noqa: E731
    return coco_eval.Detections(cat_(img, ()), cat_(cat, ()), cat_(score, ()), box=cat_(box, (4,)))


def _segm_results(json_dataset, all_boxes, all_segms):
    image_ids = _image_ids(json_dataset)
    img, cat, score, strings = [], [], [], []
    for cls_ind, cat_id in _classes(json_dataset, len(all_boxes)):
        assert len(all_boxes[cls_ind]) == len(image_ids) and len(all_segms[cls_ind]) == len(image_ids)
        for i, image_id in enumerate(image_ids):
            dets = all_boxes[cls_ind][i]
            if _empty(dets):
                continue
            rles = all_segms[cls_ind][i]
            dets = np.asarray(dets).astype(np.float64)
            for k in range(dets.shape[0]):
                c = rles[k]["counts"]
                if isinstance(c, list):
                    raise ValueError("all_segms holds compressed COCO RLEs (strings), got uncompressed counts")
                strings.append((c.encode("ascii") if isinstance(c, str) else bytes(c), tuple(int(v) for v in rles[k]["size"])))
            score.append(dets[:, -1]); img.append(np.full(len(dets), image_id)); cat.append(np.full(len(dets), cat_id))
    cat_ = lambda xs: np.concatenate(xs) if xs else np.zeros(0)  # noqa: E731
    return coco_eval.Detections(cat_(img), cat_(cat), cat_(score), strings=strings)


def _keypoint_confidence(cfg, keypoint_confidence):
    if keypoint_confidence is None:
        keypoint_confidence = cfg.KRCNN.KEYPOINT_CONFIDENCE if cfg is not None else "bbox"
    if keypoint_confidence not in ("logit", "prob", "bbox"):
        raise ValueError('KRCNN.KEYPOINT_CONFIDENCE must be "logit", "prob", or "bbox"')
    return keypoint_confidence


def _keypoint_results(json_dataset, all_boxes, all_keyps, confidence):
    image_ids = _image_ids(json_dataset)
    img, cat, score, kps = [], [], [], []
    for cls_ind, cat_id in _classes(json_dataset, len(all_keyps)):
        assert len(all_keyps[cls_ind]) == len(image_ids) and len(all_boxes[cls_ind]) == len(image_ids)
        for i, image_id in enumerate(image_ids):
            if len(all_boxes[cls_ind][i]) == 0:
                continue
            kps_dets = all_keyps[cls_ind][i]
            if len(kps_dets) == 0:
                continue
            scores = np.asarray(all_boxes[cls_ind][i])[:, -1].astype(np.float64)
            for j in range(len(kps_dets)):
                kd = np.asarray(kps_dets[j])
                if kd.shape[1] != 17:
                    raise ValueError("COCO keypoints are 17 per person, got %d" % kd.shape[1])
                xyv = np.stack([kd[0].astype(np.float64), kd[1].astype(np.float64), np.ones(17)], axis=1)
                if confidence == "bbox":
                    s = scores[j]
                else:
                    row = kd[2 if confidence == "logit" else 3].astype(np.float64)
                    s = 0.0
                    for v in row:                                          # in order, in float64
                        s += v
                    s /= kd.shape[1]
                kps.append(xyv); score.append(s); img.append(image_id); cat.append(cat_id)
    return coco_eval.Detections(img, cat, score, keypoints=np.asarray(kps, np.float64).reshape(-1, 17, 3))


def _save(result, output_dir, file_name):
    eval_file = os.path.join(output_dir, file_name)
    with open(eval_file, "wb") as f:
        pickle.dump(result, f, pickle.HIGHEST_PROTOCOL)
    logger.info("Wrote json eval results to: {}".format(eval_file))


def _log_detection_eval_metrics(json_dataset, coco_eval_result):
    """The reference's mean and per-category AP at IoU 0.50:0.95 (area all, 100 detections), then summarize()."""
    def _get_thr_ind(thr):
        ind = np.where((coco_eval_result.params.iouThrs > thr - 1e-5) & (coco_eval_result.params.iouThrs < thr + 1e-5))[0][0]
        assert np.isclose(coco_eval_result.params.iouThrs[ind], thr)
        return ind

    ind_lo, ind_hi = _get_thr_ind(0.5), _get_thr_ind(0.95)
    precision = coco_eval_result.eval["precision"][ind_lo:(ind_hi + 1), :, :, 0, 2]
    ap_default = np.mean(precision[precision > -1])
    logger.info("~~~~ Mean and per-category AP @ IoU=[{:.2f},{:.2f}] ~~~~".format(0.5, 0.95))
    logger.info("{:.1f}".format(100 * ap_default))
    for cls_ind, cls in enumerate(json_dataset.classes):
        if cls == "__background__":
            continue
        precision = coco_eval_result.eval["precision"][ind_lo:(ind_hi + 1), :, cls_ind - 1, 0, 2]
        ap = np.mean(precision[precision > -1])
        logger.info("{:.1f}".format(100 * ap))
    logger.info("~~~~ Summary metrics ~~~~")
    coco_eval_result.summarize()


def _evaluates(json_dataset):
    return json_dataset.name.find("test") == -1                          # annotations of test sets are undisclosed


def evaluate_boxes(json_dataset, all_boxes, output_dir, use_salt=True, cleanup=False, device=None):
    if not _evaluates(json_dataset):
        return None
    res = coco_eval.evaluate(json_dataset.COCO.dataset, _box_results(json_dataset, all_boxes), "bbox", device)
    _log_detection_eval_metrics(json_dataset, res)
    _save(res, output_dir, "detection_results.pkl")
    return res


def evaluate_masks(json_dataset, all_boxes, all_segms, output_dir, use_salt=True, cleanup=False, device=None):
    if not _evaluates(json_dataset):
        return None
    res = coco_eval.evaluate(json_dataset.COCO.dataset, _segm_results(json_dataset, all_boxes, all_segms), "segm", device)
    _log_detection_eval_metrics(json_dataset, res)
    _save(res, output_dir, "segmentation_results.pkl")
    return res


def evaluate_keypoints(json_dataset, all_boxes, all_keypoints, output_dir, use_salt=True, cleanup=False, cfg=None,
                       keypoint_confidence=None, device=None):
    """KRCNN.KEYPOINT_CONFIDENCE comes from `keypoint_confidence`, else from cfg.KRCNN.KEYPOINT_CONFIDENCE, else 'bbox'."""
    confidence = _keypoint_confidence(cfg, keypoint_confidence)
    if not _evaluates(json_dataset):
        return None
    res = coco_eval.evaluate(json_dataset.COCO.dataset, _keypoint_results(json_dataset, all_boxes, all_keypoints, confidence),
                             "keypoints", device)
    _save(res, output_dir, "keypoint_results.pkl")
    res.summarize()
    return res


# ---- proposal recall (lib/datasets/json_dataset_evaluator.py:236-317) ------------------------------------------------------
# Area ranges by name, in the reference's order: [side_lo², side_hi²], both ends inclusive; "unbounded" is a side of 1e5.
BOX_PROPOSAL_AREA_RANGES = OrderedDict(
    (name, (float(lo) ** 2, float(hi) ** 2))
    for name, lo, hi in (("all", 0, 1e5), ("small", 0, 32), ("medium", 32, 96), ("large", 96, 1e5), ("96-128", 96, 128),
                         ("128-256", 128, 256), ("256-512", 256, 512), ("512-inf", 512, 1e5)))
# Images packed per launch: bounds the device memory of a train-set-sized roidb.  The results do not depend on it.
BOX_PROPOSAL_CHUNK_IMAGES = 1024


def default_recall_thresholds():
    return np.arange(0.5, 0.95 + 1e-5, 0.05)


def effective_proposal_counts(num_props, limits):
    """(len(limits), N) int32: how many of each image's num_props proposals a limit keeps, len(boxes[:limit]) (None keeps all; a
    negative limit drops that many from the end, as the reference's slice does)."""
    n = np.asarray(num_props, np.int64).reshape(-1)
    out = np.empty((len(limits), n.size), np.int32)
    for k, limit in enumerate(limits):
        if limit is None:
            out[k] = n
        else:
            limit = operator.index(limit)
            out[k] = np.minimum(n, limit) if limit >= 0 else np.maximum(n + limit, 0)
    return out


def pack_roidb(roidb):
    """The reference's per-entry selection, concatenated: proposals (gt_classes == 0 rows of `boxes`, float32) and ground truth
    (gt_classes > 0 and not is_crowd: float32 boxes and float64 seg_areas), each with its (N + 1) row offsets."""
    props, gts, areas = [], [], []
    for entry in roidb:
        cls = np.asarray(entry["gt_classes"])
        rows = np.asarray(entry["boxes"])
        positive = (cls > 0) & (np.asarray(entry["is_crowd"]) == 0)
        gts.append(rows[positive].astype(np.float32).reshape(-1, 4))
        areas.append(np.asarray(entry["seg_areas"])[positive].astype(np.float64))
        props.append(rows[cls == 0].astype(np.float32).reshape(-1, 4))
    begin = lambda xs: np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int32)  # noqa: E731
    cat = lambda xs, w: np.ascontiguousarray(np.concatenate(xs)) if xs else np.zeros((0,) + w)  # noqa: E731
    return (cat(props, (4,)).astype(np.float32), begin(props), cat(gts, (4,)).astype(np.float32), cat(areas, ()).astype(np.float64),
            begin(gts))


def _box_proposal_recall(roidb, area_names, limits, thresholds, device, want_overlaps):
    """counts (L, A, T) int64, num_pos per area, and per (limit, area) the float64 gt_overlaps (unsorted) when want_overlaps, over
    the whole roidb in chunks of BOX_PROPOSAL_CHUNK_IMAGES images, one launch per chunk.  A NaN IoU raises AssertionError naming
    the first image of the first (limit, area) that has one, where the reference's `assert gt_ovr >= 0` fails."""
    import torch
    from .. import ops
    for area in area_names:
        _check_area(area)
    ranges = np.asarray([BOX_PROPOSAL_AREA_RANGES[a] for a in area_names], np.float64)
    thr = np.asarray(thresholds, np.float64).reshape(-1)
    L, A = len(limits), len(area_names)
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    counts = np.zeros((L, A, thr.size), np.int64)
    num_pos = [0] * A
    overlaps = [[[] for _ in range(A)] for _ in range(L)]
    first_error = {}
    thr_dev = torch.from_numpy(thr).to(device)
    for c0 in range(0, len(roidb), BOX_PROPOSAL_CHUNK_IMAGES):
        prop_box, prop_begin, gt_box, gt_area, gt_begin = pack_roidb(roidb[c0:c0 + BOX_PROPOSAL_CHUNK_IMAGES])
        for a in range(A):
            num_pos[a] += int(np.count_nonzero((gt_area >= ranges[a, 0]) & (gt_area <= ranges[a, 1])))
        prop_count = effective_proposal_counts(np.diff(prop_begin), limits)
        up = lambda x: torch.from_numpy(x).to(device)  # noqa: E731
        overlap, excluded, error, cnt = ops.box_proposal_match_raw(up(prop_box), up(prop_begin), up(gt_box), up(gt_area), up(gt_begin),
                                                                   up(prop_count), ranges, thr_dev)
        counts += cnt.cpu().numpy()
        error = error.cpu().numpy()
        for l, a, i in zip(*np.nonzero(error)):                 # row-major: the first image of each (l, a) comes first
            first_error.setdefault((int(l), int(a)), c0 + int(i))
        if want_overlaps:
            overlap, excluded = overlap.cpu().numpy(), excluded.cpu().numpy()
            for l in range(L):
                for a in range(A):
                    overlaps[l][a].append(overlap[l, a][~excluded[l, a]].astype(np.float64))
    if first_error:
        (l, a), i = min(first_error.items())
        raise AssertionError("roidb entry {}: a NaN IoU between its proposals and ground truth (limit {}, area '{}'); the "
                             "reference's `assert gt_ovr >= 0` fails there".format(i, limits[l], area_names[a]))
    return counts, num_pos, overlaps


def _check_area(area):
    if area not in BOX_PROPOSAL_AREA_RANGES:              # the reference's assert and message
        raise AssertionError("Unknown area range: {}".format(area))


def _recall_result(count, num_pos, thresholds, gt_overlaps):
    """The dict the reference returns.  Each recall is the int64 count over float(num_pos) as a numpy scalar division (NaN, with
    numpy's warning, when num_pos is 0), stored into an array shaped and typed like `thresholds`; ar is that array's mean."""
    denom = float(num_pos)
    recalls = np.zeros_like(thresholds)
    for k, hits in enumerate(count):
        recalls[k] = hits / denom
    return {"ar": recalls.mean(), "recalls": recalls, "thresholds": thresholds, "gt_overlaps": gt_overlaps, "num_pos": num_pos}


def evaluate_box_proposals(json_dataset, roidb, thresholds=None, area="all", limit=None, device=None):
    """Proposal recall as the reference computes it (json_dataset_evaluator.py:236-317): the reference's dict `ar`, `recalls`,
    `thresholds`, `gt_overlaps` (sorted float64) and `num_pos`, with the greedy matching and the per-threshold counts on the device.
    roidb entries need `boxes` (proposals are the gt_classes == 0 rows, in order), `gt_classes`, `is_crowd` and `seg_areas`."""
    _check_area(area)
    if thresholds is None:
        thresholds = default_recall_thresholds()
    counts, num_pos, overlaps = _box_proposal_recall(roidb, [area], [limit], thresholds, device, want_overlaps=True)
    gt_overlaps = np.sort(np.concatenate([np.zeros(0)] + overlaps[0][0]))
    return _recall_result(counts[0, 0], num_pos[0], thresholds, gt_overlaps)
