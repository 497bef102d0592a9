"""The COCO branch of the reference's task_evaluation.evaluate_all (lib/datasets/task_evaluation.py:52-70) and its box-proposal
task (evaluate_box_proposals, log_box_proposal_results), with the reference's OrderedDict result layout, so check_expected_results-style comparisons read it as they read the reference's."""
import logging
from collections import OrderedDict

from . import json_dataset_evaluator

logger = logging.getLogger(__name__)

# COCOeval.stats indices (task_evaluation.py)
COCO_AP, COCO_AP50, COCO_AP75, COCO_APS, COCO_APM, COCO_APL = range(6)


def _empty_box_results():
    return OrderedDict({"box": OrderedDict([(k, -1) for k in ["AP", "AP50", "AP75", "APs", "APm", "APl"]])})


def _empty_mask_results():
    return OrderedDict({"mask": OrderedDict([(k, -1) for k in ["AP", "AP50", "AP75", "APs", "APm", "APl"]])})


def _empty_keypoint_results():
    return OrderedDict({"keypoint": OrderedDict([(k, -1) for k in ["AP", "AP50", "AP75", "APm", "APl"]])})


def _coco_eval_to_box_results(coco_eval):
    res = _empty_box_results()
    if coco_eval is not None:
        s = coco_eval.stats
        for k, i in zip(["AP", "AP50", "AP75", "APs", "APm", "APl"], [COCO_AP, COCO_AP50, COCO_AP75, COCO_APS, COCO_APM, COCO_APL]):
            res["box"][k] = s[i]
    return res


def _coco_eval_to_mask_results(coco_eval):
    res = _empty_mask_results()
    if coco_eval is not None:
        s = coco_eval.stats
        for k, i in zip(["AP", "AP50", "AP75", "APs", "APm", "APl"], [COCO_AP, COCO_AP50, COCO_AP75, COCO_APS, COCO_APM, COCO_APL]):
            res["mask"][k] = s[i]
    return res


def _coco_eval_to_keypoint_results(coco_eval):
    res = _empty_keypoint_results()
    if coco_eval is not None:
        s = coco_eval.stats
        for k, i in zip(["AP", "AP50", "AP75", "APm", "APl"], [COCO_AP, COCO_AP50, COCO_AP75, 3, 4]):
            res["keypoint"][k] = s[i]
    return res


def _flag(cfg, section, name, default):
    try:
        return bool(getattr(getattr(cfg, section), name))
    except AttributeError:
        return default


def evaluate_all(dataset, all_boxes, all_segms, all_keyps, output_dir, cfg=None, mask_on=None, keypoints_on=None, device=None):
    """Boxes always; masks when cfg.MODEL.MASK_ON (or `mask_on`); keypoints when cfg.MODEL.KEYPOINTS_ON (or `keypoints_on`).
    Without cfg or the keywords, a task is evaluated when its results are given (not None)."""
    mask_on = _flag(cfg, "MODEL", "MASK_ON", all_segms is not None) if mask_on is None else mask_on
    keypoints_on = _flag(cfg, "MODEL", "KEYPOINTS_ON", all_keyps is not None) if keypoints_on is None else keypoints_on
    logger.info("Evaluating detections")
    coco_eval = json_dataset_evaluator.evaluate_boxes(dataset, all_boxes, output_dir, device=device)
    all_results = OrderedDict([(dataset.name, _coco_eval_to_box_results(coco_eval))])
    logger.info("Evaluating bounding boxes is done!")
    if mask_on:
        logger.info("Evaluating segmentations")
        coco_eval = json_dataset_evaluator.evaluate_masks(dataset, all_boxes, all_segms, output_dir, device=device)
        all_results[dataset.name].update(_coco_eval_to_mask_results(coco_eval))
        logger.info("Evaluating segmentations is done!")
    if keypoints_on:
        logger.info("Evaluating detections")
        coco_eval = json_dataset_evaluator.evaluate_keypoints(dataset, all_boxes, all_keyps, output_dir, cfg=cfg, device=device)
        all_results[dataset.name].update(_coco_eval_to_keypoint_results(coco_eval))
        logger.info("Evaluating keypoints is done!")
    return all_results


# ---- box proposals (lib/datasets/task_evaluation.py:151-163, 371-386) ------------------------------------------------------
_BOX_PROPOSAL_LIMITS = [100, 1000]
_BOX_PROPOSAL_AREAS = OrderedDict([("all", ""), ("small", "s"), ("medium", "m"), ("large", "l")])


def _empty_box_proposal_results():
    return OrderedDict({"box_proposal": OrderedDict([("AR{}@{:d}".format(s, limit), -1)
                                                     for limit in _BOX_PROPOSAL_LIMITS for s in _BOX_PROPOSAL_AREAS.values()])})


def evaluate_box_proposals(dataset, roidb, device=None):
    """The reference's eight keys (AR@100, ARs@100, ..., ARl@1000), each what json_dataset_evaluator.evaluate_box_proposals
    returns as `ar` for that area and limit, all eight from one launch per chunk of the roidb."""
    res = _empty_box_proposal_results()
    areas = list(_BOX_PROPOSAL_AREAS)
    thresholds = json_dataset_evaluator.default_recall_thresholds()
    counts, num_pos, _ = json_dataset_evaluator._box_proposal_recall(roidb, areas, _BOX_PROPOSAL_LIMITS, thresholds, device,
                                                                     want_overlaps=False)
    for l, limit in enumerate(_BOX_PROPOSAL_LIMITS):
        for a, (area, suffix) in enumerate(_BOX_PROPOSAL_AREAS.items()):
            stats = json_dataset_evaluator._recall_result(counts[l, a], num_pos[a], thresholds, None)
            res["box_proposal"]["AR{}@{:d}".format(suffix, limit)] = stats["ar"]
    return OrderedDict([(dataset.name, res)])


def log_box_proposal_results(results):
    """Logs each dataset's name, then one `<metric>: <value>` line per box-proposal metric, the names padded to the longest and the
    values with three decimals."""
    for name, tasks in results.items():
        metrics = tasks["box_proposal"]
        width = max(len(key) for key in metrics)
        logger.info(name)
        for key, value in metrics.items():
            logger.info("%s: %.3f", key.ljust(width), value)
