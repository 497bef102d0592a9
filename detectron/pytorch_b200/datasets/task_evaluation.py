"""The COCO branch of the reference's task_evaluation.evaluate_all (lib/datasets/task_evaluation.py:52-70), with the
reference's OrderedDict result layout, so check_expected_results-style comparisons read it as they read the reference's."""
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
