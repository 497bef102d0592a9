"""The reference's PASCAL VOC evaluator (lib/datasets/voc_dataset_evaluator.py:38-179) with every class matched in one device pass.

evaluate_boxes takes the reference's arguments, logs its lines (`VOC07 metric?`, `AP for <cls> = ...`, `Mean AP`, the results
block), pickles {'rec', 'prec', 'ap'} to <output_dir>/<cls>_pr.pkl and returns None.  Like the COCO evaluators it writes no
results files: it works on the values the reference's writer would put there (voc_eval.writer_values).  `use_salt` and `cleanup`
are accepted for the reference's signature; MATLAB evaluation is not available.
"""
import logging
import os
import pickle

import numpy as np

from . import voc_eval

logger = logging.getLogger(__name__)


def voc_info(json_dataset):
    """Year, image set and devkit paths of a `voc_<year>_<image set>` dataset; the devkit directory is json_dataset.devkit_path
    (load_json_dataset's devkit_path)."""
    year = json_dataset.name[4:8]
    image_set = json_dataset.name[9:]
    devkit_path = getattr(json_dataset, "devkit_path", None)
    if devkit_path is None or not os.path.exists(devkit_path):
        raise ValueError("Devkit directory {} not found".format(devkit_path))
    anno_path = os.path.join(devkit_path, "VOC" + year, "Annotations", "{:s}.xml")
    image_set_path = os.path.join(devkit_path, "VOC" + year, "ImageSets", "Main", image_set + ".txt")
    return dict(year=year, image_set=image_set, devkit_path=devkit_path, anno_path=anno_path, image_set_path=image_set_path)


def _image_names(json_dataset):
    """The dataset's images in sorted-id order, as names without directory and extension (the reference's roidb order)."""
    images = sorted(json_dataset.COCO.dataset.get("images", []), key=lambda im: im["id"])
    return [os.path.splitext(os.path.basename(im["file_name"]))[0] for im in images]


def evaluate_boxes(json_dataset, all_boxes, output_dir, use_salt=True, cleanup=True, use_matlab=False, device=None):
    if use_matlab:
        raise NotImplementedError("MATLAB devkit evaluation is not available; use the Python evaluation (use_matlab=False)")
    info = voc_info(json_dataset)
    image_index = voc_eval.read_image_set(info["image_set_path"])
    names = _image_names(json_dataset)
    if names != image_index[:len(names)]:
        raise ValueError("the dataset's images (sorted by id) do not match the order of {}".format(info["image_set_path"]))
    classes = [(i, c) for i, c in enumerate(json_dataset.classes) if c != "__background__"]
    use_07_metric = int(info["year"]) < 2010                             # the PASCAL VOC metric changed in 2010
    logger.info("VOC07 metric? " + ("Yes" if use_07_metric else "No"))
    recs = voc_eval.load_annotations(info["anno_path"], info["image_set_path"], image_index,
                                     os.path.join(info["devkit_path"], "annotations_cache"))
    dets = voc_eval.pack_all_boxes(all_boxes, [i for i, _ in classes], len(image_index))
    results = voc_eval.evaluate_classes(recs, image_index, [c for _, c in classes], *dets, ovthresh=0.5, use_07_metric=use_07_metric,
                                        device=device)
    if not os.path.isdir(output_dir):
        os.mkdir(output_dir)
    aps = []
    for (_, cls), (rec, prec, ap) in zip(classes, results):
        aps += [ap]
        logger.info("AP for {} = {:.4f}".format(cls, ap))
        with open(os.path.join(output_dir, cls + "_pr.pkl"), "wb") as f:
            pickle.dump({"rec": rec, "prec": prec, "ap": ap}, f, pickle.HIGHEST_PROTOCOL)
    logger.info("Mean AP = {:.4f}".format(np.mean(aps)))
    logger.info("~~~~~~~~")
    logger.info("Results:")
    for ap in aps:
        logger.info("{:.3f}".format(ap))
    logger.info("{:.3f}".format(np.mean(aps)))
    logger.info("~~~~~~~~")
    logger.info("")
    return None
