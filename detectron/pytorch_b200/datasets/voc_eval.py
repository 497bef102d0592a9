"""The reference's PASCAL VOC AP evaluation (lib/datasets/voc_eval.py:86-223) with its per-detection loop on the device.

`voc_eval(detpath, annopath, imagesetfile, classname, cachedir, ...)` keeps the reference's signature and `(rec, prec, ap)` result
and reads the results file the way the reference does; voc_dataset_evaluator.evaluate_boxes evaluates every class of all_boxes in
one device pass without writing results files.  Both go through the same stages:
  * pack (host, vectorised): the float64 values the reference reads back from its results files (writer_values), each class's
    detections in rank order -- descending score, ties in file order (image-set order, then row order), which is the reference's
    result under a stable argsort -- and the ground truth as one row range per (class, image) pair;
  * match (device, csrc/voc_eval.cu): one upload, then IoU, ovmax / jmax and the first-come claims -> tp / fp / neither;
  * curves (host): cumulative tp / fp, recall, precision and voc_ap with the reference's ufuncs, so they are bit-equal.
The annotation cache keeps the reference's path and dict (<cachedir>/<imageset>_annots.pkl) but is read and written in binary
mode, which is what lets it work on Python 3.

Differences from the reference: tied scores keep file order (numpy's default argsort leaves their order to the numpy build); a
class without detections gets empty rec / prec and AP 0.0 (the reference raises IndexError); duplicate names in the image set are
refused (the reference counts such an image's objects twice but keeps one detection list for it).
"""
import logging
import os
import pickle
import xml.etree.ElementTree as ET

import numpy as np
import torch

from .. import ops
from .coco_eval import _upload

logger = logging.getLogger(__name__)

TP, FP = 1, 0                                                            # outcome bytes of b200_voc_match (2: neither)


def parse_rec(filename):
    """The objects of one PASCAL VOC annotation file, in file order: name, pose, truncated, difficult and an integer bbox
    [xmin, ymin, xmax, ymax]."""
    objects = []
    for obj in ET.parse(filename).findall("object"):
        box = obj.find("bndbox")
        objects.append({"name": obj.find("name").text,
                        "pose": obj.find("pose").text,
                        "truncated": int(obj.find("truncated").text),
                        "difficult": int(obj.find("difficult").text),
                        "bbox": [int(box.find(k).text) for k in ("xmin", "ymin", "xmax", "ymax")]})
    return objects


def voc_ap(rec, prec, use_07_metric=False):
    """VOC AP of a precision / recall curve: the VOC07 11-point rule, or the area under the precision envelope."""
    if use_07_metric:
        ap = 0.
        for t in np.arange(0., 1.1, 0.1):
            p = 0 if np.sum(rec >= t) == 0 else np.max(prec[rec >= t])
            ap = ap + p / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.concatenate(([0.], prec, [0.]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]                       # suffix maximum, np.maximum as the reference's loop
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def read_image_set(imagesetfile):
    """Image names, one per line; duplicates are refused."""
    with open(imagesetfile, "r") as f:
        names = [x.strip() for x in f.readlines()]
    if len(set(names)) != len(names):
        raise ValueError("duplicate image names in %s" % imagesetfile)
    return names


def load_annotations(annopath, imagesetfile, imagenames, cachedir):
    """{image name: parse_rec(annopath.format(name))}, from <cachedir>/<imageset>_annots.pkl when it exists, else parsed and saved
    there."""
    if not os.path.isdir(cachedir):
        os.mkdir(cachedir)
    imageset = os.path.splitext(os.path.basename(imagesetfile))[0]
    cachefile = os.path.join(cachedir, imageset + "_annots.pkl")
    if os.path.isfile(cachefile):
        with open(cachefile, "rb") as f:
            return pickle.load(f)
    recs = {}
    for i, name in enumerate(imagenames):
        recs[name] = parse_rec(annopath.format(name))
        if i % 100 == 0:
            logger.info("Reading annotation for {:d}/{:d}".format(i + 1, len(imagenames)))
    logger.info("Saving cached annotations to {:s}".format(cachefile))
    with open(cachefile, "wb") as f:
        pickle.dump(recs, f)
    return recs


def writer_values(boxes, scores):
    """The float64 values voc_eval parses from the reference's results lines '{:.3f}' of the score and '{:.1f}' of each coordinate
    + 1.  For float32 input (the + 1 is a float32 sum under numpy 2) rint(float64(v) * 10^d) / 10^d gives them exactly: the product
    is exact, rint rounds half to even as the formatting does on the binary value, and the division rounds to the double float()
    parses.  Other dtypes go through the writer's formatting."""
    boxes = np.asarray(boxes)
    scores = np.asarray(scores)
    if boxes.dtype == np.float32 and scores.dtype == np.float32:
        return (np.rint(scores.astype(np.float64) * 1000.0) / 1000.0,
                np.rint((boxes + np.float32(1)).astype(np.float64) * 10.0) / 10.0)
    return (np.char.mod("%.3f", scores).astype(np.float64).reshape(scores.shape),
            np.char.mod("%.1f", boxes + 1).astype(np.float64).reshape(boxes.shape))


def pack_all_boxes(all_boxes, cls_inds, num_images):
    """Detections of all_boxes[c][i] for the classes cls_inds, in the order the reference writes them (class, image, row), as
    (det_class (index into cls_inds), det_image, score, box) with writer_values' float64 values."""
    arrays, det_class, det_image = [], [], []
    for k, c in enumerate(cls_inds):
        if len(all_boxes[c]) != num_images:
            raise ValueError("all_boxes[%d] has %d images, the image set %d" % (c, len(all_boxes[c]), num_images))
        for i, dets in enumerate(all_boxes[c]):
            if isinstance(dets, list):
                if len(dets):
                    raise ValueError("dets should be numpy.ndarray or empty list")
                continue
            if dets.shape[0]:
                arrays.append(dets); det_class.append(k); det_image.append(i)
    n = np.array([a.shape[0] for a in arrays], np.int64)
    det_class = np.repeat(np.asarray(det_class, np.int64), n)
    det_image = np.repeat(np.asarray(det_image, np.int64), n)
    if not arrays:
        return det_class, det_image, np.zeros(0), np.zeros((0, 4))
    if all(a.dtype == np.float32 for a in arrays):
        score, box = writer_values(np.concatenate([a[:, 0:4] for a in arrays]), np.concatenate([a[:, -1] for a in arrays]))
    else:
        parts = [writer_values(a[:, 0:4], a[:, -1]) for a in arrays]
        score, box = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    return det_class, det_image, score, box


class Packed:
    """Host arrays of one evaluation: detections in rank order within each class (class k's are cls_begin[k] .. [k + 1]), ground
    truth per (class, image) pair, npos per class."""

    def __init__(self, recs, imagenames, classes, det_class, det_image, score, box):
        C, I = len(classes), len(imagenames)
        if C * I >= 2 ** 31 or len(score) >= 2 ** 31:
            raise ValueError("more than 2^31 - 1 (class, image) pairs or detections")
        cls_index = {c: k for k, c in enumerate(classes)}
        g_cls, g_img, g_box, g_diff = [], [], [], []
        for i, name in enumerate(imagenames):
            for obj in recs[name]:
                k = cls_index.get(obj["name"])
                if k is not None:
                    g_cls.append(k); g_img.append(i); g_box.append(obj["bbox"]); g_diff.append(obj["difficult"])
        g_cls = np.asarray(g_cls, np.int64)
        g_diff = np.asarray(g_diff, np.int64) != 0
        self.npos = np.bincount(g_cls[~g_diff], minlength=C)
        g_key = g_cls * I + np.asarray(g_img, np.int64)
        g_ord = np.argsort(g_key, kind="stable")
        self.pair_gt_begin = np.searchsorted(g_key[g_ord], np.arange(C * I + 1), side="left").astype(np.int32)
        self.gt_box = np.asarray(g_box, np.float64).reshape(-1, 4)[g_ord]
        self.gt_difficult = g_diff[g_ord].astype(np.uint8)
        det_class = np.asarray(det_class, np.int64)
        order = np.lexsort((-np.asarray(score, np.float64), det_class))  # class, then descending score; lexsort is stable
        self.cls_begin = np.searchsorted(det_class[order], np.arange(C + 1), side="left")
        self.det_pair = (det_class[order] * I + np.asarray(det_image, np.int64)[order]).astype(np.int32)
        self.det_box = np.ascontiguousarray(np.asarray(box, np.float64).reshape(-1, 4)[order])


def upload(packed, device=None):
    """One host-to-device copy of the packed tables: (pair_gt_begin, gt_box, gt_difficult, det_pair, det_box) on `device`."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    D, G = packed.det_pair.size, packed.gt_difficult.size
    (pgb, gb, gd, dp, db), buf, host = _upload([packed.pair_gt_begin, packed.gt_box, packed.gt_difficult, packed.det_pair,
                                                packed.det_box], dev)
    return pgb, gb[:G], gd[:G], dp[:D], db[:D], (buf, host)


def curves(packed, outcome, use_07_metric=False):
    """[(rec, prec, ap)] per class from the outcome bytes (host, rank order) -- the reference's arithmetic, ufunc for ufunc."""
    out = []
    eps = np.finfo(np.float64).eps
    for k in range(packed.npos.size):
        o = outcome[packed.cls_begin[k]:packed.cls_begin[k + 1]]
        tp = np.cumsum((o == TP).astype(np.float64))
        fp = np.cumsum((o == FP).astype(np.float64))
        with np.errstate(divide="ignore", invalid="ignore"):             # npos = 0: rec is inf / NaN, as in the reference
            rec = tp / float(packed.npos[k])
        prec = tp / np.maximum(tp + fp, eps)
        out.append((rec, prec, voc_ap(rec, prec, use_07_metric)))
    return out


def evaluate_classes(recs, imagenames, classes, det_class, det_image, score, box, ovthresh=0.5, use_07_metric=False, device=None):
    """[(rec, prec, ap)] for each of `classes`, detections as pack_all_boxes gives them, ground truth from recs (parse_rec per
    image name)."""
    packed = Packed(recs, imagenames, classes, det_class, det_image, score, box)
    if packed.det_pair.size == 0:
        outcome = np.zeros(0, np.uint8)
    else:
        pgb, gb, gd, dp, db, _keep = upload(packed, device)
        with torch.cuda.device(dp.device):
            outcome = ops.voc_match_raw(pgb, gb, gd, dp, db, ovthresh).cpu().numpy()
    return curves(packed, outcome, use_07_metric)


def voc_eval(detpath, annopath, imagesetfile, classname, cachedir, ovthresh=0.5, use_07_metric=False, device=None):
    """rec, prec, ap of `classname`: detections from detpath.format(classname) ('<image> <score> <x1> <y1> <x2> <y2>' lines),
    annotations from annopath.format(image) via the cache in cachedir, images from imagesetfile."""
    imagenames = read_image_set(imagesetfile)
    recs = load_annotations(annopath, imagesetfile, imagenames, cachedir)
    with open(detpath.format(classname), "r") as f:
        lines = f.readlines()
    splitlines = [x.strip().split(" ") for x in lines]
    image_ids = np.array([x[0] for x in splitlines], dtype=str)
    score = np.array([float(x[1]) for x in splitlines], np.float64)
    box = np.array([[float(z) for z in x[2:]] for x in splitlines], np.float64).reshape(-1, 4)
    names = np.array(imagenames, dtype=str)
    by_name = np.argsort(names, kind="stable")
    pos = np.minimum(np.searchsorted(names[by_name], image_ids), max(names.size - 1, 0))
    if image_ids.size and (names.size == 0 or np.any(names[by_name][pos] != image_ids)):
        raise KeyError("detections on images outside %s" % imagesetfile)
    det_image = by_name[pos]
    ((rec, prec, ap),) = evaluate_classes(recs, imagenames, [classname], np.zeros(score.size, np.int64), det_image, score, box,
                                          ovthresh, use_07_metric, device)
    return rec, prec, ap
