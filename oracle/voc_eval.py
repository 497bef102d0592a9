"""PASCAL VOC detection AP restated in numpy for the tests (TEST INFRASTRUCTURE ONLY): the reference's results writer
(lib/datasets/voc_dataset_evaluator.py:58-92) and voc_eval (lib/datasets/voc_eval.py:86-223), one detection at a time.

Written for clarity, not speed.  The one deliberate difference from the reference: detections of equal score keep file order
(a stable sort), which is the order detectron/pytorch_b200/datasets/voc_eval.py uses.
"""
import numpy as np


def writer_lines(all_boxes, cls_ind, image_index):
    """The lines the reference's writer puts in one class's results file."""
    lines = []
    for im_ind, name in enumerate(image_index):
        dets = all_boxes[cls_ind][im_ind]
        if isinstance(dets, list):
            assert len(dets) == 0
            continue
        for k in range(dets.shape[0]):
            lines.append("{:s} {:.3f} {:.1f} {:.1f} {:.1f} {:.1f}\n".format(
                name, dets[k, -1], dets[k, 0] + 1, dets[k, 1] + 1, dets[k, 2] + 1, dets[k, 3] + 1))
    return lines


def parse_lines(lines):
    """(image names, scores, boxes (n, 4)) as float64, read back with float()."""
    fields = [ln.strip().split(" ") for ln in lines]
    names = [f[0] for f in fields]
    scores = np.array([float(f[1]) for f in fields], np.float64)
    boxes = np.array([[float(v) for v in f[2:6]] for f in fields], np.float64).reshape(-1, 4)
    return names, scores, boxes


def overlaps(box, gts):
    """IoU of one box against rows of gts, in the reference's float64 operation order."""
    iw = np.maximum(np.minimum(gts[:, 2], box[2]) - np.maximum(gts[:, 0], box[0]) + 1., 0.)
    ih = np.maximum(np.minimum(gts[:, 3], box[3]) - np.maximum(gts[:, 1], box[1]) + 1., 0.)
    inters = iw * ih
    uni = ((box[2] - box[0] + 1.) * (box[3] - box[1] + 1.) + (gts[:, 2] - gts[:, 0] + 1.) * (gts[:, 3] - gts[:, 1] + 1.)) - inters
    with np.errstate(divide="ignore", invalid="ignore"):
        return inters / uni


def average_precision(rec, prec, use_07_metric):
    if use_07_metric:                                                    # VOC07: 11 recall thresholds 0, 0.1, ..., 1
        ap = 0.
        for t in np.arange(0., 1.1, 0.1):
            above = rec >= t
            ap = ap + (np.max(prec[above]) if np.sum(above) > 0 else 0) / 11.
        return ap
    r = np.concatenate(([0.], rec, [1.]))
    p = np.concatenate(([0.], prec, [0.]))
    for i in range(p.size - 2, -1, -1):                                  # precision envelope, right to left
        p[i] = np.maximum(p[i], p[i + 1])
    steps = np.where(r[1:] != r[:-1])[0]
    return np.sum((r[steps + 1] - r[steps]) * p[steps + 1])


def class_ground_truth(recs, imagenames, classname):
    """{image name: (boxes float64 (g, 4), difficult bool (g,))} of one class, and npos (its non-difficult objects)."""
    gt, npos = {}, 0
    for name in imagenames:
        objs = [o for o in recs[name] if o["name"] == classname]
        boxes = np.array([o["bbox"] for o in objs], np.float64).reshape(-1, 4)
        difficult = np.array([o["difficult"] for o in objs], np.int64) != 0
        gt[name] = (boxes, difficult)
        npos += int(np.count_nonzero(~difficult))
    return gt, npos


def outcomes(names, scores, boxes, gt, ovthresh=0.5):
    """(tp, fp) per detection in rank order (descending score, ties in file order)."""
    order = np.argsort(-scores, kind="stable")
    claimed = {name: np.zeros(len(d), bool) for name, (_, d) in gt.items()}
    tp, fp = np.zeros(order.size), np.zeros(order.size)
    for r, d in enumerate(order):
        gboxes, difficult = gt[names[d]]
        best, j = -np.inf, -1
        if len(gboxes):
            ov = overlaps(boxes[d], gboxes)
            best, j = np.max(ov), int(np.argmax(ov))
        if not best > ovthresh:
            fp[r] = 1.
        elif difficult[j]:
            pass                                                         # a difficult box: neither tp nor fp
        elif claimed[names[d]][j]:
            fp[r] = 1.                                                   # the box was found by a higher-ranked detection
        else:
            tp[r] = 1.
            claimed[names[d]][j] = True
    return tp, fp


def voc_eval(lines, recs, imagenames, classname, ovthresh=0.5, use_07_metric=False):
    """rec, prec, ap of one class from its results-file lines and the parsed annotations {image name: objects}."""
    names, scores, boxes = parse_lines(lines)
    gt, npos = class_ground_truth(recs, imagenames, classname)
    tp, fp = outcomes(names, scores, boxes, gt, ovthresh)
    tp, fp = np.cumsum(tp), np.cumsum(fp)
    with np.errstate(divide="ignore", invalid="ignore"):
        rec = tp / float(npos)
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    return rec, prec, average_precision(rec, prec, use_07_metric)
