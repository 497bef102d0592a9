"""Proposal recall in plain numpy, as the reference's json_dataset_evaluator.evaluate_box_proposals defines it
(lib/datasets/json_dataset_evaluator.py:236-317), for the tests and tools.  The product never imports it.

The definition, per image: the proposals are the rows of `boxes` whose class is 0, cut to `limit` with Python slicing (an image with
no such row is left out, though its ground truth still counts as positives); the positives are the rows with a class > 0 that are not
crowd and whose seg_area lies in the closed area range.  With the IoU matrix M (proposals x positives), min(P, G) rounds each take the
column whose maximum is largest (first column on ties), take that column's first maximal row, record the value, and strike out that
row and that column; the positives never reached record 0.  Recall at t is the fraction of all positives whose recorded value is >= t.
A NaN in M makes the first round's maximum NaN, which the reference refuses with an AssertionError; so does this restatement.
"""
import numpy as np

from oracle.targets import bbox_overlaps

AREA_SIDES = (("all", 0, 1e5), ("small", 0, 32), ("medium", 32, 96), ("large", 96, 1e5), ("96-128", 96, 128), ("128-256", 128, 256),
              ("256-512", 256, 512), ("512-inf", 512, 1e5))
AREA_RANGE = {name: (float(lo) ** 2, float(hi) ** 2) for name, lo, hi in AREA_SIDES}


def overlaps(boxes, query):
    """bbox_overlaps with the compiled Cython's NaN behaviour.  Its min / max are the selects `q < b ? q : b` / `q > b ? q : b` (b the
    boxes row), which return b when either is NaN.  A NaN in a boxes row therefore makes iw or ih NaN and the IoU 0, as bbox_overlaps
    (np.minimum / np.maximum propagate NaN) gives it too; a NaN only in a query row leaves iw and ih finite, and the union NaN makes the
    IoU NaN whenever iw > 0 and ih > 0, where bbox_overlaps gives 0."""
    b = np.asarray(boxes, np.float32); q = np.asarray(query, np.float32)
    out = bbox_overlaps(b, q)
    if out.size == 0:
        return out
    sel = np.isnan(q).any(1)[None, :] & ~np.isnan(b).any(1)[:, None]
    if sel.any():
        f64 = np.float64
        pick_min = lambda bb, qq: np.where(qq < bb, qq, bb)  # noqa: E731
        pick_max = lambda bb, qq: np.where(qq > bb, qq, bb)  # noqa: E731
        iw = ((pick_min(b[:, None, 2], q[None, :, 2]) - pick_max(b[:, None, 0], q[None, :, 0])).astype(f64) + 1.0).astype(np.float32)
        ih = ((pick_min(b[:, None, 3], q[None, :, 3]) - pick_max(b[:, None, 1], q[None, :, 1])).astype(f64) + 1.0).astype(np.float32)
        out[sel & (iw > 0) & (ih > 0)] = np.nan
    return out


def split_entry(entry, area, limit):
    """(proposals kept by `limit` or None when the image has none at all, the positives in `area`) of one roidb entry."""
    lo, hi = AREA_RANGE[area]
    cls = entry["gt_classes"]
    rows = entry["boxes"]
    pos = rows[(cls > 0) & (entry["is_crowd"] == 0)]
    pos_area = entry["seg_areas"][(cls > 0) & (entry["is_crowd"] == 0)]
    pos = pos[(pos_area >= lo) & (pos_area <= hi)]
    props = rows[cls == 0]
    if len(props) == 0:
        return None, pos
    return props[:limit], pos


def greedy_coverage(m):
    """The recorded value of every round on the IoU matrix m (P x G), then zeros for the positives no round reached: G values."""
    m = np.array(m, dtype=np.float32)
    recorded = np.zeros(m.shape[1])
    for r in range(min(m.shape)):
        best = m.max(axis=0)                   # NaN propagates, as in the reference
        col = int(np.argmax(best))
        if not best[col] >= 0:
            raise AssertionError("NaN IoU in the matching: the reference's assert fails here")
        row = int(np.argmax(m[:, col]))
        recorded[r] = m[row, col]
        m[row, :] = -1
        m[:, col] = -1
    return recorded


def recall_summary(gt_overlaps, num_pos, thresholds):
    """ar / recalls as the reference computes them from the sorted overlaps: numpy int64 hits over float(num_pos), stored in an array
    shaped and typed like `thresholds`."""
    recalls = np.zeros_like(thresholds)
    for k, t in enumerate(thresholds):
        recalls[k] = np.int64(np.count_nonzero(gt_overlaps >= t)) / float(num_pos)
    return {"ar": recalls.mean(), "recalls": recalls, "thresholds": thresholds, "gt_overlaps": gt_overlaps, "num_pos": num_pos}


def evaluate_box_proposals(roidb, thresholds=None, area="all", limit=None):
    if area not in AREA_RANGE:
        raise AssertionError("Unknown area range: {}".format(area))
    values, num_pos = [np.zeros(0)], 0
    for entry in roidb:
        props, pos = split_entry(entry, area, limit)
        num_pos += len(pos)
        if props is not None:
            values.append(greedy_coverage(overlaps(props, pos)))
    if thresholds is None:
        thresholds = np.arange(0.5, 0.95 + 1e-5, 0.05)
    return recall_summary(np.sort(np.concatenate(values)), num_pos, thresholds)
