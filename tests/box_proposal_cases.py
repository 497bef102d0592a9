"""Seeded synthetic roidbs for proposal recall (tests/test_box_proposals.py, tests/golden/make_golden_box_proposals.py,
tools/box_proposals_probe.py).

An entry is what evaluate_box_proposals reads of a reference roidb entry: `boxes` (float32 rows: ground truth and proposals, the
proposals being the gt_classes == 0 rows in order), `gt_classes`, `is_crowd` and `seg_areas` (float32, as JsonDataset stores them).
"""
import numpy as np

AREA_BOUNDS = [1024.0, 9216.0, 16384.0, 65536.0, 262144.0, 1e10]
LIMITS = [None, 1000, 100, 7, 0, -3]
CUSTOM_THRESHOLDS = np.array([-0.5, 0.0, 0.25, 0.5, 0.75, 1.0, 1.0000001], np.float64)


def entry(gt_boxes, gt_classes, is_crowd, seg_areas, props, order=None):
    """One roidb entry: ground-truth rows then proposal rows (class 0, not crowd, area 0), optionally permuted by `order`."""
    gt_boxes = np.asarray(gt_boxes, np.float32).reshape(-1, 4)
    props = np.asarray(props, np.float32).reshape(-1, 4)
    boxes = np.concatenate([gt_boxes, props])
    cls = np.concatenate([np.asarray(gt_classes, np.int32).reshape(-1), np.zeros(len(props), np.int32)])
    crowd = np.concatenate([np.asarray(is_crowd, np.bool_).reshape(-1), np.zeros(len(props), np.bool_)])
    areas = np.concatenate([np.asarray(seg_areas, np.float32).reshape(-1), np.zeros(len(props), np.float32)])
    if order is not None:
        boxes, cls, crowd, areas = boxes[order], cls[order], crowd[order], areas[order]
    return {"boxes": boxes, "gt_classes": cls, "is_crowd": crowd, "seg_areas": areas}


def _random_gts(rng, g, size=640.0):
    x1 = rng.uniform(0, size * 0.8, g); y1 = rng.uniform(0, size * 0.8, g)
    w = np.exp(rng.uniform(np.log(2.0), np.log(size * 0.7), g)); h = w * np.exp(rng.uniform(-1.0, 1.0, g))
    return np.round(np.stack([x1, y1, x1 + w, y1 + h], 1) * 2) / 2


def _jittered(rng, gts, n, size=640.0):
    """n proposals: most jittered from a gt by a random relative scale (IoUs across [0, 1]), some uniform, some exact copies."""
    if n == 0:
        return np.zeros((0, 4))
    out = _random_gts(rng, n, size)
    if len(gts):
        k = rng.randint(0, len(gts), n)
        g = gts[k]
        wh = np.concatenate([g[:, 2:4] - g[:, 0:2] + 1] * 2, 1)
        s = rng.choice([0.0, 0.02, 0.1, 0.3, 0.8], n)[:, None]
        jit = g + rng.standard_normal((n, 4)) * wh * s
        jit[:, 2:4] = np.maximum(jit[:, 2:4], jit[:, 0:2])
        pick = rng.uniform(size=n) < 0.85
        out[pick] = np.round(jit[pick] * 4) / 4
    return out


def coco_like(seed=1, n_images=40, max_gt=30, max_props=2500):
    """0 .. max_gt gts per image (some crowd, some class 0), 0 .. max_props proposals, rows of some images shuffled."""
    rng = np.random.RandomState(seed)
    roidb = []
    for i in range(n_images):
        g = rng.randint(0, max_gt + 1)
        gts = _random_gts(rng, g)
        cls = rng.randint(1, 81, g)
        cls[rng.uniform(size=g) < 0.05] = 0
        crowd = rng.uniform(size=g) < 0.1
        wh = gts[:, 2:4] - gts[:, 0:2] + 1
        areas = wh[:, 0] * wh[:, 1] * rng.uniform(0.4, 1.0, g)
        n = 0 if i % 13 == 5 else rng.randint(0, max_props + 1)
        props = _jittered(rng, gts, n)
        order = rng.permutation(g + n) if i % 4 == 3 else None
        roidb.append(entry(gts, cls, crowd, areas, props, order))
    return roidb


def area_boundaries(seed=2):
    """seg_areas exactly at every range boundary, and one float32 ulp on either side."""
    rng = np.random.RandomState(seed)
    roidb = []
    for b in AREA_BOUNDS:
        b32 = np.float32(b)
        areas = [np.nextafter(b32, np.float32(0)), b32, np.nextafter(b32, np.float32(np.inf))]
        gts = _random_gts(rng, 3)
        roidb.append(entry(gts, [1, 2, 3], [0, 0, 0], areas, _jittered(rng, gts, 20)))
    return roidb


def ties(seed=3):
    """Duplicate proposals, duplicate gts and symmetric layouts where the first-index rules decide."""
    rng = np.random.RandomState(seed)
    sq = [10, 10, 49, 49]
    roidb = [
        # two identical gts, two identical proposals on them, a third proposal shifted
        entry([sq, sq], [1, 1], [0, 0], [1600, 1600], [sq, sq, [12, 10, 51, 49]]),
        # one proposal straddling two mirror-image gts: equal IoU with both, the first gt wins it
        entry([[0, 0, 19, 19], [20, 0, 39, 19]], [1, 2], [0, 0], [400, 400], [[10, 0, 29, 19], [100, 100, 110, 110]]),
        # a gt covered equally by two proposals: the first proposal is taken
        entry([[10, 10, 29, 29]], [1], [0], [400], [[5, 10, 24, 29], [15, 10, 34, 29]]),
        # a grid of equal-size gts with every proposal a copy: all IoUs 1 or 0
        entry([[x, y, x + 9, y + 9] for x in (0, 20) for y in (0, 20)], [1, 2, 3, 4], [0] * 4, [100] * 4,
              [[x, y, x + 9, y + 9] for x in (20, 0) for y in (20, 0)] * 2),
        # P < G with many equal IoUs
        entry([sq] * 5, [1] * 5, [0] * 5, [1600] * 5, [[10, 10, 49, 29]] * 3),
    ]
    gts = np.round(_random_gts(rng, 12) / 8) * 8
    props = np.concatenate([gts[rng.randint(0, 12, 30)], np.round(_jittered(rng, gts, 60) / 8) * 8])
    roidb.append(entry(np.concatenate([gts, gts[:4]]), rng.randint(1, 5, 16), np.zeros(16), np.full(16, 2000.0), props))
    return roidb


def on_threshold():
    """IoUs exactly 0.5 and 0.75 (100 x 100 gt, proposals keeping 50 / 75 of its rows), and exactly 1."""
    g = [0, 0, 99, 99]
    return [entry([g], [1], [0], [10000], [[0, 0, 99, 49]]),
            entry([g], [1], [0], [10000], [[0, 0, 99, 74]]),
            entry([g, [200, 200, 299, 299]], [1, 1], [0, 0], [10000, 10000], [[200, 200, 299, 299], [0, 50, 99, 99]])]


def shapes():
    """P < G, an image without proposals, one without valid gts (crowd / background only), one without any gt."""
    g3 = [[0, 0, 9, 9], [30, 30, 59, 59], [100, 0, 199, 99]]
    return [entry(g3, [1, 2, 3], [0, 0, 0], [100, 900, 10000], [[0, 0, 9, 9]]),
            entry(g3, [1, 2, 3], [0, 0, 0], [100, 900, 10000], []),
            entry(g3, [0, 2, 3], [0, 1, 1], [100, 900, 10000], [[0, 0, 9, 9], [30, 30, 59, 59]]),
            entry([], [], [], [], [[0, 0, 9, 9]]),
            entry(g3[:2], [4, 5], [0, 0], [5000, 20000], [[1, 1, 9, 9], [31, 30, 59, 59], [0, 0, 5, 5]])]


def no_positives():
    """Every gt crowd or background: num_pos == 0, ar NaN."""
    return [entry([[0, 0, 9, 9]], [1], [1], [100], [[0, 0, 9, 9]]),
            entry([[0, 0, 9, 9]], [0], [0], [100], [[0, 0, 9, 9]]),
            entry([], [], [], [], [])]


def nan_gt():
    """A NaN ground-truth coordinate: its IoUs are NaN (the union is), and the reference's assert fails wherever that gt is in range
    and the limit keeps a proposal."""
    return [entry([[0, 0, 9, 9]], [1], [0], [100], [[0, 0, 9, 9]]),
            entry([[0, 0, 9, 9], [50, 50, 59, np.nan]], [1, 1], [0, 0], [100, 100], [[0, 0, 9, 9], [1, 1, 9, 9], [50, 50, 59, 59]])]


def nan_proposal():
    """A NaN proposal coordinate: the compiled Cython's min / max return it, so iw or ih is NaN and the IoU 0; nothing raises."""
    return [entry([[0, 0, 9, 9], [50, 50, 59, 59]], [1, 1], [0, 0], [100, 100],
                  [[1, 1, 9, np.nan], [np.nan, 0, 9, 9], [50, 50, 59, 59], [0, 0, 9, 9]])]


CASES = {"coco_like": coco_like, "area_boundaries": area_boundaries, "ties": ties, "on_threshold": on_threshold, "shapes": shapes,
         "no_positives": no_positives, "nan_gt": nan_gt,
         "nan_proposal": nan_proposal}
AREA_NAMES = ["all", "small", "medium", "large", "96-128", "128-256", "256-512", "512-inf"]
THRESHOLD_SETS = {"default": None, "custom": CUSTOM_THRESHOLDS}


def load_golden(g, case, tname, area, limit):
    """The reference's result for one (case, threshold set, area, limit): None if it raised, else its dict."""
    a, l = AREA_NAMES.index(area), LIMITS.index(limit)
    p = "%s/%s/" % (case, tname)
    if g[p + "raised"][a, l]:
        return None
    k = a * len(LIMITS) + l
    b = g[p + "gt_overlaps_begin"]
    return {"ar": g[p + "ar"][a, l], "recalls": g[p + "recalls"][a, l], "thresholds": g[p + "thresholds"], "num_pos": int(g[p + "num_pos"][a, l]),
            "gt_overlaps": g[p + "gt_overlaps"][b[k]:b[k + 1]]}


def pack(roidb):
    """Flat arrays of a roidb (rows of all entries with their offsets), for the golden file."""
    begin = np.concatenate([[0], np.cumsum([len(e["boxes"]) for e in roidb])]).astype(np.int64)
    cat = lambda k, dt: np.concatenate([e[k] for e in roidb]).astype(dt) if roidb else np.zeros(0, dt)  # noqa: E731
    return {"row_begin": begin, "boxes": cat("boxes", np.float32).reshape(-1, 4), "gt_classes": cat("gt_classes", np.int32),
            "is_crowd": cat("is_crowd", np.bool_), "seg_areas": cat("seg_areas", np.float32)}


def unpack(arrays):
    b = arrays["row_begin"]
    return [{k: arrays[k][b[i]:b[i + 1]] for k in ("boxes", "gt_classes", "is_crowd", "seg_areas")} for i in range(len(b) - 1)]


def scale_set(seed=7, n_images=5000, props=(1000, 2000), gt_mean=7.3, max_gt=None, size=640.0):
    """A COCO-minival-shaped roidb: n_images images, props[0] .. props[1] proposals each, Poisson gt counts around gt_mean (capped at
    max_gt, or a fixed max_gt-heavy tail when gt_mean is None), proposals jittered from the gts."""
    rng = np.random.RandomState(seed)
    roidb = []
    for i in range(n_images):
        g = int(rng.poisson(gt_mean)) if gt_mean is not None else int(rng.randint(0, max_gt + 1))
        if max_gt is not None:
            g = min(g, max_gt)
        gts = _random_gts(rng, g, size)
        wh = gts[:, 2:4] - gts[:, 0:2] + 1
        n = int(rng.randint(props[0], props[1] + 1))
        roidb.append(entry(gts, rng.randint(1, 81, g), rng.uniform(size=g) < 0.01, wh[:, 0] * wh[:, 1] * 0.7, _jittered(rng, gts, n, size)))
    return roidb
