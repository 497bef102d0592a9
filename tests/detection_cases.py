"""Seeded inputs of the detection post-processing tests (box_results_with_nms_and_limit, lib/core/test.py:732-790) -- inputs
only; expected values come from tests/golden/detections.npz (the reference's own function) and oracle/detections.py.

Every case is (scores (R, K), boxes (R, 4K), params) with params the cfg.TEST values it runs with.  No case has two
candidates of one class with equal scores and overlapping boxes: the reference orders by an unstable argsort, so with such
ties its classic NMS is not a function of its inputs (check_no_overlapping_ties)."""
import numpy as np

from oracle import detections as O
from tests import cases

f32 = np.float32

# (soft_nms, soft_method, bbox_vote, vote_scoring): every configuration of tests/cases.py plus soft-NMS "hard"
ALL_CONFIGS = cases.DETECTION_CONFIGS + ((True, "hard", False, "ID"),)
CLASSIC, SOFT_HARD, VOTE_ID, VOTE_AVG = (False, "linear", False, "ID"), (True, "hard", False, "ID"), (False, "linear", True, "ID"), \
    (False, "linear", True, "AVG")
BOUNDARY_CONFIGS = (CLASSIC, SOFT_HARD, VOTE_ID)
DEFAULTS = dict(score_thresh=0.05, nms=0.5, detections_per_im=100, vote_th=0.8)
COCO_SEEDS = (0, 1)
SWEEP_SEEDS = tuple(range(10, 16))


def _params(**kw):
    p = dict(DEFAULTS)
    p.update(kw)
    return p


def coco_case(seed, R=1000, K=81, im_w=1333, im_h=800):
    """COCO-scale detection head output: 70 objects x ~14 jittered proposals, each object with one or two strong classes,
    boxes clipped to the image like the detector's (so border coordinates are integers)."""
    rng = np.random.RandomState(1000 + seed)
    n_obj = 70
    obj = rng.randint(0, n_obj, R)
    cx, cy = rng.uniform(0, im_w, n_obj)[obj], rng.uniform(0, im_h, n_obj)[obj]
    w, h = rng.uniform(20, 400, n_obj)[obj], rng.uniform(20, 400, n_obj)[obj]
    boxes = np.zeros((R, 4 * K), f32)
    for j in range(K):
        jx, jy = cx + rng.normal(0, 0.07, R) * w, cy + rng.normal(0, 0.07, R) * h
        jw, jh = w * (1 + rng.normal(0, 0.1, R)), h * (1 + rng.normal(0, 0.1, R))
        b = np.stack([jx - jw / 2, jy - jh / 2, jx + jw / 2, jy + jh / 2], 1)
        b[:, 0::2] = np.clip(b[:, 0::2], 0, im_w - 1); b[:, 1::2] = np.clip(b[:, 1::2], 0, im_h - 1)
        boxes[:, 4 * j:4 * j + 4] = b
    logits = rng.standard_normal((R, K)) * 1.5
    c1, c2 = rng.randint(1, K, n_obj), rng.randint(1, K, n_obj)
    logits[np.arange(R), c1[obj]] += rng.uniform(3, 7, R)
    second = rng.rand(n_obj)[obj] < 0.5
    logits[np.nonzero(second)[0], c2[obj][second]] += rng.uniform(2, 5, second.sum())
    e = np.exp(logits - logits.max(1, keepdims=True))
    return (e / e.sum(1, keepdims=True)).astype(f32), boxes


def _image(dets_by_class, K, rng, R_min=0, im_w=1333, im_h=800):
    """scores (R, K), boxes (R, 4K) holding the given detections of each class (one row each) and nothing else above
    0.05: the other entries are low scores (<= 0.04) with random boxes."""
    rows = [(j, d) for j in sorted(dets_by_class) for d in dets_by_class[j]]
    R = max(len(rows), R_min)
    scores = rng.uniform(0.001, 0.04, (R, K)).astype(f32)
    x1, y1 = rng.uniform(0, im_w - 100, (R, K)), rng.uniform(0, im_h - 100, (R, K))
    boxes = np.stack([x1, y1, x1 + rng.uniform(5, 100, (R, K)), y1 + rng.uniform(5, 100, (R, K))], 2).reshape(R, 4 * K).astype(f32)
    perm = rng.permutation(R)
    for r, (j, d) in zip(perm, rows):
        boxes[r, 4 * j:4 * j + 4] = d[:4]
        scores[r, j] = d[4]
    return scores, boxes


def k201_case(seed=0, R=400, K=201):
    """201 classes (200 problems: two soft-NMS / voting chunks of 128, four NMS chunks of 64) with classes 1-64 empty, so the
    first NMS chunk has no candidate at all."""
    scores, boxes = coco_case(seed, R=R, K=K)
    scores[:, 1:65] = np.minimum(scores[:, 1:65], f32(0.04))
    return scores, boxes


def sparse_case(seed=0, K=81, R=300):
    """Most classes empty; classes 3, 17, 40 have one candidate each, class 7 two far apart, class 60 a cluster.  Scores of
    exactly float32(0.05) are not candidates (`> SCORE_THRESH` in float32); the next float32 up is."""
    rng = np.random.RandomState(2000 + seed)
    at, above = f32(0.05), np.nextafter(f32(0.05), f32(1))
    d = {3: [[10, 10, 60, 90, 0.7]], 17: [[0, 0, 1332, 799, above]], 40: [[500.5, 300.25, 501.5, 300.75, 0.3]],
         7: [[100, 100, 200, 200, 0.6], [700, 500, 800, 600, 0.55]],
         60: [[300 + 3 * i, 200 + 2 * i, 400 + 3 * i, 330 + 2 * i, 0.9 - 0.03 * i] for i in range(12)],
         22: [[50, 50, 150, 150, at]], 23: [[60, 60, 160, 160, at], [600, 400, 700, 500, 0.2]]}
    scores, boxes = _image({j: [np.asarray(r, f32) for r in v] for j, v in d.items()}, K, rng, R_min=R)
    scores[rng.randint(0, R, 20), rng.randint(1, K, 20)] = at
    return scores, boxes


def empty_case(seed=0, K=81, R=300):
    """No score above the threshold (some equal to float32(0.05))."""
    rng = np.random.RandomState(3000 + seed)
    scores, boxes = _image({}, K, rng, R_min=R)
    scores[rng.randint(0, R, 40), rng.randint(0, K, 40)] = f32(0.05)
    return scores, boxes


def _ulp(t, k):
    v = f32(t)
    for _ in range(abs(k)):
        v = np.nextafter(v, f32(np.inf) if k > 0 else f32(-np.inf))
    return v


def pair_at(t, k, rng, iou=O.nms_iou):
    """A pair of float boxes (A, B) with iou(A, B) == float32(t) moved k ulps (random search around the analytic shift).
    iou: the overlap arithmetic the pair is built for, vectorized over rows (cython_nms.nms's by default)."""
    target = _ulp(t, k)
    for _ in range(200):
        n = 20000
        w, h = rng.uniform(30, 300, n), rng.uniform(30, 300, n)
        x0, y0 = rng.uniform(0, 900, n), rng.uniform(0, 400, n)
        dx = w * (1 - t) / (1 + t) + rng.uniform(-0.02, 0.02, n)
        A = np.stack([x0, y0, x0 + w - 1, y0 + h - 1], 1).astype(f32)
        B = np.stack([x0 + dx, y0, x0 + dx + w - 1, y0 + h - 1], 1).astype(f32)
        hit = np.nonzero(iou(A, B) == target)[0]
        if len(hit):
            return A[hit[0]], B[hit[0]]
    raise AssertionError("no pair at %r %+d ulp" % (t, k))


def _integer_pair(t, x0, y0):
    """A 100 x 100 box and a box inside it with 100 * t of its rows: IoU exactly 100 t / 100 in float32."""
    A = np.array([x0, y0, x0 + 99, y0 + 99], f32)
    return A, np.array([x0, y0, x0 + 99, y0 + round(100 * t) - 1], f32)


def nms_threshold_case(t, seed=0, K=12):
    """Same-class pairs whose Cython-NMS IoU is exactly float32(t) (integer boxes, and float boxes), 1 ulp above and 1 ulp
    below it, and a chain A > B > C where B sits exactly at the threshold to A and C overlaps B but not A: the reference
    drops B and so keeps C."""
    rng = np.random.RandomState(4000 + seed + int(round(100 * t)))
    d = {}
    A, B = _integer_pair(t, 100, 100)
    d[1] = [np.r_[A, 0.9], np.r_[B, 0.8]]
    A, B = _integer_pair(t, 0, 700)                                   # the lower box scores higher
    d[2] = [np.r_[B, 0.7], np.r_[A, 0.6]]
    for j, k in ((3, 0), (4, 1), (5, -1), (6, 0), (7, 1), (8, -1)):
        A, B = pair_at(t, k, rng)
        d[j] = [np.r_[A, 0.95 - 0.01 * j], np.r_[B, 0.5 - 0.01 * j]]
    A, B = _integer_pair(t, 400, 200)
    C = B + np.array([-10, 2, -10, 2], f32)
    assert O.nms_iou(A, C) < f32(t) <= O.nms_iou(B, C)
    d[9] = [np.r_[A, 0.9], np.r_[B, 0.85], np.r_[C, 0.8]]
    A, B = pair_at(t, 0, rng)
    C = B + np.array([0.3 * (B[2] - B[0]), 0, 0.3 * (B[2] - B[0]), 0], f32)
    if O.nms_iou(A, C) < f32(t) <= O.nms_iou(B, C):
        d[10] = [np.r_[A, 0.9], np.r_[B, 0.85], np.r_[C, 0.8]]
    return _image({j: [np.asarray(r, f32) for r in v] for j, v in d.items()}, K, rng)


def vote_threshold_case(seed=0, K=6, vote_th=0.8):
    """A kept box and a box it suppresses whose bbox_overlaps IoU is exactly float32(VOTE_TH) (votes), 1 ulp below it
    (does not vote) and 1 ulp above it."""
    rng = np.random.RandomState(5000 + seed)
    d = {}
    A, B = _integer_pair(vote_th, 100, 100)
    assert O.overlaps(A, B) == f32(vote_th)
    d[1] = [np.r_[A, 0.9], np.r_[B, 0.6]]
    for j, k in ((2, 0), (3, -1), (4, 1)):
        A, B = pair_at(vote_th, k, rng, iou=O.overlaps)
        d[j] = [np.r_[A, 0.9], np.r_[B, 0.7], np.r_[B + f32(150), 0.3]]
    return _image({j: [np.asarray(r, f32) for r in v] for j, v in d.items()}, K, rng)


def dpi_ties_case(seed=0, K=81):
    """~130 candidates after NMS, six of them (in six classes) sharing the 100th-best score: the reference keeps all six."""
    rng = np.random.RandomState(6000 + seed)
    d = {}
    s = np.sort(rng.uniform(0.1, 0.99, 130).astype(f32))[::-1]
    assert len(np.unique(s)) == 130
    tie = s[97]
    s[94:100] = tie
    for i in range(130):
        j = 1 + i % (K - 1)
        x, y = 10 * (i // (K - 1)) * 30, 0
        d.setdefault(j, []).append(np.asarray([x + 5, y + 5, x + 200, y + 150, s[i]], f32))
    return _image(d, K, rng)


def check_no_overlapping_ties(scores, boxes, score_thresh, K):
    """No two candidates of one class with equal scores and boxes that overlap (see the module docstring)."""
    for j in range(1, K):
        inds = np.nonzero(scores[:, j] > f32(score_thresh))[0]
        s = scores[inds, j]
        b = boxes[inds, 4 * j:4 * j + 4]
        vals, counts = np.unique(s, return_counts=True)
        for v in vals[counts > 1]:
            tied = b[s == v]
            for a in range(len(tied)):
                assert np.all(O.nms_iou(tied[a], tied[a + 1:]) <= 0), "class %d: overlapping boxes tie at score %r" % (j, v)


def detection_cases():
    """name -> (scores, boxes, K, params, configs) for every golden case."""
    out = {}
    for seed in COCO_SEEDS:
        s, b = coco_case(seed)
        out["coco%d" % seed] = (s, b, 81, _params(), ALL_CONFIGS)
    s, b = k201_case()
    out["k201"] = (s, b, 201, _params(), ALL_CONFIGS)
    s, b = sparse_case()
    out["sparse"] = (s, b, 81, _params(), ALL_CONFIGS)
    s, b = empty_case()
    out["empty"] = (s, b, 81, _params(), ALL_CONFIGS)
    for t in (0.3, 0.5, 0.7):
        s, b = nms_threshold_case(t)
        out["nms%d" % round(100 * t)] = (s, b, 12, _params(nms=t), BOUNDARY_CONFIGS)
    s, b = vote_threshold_case()
    out["vote80"] = (s, b, 6, _params(), (VOTE_ID, VOTE_AVG))
    s, b = dpi_ties_case()
    for dpi in (100, 0, 1000):
        out["ties_dpi%d" % dpi] = (s, b, 81, _params(detections_per_im=dpi), (CLASSIC, VOTE_ID))
    for name, (s, b, K, p, _) in out.items():
        assert s.shape[1] == K and b.shape[1] == 4 * K, name
        check_no_overlapping_ties(s, b, p["score_thresh"], K)
    return out
