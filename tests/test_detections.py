"""SURVEY.md 8f N3: test-time detection post-processing on the device (per-class NMS in one batched launch pair, soft-NMS,
box voting, the per-image limit) against golden outputs of the REFERENCE'S OWN function -- lib/core/test.py:732-790 with
lib/utils/boxes.py and the Cython routines built from its .pyx -- run unmodified on the seeded inputs of tests/cases.py and
tests/detection_cases.py (tests/golden/make_golden_detections.py -> detections.npz), and against oracle/detections.py.

Classic NMS and soft-NMS are compared bit for bit.  Box voting is a weighted average: the reference averages in float32
(np.average), the device and the oracle in float64, so the device must be within one float32 ulp of the oracle, and the
oracle within the float32 error of np.average of the golden."""
import os
import types

import numpy as np
import pytest

from oracle import detections as O
from tests import cases
from tests import detection_cases as DC

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "detections.npz")
f32 = np.float32


def _golden_case(g, name, k, K):
    arr, cnt = g["%s_c%d" % (name, k)], g["%s_c%d_counts" % (name, k)]
    off = np.concatenate([[0], np.cumsum(cnt)])
    return [None] + [arr[off[j]:off[j + 1]] for j in range(K - 1)]


def _oracle(scores, boxes, K, p, config):
    soft, method, vote, scoring = config
    return O.box_results_with_nms_and_limit(scores, boxes, K, p["score_thresh"], p["nms"], p["detections_per_im"], soft, 0.5, method,
                                            vote, p["vote_th"], scoring)


def _kw(K, p, config):
    soft, method, vote, scoring = config
    return dict(num_classes=K, score_thresh=p["score_thresh"], nms=p["nms"], detections_per_im=p["detections_per_im"], soft_nms=soft,
                soft_method=method, bbox_vote=vote, vote_th=p["vote_th"], vote_scoring=scoring)


def _cfg(K, p, config):
    """A stand-in for the reference's cfg object with the fields box_results_with_nms_and_limit reads."""
    soft, method, vote, scoring = config
    ns = types.SimpleNamespace
    return ns(MODEL=ns(NUM_CLASSES=K),
              TEST=ns(SCORE_THRESH=p["score_thresh"], NMS=p["nms"], DETECTIONS_PER_IM=p["detections_per_im"],
                      SOFT_NMS=ns(ENABLED=soft, SIGMA=0.5, METHOD=method),
                      BBOX_VOTE=ns(ENABLED=vote, VOTE_TH=p["vote_th"], SCORING_METHOD=scoring)))


def _within_f32_average_error(golden, exact, what):
    """golden: a float32 np.average of n rows; exact: the same in float64.  Pairwise float32 summation is within
    (log2 n + 2) eps of the largest magnitude involved; n <= 1000 here."""
    if len(golden) == 0:
        return
    bound = 12 * np.finfo(f32).eps * max(1.0, float(np.abs(exact).max()))
    err = np.abs(golden.astype(np.float64) - exact).max()
    assert err <= bound, (what, err, bound)


def _within_one_ulp(ours, exact, what):
    """ours (float32) is within one float32 ulp of the float64 value."""
    ref = exact.astype(f32)
    ulp = np.spacing(np.maximum(np.abs(ref), np.finfo(f32).tiny))
    bad = np.abs(ours.astype(np.float64) - exact) > ulp
    assert not bad.any(), (what, ours[bad][:4], exact[bad][:4])


def _compare(ours_cls, gold_cls, K, config, what):
    vote = config[2]
    for j in range(1, K):
        a, b = gold_cls[j], np.asarray(ours_cls[j]).reshape(-1, 5)
        assert a.shape == b.shape, (what, j, a.shape, b.shape)
        if vote:
            np.testing.assert_allclose(b, a, rtol=1e-5, atol=2e-3)
        else:
            assert b.dtype == np.float32 and np.array_equal(a, b), (what, j)


# ------------------------------------------------------------------------------------------------ CPU: cases and oracle
def test_cases_sit_on_the_boundaries_they_name():
    cs = DC.detection_cases()
    assert {"coco0", "coco1", "k201", "sparse", "empty", "nms30", "nms50", "nms70", "vote80", "ties_dpi100", "ties_dpi0",
            "ties_dpi1000"} <= set(cs)
    for t in (0.3, 0.5, 0.7):
        s, b, K, p, _ = cs["nms%d" % round(100 * t)]
        found = set()
        for j in range(1, K):
            inds = np.nonzero(s[:, j] > f32(0.05))[0]
            d = b[inds, 4 * j:4 * j + 4]
            for x in range(len(d)):
                for y in range(x + 1, len(d)):
                    v = O.nms_iou(d[x], d[y])
                    for k in (-1, 0, 1):
                        if v == DC._ulp(t, k):
                            found.add(k)
        assert found == {-1, 0, 1}, (t, found)
    s, b, K, p, _ = cs["k201"]
    counts = (s[:, 1:] > f32(0.05)).sum(0)
    assert counts[:64].sum() == 0 and (counts[64:] > 0).sum() > 128
    s, b, K, p, _ = cs["empty"]
    assert not (s[:, 1:] > f32(0.05)).any() and (s == f32(0.05)).any()
    s, b, K, p, _ = cs["sparse"]
    counts = (s[:, 1:] > f32(0.05)).sum(0)
    assert (counts == 0).sum() > 70 and (counts == 1).sum() >= 3 and (s == f32(0.05)).any()
    for seed in DC.COCO_SEEDS:
        s, _ = DC.coco_case(seed)
        assert s.shape == (1000, 81) and ((s[:, 1:] > f32(0.05)).sum(0) > 0).sum() > 64


def test_oracle_reproduces_every_golden():
    g = np.load(GOLDEN)
    for name, (s, b, K, p, configs) in DC.detection_cases().items():
        for k, config in enumerate(configs):
            gold = _golden_case(g, name, k, K)
            ora = _oracle(s, b, K, p, config)
            for j in range(1, K):
                assert gold[j].shape == ora[j].shape, (name, config, j)
                if config[2]:
                    _within_f32_average_error(gold[j], ora[j], (name, config, j))
                else:
                    assert np.array_equal(gold[j], ora[j]), (name, config, j)
    for seed in cases.DETECTION_SEEDS:
        s, b = cases.detection_case(seed)
        for k, config in enumerate(cases.DETECTION_CONFIGS):
            ora = _oracle(s, b, 21, DC.DEFAULTS, config)
            for j in range(1, 21):
                gold = g["s%d_c%d_j%d" % (seed, k, j)]
                assert gold.shape == ora[j].shape
                if config[2]:
                    _within_f32_average_error(gold, ora[j], (seed, config, j))
                else:
                    assert np.array_equal(gold, ora[j]), (seed, config, j)


def test_oracle_nms_boundaries_and_tie_rule():
    """Cython NMS: suppress at IoU >= float32(thresh), so exactly 0.5 suppresses and 0.7 (7/10 rounds to float32(0.7))
    too; tied scores go lower index first -- the rule the device follows where the reference's argsort is unstable."""
    A, B = DC._integer_pair(0.5, 0, 0)
    assert list(O.nms(np.array([np.r_[A, 0.9], np.r_[B, 0.8]], f32), 0.5)) == [0]
    A, B = DC._integer_pair(0.7, 0, 0)
    assert O.nms_iou(A, B) == f32(0.7) and list(O.nms(np.array([np.r_[A, 0.9], np.r_[B, 0.8]], f32), 0.7)) == [0]
    tie = np.array([np.r_[B, 0.8], np.r_[A, 0.8], np.r_[A + f32(500), 0.8]], f32)
    assert list(O.nms(tie, 0.5)) == [0, 2]
    assert list(O.nms(tie[[1, 0, 2]], 0.5)) == [0, 2]


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_box_results_with_nms_and_limit_matches_the_reference():
    from detectron.pytorch_b200.core.test import box_results_with_nms_and_limit as ours
    g = np.load(GOLDEN)
    checked = 0
    for seed in cases.DETECTION_SEEDS:
        scores, boxes = cases.detection_case(seed)
        for k, (soft, method, vote, scoring) in enumerate(cases.DETECTION_CONFIGS):
            os_, ob, oc = ours(scores, boxes, num_classes=21, score_thresh=0.05, nms=0.5, detections_per_im=100, soft_nms=soft,
                               soft_method=method, bbox_vote=vote, vote_th=0.8, vote_scoring=scoring)
            assert len(oc) == 21
            for j in range(1, 21):
                a, b = g["s%d_c%d_j%d" % (seed, k, j)], np.asarray(oc[j]).reshape(-1, 5)
                assert a.shape == b.shape, (seed, soft, method, vote, scoring, j, a.shape, b.shape)
                if vote:      # numpy averages in float32 pairwise order; ours accumulates in fp64
                    np.testing.assert_allclose(b, a, rtol=1e-4, atol=2e-3)
                else:
                    assert np.array_equal(a, b), (seed, soft, method, j)
            n = int(g["s%d_c%d_n" % (seed, k)])
            assert os_.shape == (n,) and ob.shape == (n, 4)
            checked += 1
    assert checked == 18


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DC.detection_cases()))
def test_every_golden_case_numpy_cuda_and_cfg(name):
    """Every new golden case and configuration, through numpy inputs, CUDA-tensor inputs and a cfg object; voting also
    within one float32 ulp of the float64 oracle."""
    import torch
    from detectron.pytorch_b200.core.test import box_results_with_nms_and_limit as ours
    g = np.load(GOLDEN)
    s, b, K, p, configs = DC.detection_cases()[name]
    S, B = torch.from_numpy(s).cuda(), torch.from_numpy(b).cuda()
    for k, config in enumerate(configs):
        gold = _golden_case(g, name, k, K)
        n = int(sum(len(x) for x in gold[1:]))
        runs = (ours(s, b, **_kw(K, p, config)), ours(S, B, **_kw(K, p, config)), ours(s, b, cfg=_cfg(K, p, config)))
        for r, (os_, ob, oc) in enumerate(runs):
            what = (name, config, ("numpy", "cuda", "cfg")[r])
            assert len(oc) == K and os_.shape == (n,) and ob.shape == (n, 4), what
            _compare(oc, gold, K, config, what)
            assert np.array_equal(runs[0][2][K - 1], oc[K - 1]) and all(np.array_equal(runs[0][2][j], oc[j]) for j in range(1, K))
        if config[2]:
            ora = _oracle(s, b, K, p, config)
            for j in range(1, K):
                _within_one_ulp(runs[0][2][j], ora[j], (name, config, j))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", DC.SWEEP_SEEDS)
def test_coco_scale_sweep_against_the_oracle(seed):
    """More seeded COCO-scale images (81 classes, 1000 detections: two NMS chunks) against oracle/detections.py, every
    configuration: NMS and soft-NMS bit for bit, voting within one float32 ulp of float64."""
    from detectron.pytorch_b200.core.test import box_results_with_nms_and_limit as ours
    s, b = DC.coco_case(seed)
    DC.check_no_overlapping_ties(s, b, 0.05, 81)
    for nms in (0.3, 0.5, 0.7):
        p = DC._params(nms=nms)
        for config in (DC.ALL_CONFIGS if nms == 0.5 else (DC.CLASSIC, DC.SOFT_HARD, DC.VOTE_ID)):
            _, _, oc = ours(s, b, **_kw(81, p, config))
            ora = _oracle(s, b, 81, p, config)
            for j in range(1, 81):
                o = np.asarray(oc[j]).reshape(-1, 5)
                assert o.shape == ora[j].shape, (seed, nms, config, j)
                if config[2]:
                    _within_one_ulp(o, ora[j], (seed, nms, config, j))
                else:
                    assert np.array_equal(o, ora[j]), (seed, nms, config, j)


@pytest.mark.gpu
def test_ties_keep_the_lower_index():
    """Two overlapping boxes of one class with equal scores: the device keeps the lower detection index (score-sorted
    stable), in box_results_with_nms_and_limit and in utils.boxes.nms, like the oracle."""
    from detectron.pytorch_b200.core.test import box_results_with_nms_and_limit as ours
    from detectron.pytorch_b200.utils.boxes import nms as boxes_nms
    A, B = DC._integer_pair(0.7, 10, 10)
    for first, second in ((A, B), (B, A)):
        dets = np.array([np.r_[first, 0.8], np.r_[second, 0.8], np.r_[A + f32(300), 0.8]], f32)
        assert list(boxes_nms(dets, 0.5)) == list(O.nms(dets, 0.5)) == [0, 2]
        scores = np.array([[0.1, 0.8], [0.1, 0.8], [0.1, 0.8]], f32)
        _, _, oc = ours(scores, np.tile(dets[:, :4], (1, 2)), num_classes=2)
        assert np.array_equal(oc[1], dets[[0, 2]])


@pytest.mark.gpu
@pytest.mark.parametrize("t", (0.3, 0.5, 0.7))
def test_utils_boxes_nms_is_the_cython_nms(t):
    """utils.boxes.nms (the stand-in for cython_nms.nms): unsorted rows of the boundary cases, kept indices ascending."""
    from detectron.pytorch_b200.utils.boxes import nms as boxes_nms
    s, b, K, p, _ = DC.detection_cases()["nms%d" % round(100 * t)]
    rows = []
    for j in range(1, K):
        inds = np.nonzero(s[:, j] > f32(0.05))[0]
        rows.append(np.hstack([b[inds, 4 * j:4 * j + 4], s[inds, j][:, None]]))
    for dets in rows + [np.concatenate(rows).astype(f32)]:
        dets = np.ascontiguousarray(dets, f32)
        assert list(boxes_nms(dets, t)) == list(O.nms(dets, t)), dets
    assert boxes_nms(np.zeros((0, 5), f32), t) == []


def band_case(t, seed=0):
    """Score-sorted boxes for the proposal NMS whose pairs sit where the division-free screen of the mask kernel cannot
    decide: IoU within a few float32 ulps of the threshold (float and integer boxes), boxes with coordinates near 2^33
    (denominators above 2^62), and pairs whose fused denominator is 0 or negative, below 2^-62 (boxes of negative width;
    with the +1 convention a positive area is at least 2^-48, so a positive denominator cannot get below 2^-62).  Pairs are spread over a grid, so they land in diagonal and off-diagonal 64 x 64 tiles."""
    rng = np.random.RandomState(7000 + seed + int(round(100 * t)))
    boxes = []
    for p in range(240):
        gx, gy = (p % 20) * 700.0, (p // 20) * 700.0
        w, h = rng.uniform(30, 300), rng.uniform(30, 300)
        kind = p % 6
        if kind == 5:                                          # integer boxes: IoU exactly t
            A, B = DC._integer_pair(t, gx, gy)
        elif kind == 4:                                        # huge boxes: denominators ~2^66
            s = 2.0 ** 32
            dx = s * (1 - t) / (1 + t) * (1 + rng.uniform(-2e-6, 2e-6))
            A = np.array([gx * s, gy * s, gx * s + s, gy * s + s], f32)
            B = np.array([gx * s + dx, gy * s, gx * s + dx + s, gy * s + s], f32)
        elif kind == 3 and p % 4 == 1:                         # den = fma(bw, bh, Sa) - inter exactly 0: areas -+20 * 2^-48
            e = 2.0 ** -24
            A = np.array([0, 0, -1 - 4 * e, -1 + 5 * e], f32)
            B = np.array([0, 0, -1 + 4 * e, -1 + 5 * e], f32)
        elif kind == 3:                                        # negative den: a box of negative width against a small one
            A = np.array([gx, gy, gx - 10, gy + 20], f32)
            B = np.array([gx, gy, gx + 5, gy + 5], f32)
        else:
            dx = w * (1 - t) / (1 + t) + rng.uniform(-2e-4, 2e-4)
            A = np.array([gx, gy, gx + w - 1, gy + h - 1], f32)
            B = np.array([gx + dx, gy, gx + dx + w - 1, gy + h - 1], f32)
        boxes += [A, B]
    b = np.array(boxes, f32)
    order = rng.permutation(len(b))
    b = b[order]
    return np.concatenate([b, np.linspace(1.0, 0.01, len(b)).astype(f32)[:, None]], axis=1)


def _screen_undecided(b, t):
    """(pairs in the +-2^-18 band of the screen, pairs with a denominator outside [2^-62, 2^62)) of the proposal NMS's
    IoU, restated in float64 (the fused area: bw * bh + Sa rounded once)."""
    x = b[:, :4].astype(f32)
    bw, bh = (x[:, 2] - x[:, 0]) + f32(1), (x[:, 3] - x[:, 1]) + f32(1)
    Sa = bw * bh
    i, j = np.triu_indices(len(x), 1)
    w = np.maximum((np.minimum(x[i, 2], x[j, 2]) - np.maximum(x[i, 0], x[j, 0])) + f32(1), f32(0))
    h = np.maximum((np.minimum(x[i, 3], x[j, 3]) - np.maximum(x[i, 1], x[j, 1])) + f32(1), f32(0))
    inter = (w * h).astype(np.float64)
    den = (bw[j].astype(np.float64) * bh[j] + Sa[i]).astype(f32).astype(np.float64) - inter
    out = ~((den >= 2.0 ** -62) & (den < 2.0 ** 62))
    with np.errstate(divide="ignore", invalid="ignore"):
        q = inter / den
    band = ~out & (np.abs(q / t - 1.0) <= 2.0 ** -18)
    return int(band.sum()), int(out.sum())


def test_band_case_reaches_the_exact_fallback():
    for t in (0.3, 0.5, 0.7):
        in_band, out_of_range = _screen_undecided(band_case(t), t)
        assert in_band >= 50 and out_of_range >= 20, (t, in_band, out_of_range)


@pytest.mark.gpu
@pytest.mark.parametrize("t", (0.3, 0.5, 0.7))
def test_nms_threshold_band_pairs(t):
    """Pairs the mask kernel's screen leaves to the exact re-evaluation, through the proposal NMS (nms_gpu,
    ops.nms_batched_raw: CUDA semantics, against oracle/cpu.py) and the Cython flavour (ops.nms_batched_raw(cython=True),
    against oracle/detections.py)."""
    import torch
    from detectron.pytorch_b200 import ops
    from detectron.pytorch_b200.model.nms.nms_gpu import nms_gpu
    from oracle import cpu as OC
    b = band_case(t)
    d = torch.from_numpy(b).cuda()
    assert np.array_equal(nms_gpu(d, t).cpu().numpy().reshape(-1), OC.nms_cuda(b, t))
    parts = [b[:100], b[100:101], b[101:300], b[300:]]
    counts = [len(x) for x in parts]
    off = np.concatenate([[0], np.cumsum(counts)])
    for cython in (False, True):
        keep, num = ops.nms_batched_raw(d, counts, t, cython=cython)
        keep, num = keep.cpu().numpy(), num.cpu().numpy()
        for q, x in enumerate(parts):
            ref = O.nms(x, t) if cython else OC.nms_cuda(x, t)
            assert np.array_equal(keep[off[q]:off[q] + num[q]], ref), (t, cython, q)


def test_detection_batches_validate_on_the_host():
    import ctypes
    from detectron.pytorch_b200 import _lib
    lib = _lib.load()
    counts = (ctypes.c_int * 2)(3, 4)
    assert lib.b200_soft_nms_batched(None, ctypes.cast(counts, ctypes.c_void_p), 2, ctypes.c_float(0.5), ctypes.c_float(0.3),
                                     ctypes.c_float(0.001), 1, None, None, None) == -1
    assert lib.b200_box_voting_batched(None, ctypes.cast(counts, ctypes.c_void_p), None, ctypes.cast(counts, ctypes.c_void_p), 2,
                                       ctypes.c_float(0.8), 9, ctypes.c_float(1.0), None, None) == -1
    assert lib.b200_nms_batched_cython(None, ctypes.cast(counts, ctypes.c_void_p), 2, 5, ctypes.c_float(0.5), None, None, None, 0,
                                       None) == -1
