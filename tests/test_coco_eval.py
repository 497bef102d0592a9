"""COCO box, mask and keypoint evaluation: the numpy restatement of COCOeval (oracle/cocoeval.py) against hand-derived answers
on the CPU, and the device evaluators (detectron/pytorch_b200/datasets) against the restatement on the GPU."""
import copy
import os

import numpy as np
import pytest

from oracle import cocoeval as C
from oracle import masks as OM
from oracle import segms as OS
from tests import coco_eval_cases as CC


def _dataset(anns, h=100, w=100, n_images=1, cats=(1,)):
    return {"images": [{"id": i + 1, "height": h, "width": w} for i in range(n_images)],
            "annotations": anns, "categories": [{"id": c, "name": "c%d" % c} for c in cats]}


def _gt(aid, img, box, cat=1, crowd=0, area=None, **kw):
    a = {"id": aid, "image_id": img, "category_id": cat, "iscrowd": crowd, "bbox": list(map(float, box)),
         "area": float(box[2] * box[3] if area is None else area)}
    a.update(kw)
    return a


def _det(img, box, score, cat=1):
    return {"image_id": img, "category_id": cat, "bbox": list(map(float, box)), "score": score}


def _run(ds, res, t="bbox"):
    return CC.oracle_eval(ds, res, t)


# ---- CPU: the restatement on hand-derived answers -------------------------------------------------------------------------
def test_perfect_detection_ap_one():
    ev = _run(_dataset([_gt(1, 1, [10, 10, 40, 40])]), [_det(1, [10, 10, 40, 40], .9)])
    assert np.allclose([ev.stats[0], ev.stats[1], ev.stats[8]], 1.0)               # pr = tp / (tp + fp + eps)


def test_iou_06_gives_three_of_ten_thresholds():
    # det [10, 10, 40, 40] vs gt [10, 10, 40, 24]: i = 40 * 24, u = 1600 -> IoU 0.6
    ev = _run(_dataset([_gt(1, 1, [10, 10, 40, 24])]), [_det(1, [10, 10, 40, 40], .9)])
    assert C.bb_iou([[10, 10, 40, 40]], [[10, 10, 40, 24]], [0])[0, 0] == 0.6
    assert np.isclose(ev.stats[0], 0.3) and np.isclose(ev.stats[1], 1.0) and ev.stats[2] == 0.0


def test_detection_in_crowd_region_is_neither_tp_nor_fp():
    ds = _dataset([_gt(1, 1, [10, 10, 20, 20]), _gt(2, 1, [50, 50, 40, 40], crowd=1)])
    ev = _run(ds, [_det(1, [10, 10, 20, 20], .5), _det(1, [55, 55, 10, 10], .9)])
    assert np.isclose(ev.stats[0], 1.0)                                   # the crowd det (higher score) is ignored


def test_gt_outside_area_range_makes_its_match_ignored():
    # areas 2500 (medium) and 100 (small); the detection on the out-of-range gt always has the higher score, so counting it
    # as a false positive would halve the precision at full recall
    ds = _dataset([_gt(1, 1, [0, 0, 50, 50]), _gt(2, 1, [60, 60, 10, 10])])
    ev = _run(ds, [_det(1, [0, 0, 50, 50], .8), _det(1, [60, 60, 10, 10], .9)])
    assert np.allclose(ev.eval["precision"][:, :, 0, 2, 2], 1.0)           # medium: the small det matched an ignored gt
    ev = _run(ds, [_det(1, [0, 0, 50, 50], .9), _det(1, [60, 60, 10, 10], .8)])
    assert np.allclose(ev.eval["precision"][:, :, 0, 1, 2], 1.0)           # small: the medium det matched an ignored gt
    ev = _run(_dataset([_gt(1, 1, [60, 60, 10, 10])]), [_det(1, [0, 0, 50, 50], .9), _det(1, [60, 60, 10, 10], .8)])
    assert np.allclose(ev.eval["precision"][:, :, 0, 1, 2], 1.0)           # small: an unmatched medium det is ignored too
    assert np.allclose(ev.eval["precision"][:, 0, 0, 0, 2], 0.5)           # all: it is a false positive


def test_tie_scores_across_images_keep_image_order():
    ds = _dataset([_gt(1, 1, [0, 0, 10, 10]), _gt(2, 2, [0, 0, 10, 10])], n_images=2)
    ev = _run(ds, [_det(1, [50, 50, 10, 10], .5), _det(2, [0, 0, 10, 10], .5)])   # image 1's fp before image 2's tp
    assert ev.eval["precision"][0, 0, 0, 0, 2] == 0.5
    assert ev.eval["scores"][0, 0, 0, 0, 2] == 0.5
    ev2 = _run(ds, [_det(2, [0, 0, 10, 10], .5), _det(1, [50, 50, 10, 10], .5)])
    assert ev2.eval["precision"][0, 0, 0, 0, 2] == 0.5                    # results order does not change the image order


def test_category_without_gt_is_minus_one_and_excluded():
    ds = _dataset([_gt(1, 1, [10, 10, 40, 40])], cats=(1, 2))
    ev = _run(ds, [_det(1, [10, 10, 40, 40], .9), _det(1, [10, 10, 40, 40], .9, cat=2)])
    assert np.all(ev.eval["precision"][:, :, 1] == -1) and np.all(ev.eval["recall"][:, 1] == -1)
    assert np.isclose(ev.stats[0], 1.0)


def test_two_polygon_object_is_union():
    a = [10.0, 10.0, 30.0, 10.0, 30.0, 30.0, 10.0, 30.0]
    b = [20.0, 20.0, 40.0, 20.0, 40.0, 40.0, 20.0, 40.0]                   # overlaps a: an even-odd fill would cut a hole
    rles = C.mask.frPyObjects([a, b], 50, 50)
    u = C.mask.merge(rles)
    dense = OM.rle_decode(C.counts_of(u), 50, 50)
    want = np.maximum(OM.rle_decode(OM.rle_fr_poly(a, 50, 50), 50, 50), OM.rle_decode(OM.rle_fr_poly(b, 50, 50), 50, 50))
    assert np.array_equal(dense, want) and dense[25, 25] == 1


def test_oks_zero_visible_uses_expanded_box():
    gt = {"keypoints": [0.0] * 51, "bbox": [10.0, 10.0, 20.0, 20.0], "area": 400.0}
    inside = {"keypoints": [v for _ in range(17) for v in (5.0, 5.0, 1)]}  # inside [-10, 50]: every distance 0
    outside = {"keypoints": [v for _ in range(17) for v in (60.0, 20.0, 1)]}
    o = C.oks([inside, outside], [gt])
    assert o[0, 0] == 1.0
    sig = C.KPT_OKS_SIGMAS
    e = (10.0 ** 2) / ((sig * 2) ** 2) / (400.0 + np.spacing(1)) / 2
    assert o[1, 0] == np.sum(np.exp(-e)) / 17


def test_max_dets_truncation():
    gts = [_gt(i + 1, 1, [i * 9, 0, 8, 8]) for i in range(11)]
    dets = [_det(1, [i * 9, 0, 8, 8], 1.0 - i * .01) for i in range(11)]
    ev = _run(_dataset(gts, w=120), dets)
    assert np.isclose(ev.stats[6], 1 / 11) and np.isclose(ev.stats[7], 10 / 11) and np.isclose(ev.stats[8], 1.0)


def test_restated_rasteriser_and_string_codec():
    rng = np.random.RandomState(3)
    for it in range(60):
        k, h, w = rng.randint(3, 40), rng.randint(5, 60), rng.randint(5, 60)
        xy = rng.uniform(-5, 70, 2 * k)
        if it % 5 == 0:
            xy = np.round(xy)
        assert np.array_equal(OM.rle_decode(OM.rle_fr_poly(xy, h, w), h, w), OM.rle_decode(C.rle_fr_poly(xy, h, w), h, w))
        m = (rng.rand(h, w) > .5).astype(np.uint8)
        assert np.array_equal(C.rle_fr_string(OS.rle_string(OS.rle_counts(m))), OS.rle_counts(m))


def test_rle_iou_equals_dense():
    ds, _, all_segms, _ = CC.make_set(5, n_images=3)
    coco = C.COCO(copy.deepcopy(ds))
    img = ds["images"][0]
    h, w = img["height"], img["width"]
    gts = [coco.annToRLE(a) for a in coco.imgToAnns[img["id"]]]
    crowd = [a["iscrowd"] for a in coco.imgToAnns[img["id"]]]
    dts = [r for cls in all_segms for r in cls[sorted(i["id"] for i in ds["images"]).index(img["id"])]]
    o = C.rle_iou(dts, gts, crowd)
    D = [OM.rle_decode(C.counts_of(r), h, w).astype(bool) for r in dts]
    G = [OM.rle_decode(C.counts_of(r), h, w).astype(bool) for r in gts]
    for d in range(len(D)):
        for g in range(len(G)):
            i = int((D[d] & G[g]).sum())
            u = int(D[d].sum()) if crowd[g] else int((D[d] | G[g]).sum())
            assert o[d, g] == (0.0 if i == 0 else i / u)


# ---- GPU: the device evaluators against the restatement ------------------------------------------------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "coco_eval.npz")
GOLDEN_CASES = ["bbox", "segm", "kp_bbox", "kp_logit", "kp_prob"]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_oracle_equals_reference_goldens(golden, case):
    """The restatement, fed by the restated writers, gives what the unmodified reference evaluator gave over it."""
    ds, ab, asg, ak, t, conf, want = CC.load_golden(golden, case)
    res = CC.results(ds, ab, asg, ak, t, conf or "bbox")
    assert res == want["results"]
    ora = CC.oracle_eval(ds, res, t)
    for k in ("precision", "recall", "scores"):
        assert np.array_equal(ora.eval[k], want[k]), k
    assert np.array_equal(np.asarray(ora.stats), want["stats"])


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_evaluator_inputs_equal_reference_writers(golden, case):
    """The evaluators' host conversion of all_boxes / all_segms / all_keyps equals the results list the reference's writers
    wrote, value for value and in order (no GPU: this is the host side of evaluate_*)."""
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    ds, ab, asg, ak, t, conf, want = CC.load_golden(golden, case)
    jd = J.load_json_dataset("coco_synthetic_val", ds)
    if t == "bbox":
        d = J._box_results(jd, ab)
        assert np.array_equal(d.box, np.array([r["bbox"] for r in want["results"]], np.float64).reshape(-1, 4))
    elif t == "segm":
        d = J._segm_results(jd, ab, asg)
        assert [(s.decode(), list(hw)) for s, hw in d.strings] == [(r["segmentation"]["counts"], r["segmentation"]["size"])
                                                                   for r in want["results"]]
    else:
        d = J._keypoint_results(jd, ab, ak, conf)
        assert np.array_equal(d.keypoints, np.array([r["keypoints"] for r in want["results"]], np.float64).reshape(-1, 17, 3))
    assert d.image_id.tolist() == [r["image_id"] for r in want["results"]]
    assert d.category_id.tolist() == [r["category_id"] for r in want["results"]]
    assert np.array_equal(d.score, np.array([r["score"] for r in want["results"]], np.float64))


def _device_eval(ds, all_boxes, all_segms, all_keyps, t, confidence="bbox"):
    from detectron.pytorch_b200.datasets import coco_eval as DE
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    jd = J.load_json_dataset("coco_synthetic_val", ds)
    if t == "bbox":
        dets = J._box_results(jd, all_boxes)
    elif t == "segm":
        dets = J._segm_results(jd, all_boxes, all_segms)
    else:
        dets = J._keypoint_results(jd, all_boxes, all_keyps, confidence)
    res = DE.evaluate(ds, dets, t)
    res.summarize(out=None)
    return res


def _assert_same(dev, ora, exact=True):
    for key in ("precision", "recall", "scores"):
        a, b = dev.eval[key], ora.eval[key]
        assert a.shape == b.shape and a.dtype == np.float64
        if exact:
            assert np.array_equal(a, b), (key, np.argwhere(a != b)[:5])
        else:
            np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)
    assert np.array_equal(np.asarray(dev.stats), np.asarray(ora.stats))


@pytest.mark.gpu
@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_device_equals_oracle_small(iou_type, seed):
    ds, ab, asg, ak = CC.make_set(seed)
    ora = CC.oracle_eval(ds, CC.results(ds, ab, asg, ak, iou_type), iou_type)
    dev = _device_eval(ds, ab, asg, ak, iou_type)
    _assert_same(dev, ora)


OKS_ULP_TOL = 4e-15                                                       # CUDA exp vs numpy exp: a few ulp of OKS <= 1


def _oks_margins_ok(ora, tol=OKS_ULP_TOL):
    """Precondition for bit-equal keypoint arrays when OKS differs by up to `tol`: no OKS within `tol` of a threshold, and
    in no row two candidates at or above the lowest threshold within `tol` of each other (greedy matching compares them,
    and the later of two equal values wins).  Ties at exactly 1.0 are allowed: here they are detections inside the expanded
    box of persons without visible keypoints, every distance 0 and every term exp(-0) = 1 on both sides (a non-zero distance
    between these float32 coordinates gives e > 5e-16, so exp(-e) < 1 in numpy and in CUDA alike)."""
    thr = ora.params.iouThrs
    for v in ora.ious.values():
        if not len(v):
            continue
        v = np.asarray(v)
        if np.min(np.abs(v[..., None] - thr)) <= tol:
            return False
        for row in v:
            c = np.sort(row[row >= thr[0] - tol])
            c = np.concatenate([c[c < 1.0], c[c == 1.0][:1]])
            if c.size > 1 and np.min(np.diff(c)) <= tol:
                return False
    return True


@pytest.mark.gpu
@pytest.mark.parametrize("confidence", ["bbox", "logit", "prob"])
def test_device_keypoints_within_tolerance(confidence):
    import torch  # noqa: F401
    from detectron.pytorch_b200.datasets import coco_eval as DE  # noqa: F401
    ds, ab, asg, ak = CC.make_set(7, keypoints=True, masks=False)
    res = CC.results(ds, ab, asg, ak, "keypoints", confidence)
    ora = CC.oracle_eval(ds, res, "keypoints")
    assert _oks_margins_ok(ora)
    dev = _device_eval(ds, ab, asg, ak, "keypoints", confidence)
    _assert_same(dev, ora)


@pytest.mark.gpu
def test_device_oks_matrix_within_tolerance():
    import torch
    from detectron.pytorch_b200 import ops
    rng = np.random.RandomState(11)
    D, G = 50, 30
    det = np.stack([rng.uniform(0, 100, (D, 17)), rng.uniform(0, 100, (D, 17)), np.ones((D, 17))], 2)
    v = rng.choice([0, 1, 2], (G, 17))
    v[:5] = 0
    gtk = np.stack([rng.uniform(0, 100, (G, 17)), rng.uniform(0, 100, (G, 17)), v], 2)
    box = np.column_stack([rng.uniform(0, 50, (G, 2)), rng.uniform(5, 50, (G, 2))])
    area = rng.uniform(10, 5000, G)
    want = C.oks([{"keypoints": d.reshape(-1).tolist()} for d in det],
                 [{"keypoints": g.reshape(-1).tolist(), "bbox": b.tolist(), "area": a} for g, b, a in zip(gtk, box, area)])
    cu = lambda a, dt=torch.float64: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)  # noqa: E731
    ious = torch.empty(D * G, dtype=torch.float64, device="cuda")
    ops.coco_oks_raw((C.KPT_OKS_SIGMAS * 2) ** 2, cu([0, G], torch.int32), cu([0, D], torch.int32), cu([0], torch.int64),
                     cu(np.arange(D), torch.int32), cu(det), cu(gtk), cu(box), cu(area), ious)
    got = ious.cpu().numpy().reshape(D, G)
    np.testing.assert_allclose(got, want, rtol=0, atol=OKS_ULP_TOL)


@pytest.mark.gpu
def test_device_empty_results_and_edge_images():
    ds, ab, asg, ak = CC.make_set(3)
    empty = [[[] for _ in cls] for cls in ab]
    for t in ("bbox", "segm"):
        dev = _device_eval(ds, empty, [[[] for _ in cls] for cls in asg], ak, t)
        k_has = np.array([any(a["category_id"] == c["id"] for a in ds["annotations"])
                          for c in sorted(ds["categories"], key=lambda c: c["id"])])
        assert np.all(dev.eval["precision"][:, :, k_has, 0] == 0) and np.all(dev.eval["precision"][:, :, ~k_has] == -1)
        assert np.all(dev.eval["recall"][:, k_has, 0] == 0)


@pytest.mark.gpu
def test_evaluate_all_result_layout(tmp_path):
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    from detectron.pytorch_b200.datasets import task_evaluation as TE
    ds, ab, asg, ak = CC.make_set(4, keypoints=True)
    jd = J.load_json_dataset("coco_synthetic_val", ds)
    out = TE.evaluate_all(jd, ab, asg, ak, str(tmp_path), mask_on=True, keypoints_on=True)
    r = out["coco_synthetic_val"]
    assert list(r) == ["box", "mask", "keypoint"]
    assert list(r["box"]) == ["AP", "AP50", "AP75", "APs", "APm", "APl"] and list(r["keypoint"]) == ["AP", "AP50", "AP75", "APm", "APl"]
    ora = CC.oracle_eval(ds, CC.results(ds, ab, asg, ak, "bbox"), "bbox")
    assert r["box"]["AP"] == ora.stats[0]
    for f in ("detection_results.pkl", "segmentation_results.pkl", "keypoint_results.pkl"):
        assert (tmp_path / f).exists()


@pytest.mark.gpu
def test_device_equals_oracle_coco_scale():
    import sys
    import time
    ds, ab, asg = CC.coco_scale_set()
    for t in ("bbox", "segm"):
        t0 = time.perf_counter()
        dev = _device_eval(ds, ab, asg, None, t)
        t1 = time.perf_counter()
        sys.stderr.write("coco scale %s: device %.2f s\n" % (t, t1 - t0)); sys.stderr.flush()
        ora = CC.oracle_eval(ds, CC.results(ds, ab, asg, None, t), t)
        sys.stderr.write("coco scale %s: oracle %.2f s\n" % (t, time.perf_counter() - t1)); sys.stderr.flush()
        _assert_same(dev, ora)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_device_equals_reference_goldens(golden, case):
    ds, ab, asg, ak, t, conf, want = CC.load_golden(golden, case)
    if t == "keypoints":                                                   # CUDA's exp: bit-equal only away from ties
        assert _oks_margins_ok(CC.oracle_eval(ds, CC.results(ds, ab, asg, ak, t, conf), t))
    dev = _device_eval(ds, ab, asg, ak, t, conf or "bbox")
    for k in ("precision", "recall", "scores"):
        assert np.array_equal(dev.eval[k], want[k]), (k, np.argwhere(dev.eval[k] != want[k])[:5])
    assert np.array_equal(np.asarray(dev.stats), want["stats"])


@pytest.mark.gpu
def test_device_masks_in_several_chunks(monkeypatch):
    """A bitmap budget of a few images per chunk gives the same arrays as one chunk."""
    from detectron.pytorch_b200.datasets import coco_eval as DE
    ds, ab, asg, ak = CC.make_set(9, n_images=16)
    one = _device_eval(ds, ab, asg, ak, "segm")
    monkeypatch.setattr(DE, "MASK_CHUNK_WORDS", 40 * 200 * 200 // 32)
    many = _device_eval(ds, ab, asg, ak, "segm")
    _assert_same(many, one)
    _assert_same(many, CC.oracle_eval(ds, CC.results(ds, ab, asg, ak, "segm"), "segm"))
