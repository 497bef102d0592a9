"""PASCAL VOC detection AP: the numpy restatement (oracle/voc_eval.py) against hand-derived answers and the reference's goldens on
the CPU, the evaluator's host side against the reference's writer and parser, and the device evaluation
(detectron/pytorch_b200/datasets/voc_eval.py) against the goldens and the restatement on the GPU."""
import os
import pickle
import sys
import types

import numpy as np
import pytest

from oracle import voc_eval as O
from tests import voc_eval_cases as VC

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voc_eval.npz")
GOLDEN_CASES = ["voc07", "voc12", "ties", "edge07", "edge12"]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _same_ap(a, b):
    return float(a) == float(b) or (np.isnan(a) and np.isnan(b))


# ---- CPU: the restatement on hand-derived answers -------------------------------------------------------------------------
def _recs(*objs):
    return {"img": [{"name": "c", "pose": "Unspecified", "truncated": 0, "difficult": d, "bbox": list(b)} for b, d in objs]}


def _lines(*dets):
    return ["img {:.3f} {:.1f} {:.1f} {:.1f} {:.1f}\n".format(s, *b) for b, s in dets]


def test_oracle_iou_exactly_half_is_fp():
    # (10, 10, 29, 19) inside (10, 10, 29, 29): inters 20 * 10 = 200, union 400 + 200 - 200 = 400
    assert O.overlaps(np.array([10., 10., 29., 19.]), np.array([[10., 10., 29., 29.]]))[0] == 0.5
    rec, prec, ap = O.voc_eval(_lines(((10, 10, 29, 19), .9)), _recs(((10, 10, 29, 29), 0)), ["img"], "c")
    assert rec.tolist() == [0.0] and prec.tolist() == [0.0] and ap == 0.0


def test_oracle_match_to_difficult_box_is_neither():
    rec, prec, ap = O.voc_eval(_lines(((10, 10, 29, 29), .9), ((50, 50, 60, 60), .8)),
                               _recs(((10, 10, 29, 29), 1), ((100, 100, 120, 120), 0)), ["img"], "c")
    assert rec.tolist() == [0.0, 0.0] and prec.tolist() == [0.0, 0.0]         # tp 0, fp 0 then 1: 0 / eps, 0 / 1


def test_oracle_two_detections_on_one_box():
    rec, prec, ap = O.voc_eval(_lines(((10, 10, 29, 29), .8), ((11, 10, 29, 29), .9)), _recs(((10, 10, 29, 29), 0)), ["img"], "c")
    assert rec.tolist() == [1.0, 1.0] and prec.tolist() == [1.0, 0.5]          # the higher score claims it


def test_oracle_ap_rules_on_three_points():
    # npos 2, outcomes tp, fp, tp: rec (.5, .5, 1), prec (1, .5, 2/3)
    rec, prec = np.array([.5, .5, 1.]), np.array([1., .5, 2 / 3])
    assert np.isclose(O.average_precision(rec, prec, False), .5 * 1 + .5 * (2 / 3))          # area under the envelope: 5/6
    assert np.isclose(O.average_precision(rec, prec, True), (6 * 1 + 5 * (2 / 3)) / 11)     # t = 0 .. .5 -> 1, .6 .. 1 -> 2/3
    got = O.voc_eval(_lines(((10, 10, 29, 29), .9), ((200, 200, 220, 220), .8), ((40, 40, 59, 59), .7)),
                     _recs(((10, 10, 29, 29), 0), ((40, 40, 59, 59), 0)), ["img"], "c")
    assert np.array_equal(got[0], rec) and np.array_equal(got[1], prec)


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_oracle_equals_reference_goldens(golden, case):
    name, classes, names, xmls, ab, want = VC.load_golden(golden, case)
    for cls in classes[1:]:
        assert O.writer_lines(ab, classes.index(cls), names) == want["lines"][cls].splitlines(keepends=True)
        rec, prec, ap = O.voc_eval(want["lines"][cls].splitlines(), want["recs"], names, cls,
                                   use_07_metric=int(name[4:8]) < 2010)
        wrec, wprec, wap = want["curves"][cls]
        assert _same(rec, wrec) and _same(prec, wprec) and _same_ap(ap, wap), cls


# ---- CPU: the evaluator's host side ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_host_values_equal_reference_writer(golden, case):
    """pack_all_boxes' float64 values equal float() of every line the reference's writer wrote, in the same order."""
    from detectron.pytorch_b200.datasets import voc_eval as V
    name, classes, names, xmls, ab, want = VC.load_golden(golden, case)
    det_class, det_image, score, box = V.pack_all_boxes(ab, list(range(1, len(classes))), len(names))
    lines = [ln for cls in classes[1:] for ln in want["lines"][cls].splitlines()]
    assert len(lines) == score.size
    assert [names[i] for i in det_image] == [ln.split(" ")[0] for ln in lines]
    assert np.array_equal(score, np.array([float(ln.split(" ")[1]) for ln in lines]))
    assert np.array_equal(box, np.array([[float(v) for v in ln.split(" ")[2:]] for ln in lines]))
    counts = [len(want["lines"][cls].splitlines()) for cls in classes[1:]]
    assert np.array_equal(det_class, np.repeat(np.arange(len(counts)), counts))


def test_host_values_other_dtypes_use_writer_formatting():
    from detectron.pytorch_b200.datasets import voc_eval as V
    rng = np.random.RandomState(4)
    for dt in (np.float64, np.float16):
        dets = (np.round(rng.uniform(0, 500, (200, 5)) * 20) / 20).astype(dt)
        dets[:, 4] = rng.uniform(0, 1, 200).astype(dt)
        score, box = V.writer_values(dets[:, 0:4], dets[:, -1])
        for k in range(200):
            line = "{:.3f} {:.1f} {:.1f} {:.1f} {:.1f}".format(dets[k, -1], dets[k, 0] + 1, dets[k, 1] + 1, dets[k, 2] + 1, dets[k, 3] + 1)
            assert [score[k]] + box[k].tolist() == [float(v) for v in line.split(" ")]


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_parse_rec_equals_reference(golden, case, tmp_path):
    from detectron.pytorch_b200.datasets import voc_eval as V
    name, classes, names, xmls, ab, want = VC.load_golden(golden, case)
    for n, text in zip(names, xmls):
        p = tmp_path / (n + ".xml")
        p.write_text(text)
        assert V.parse_rec(str(p)) == want["recs"][n]


def _voc_dataset(tmp_path, classes, names, recs, ds_name="voc_2007_test", image_set_names=None):
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    devkit = VC.write_devkit(str(tmp_path / "VOCdevkit"), ds_name, image_set_names or names, [VC.xml_text(n, recs.get(n, []))
                                                                                              for n in (image_set_names or names)])
    return J.load_json_dataset(ds_name, VC.dataset_dict(classes, names), devkit_path=devkit)


def test_evaluate_boxes_refuses_bad_inputs(tmp_path):
    from detectron.pytorch_b200.datasets import voc_dataset_evaluator as E
    classes, names, recs, ab = VC.make_set(3, n_images=4)
    jd = _voc_dataset(tmp_path / "a", classes, names, recs)
    with pytest.raises(NotImplementedError):
        E.evaluate_boxes(jd, ab, str(tmp_path / "out"), use_matlab=True)
    swapped = [names[1], names[0]] + names[2:]
    jd = _voc_dataset(tmp_path / "b", classes, names, recs, image_set_names=swapped)
    with pytest.raises(ValueError, match="order"):
        E.evaluate_boxes(jd, ab, str(tmp_path / "out"))
    jd = _voc_dataset(tmp_path / "c", classes, names, recs, image_set_names=names + [names[0]])
    with pytest.raises(ValueError, match="duplicate"):
        E.evaluate_boxes(jd, ab, str(tmp_path / "out"))
    assert not (tmp_path / "out").exists()


def test_install_reference_aliases_repoints_voc_eval(monkeypatch):
    import detectron.pytorch_b200 as pkg
    from detectron.pytorch_b200.datasets import voc_eval as V
    ref_eval = types.ModuleType("datasets.voc_eval")
    ref_eval.voc_eval = lambda *a, **k: None
    ref_evaluator = types.ModuleType("datasets.voc_dataset_evaluator")
    ref_evaluator.voc_eval = ref_eval.voc_eval
    ref_pkg = types.ModuleType("datasets")
    ref_pkg.voc_eval, ref_pkg.voc_dataset_evaluator = ref_eval, ref_evaluator
    for m in (ref_pkg, ref_eval, ref_evaluator):
        monkeypatch.setitem(sys.modules, m.__name__, m)
    installed = pkg.install_reference_aliases(voc=True)
    assert "datasets.voc_eval.voc_eval" in installed and "datasets.voc_dataset_evaluator.voc_eval" in installed
    assert ref_eval.voc_eval is V.voc_eval and ref_evaluator.voc_eval is V.voc_eval


def test_class_without_detections_gets_empty_curve():
    """No device work when there is nothing to match: empty rec / prec and AP 0.0 under both rules."""
    from detectron.pytorch_b200.datasets import voc_eval as V
    recs = {"a": [{"name": "c", "pose": "", "truncated": 0, "difficult": 0, "bbox": [1, 1, 5, 5]}]}
    for use_07 in (True, False):
        ((rec, prec, ap),) = V.evaluate_classes(recs, ["a"], ["c"], np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0),
                                                np.zeros((0, 4)), use_07_metric=use_07)
        assert rec.size == 0 and prec.size == 0 and ap == 0.0


# ---- GPU: the device evaluation -------------------------------------------------------------------------------------------
def _read_pr(out_dir, cls):
    with open(os.path.join(out_dir, cls + "_pr.pkl"), "rb") as f:
        return pickle.load(f)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_device_equals_reference_goldens(golden, case, tmp_path):
    from detectron.pytorch_b200.datasets import json_dataset_evaluator as J
    from detectron.pytorch_b200.datasets import voc_dataset_evaluator as E
    name, classes, names, xmls, ab, want = VC.load_golden(golden, case)
    devkit = VC.write_devkit(str(tmp_path / "VOCdevkit"), name, names, xmls)
    jd = J.load_json_dataset(name, VC.dataset_dict(classes, names), devkit_path=devkit)
    assert E.evaluate_boxes(jd, ab, str(tmp_path / "out")) is None
    for cls in classes[1:]:
        r = _read_pr(str(tmp_path / "out"), cls)
        wrec, wprec, wap = want["curves"][cls]
        assert _same(r["rec"], wrec) and _same(r["prec"], wprec) and _same_ap(r["ap"], wap), cls


def _oracle_curves(classes, names, recs, ab):
    """{cls: (rec, prec, ap07, ap_area)} from the restated writer and loop."""
    out = {}
    for c, cls in enumerate(classes[1:], start=1):
        lines = O.writer_lines(ab, c, names)
        rec, prec, _ = O.voc_eval(lines, recs, names, cls)
        out[cls] = (rec, prec, O.average_precision(rec, prec, True), O.average_precision(rec, prec, False))
    return out


def _check_device_against_oracle(classes, names, recs, ab):
    from detectron.pytorch_b200.datasets import voc_eval as V
    want = _oracle_curves(classes, names, recs, ab)
    dets = V.pack_all_boxes(ab, list(range(1, len(classes))), len(names))
    for rule, use_07 in ((2, True), (3, False)):
        got = V.evaluate_classes(recs, names, classes[1:], *dets, use_07_metric=use_07)
        for cls, (rec, prec, ap) in zip(classes[1:], got):
            assert _same(rec, want[cls][0]) and _same(prec, want[cls][1]) and _same_ap(ap, want[cls][rule]), (cls, use_07)


@pytest.mark.gpu
def test_device_equals_oracle_voc2007_test_scale():
    classes, names, recs, ab = VC.scale_set()
    assert len(names) == 4952 and len(classes) == 21
    assert sum(len(a) for cls in ab for a in cls) == 4952 * 100
    assert any(o["difficult"] for objs in recs.values() for o in objs)
    _check_device_against_oracle(classes, names, recs, ab)


@pytest.mark.gpu
def test_device_equals_oracle_one_class_long_curve():
    classes, names, recs, ab = VC.make_set(11, n_images=3000, n_classes=1, objs_per_image=4.0, dets_per_image=20, ties=True)
    assert sum(len(v) for v in recs.values()) > 10000
    _check_device_against_oracle(classes, names, recs, ab)


@pytest.mark.gpu
def test_file_voc_eval_equals_evaluate_boxes(tmp_path):
    from detectron.pytorch_b200.datasets import voc_dataset_evaluator as E
    from detectron.pytorch_b200.datasets import voc_eval as V
    classes, names, recs, ab = VC.make_set(12, n_images=40, n_classes=6, dets_per_image=30, ties=True)
    jd = _voc_dataset(tmp_path, classes, names, recs, ds_name="voc_2012_trainval")
    E.evaluate_boxes(jd, ab, str(tmp_path / "out"))
    info = E.voc_info(jd)
    for c, cls in enumerate(classes[1:], start=1):
        det_file = tmp_path / ("det_%s.txt" % cls)
        det_file.write_text("".join(O.writer_lines(ab, c, names)))
        rec, prec, ap = V.voc_eval(str(tmp_path / "det_{:s}.txt"), info["anno_path"], info["image_set_path"], cls,
                                   str(tmp_path / "cache"))
        r = _read_pr(str(tmp_path / "out"), cls)
        assert _same(rec, r["rec"]) and _same(prec, r["prec"]) and _same_ap(ap, r["ap"]), cls
    assert (tmp_path / "cache" / "trainval_annots.pkl").exists()
