"""Golden proposal-recall results, produced by the UNMODIFIED reference evaluator on the CPU.

    python tests/golden/make_golden_box_proposals.py      # writes tests/golden/box_proposals.npz (needs a reference checkout)

The reference's json_dataset_evaluator.evaluate_box_proposals and task_evaluation.evaluate_box_proposals run as they are, on the seeded
roidbs of tests/box_proposal_cases.py.  Outside patches only, none of which touches a reference file:
  * utils.cython_bbox / utils.cython_nms: the reference's own .pyx files built with the installed Cython
    (tests/golden/make_golden_proposals.build_cython, with its numpy 2 dtype patch of cython_nms);
  * pycocotools is not installed: `pycocotools.cocoeval` and `pycocotools.coco` are oracle/cocoeval.py's restatement and
    `pycocotools.mask` an empty module (task_evaluation imports the Cityscapes evaluator, which imports it; nothing here calls it);
  * oracle/refmodel.py's import shims for today's torch (core.config's imports).
For every case and threshold set (default, custom) the file stores, per (area name, limit of tests/box_proposal_cases.LIMITS), ar,
recalls, num_pos, gt_overlaps (concatenated, with offsets) and whether the reference raised, and the returned thresholds; and per case
task_evaluation's eight keys and values in order.  tests/box_proposal_cases.load_golden reads a result back.
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import cocoeval as OC  # noqa: E402
from oracle import refmodel  # noqa: E402
from oracle.refpath import reference_dir  # noqa: E402
from tests import box_proposal_cases as BC  # noqa: E402
from tests.golden import make_golden_proposals as MP  # noqa: E402


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def reference_evaluators(tmp):
    ref = reference_dir()
    assert ref is not None, "no reference checkout (set DETECTRON_REFERENCE)"
    MP.build_cython(tmp)
    sys.path.insert(0, tmp)
    import cython_bbox
    import cython_nms
    sys.modules["utils.cython_bbox"] = cython_bbox
    sys.modules["utils.cython_nms"] = cython_nms
    if not hasattr(np, "float"):
        np.float = float
    _stub("pycocotools.cocoeval", COCOeval=OC.COCOeval)
    _stub("pycocotools.coco", COCO=OC.COCO)
    _stub("pycocotools.mask")
    pc = _stub("pycocotools")
    pc.mask, pc.coco, pc.cocoeval = sys.modules["pycocotools.mask"], sys.modules["pycocotools.coco"], sys.modules["pycocotools.cocoeval"]
    refmodel._install_compat()
    sys.path.insert(0, os.path.join(ref, "lib"))
    import utils  # noqa: F401  (the reference's package, so the modules above sit inside it)
    sys.modules["utils"].cython_bbox = cython_bbox
    sys.modules["utils"].cython_nms = cython_nms
    import datasets.json_dataset_evaluator as E
    import datasets.task_evaluation as T
    return E, T


class StubDataset:
    def __init__(self, name):
        self.name = name


def main(out_path):
    gold = {}
    with tempfile.TemporaryDirectory() as tmp:
        E, T = reference_evaluators(tmp)
        for case, make in BC.CASES.items():
            roidb = make()
            for k, v in BC.pack(roidb).items():
                gold[case + "/in/" + k] = v
            for tname, thr in BC.THRESHOLD_SETS.items():
                shape = (len(BC.AREA_NAMES), len(BC.LIMITS))
                raised, ar, num_pos = np.zeros(shape, np.bool_), np.full(shape, np.nan), np.zeros(shape, np.int64)
                recalls, overlaps, thresholds = [], [], None
                for a, area in enumerate(BC.AREA_NAMES):
                    for l, limit in enumerate(BC.LIMITS):
                        try:
                            r = E.evaluate_box_proposals(None, roidb, thresholds=None if thr is None else thr.copy(), area=area, limit=limit)
                        except AssertionError:
                            raised[a, l] = True
                            recalls.append(np.full(len(thr) if thr is not None else 10, np.nan)); overlaps.append(np.zeros(0))
                            continue
                        ar[a, l], num_pos[a, l], thresholds = r["ar"], r["num_pos"], r["thresholds"]
                        recalls.append(r["recalls"]); overlaps.append(r["gt_overlaps"])
                g = "%s/%s/" % (case, tname)
                gold.update({g + "raised": raised, g + "ar": ar, g + "num_pos": num_pos, g + "thresholds": np.asarray(thresholds),
                             g + "recalls": np.stack(recalls).reshape(shape + (-1,)), g + "gt_overlaps": np.concatenate(overlaps),
                             g + "gt_overlaps_begin": np.concatenate([[0], np.cumsum([o.size for o in overlaps])]).astype(np.int64)})
            try:
                res = T.evaluate_box_proposals(StubDataset(case), roidb)[case]["box_proposal"]
                gold[case + "/task/raised"] = np.asarray(False)
                gold[case + "/task/keys"] = np.frombuffer(json.dumps(list(res.keys())).encode(), np.uint8)
                gold[case + "/task/values"] = np.asarray(list(res.values()), np.float64)
            except AssertionError:
                gold[case + "/task/raised"] = np.asarray(True)
            print(case, len(roidb), "images")
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "box_proposals.npz"))
