"""Golden COCO evaluation results, produced by the UNMODIFIED reference evaluator on the CPU.

    python tests/golden/make_golden_coco_eval.py      # writes tests/golden/coco_eval.npz (needs a reference checkout)

The reference's json_dataset_evaluator.evaluate_boxes / evaluate_masks / evaluate_keypoints run as they are: their results
writers (_write_coco_bbox_results_file, _write_coco_segms_results_file, _write_coco_keypoint_results_file) write the JSON file,
_do_*_eval reads it back through `COCO.loadRes`, and _log_detection_eval_metrics / summarize() fill `stats`.  pycocotools is not
installed, so it is replaced from outside: `pycocotools.cocoeval.COCOeval` and the dataset's `COCO` are oracle/cocoeval.py's
restatement.  These goldens therefore pin the reference's glue (the + 1 of xyxy_to_xywh, the class-to-category mapping, the
keypoint score under each KRCNN.KEYPOINT_CONFIDENCE) together with the restatement, not pycocotools' binary.

Other outside shims, none of which touches a reference file:
  * `np.float` (removed in numpy 2; the writers call `.astype(np.float)`) is aliased to `float`;
  * `utils.cython_bbox` / `utils.cython_nms` (imported by utils.boxes, unused by xyxy_to_xywh) are placeholders;
  * oracle/refmodel.py's import shims for today's torch (torch._six and the collections aliases core.config's imports need);
  * the keypoint writer's `kps_score = 0; kps_score += kps_dets[j][score_index, k]` is a float32 sum under numpy 2 (a Python
    int plus an np.float32 scalar stays float32, NEP 50), and json.dump rejects np.float32.  Under numpy 1, the version the
    reference was written for, the sum is float64.  The writer is handed float64 copies of all_keyps (exact widening of the
    float32 values), which gives numpy 1's float64 in-order sum and score; x and y go through float() either way.

Each case stores its inputs (the annotation dict as JSON, the detections as flat arrays with their (class, image) slots), the
results list the reference wrote (as JSON), and `precision`, `recall`, `scores` and `stats`; tests/coco_eval_cases.load_golden
reads a case back.
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
from tests import coco_eval_cases as CC  # noqa: E402

CASES = [  # name, iou type, KEYPOINT_CONFIDENCE, make_set arguments
    ("bbox", "bbox", None, dict(seed=21, n_images=8, n_cats=4, dets_per_image=30)),
    ("segm", "segm", None, dict(seed=22, n_images=8, n_cats=4, dets_per_image=30)),
    ("kp_bbox", "keypoints", "bbox", dict(seed=23, n_images=8, n_cats=2, dets_per_image=25, keypoints=True, masks=False, vertices=(6, 12))),
    ("kp_logit", "keypoints", "logit", dict(seed=24, n_images=8, n_cats=2, dets_per_image=25, keypoints=True, masks=False, vertices=(6, 12))),
    ("kp_prob", "keypoints", "prob", dict(seed=25, n_images=8, n_cats=2, dets_per_image=25, keypoints=True, masks=False, vertices=(6, 12))),
]


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def reference_evaluator():
    ref = reference_dir()
    assert ref is not None, "no reference checkout (set DETECTRON_REFERENCE)"
    if not hasattr(np, "float"):
        np.float = float
    _stub("utils.cython_bbox", bbox_overlaps=None)
    _stub("utils.cython_nms", nms=None, soft_nms=None)
    _stub("pycocotools.cocoeval", COCOeval=OC.COCOeval)
    _stub("pycocotools.coco", COCO=OC.COCO)
    _stub("pycocotools")
    refmodel._install_compat()                                          # torch._six, collections aliases, yaml (core.config needs them)
    sys.path.insert(0, os.path.join(ref, "lib"))
    import utils  # noqa: F401  (the reference's package, so the stubs above sit inside it)
    sys.modules["utils"].cython_bbox = sys.modules["utils.cython_bbox"]
    sys.modules["utils"].cython_nms = sys.modules["utils.cython_nms"]
    from core.config import cfg
    import datasets.json_dataset_evaluator as E
    return E, cfg


class StubJsonDataset:
    """The reference's JsonDataset as its evaluators read it (json_dataset.py:69-80), over the restated COCO."""

    def __init__(self, name, dataset):
        self.name = name
        self.COCO = OC.COCO(dataset)
        category_ids = self.COCO.getCatIds()
        categories = [c["name"] for c in self.COCO.loadCats(category_ids)]
        self.category_to_id_map = dict(zip(categories, category_ids))
        self.classes = ["__background__"] + categories


def _text(s):
    return np.frombuffer(s.encode("utf-8"), np.uint8)


def flatten(per_class, width):
    """all_boxes-style [cls][img] lists -> (rows, slot (n, 2) = (cls, img))."""
    rows, slots = [], []
    for c, imgs in enumerate(per_class):
        for i, v in enumerate(imgs):
            for r in (v if len(v) else []):
                rows.append(np.asarray(r)); slots.append((c, i))
    return (np.stack(rows) if rows else np.zeros((0,) + width, np.float32)), np.asarray(slots, np.int64).reshape(-1, 2)


def main(out_path):
    E, cfg = reference_evaluator()
    gold = {}
    for name, t, conf, kw in CASES:
        ds, ab, asg, ak = CC.make_set(**kw)
        ds_json = json.dumps(ds)
        jd = StubJsonDataset("coco_synthetic_val", json.loads(ds_json))
        with tempfile.TemporaryDirectory() as tmp:
            if t == "bbox":
                ev = E.evaluate_boxes(jd, ab, tmp, use_salt=False)
                res_file = os.path.join(tmp, "bbox_coco_synthetic_val_results.json")
            elif t == "segm":
                ev = E.evaluate_masks(jd, ab, asg, tmp, use_salt=False)
                res_file = os.path.join(tmp, "segmentations_coco_synthetic_val_results.json")
            else:
                cfg.KRCNN.KEYPOINT_CONFIDENCE = conf
                ak64 = [[[np.asarray(k, np.float64) for k in v] for v in imgs] for imgs in ak]
                ev = E.evaluate_keypoints(jd, ab, ak64, tmp, use_salt=False)
                res_file = os.path.join(tmp, "keypoints_coco_synthetic_val_results.json")
            with open(res_file) as f:
                written = f.read()
        boxes, box_slot = flatten(ab, (5,))
        g = name + "/"
        gold.update({g + "iou_type": np.asarray(t), g + "confidence": np.asarray(conf or ""), g + "dataset": _text(ds_json),
                     g + "num_classes": np.asarray(len(ab)), g + "num_images": np.asarray(len(ds["images"])),
                     g + "boxes": boxes.astype(np.float32), g + "box_slot": box_slot, g + "results": _text(written),
                     g + "precision": ev.eval["precision"], g + "recall": ev.eval["recall"], g + "scores": ev.eval["scores"],
                     g + "stats": np.asarray(ev.stats, np.float64)})
        if t == "segm":
            gold[g + "segms"] = _text(json.dumps(asg))
        if t == "keypoints":
            kps, kp_slot = flatten(ak, (4, 17))
            gold[g + "keypoints"] = kps.astype(np.float32); gold[g + "kp_slot"] = kp_slot
        print(name, "stats", np.round(ev.stats, 4))
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "coco_eval.npz"))
