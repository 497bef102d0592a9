"""Golden PASCAL VOC evaluation results, produced by the UNMODIFIED reference evaluator on the CPU.

    python tests/golden/make_golden_voc_eval.py      # writes tests/golden/voc_eval.npz (needs a reference checkout)

The reference's voc_dataset_evaluator.evaluate_boxes runs as it is: _write_voc_results_files writes one results file per class,
_do_python_eval calls voc_eval per class (annotation cache, file parsing, the per-detection loop, voc_ap) and save_object pickles
{'rec', 'prec', 'ap'}.  Each case is a seeded synthetic set (tests/voc_eval_cases.py) laid out in a temporary VOCdevkit with XML
annotations and an image-set file.  Only outside patches, none of which touches a reference file:
  * voc_eval's module globals get an `open` that opens `.pkl` paths in binary mode (the reference pickles its annotation cache
    into a text-mode file, which Python 3 refuses);
  * the catalog (datasets.dataset_catalog.DATASETS) gets an entry pointing the dataset's DEVKIT_DIR at the temporary devkit;
  * the dataset is a stub with `name`, `classes` and get_roidb() entries holding `image`;
  * for the tie case only, voc_eval's `np` is a proxy whose argsort is stable, so tied scores keep file order (numpy's default
    argsort leaves their order to the numpy build and the CPU);
  * oracle/refmodel.py's import shims for today's torch (core.config imports torch and the collections aliases).
Each case stores its inputs (dataset name, classes, image names, XML texts, all_boxes as flat float32 rows with their (class, image)
slots), the lines the writer wrote per class, the annotation cache's records and rec / prec / ap per class;
tests/voc_eval_cases.load_golden reads a case back.
"""
import builtins
import json
import os
import pickle
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402
from oracle.refpath import reference_dir  # noqa: E402
from tests import voc_eval_cases as VC  # noqa: E402

CASES = [  # name, dataset name, set, stable argsort
    ("voc07", "voc_2007_test", lambda: VC.make_set(31, n_images=14, n_classes=5), False),
    ("voc12", "voc_2012_trainval", lambda: VC.make_set(32, n_images=14, n_classes=5), False),
    ("ties", "voc_2007_trainval", lambda: VC.make_set(33, n_images=14, n_classes=4, ties=True), True),
    ("edge07", "voc_2007_test", lambda: VC.edge_set(34), False),
    ("edge12", "voc_2012_trainval", lambda: VC.edge_set(34), False),
]


def _binary_pkl_open(path, mode="r", *args, **kwargs):
    if str(path).endswith(".pkl") and "b" not in mode:
        mode += "b"
    return builtins.open(path, mode, *args, **kwargs)


class _StableArgsortNumpy:
    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def argsort(a, *args, **kwargs):
        return np.argsort(a, kind="stable")


class StubDataset:
    def __init__(self, name, classes, names):
        self.name, self.classes, self._names = name, classes, names

    def get_roidb(self):
        return [{"image": os.path.join("JPEGImages", n + ".jpg")} for n in self._names]


def reference_evaluator():
    ref = reference_dir()
    assert ref is not None, "no reference checkout (set DETECTRON_REFERENCE)"
    refmodel._install_compat()
    sys.path.insert(0, os.path.join(ref, "lib"))
    import datasets.dataset_catalog as catalog
    import datasets.voc_dataset_evaluator as E
    import datasets.voc_eval as V
    V.open = _binary_pkl_open
    return E, V, catalog


def _text(obj):
    return np.frombuffer(json.dumps(obj).encode("utf-8"), np.uint8)


def main(out_path):
    E, V, catalog = reference_evaluator()
    gold = {}
    for case, ds_name, make, stable in CASES:
        classes, names, recs, ab = make()
        xmls = [VC.xml_text(n, recs[n]) for n in names]
        V.np = _StableArgsortNumpy() if stable else np
        with tempfile.TemporaryDirectory() as tmp:
            devkit = VC.write_devkit(os.path.join(tmp, "VOCdevkit"), ds_name, names, xmls)
            catalog.DATASETS[ds_name] = {catalog.DEVKIT_DIR: devkit}
            out = os.path.join(tmp, "out")
            E.evaluate_boxes(StubDataset(ds_name, classes, names), ab, out, use_salt=False, cleanup=True)
            lines, rec, prec, ap, begin = {}, [], [], [], [0]
            for cls in classes[1:]:
                with open(os.path.join(out, "comp4_det_%s_%s.txt" % (ds_name[9:], cls))) as f:
                    lines[cls] = f.read()
                with open(os.path.join(out, cls + "_pr.pkl"), "rb") as f:
                    r = pickle.load(f)
                rec.append(np.asarray(r["rec"], np.float64)); prec.append(np.asarray(r["prec"], np.float64)); ap.append(float(r["ap"]))
                begin.append(begin[-1] + rec[-1].size)
            with open(os.path.join(devkit, "annotations_cache", ds_name[9:] + "_annots.pkl"), "rb") as f:
                ref_recs = pickle.load(f)
        V.np = np
        rows, slots = [], []
        for c, imgs in enumerate(ab):
            for i, v in enumerate(imgs):
                for r in (v if len(v) else []):
                    rows.append(np.asarray(r)); slots.append((c, i))
        g = case + "/"
        gold.update({g + "dataset_name": np.asarray(ds_name), g + "classes": _text(classes), g + "names": _text(names),
                     g + "xml": _text(xmls), g + "boxes": np.stack(rows).astype(np.float32),
                     g + "box_slot": np.asarray(slots, np.int64).reshape(-1, 2), g + "lines": _text(lines), g + "recs": _text(ref_recs),
                     g + "rec": np.concatenate(rec), g + "prec": np.concatenate(prec), g + "ap": np.asarray(ap, np.float64),
                     g + "curve_begin": np.asarray(begin, np.int64)})
        print(case, ds_name, "AP", np.round(ap, 4))
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "voc_eval.npz"))
