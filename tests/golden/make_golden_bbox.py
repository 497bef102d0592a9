"""Golden vectors for the box head's decode and test-time augmentation, produced by the UNMODIFIED reference functions
core.test.im_detect_bbox / im_detect_bbox_aug / im_detect_all on the CPU with cv2's IPP off.

    python oracle/make_reflib.py                       # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_bbox.py            # writes tests/golden/detect_bbox.npz

The model is tests/bbox_cases.py's record / replay stand-in: its outputs are generated from (seed, call index), so only what
the reference did with them is stored, per case <name>:
  <name>/calls        the model calls in order ("data <shape> <sha256 of the data blob> <rois keys>");
  <name>/c<i>/<key>   im_info and every rois / FPN blob of call i, in full;
  <name>/scores, <name>/boxes, <name>/im_scale   im_detect_bbox_aug's (or, without BBOX_AUG, im_detect_bbox's) result;
  <name>/cls_boxes, <name>/cls_counts            im_detect_all's cls_boxes (MASK_ON off) stacked over classes 1..K-1, and
                                                 the row count of each class (cases with im_detect_all).
Shims applied from outside, for today's numpy / torch and a CPU-only run: np.float / np.int (refmodel), torch.Tensor.cuda as
the identity.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402
from tests import bbox_cases as cases  # noqa: E402


def main(out_path):
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    import cv2
    import torch
    cv2.ipp.setUseIPP(False)
    torch.Tensor.cuda = lambda self, *a, **k: self
    cfg = refmodel.setup(use_b200_ops=False)
    import core.test as ref_test
    gold = {}
    for name, case in sorted(cases.CASES.items()):
        cases.configure(cfg, case)
        im = cases.image(case["seed"])
        props = None if case["faster"] else cases.proposals(case["seed"], case["R"])
        model = cases.ReplayModel(case, to_numpy=lambda t: t.numpy() if torch.is_tensor(t) else t, wrap=torch.from_numpy)
        if cfg.TEST.BBOX_AUG.ENABLED:
            scores, boxes, im_scale, _ = ref_test.im_detect_bbox_aug(model, im, props)
        else:
            scores, boxes, im_scale, _ = ref_test.im_detect_bbox(model, im, cfg.TEST.SCALE, cfg.TEST.MAX_SIZE, props)
        gold[name + "/calls"] = np.array(model.calls)
        for i, blobs in enumerate(model.blobs):
            for k, v in blobs.items():
                gold["%s/c%d/%s" % (name, i, k)] = v
        gold[name + "/scores"] = np.asarray(scores)
        gold[name + "/boxes"] = np.asarray(boxes)
        gold[name + "/im_scale"] = np.asarray(im_scale, dtype=np.float64)
        if case["im_detect_all"]:
            model = cases.ReplayModel(case, to_numpy=lambda t: t.numpy() if torch.is_tensor(t) else t, wrap=torch.from_numpy)
            cls_boxes, _, _ = ref_test.im_detect_all(model, im, props)
            gold[name + "/cls_boxes"] = np.vstack([np.asarray(b, np.float32).reshape(-1, 5) for b in cls_boxes[1:]])
            gold[name + "/cls_counts"] = np.array([len(b) for b in cls_boxes[1:]], dtype=np.int64)
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "detect_bbox.npz"))
