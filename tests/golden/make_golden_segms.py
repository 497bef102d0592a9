"""Golden run-length encodings of the test-time mask paste, produced by the UNMODIFIED reference function
core.test.segm_results (lib/core/test.py:793-847) on the CPU.

    python oracle/make_reflib.py                  # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_segms.py      # writes tests/golden/segms.npz

pycocotools is not needed: the reference's `mask_util` is replaced, from outside, by a recorder whose encode() stores the
uncompressed column-major counts of the full-image mask it is handed and returns an empty string.  Every case of
tests/segm_cases.py (SEGM_CASES) is recorded twice, with cv2's IPP resize on and off: key "c<case>_ipp<0|1>_counts" holds
the counts of all detections back to back (uint32), "..._offs" the (D + 1,) offsets into them.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402
from tests import segm_cases as cases  # noqa: E402


def _counts(a):
    flat = np.asarray(a).ravel(order="F").astype(np.int8)
    change = np.flatnonzero(np.diff(np.concatenate([[0], flat])))       # positions whose value differs from the previous
    return np.diff(np.concatenate([[0], change, [flat.size]])).astype(np.uint32)


def main(out_path):
    import cv2
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import core.test as ref_test
    recorded = []

    def encode(arr):
        assert arr.ndim == 3 and arr.shape[2] == 1 and arr.dtype == np.uint8
        recorded.append(_counts(arr[:, :, 0]))
        return [{"counts": b""}]

    ref_test.mask_util = types.SimpleNamespace(encode=encode)
    gold = {}
    for k, (seed, im_h, im_w, M, cls_specific) in enumerate(cases.SEGM_CASES):
        cls_boxes, masks, ref_boxes = cases.segm_case(seed, im_h, im_w, M, cls_specific)
        cfg.MODEL.NUM_CLASSES = cases.SEGM_NUM_CLASSES
        cfg.MRCNN.RESOLUTION = M; cfg.MRCNN.CLS_SPECIFIC_MASK = cls_specific; cfg.MRCNN.THRESH_BINARIZE = 0.5
        for ipp in (0, 1):
            cv2.ipp.setUseIPP(bool(ipp))
            del recorded[:]
            segms = ref_test.segm_results(cls_boxes, masks, ref_boxes, im_h, im_w)
            assert len(segms) == cases.SEGM_NUM_CLASSES and len(recorded) == ref_boxes.shape[0]
            gold["c%d_ipp%d_counts" % (k, ipp)] = np.concatenate(recorded)
            gold["c%d_ipp%d_offs" % (k, ipp)] = np.concatenate([[0], np.cumsum([len(r) for r in recorded])]).astype(np.int64)
    cv2.ipp.setUseIPP(True)
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "segms.npz"))
