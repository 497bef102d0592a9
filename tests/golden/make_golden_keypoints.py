"""Golden keypoints of the Keypoint R-CNN test-time step, produced by the UNMODIFIED reference function
core.test.keypoint_results (lib/core/test.py:850-866) on the CPU.

    python oracle/make_reflib.py                     # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_keypoints.py     # writes tests/golden/keypoints.npz

The reference's utils.keypoints.heatmaps_to_keypoints and nms_oks are wrapped, from outside, by recorders that call the
originals and keep their results.  Every case of tests/keypoint_cases.py (KEYPOINT_CASES) runs twice, with cv2's IPP on
and off, and the two runs must agree exactly (for 17 channels cv2 never hands the resize to IPP).  Keys per case k:
"c<k>_xy" the (D, 4, 17) xy_preds of all detections, "c<k>_keep" the OKS NMS keep list (cases with NMS_OKS only) and
"c<k>_boxes" cls_boxes[1] after keypoint_results (filtered in place when NMS_OKS is on).

KRCNN.INFERENCE_MIN_SIZE = 0, the reference's default, cannot run on cv2 4.13: the sizes it hands cv2.resize are
np.float32 and cv2 rejects them ("Can't parse 'dsize'").  The cases use 1 instead.  Box sides are clamped to >= 1 before
the minimum applies, so min_size = 1 gives the same heatmap sizes as 0, and the float32 corrections w / map_w are the
same numbers (a float32 divided by an equal int or float32).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402
from tests import keypoint_cases as cases  # noqa: E402


def main(out_path):
    import cv2
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import core.test as ref_test
    kpu = ref_test.keypoint_utils
    h2k, nms = kpu.heatmaps_to_keypoints, kpu.nms_oks
    rec = {}

    def rec_h2k(maps, rois):
        rec["xy"] = h2k(maps, rois)
        return rec["xy"]

    def rec_nms(kp, rois, thresh):
        assert thresh == 0.3
        rec["keep"] = nms(kp, rois, thresh)
        return rec["keep"]

    kpu.heatmaps_to_keypoints, kpu.nms_oks = rec_h2k, rec_nms
    gold = {}
    for k, (seed, D, min_size, nms_oks) in enumerate(cases.KEYPOINT_CASES):
        cfg.MODEL.NUM_CLASSES = cases.KP_NUM_CLASSES
        cfg.KRCNN.NUM_KEYPOINTS = cases.KP_NUM_KEYPOINTS
        cfg.KRCNN.HEATMAP_SIZE = cases.KP_HEATMAP_SIZE
        cfg.KRCNN.INFERENCE_MIN_SIZE = min_size
        cfg.KRCNN.NMS_OKS = nms_oks
        runs = []
        for ipp in (0, 1):
            cv2.ipp.setUseIPP(bool(ipp))
            rec.clear()
            cls_boxes, maps, ref_boxes = cases.keypoint_case(seed, D, min_size, nms_oks)
            cls_keyps = ref_test.keypoint_results(cls_boxes, maps, ref_boxes)
            keep = np.asarray(rec["keep"] if nms_oks else np.arange(D), dtype=np.int64)
            assert len(cls_keyps) == cases.KP_NUM_CLASSES and cls_keyps[0] == []
            assert np.array_equal(np.stack(cls_keyps[1]), rec["xy"][keep])
            runs.append((rec["xy"], keep, cls_boxes[1]))
        for a, b in zip(*runs):
            assert np.array_equal(a, b), "case %d: IPP on and off differ" % k
        xy, keep, boxes = runs[0]
        gold["c%d_xy" % k] = xy
        gold["c%d_boxes" % k] = boxes
        if nms_oks:
            assert 0 < len(keep) < D, "case %d: the OKS NMS should keep some detections and drop others" % k
            gold["c%d_keep" % k] = keep
    cv2.ipp.setUseIPP(True)
    kpu.heatmaps_to_keypoints, kpu.nms_oks = h2k, nms
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "keypoints.npz"))
