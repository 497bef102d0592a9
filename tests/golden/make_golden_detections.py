"""Golden vectors for the test-time detection post-processing, produced by the UNMODIFIED reference function
core.test.box_results_with_nms_and_limit (with the Cython NMS / soft-NMS built from its .pyx) on the CPU.

    python oracle/make_reflib.py                       # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_detections.py      # writes tests/golden/detections.npz

Inputs are seeded, so only the reference OUTPUTS are stored:
  * tests/cases.py (detection_case, DETECTION_CONFIGS; VOC's 21 classes): key "s<seed>_c<config>_j<class>" holds the (n, 5)
    detections of class j, "s<seed>_c<config>_n" the total kept;
  * tests/detection_cases.py (COCO scale, 201 classes, sparse and empty images, the NMS / voting / per-image-limit
    boundaries): key "<case>_c<config>" holds the detections of classes 1 .. K-1 one after the other, "<case>_c<config>_counts"
    how many each class has; config indexes the case's own list.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402
from tests import cases      # noqa: E402
from tests import detection_cases  # noqa: E402


def main(out_path):
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import core.test as ref_test
    cfg.MODEL.NUM_CLASSES = 21
    cfg.TEST.SCORE_THRESH = 0.05; cfg.TEST.NMS = 0.5; cfg.TEST.DETECTIONS_PER_IM = 100; cfg.TEST.BBOX_VOTE.VOTE_TH = 0.8
    gold = {}
    for seed in cases.DETECTION_SEEDS:
        scores, boxes = cases.detection_case(seed)
        for k, (soft, method, vote, scoring) in enumerate(cases.DETECTION_CONFIGS):
            cfg.TEST.SOFT_NMS.ENABLED = soft; cfg.TEST.SOFT_NMS.METHOD = method
            cfg.TEST.BBOX_VOTE.ENABLED = vote; cfg.TEST.BBOX_VOTE.SCORING_METHOD = scoring
            rs, rb, rc = ref_test.box_results_with_nms_and_limit(scores, boxes)
            assert len(rc) == 21 and rs.shape[0] == rb.shape[0]
            for j in range(1, 21):
                gold["s%d_c%d_j%d" % (seed, k, j)] = np.asarray(rc[j]).reshape(-1, 5)
            gold["s%d_c%d_n" % (seed, k)] = np.array(rs.shape[0], dtype=np.int64)
    for name, (scores, boxes, K, p, configs) in detection_cases.detection_cases().items():
        cfg.MODEL.NUM_CLASSES = K
        cfg.TEST.SCORE_THRESH = p["score_thresh"]; cfg.TEST.NMS = p["nms"]; cfg.TEST.DETECTIONS_PER_IM = p["detections_per_im"]
        cfg.TEST.BBOX_VOTE.VOTE_TH = p["vote_th"]
        for k, (soft, method, vote, scoring) in enumerate(configs):
            cfg.TEST.SOFT_NMS.ENABLED = soft; cfg.TEST.SOFT_NMS.METHOD = method
            cfg.TEST.BBOX_VOTE.ENABLED = vote; cfg.TEST.BBOX_VOTE.SCORING_METHOD = scoring
            rs, rb, rc = ref_test.box_results_with_nms_and_limit(scores, boxes)
            assert len(rc) == K and rs.shape[0] == rb.shape[0]
            per_class = [np.asarray(rc[j], dtype=np.float32).reshape(-1, 5) for j in range(1, K)]
            gold["%s_c%d" % (name, k)] = np.concatenate(per_class, axis=0)
            gold["%s_c%d_counts" % (name, k)] = np.array([len(c) for c in per_class], dtype=np.int64)
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "detections.npz"))
