"""Golden C4 training blobs (GenerateProposalLabelsOp, FPN off), produced by the UNMODIFIED reference code on the CPU.

    python oracle/make_reflib.py                            # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_proposal_labels.py      # writes tests/golden/proposal_labels.npz

The reference's modeling.generate_proposal_labels.GenerateProposalLabelsOp runs as it is: json_dataset.add_proposals(...,
crowd_thresh=0) and roi_data.fast_rcnn.add_fast_rcnn_blobs on roidb entries built as json_dataset._add_gt_annotations leaves
them (make_golden_fast_rcnn_roidb.gt_entry).  numpy.random.choice is wrapped from outside only to record the positions it
picks, and utils.segms' `mask_util` is replaced by oracle/masks.py's pycocotools restatement, as in make_golden_masks.py.

Cases (key prefix "<case>/"): see CASES.  Each stores its inputs (rpn_rois, im_info, per image gt / gt_classes / is_crowd,
packed polygons and keypoints), the recorded draws and every output blob ("blob_<name>").
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle import masks as OM  # noqa: E402
from oracle import refmodel  # noqa: E402
from tests import fast_rcnn_roidb_cases as C  # noqa: E402
import make_golden_fast_rcnn_roidb as FG  # noqa: E402
import make_golden_keypoint_targets as KT  # noqa: E402
import make_golden_masks as MM  # noqa: E402

# name -> (roster layout, extra TRAIN / MODEL keys).  "two": the two training-branch images at scales 1.667 and 0.8, their
# proposals interleaved in rpn_rois; "sparse": those two plus an image whose only object is a crowd region away from every
# proposal (no fg; the reference cannot sample an image without ground truth) and an image with ground truth but no proposal.
CASES = {
    "two": ("two", {}),
    "agnostic": ("two", dict(CLS_AGNOSTIC_BBOX_REG=True)),
    "sparse": ("sparse", {}),
    "mask": ("two", C.TRAIN_MASK),
    "kp": ("two", C.TRAIN_KEYPOINTS),
}


def rosters(layout):
    """Per image (gt, classes, crowd, proposals in image coordinates, scale, (h, w))."""
    base = [(gt, cl, cr, p, s, hw) for (gt, cl, cr, p), s, hw in zip(C.train_rosters(), C.TRAIN_SCALES, C.TRAIN_IM_INFO)]
    if layout == "two":
        return base
    rng = np.random.RandomState(31)
    no_gt = (np.asarray([C.CROWD_BOX], np.float32), np.ones(1, np.int32), np.ones(1, bool),
             C._random_boxes(rng, 300, 10, 200, 900).astype(np.float32), 1.25, (750.0, 1000.0))
    gt, cl, cr, _ = C.train_rosters()[0]
    no_props = (gt, cl, cr, np.zeros((0, 4), np.float32), 1.0, (600.0, 1000.0))
    return [base[0], no_gt, base[1], no_props]


def rpn_rois(ros):
    rng = np.random.RandomState(17)
    props = np.concatenate([np.hstack([np.full((p.shape[0], 1), i, np.float32), p * np.float32(s)]).astype(np.float32)
                            for i, (_, _, _, p, s, _) in enumerate(ros)])
    return props[rng.permutation(props.shape[0])]


def main(out_path):
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import torch
    import utils.segms as segm_utils
    import modeling.generate_proposal_labels as GPL
    segm_utils.mask_util = types.SimpleNamespace(frPyObjects=OM.frPyObjects, decode=OM.decode)
    np.random.choice = KT.recording_choice
    gold = {}
    try:
        for name, (layout, extra) in CASES.items():
            ros = rosters(layout)
            t = dict(C.TRAIN_CFG, **{k: v for k, v in extra.items() if k in C.TRAIN_CFG})
            FG.set_train_cfg(cfg, t)
            cfg.FPN.FPN_ON = False; cfg.FPN.MULTILEVEL_ROIS = False; cfg.FPN.MULTILEVEL_RPN = False
            if extra.get("MASK_ON"):
                cfg.MODEL.MASK_ON = True; cfg.MRCNN.RESOLUTION = extra["MRCNN_RESOLUTION"]; cfg.MRCNN.CLS_SPECIFIC_MASK = extra["CLS_SPECIFIC_MASK"]
            if extra.get("KEYPOINTS_ON"):
                cfg.MODEL.KEYPOINTS_ON = True; cfg.KRCNN.HEATMAP_SIZE = extra["HEATMAP_SIZE"]
                cfg.KRCNN.NUM_KEYPOINTS = extra["NUM_KEYPOINTS"]; cfg.TRAIN.IMS_PER_BATCH = extra["IMS_PER_BATCH"]
            rng = np.random.RandomState(23)
            g = name + "/"
            roidb = []
            for i, (gt, cl, cr, _, _, _) in enumerate(ros):
                s = []
                for b, c in zip(gt, cr):
                    cx, cy, rx, ry = (b[0] + b[2]) / 2, (b[1] + b[3]) / 2, (b[2] - b[0]) / 2, (b[3] - b[1]) / 2
                    s.append(dict(FG.CROWD_RLE) if c else
                             [MM.star(rng, cx, cy, rx, ry, int(rng.randint(3, 30))) for _ in range(int(rng.randint(1, 3)))])
                kps = (np.stack([KT.keypoints_in(rng, b, C.TRAIN_KEYPOINTS["NUM_KEYPOINTS"], n_out=2) for b in gt]) if len(gt)
                       else np.zeros((0, 3, C.TRAIN_KEYPOINTS["NUM_KEYPOINTS"]), np.int32))
                pb, cb, co = MM.pack(s)
                gold.update({g + "gt_%d" % i: gt, g + "gt_classes_%d" % i: cl, g + "is_crowd_%d" % i: cr, g + "poly_begin_%d" % i: pb,
                             g + "coord_begin_%d" % i: cb, g + "coords_%d" % i: co, g + "gt_keypoints_%d" % i: kps})
                roidb.append(FG.gt_entry(gt, cl, cr, t["NUM_CLASSES"], segms=s, gt_keypoints=kps))
            rr = rpn_rois(ros)
            im_info = np.asarray([[h, w, s] for (_, _, _, _, s, (h, w)) in ros], np.float32)
            gold.update({g + "rpn_rois": rr, g + "im_info": im_info, g + "num_images": np.int64(len(ros))})
            del KT._picks[:]
            np.random.seed(5)
            blobs = GPL.GenerateProposalLabelsOp().forward(rr, roidb, torch.from_numpy(im_info))
            for i, (fg_c, bg_c, kp_c) in enumerate(FG.split_draws(roidb, t["FG_THRESH"], t["BG_THRESH_HI"], t["BG_THRESH_LO"])):
                gold[g + "fg_choice_%d" % i] = fg_c; gold[g + "bg_choice_%d" % i] = bg_c
                if kp_c is not None:
                    gold[g + "kp_choice_%d" % i] = kp_c
            for k, v in blobs.items():
                gold[g + "blob_" + k] = np.asarray(v)
            print(name, {k: np.asarray(v).shape for k, v in blobs.items()})
    finally:
        np.random.choice = KT._orig_choice
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "proposal_labels.npz"))
