"""Golden Fast R-CNN training targets on crowd objects, identical ground-truth boxes, threshold edges, empty minibatches and
large rosters, produced by the UNMODIFIED reference code on the CPU.

    python oracle/make_reflib.py                           # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_fast_rcnn_roidb.py     # writes tests/golden/fast_rcnn_roidb.npz

Each image's roidb entry is built as json_dataset._add_gt_annotations leaves it (a ground-truth row maps to itself with
overlap 1 for its class, a crowd row has overlap -1 for every class); the reference's own _merge_proposal_boxes_into_roidb,
_add_class_assignments and roi_data.fast_rcnn._sample_rois then run as they are.  numpy.random.choice is wrapped from outside
only to record the positions it picks (make_golden_keypoint_targets.recording_choice, tagged by the calling function); a
draw happens only for a non-empty index set, so an image without fg (bg) candidates has an empty fg (bg) choice.  The inputs
come from tests/fast_rcnn_roidb_cases.py.

Per-image cases (key prefix "<case>/"): fast_rcnn_roidb_cases.CASES.
"train/<call>/": CollectAndDistributeFpnRpnProposalsOp.forward in training mode on one roster of two images with crowd
objects and identical gt boxes, FPN levels 2-6: <call> = "frcn" (Fast R-CNN blobs only), "mask" (MODEL.MASK_ON; crowd
segmentations are RLE stand-ins, as in make_golden_masks.py) and "kp" (MODEL.KEYPOINTS_ON; every object, the crowd ones
included, has keypoints).  matplotlib and pycocotools are absent here: oracle/refmodel.py registers stand-in modules from
outside, and utils.segms' `mask_util` is replaced by oracle/masks.py as in make_golden_masks.py.
"""
import os
import sys
import types

import numpy as np
import scipy.sparse

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle import masks as OM  # noqa: E402
from oracle import refmodel  # noqa: E402
from tests import fast_rcnn_roidb_cases as C  # noqa: E402
import make_golden_keypoint_targets as KT  # noqa: E402
import make_golden_masks as MM  # noqa: E402

CROWD_RLE = {"counts": "crowd", "size": [600, 800]}


def gt_entry(boxes, classes, crowd, num_classes, **extra):
    """A roidb entry as json_dataset._add_gt_annotations leaves it."""
    G = boxes.shape[0]
    ov = np.zeros((G, num_classes), np.float32)
    for i in range(G):
        if crowd[i]:
            ov[i, :] = -1.0
        else:
            ov[i, classes[i]] = 1.0
    return dict(boxes=boxes.astype(np.float32), gt_classes=classes.astype(np.int32), seg_areas=np.zeros(G, np.float32),
                gt_overlaps=scipy.sparse.csr_matrix(ov), is_crowd=np.asarray(crowd, bool), box_to_gt_ind_map=np.arange(G, dtype=np.int32),
                **extra)


def split_draws(entries, fg_thresh, bg_hi, bg_lo):
    """Per image (fg_choice, bg_choice, keypoint choice or None) from the recorded draws: _sample_rois draws fg, then bg,
    each only from a non-empty set; add_keypoint_rcnn_blobs draws after them when it has more candidates than it keeps."""
    picks = list(KT._picks)
    empty = np.zeros(0, np.int64)
    out = []
    for e in entries:
        mo = e["max_overlaps"]
        fg = empty if not (mo >= np.float32(fg_thresh)).any() else picks.pop(0)
        bg = empty if not ((mo < np.float32(bg_hi)) & (mo >= np.float32(bg_lo))).any() else picks.pop(0)
        kp = picks.pop(0) if picks and picks[0][0] == "add_keypoint_rcnn_blobs" else None
        assert not isinstance(fg, tuple) or fg[0] == "_sample_rois"
        assert not isinstance(bg, tuple) or bg[0] == "_sample_rois"
        out.append((fg[1] if isinstance(fg, tuple) else fg, bg[1] if isinstance(bg, tuple) else bg, None if kp is None else kp[1]))
    assert not picks, [f for f, _ in picks]
    return out


def set_train_cfg(cfg, t):
    cfg.MODEL.NUM_CLASSES = t["NUM_CLASSES"]; cfg.MODEL.CLS_AGNOSTIC_BBOX_REG = t["CLS_AGNOSTIC_BBOX_REG"]
    cfg.MODEL.BBOX_REG_WEIGHTS = tuple(t["BBOX_REG_WEIGHTS"])
    cfg.TRAIN.BATCH_SIZE_PER_IM = t["BATCH_SIZE_PER_IM"]; cfg.TRAIN.FG_FRACTION = t["FG_FRACTION"]; cfg.TRAIN.FG_THRESH = t["FG_THRESH"]
    cfg.TRAIN.BG_THRESH_HI = t["BG_THRESH_HI"]; cfg.TRAIN.BG_THRESH_LO = t["BG_THRESH_LO"]
    cfg.MODEL.MASK_ON = False; cfg.MODEL.KEYPOINTS_ON = False


def image_cases(cfg):
    import datasets.json_dataset as JD
    import roi_data.fast_rcnn as FR
    gold = {}
    for name in C.CASES:
        gt, classes, crowd, props, t = C.image_case(name)
        set_train_cfg(cfg, t)
        entry = gt_entry(gt, classes, crowd, t["NUM_CLASSES"])
        JD._merge_proposal_boxes_into_roidb([entry], [props])
        JD._add_class_assignments([entry])
        del KT._picks[:]
        np.random.seed(C.CASES[name][0])
        blobs = FR._sample_rois(entry, t["im_scale"], t["batch_idx"])
        fg_c, bg_c, _ = split_draws([entry], t["FG_THRESH"], t["BG_THRESH_HI"], t["BG_THRESH_LO"])[0]
        g = name + "/"
        gold.update({g + "gt": gt, g + "gt_classes": classes, g + "is_crowd": crowd, g + "prop": props,
                     g + "max_overlaps": entry["max_overlaps"].astype(np.float32), g + "max_classes": entry["max_classes"].astype(np.int32),
                     g + "box_to_gt": entry["box_to_gt_ind_map"].astype(np.int32), g + "fg_choice": fg_c, g + "bg_choice": bg_c})
        for k in ("labels_int32", "rois", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights"):
            gold[g + k] = np.asarray(blobs[k])
        print(name, "rows", entry["boxes"].shape[0], "fg", fg_c.size, "bg", bg_c.size, "targets", blobs["bbox_targets"].shape)
    return gold


def training_branch(cfg):
    import torch
    import modeling.collect_and_distribute_fpn_rpn_proposals as CD
    gold = {}
    rng = np.random.RandomState(23)
    rosters = C.train_rosters()
    segms, kps = [], []
    for i, (gt, classes, crowd, _) in enumerate(rosters):
        s = []
        for b, c in zip(gt, crowd):                                          # one or two polygons inside each box
            cx, cy, rx, ry = (b[0] + b[2]) / 2, (b[1] + b[3]) / 2, (b[2] - b[0]) / 2, (b[3] - b[1]) / 2
            s.append(dict(CROWD_RLE) if c else [MM.star(rng, cx, cy, rx, ry, int(rng.randint(3, 30))) for _ in range(int(rng.randint(1, 3)))])
        segms.append(s)
        kps.append(np.stack([KT.keypoints_in(rng, b, C.TRAIN_KEYPOINTS["NUM_KEYPOINTS"], n_out=2) for b in gt]))
        pb, cb, co = MM.pack(s)
        gold.update({"train/gt_%d" % i: gt, "train/gt_classes_%d" % i: classes, "train/is_crowd_%d" % i: crowd,
                     "train/poly_begin_%d" % i: pb, "train/coord_begin_%d" % i: cb, "train/coords_%d" % i: co,
                     "train/gt_keypoints_%d" % i: kps[i]})
    roi_inputs, score_inputs = C.train_rpn_inputs()
    for l in range(5):
        gold["train/rpn_rois_%d" % l] = roi_inputs[l]; gold["train/rpn_probs_%d" % l] = score_inputs[l]
    im_info = C.train_im_info()
    gold["train/im_info"] = im_info
    t = C.TRAIN_CFG
    for call, extra in (("frcn", {}), ("mask", C.TRAIN_MASK), ("kp", C.TRAIN_KEYPOINTS)):
        set_train_cfg(cfg, t)
        cfg.FPN.FPN_ON = True; cfg.FPN.MULTILEVEL_ROIS = True; cfg.FPN.MULTILEVEL_RPN = True
        cfg.TRAIN.RPN_POST_NMS_TOP_N = C.TRAIN_POST_NMS_TOP_N
        if extra.get("MASK_ON"):
            cfg.MODEL.MASK_ON = True; cfg.MRCNN.RESOLUTION = extra["MRCNN_RESOLUTION"]; cfg.MRCNN.CLS_SPECIFIC_MASK = extra["CLS_SPECIFIC_MASK"]
        if extra.get("KEYPOINTS_ON"):
            cfg.MODEL.KEYPOINTS_ON = True; cfg.KRCNN.HEATMAP_SIZE = extra["HEATMAP_SIZE"]
            cfg.KRCNN.NUM_KEYPOINTS = extra["NUM_KEYPOINTS"]; cfg.TRAIN.IMS_PER_BATCH = extra["IMS_PER_BATCH"]
        roidb = [gt_entry(gt, classes, crowd, t["NUM_CLASSES"], segms=segms[i], gt_keypoints=kps[i])
                 for i, (gt, classes, crowd, _) in enumerate(rosters)]
        op = CD.CollectAndDistributeFpnRpnProposalsOp()
        op.train()
        del KT._picks[:]
        np.random.seed(5)
        blobs = op.forward(roi_inputs + score_inputs, roidb, torch.from_numpy(im_info))
        g = "train/%s/" % call
        for i, (fg_c, bg_c, kp_c) in enumerate(split_draws(roidb, t["FG_THRESH"], t["BG_THRESH_HI"], t["BG_THRESH_LO"])):
            gold[g + "fg_choice_%d" % i] = fg_c; gold[g + "bg_choice_%d" % i] = bg_c
            if kp_c is not None:
                gold[g + "kp_choice_%d" % i] = kp_c
        for k, v in blobs.items():
            gold[g + "blob_" + k] = np.asarray(v)
        print("train", call, {k: np.asarray(v).shape for k, v in blobs.items()})
    return gold


def main(out_path):
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import utils.segms as segm_utils
    segm_utils.mask_util = types.SimpleNamespace(frPyObjects=OM.frPyObjects, decode=OM.decode)
    np.random.choice = KT.recording_choice
    try:
        gold = image_cases(cfg)
        gold.update(training_branch(cfg))
    finally:
        np.random.choice = KT._orig_choice
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "fast_rcnn_roidb.npz"))
