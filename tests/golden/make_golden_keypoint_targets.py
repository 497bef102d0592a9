"""Golden Keypoint R-CNN training targets (add_keypoint_rcnn_blobs), produced by the UNMODIFIED reference code on the CPU.

    python oracle/make_reflib.py                          # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_keypoint_targets.py   # writes tests/golden/keypoint_targets.npz

Each image's roidb is built like json_dataset._add_gt_annotations (a ground-truth row maps to itself with overlap 1, a crowd
row has overlap -1) and merged with its proposals by the reference's own _merge_proposal_boxes_into_roidb and
_add_class_assignments; roi_data.keypoint_rcnn.add_keypoint_rcnn_blobs and finalize_keypoint_minibatch then run as they are.
numpy.random.choice is wrapped from outside to record the positions it picks, tagged by the calling function: the keypoint
draw happens only when an image has more candidates than fg_rois_per_image.

Single-image cases (key prefix "<case>/"):
  hs56_k17       HS 56, K 17, no subsampling; keypoints exactly on x1 / y1 / x2 / y2, outside the box, v = 0, 1 and 2;
                 a crowd person with visible keypoints; two identical gt boxes with different keypoints; a zero-width gt box
                 with a keypoint on it and keypoints off it
  hs56_k17_sub   the same image with fg_rois_per_image 16: the keypoint draw
  hs64_k5        HS 64, K 5
  fg0            FG_THRESH 0: proposals without overlap map to -1, which selects the last person for the candidate test and
                 gives an all -1 keypoint row (weights 0) once selected
  nocand         no visible keypoint anywhere: no candidate, empty blobs
"train/": CollectAndDistributeFpnRpnProposalsOp.forward in training mode with MODEL.KEYPOINTS_ON, two images over five RPN
levels, without crowd objects or duplicated gt boxes; make_golden_fast_rcnn_roidb.py runs the training branch with KEYPOINTS_ON
on both.
"""
import os
import sys

import numpy as np
import scipy.sparse

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402

NUM_CLASSES = 2          # background + person, as the keypoint baselines
_picks = []
_orig_choice = np.random.choice


def recording_choice(a, size=None, replace=True, p=None):
    sel = _orig_choice(a, size=size, replace=replace, p=p)
    pos = {int(v): i for i, v in enumerate(np.asarray(a))}
    _picks.append((sys._getframe(1).f_code.co_name, np.asarray([pos[int(v)] for v in np.atleast_1d(sel)], np.int64)))
    return sel


def keypoints_in(rng, box, K, n_out=0):
    """(3, K) int32: integer keypoints inside the box (some of them outside when n_out > 0), v in {0, 1, 2}."""
    x1, y1, x2, y2 = box
    kx = rng.randint(int(np.ceil(x1)), int(np.floor(x2)) + 1, K)
    ky = rng.randint(int(np.ceil(y1)), int(np.floor(y2)) + 1, K)
    v = rng.choice([0, 1, 2], K, p=[0.3, 0.2, 0.5])
    for k in rng.choice(K, n_out, replace=False):
        kx[k] = int(x2) + rng.randint(2, 40) if rng.rand() < 0.5 else int(x1) - rng.randint(2, 40)
    return np.stack([kx, ky, v]).astype(np.int32)


def gt_entry(boxes, keypoints, crowd):
    """A roidb entry as json_dataset._add_gt_annotations leaves it (every object is a person, class 1)."""
    G = boxes.shape[0]
    ov = np.zeros((G, NUM_CLASSES), np.float32)
    for i in range(G):
        if crowd[i]:
            ov[i, :] = -1.0
        else:
            ov[i, 1] = 1.0
    return dict(boxes=boxes.astype(np.float32), gt_classes=np.ones(G, np.int32), seg_areas=np.zeros(G, np.float32),
                gt_overlaps=scipy.sparse.csr_matrix(ov), is_crowd=np.asarray(crowd, bool), box_to_gt_ind_map=np.arange(G, dtype=np.int32),
                gt_keypoints=keypoints.astype(np.int32), segms=[[] for _ in range(G)])


def proposals_near(rng, boxes, n, sigma=0.15):
    src = rng.randint(0, boxes.shape[0], n)
    wh = np.maximum(boxes[src, 2:] - boxes[src, :2], 4.0)
    p = boxes[src] + rng.standard_normal((n, 4)) * np.concatenate([wh, wh], 1) * sigma
    p[:, 2:] = np.maximum(p[:, 2:], p[:, :2])
    return p.astype(np.float32)


def image_case(seed, K, im_w=1333, im_h=800, n_prop=300, all_hidden=False, far_kp=False):
    """Ground truth (boxes, keypoints, crowd flags) with the special rows of the module docstring, and proposals."""
    rng = np.random.RandomState(seed)
    boxes, kps, crowd = [], [], []
    for _ in range(5):
        x1, y1 = rng.uniform(20, im_w - 300), rng.uniform(20, im_h - 300)
        b = np.asarray([x1, y1, x1 + rng.uniform(40, 280), y1 + rng.uniform(60, 280)], np.float32)
        boxes.append(b); kps.append(keypoints_in(rng, b, K, n_out=2)); crowd.append(0)
    # keypoints exactly on the four edges of box 0 (its corners are integers so that int32 keypoints can reach them)
    boxes[0] = np.round(boxes[0]).astype(np.float32)
    x1, y1, x2, y2 = boxes[0].astype(int)
    on = [(x1, (y1 + y2) // 2, 2), (x2, (y1 + y2) // 2, 1), ((x1 + x2) // 2, y1, 2), ((x1 + x2) // 2, y2, 2), (x2, y2, 2), (x1, y1, 1),
          (x2 + 1, y2, 2), (x1 - 1, y1, 2)]
    for k, (x, y, v) in enumerate(on[:K]):
        kps[0][:, k] = (x, y, v)
    # the crowd person: visible keypoints inside its box
    b = np.asarray([900, 100, 1100, 380], np.float32)
    boxes.append(b); kp = keypoints_in(rng, b, K); kp[2] = 2; kps.append(kp); crowd.append(1)
    # two identical gt boxes, different keypoints
    b = np.asarray([300.5, 450.25, 520.75, 700.5], np.float32)
    for _ in range(2):
        boxes.append(b.copy()); kps.append(keypoints_in(rng, b, K)); crowd.append(0)
    # a zero-width gt box: a keypoint on x1 == x2, the others off it
    b = np.asarray([640, 500, 640, 620], np.float32)
    kp = keypoints_in(rng, np.asarray([600, 500, 680, 620], np.float32), K)
    kp[:, 0] = (640, 560, 2); kp[:, 1 % K] = (641, 530, 2); kp[2] = np.maximum(kp[2], 1)
    boxes.append(b); kps.append(kp); crowd.append(0)
    if far_kp:                                                  # the last person has a visible keypoint far from every box
        kps[-1][:, K - 1] = (1250, 760, 2)
    boxes = np.stack(boxes).astype(np.float32)
    kps = np.stack(kps).astype(np.int32)
    if all_hidden:
        kps[:, 2, :] = 0
    props = proposals_near(rng, boxes, n_prop)
    props = np.concatenate([props, [[1200, 700, 1300, 790], [1240, 750, 1260, 770], [1251, 700, 1300, 790], [1100, 720, 1250, 780]]])
    props[:, 0::2] = np.clip(props[:, 0::2], 0, im_w - 1); props[:, 1::2] = np.clip(props[:, 1::2], 0, im_h - 1)
    return boxes, kps, np.asarray(crowd, np.int32), props.astype(np.float32)


def merged_roidb(boxes, kps, crowd, props):
    import datasets.json_dataset as JD
    entry = gt_entry(boxes, kps, crowd)
    JD._merge_proposal_boxes_into_roidb([entry], [props])
    JD._add_class_assignments([entry])
    return entry


def main(out_path):
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import roi_data.keypoint_rcnn as ref_kp
    gold = {}
    cases = [("hs56_k17", 1, 56, 17, 0.5, 512, {}), ("hs56_k17_sub", 1, 56, 17, 0.5, 16, {}), ("hs64_k5", 2, 64, 5, 0.5, 512, {}),
             ("fg0", 3, 56, 17, 0.0, 512, dict(far_kp=True)), ("nocand", 4, 56, 17, 0.5, 64, dict(all_hidden=True))]
    np.random.choice = recording_choice
    try:
        for name, seed, HS, K, fg_thresh, fg_per_im, kw in cases:
            boxes, kps, crowd, props = image_case(seed, K, **kw)
            entry = merged_roidb(boxes, kps, crowd, props)
            cfg.KRCNN.HEATMAP_SIZE = HS; cfg.KRCNN.NUM_KEYPOINTS = K; cfg.TRAIN.FG_THRESH = fg_thresh
            blobs = {}
            im_scale = np.float32(1.25)
            del _picks[:]
            np.random.seed(seed)
            ref_kp.add_keypoint_rcnn_blobs(blobs, entry, fg_per_im, None, im_scale, 1)
            blobs = {k: [v] for k, v in blobs.items()}
            blobs = {k: np.concatenate(v) for k, v in blobs.items()}
            valid = ref_kp.finalize_keypoint_minibatch(blobs, True)
            kp_picks = [p for f, p in _picks if f == "add_keypoint_rcnn_blobs"]
            g = name + "/"
            gold.update({g + "cfg": np.asarray([HS, K, fg_per_im], np.int64), g + "fg_thresh": np.asarray(fg_thresh, np.float64),
                         g + "im_scale": np.asarray(im_scale), g + "gt_boxes": boxes, g + "gt_keypoints": kps, g + "is_crowd": crowd,
                         g + "boxes": entry["boxes"], g + "max_overlaps": entry["max_overlaps"],
                         g + "box_to_gt_ind_map": entry["box_to_gt_ind_map"], g + "gt_classes": entry["gt_classes"],
                         g + "valid": np.asarray(bool(valid))})
            if kp_picks:
                gold[g + "choice"] = kp_picks[0]
            for k in ("keypoint_rois", "keypoint_locations_int32", "keypoint_weights", "keypoint_loss_normalizer"):
                gold[g + k] = np.asarray(blobs[k])
            print(name, {k: (np.asarray(blobs[k]).shape, np.asarray(blobs[k]).dtype) for k in blobs}, "draw" if kp_picks else "no draw")
        gold.update(training_branch(cfg))
    finally:
        np.random.choice = _orig_choice
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


def training_branch(cfg):
    """The reference's CollectAndDistributeFpnRpnProposalsOp.forward in TRAINING mode with MODEL.KEYPOINTS_ON: proposals of two
    images spread over five RPN levels, the labels / targets and the keypoint blobs with their FPN distribution."""
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden_targets import make_case
    import modeling.collect_and_distribute_fpn_rpn_proposals as CD
    K, HS = 17, 56
    cfg.FPN.FPN_ON = True; cfg.FPN.MULTILEVEL_ROIS = True; cfg.FPN.MULTILEVEL_RPN = True
    cfg.MODEL.NUM_CLASSES = NUM_CLASSES; cfg.MODEL.MASK_ON = False; cfg.MODEL.KEYPOINTS_ON = True
    cfg.MODEL.CLS_AGNOSTIC_BBOX_REG = False; cfg.KRCNN.NUM_KEYPOINTS = K; cfg.KRCNN.HEATMAP_SIZE = HS
    cfg.TRAIN.FG_THRESH = 0.5; cfg.TRAIN.BATCH_SIZE_PER_IM = 128; cfg.TRAIN.RPN_POST_NMS_TOP_N = 600; cfg.TRAIN.IMS_PER_BATCH = 2
    out = {}
    scales = np.asarray([1.5, 1.25], np.float32)
    im_info = torch.from_numpy(np.stack([[800, 1216, scales[0]], [768, 1333, scales[1]]]).astype(np.float32))
    rng = np.random.RandomState(17)
    roidb, all_props = [], []
    for i in range(2):
        gt, _, prop = make_case(40 + i, 6 + i, 500, NUM_CLASSES, im_w=800.0, im_h=520.0)
        kps = np.stack([keypoints_in(rng, b, K, n_out=2) for b in gt])
        roidb.append(gt_entry(gt, kps, np.zeros(gt.shape[0], np.int32)))
        all_props.append(np.hstack([np.full((prop.shape[0], 1), i, np.float32), prop * scales[i]]).astype(np.float32))
        out.update({"train/gt_%d" % i: gt, "train/gt_keypoints_%d" % i: kps})
    props = np.concatenate(all_props)
    props = props[rng.permutation(props.shape[0])]
    scores = ((rng.permutation(props.shape[0]) + 0.5) / props.shape[0]).astype(np.float32)
    bounds = np.linspace(0, props.shape[0], 6).astype(int)
    roi_inputs = [props[bounds[l]:bounds[l + 1]] for l in range(5)]
    score_inputs = [scores[bounds[l]:bounds[l + 1]].reshape(-1, 1) for l in range(5)]
    op = CD.CollectAndDistributeFpnRpnProposalsOp()
    op.train()
    del _picks[:]
    np.random.seed(5)
    blobs = op.forward(roi_inputs + score_inputs, roidb, im_info)
    # per image: the fg draw, the bg draw (_sample_rois), then the keypoint draw when there are more candidates
    per_image = []
    for f, p in _picks:
        if f == "add_keypoint_rcnn_blobs":
            per_image[-1]["kp"] = p
        elif not per_image or "bg" in per_image[-1]:
            per_image.append({"fg": p})
        else:
            per_image[-1]["bg"] = p
    assert len(per_image) == 2 and all("fg" in c and "bg" in c for c in per_image), [f for f, _ in _picks]
    for l in range(5):
        out["train/rpn_rois_%d" % l] = roi_inputs[l]; out["train/rpn_probs_%d" % l] = score_inputs[l]
    for i, c in enumerate(per_image):
        out["train/fg_choice_%d" % i] = c["fg"]; out["train/bg_choice_%d" % i] = c["bg"]
        if "kp" in c:
            out["train/kp_choice_%d" % i] = c["kp"]
    out["train/im_info"] = im_info.numpy()
    for k, v in blobs.items():
        out["train/blob_" + k] = np.asarray(v)
    print("training branch blobs:", {k: np.asarray(v).shape for k, v in blobs.items()},
          "keypoint draws:", [("kp" in c) for c in per_image])
    return out


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "keypoint_targets.npz"))
