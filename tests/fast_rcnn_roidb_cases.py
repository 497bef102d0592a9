"""Seeded inputs of the Fast R-CNN roidb tests (json_dataset._add_gt_annotations / _merge_proposal_boxes_into_roidb /
_add_class_assignments, roi_data.fast_rcnn._sample_rois) -- inputs only, expected values come from the golden file
tests/golden/fast_rcnn_roidb.npz and from oracle/targets.py.

Every image keeps x >= RESERVED_X free of random ground truth, so that the special boxes placed there have exactly the
overlaps their comments state:
  * CROWD_BOX, the first crowd object of an image: proposals jittered around it overlap it and nothing else;
  * EDGE_BOX, a 100 x 100 ground-truth box (+1 convention), and EDGE_PROPOSALS, at IoU exactly 0.5, just below 0.5, 0.49,
    exactly 0.6, exactly 0.1, sharing one pixel column (iw = 1), one pixel apart (iw = 0), zero width, zero height, and far
    from everything (IoU 0).
Identical ground-truth boxes (`dups`) carry different classes, and every group gets a proposal equal to it: the reference
gives each ground-truth row its own class, a proposal the first maximum.
"""
import numpy as np

from oracle.targets import bbox_overlaps

IM_W, IM_H = 1333.0, 800.0
RESERVED_X = 1050.0
CROWD_BOX = (1100.0, 400.0, 1299.0, 599.0)
EDGE_BOX = (1100.0, 100.0, 1199.0, 199.0)
EDGE_PROPOSALS = ((1100.0, 100.0, 1199.0, 149.0),              # 100 x 50: IoU exactly 0.5
                  (1100.0, 100.0, 1199.0, 149.0 - 1 / 64.0),   # IoU 0.49984375, just below 0.5
                  (1100.0, 100.0, 1199.0, 148.0),              # IoU 0.49
                  (1100.0, 100.0, 1199.0, 159.0),              # IoU float32(0.6): fg at FG_THRESH 0.6
                  (1100.0, 100.0, 1199.0, 109.0),              # IoU float32(0.1): bg at BG_THRESH_LO 0.1
                  (1199.0, 100.0, 1260.0, 199.0),              # shares the column x = 1199: iw = 1
                  (1200.0, 100.0, 1260.0, 199.0),              # one pixel to the right: iw = 0, IoU 0
                  (1150.0, 120.0, 1150.0, 160.0),              # zero width, inside EDGE_BOX
                  (1120.0, 150.0, 1180.0, 150.0),              # zero height, inside EDGE_BOX
                  (1250.0, 250.0, 1320.0, 300.0))              # touches nothing
# (FG_THRESH, BG_THRESH_HI, BG_THRESH_LO): the defaults, and a gap between background and foreground
SETTINGS = {"std": (0.5, 0.5, 0.0), "gap": (0.6, 0.5, 0.1)}
BBOX_REG_WEIGHTS = (10.0, 10.0, 5.0, 5.0)

# name: (seed, kind, G, roidb rows, NUM_CLASSES, CLS_AGNOSTIC_BBOX_REG, BATCH_SIZE_PER_IM, setting, im_scale, batch_idx)
#   kind "mixed": crowd objects, identical gt boxes, EDGE_BOX and its proposals, jittered and random proposals
#   kind "crowd_only": one crowd object and proposals around it; "no_fg": crowd objects only, proposals below IoU 0.5;
#   "no_bg": every proposal at IoU >= 0.6; "empty": crowd objects only, proposals at IoU 0 or in [0.5, 0.6) (nothing is
#   sampled with the "gap" setting), or no proposal at all
CASES = {
    "mixed_std":      (1, "mixed", 10, 400, 81, False, 64, "std", 1.6666666, 0),
    "mixed_gap":      (1, "mixed", 10, 400, 81, False, 64, "gap", 0.8, 3),
    "mixed_agnostic": (2, "mixed", 10, 400, 81, True, 128, "gap", 1.6666666, 3),
    "few_fg":         (3, "mixed", 8, 300, 81, False, 1024, "std", 0.8, 0),
    "crowd_only_std": (4, "crowd_only", 1, 60, 81, False, 64, "std", 1.6666666, 3),
    "crowd_only_gap": (4, "crowd_only", 1, 60, 81, False, 64, "gap", 0.8, 0),
    "no_fg":          (5, "no_fg", 3, 200, 81, False, 128, "gap", 0.8, 3),
    "no_bg":          (6, "no_bg", 5, 150, 81, False, 512, "std", 1.6666666, 0),
    "empty_gap":      (7, "empty", 2, 120, 81, False, 128, "gap", 0.8, 3),
    "empty_no_props": (8, "empty", 2, 2, 81, False, 128, "std", 1.6666666, 0),
    "g300":           (9, "mixed", 300, 1800, 81, False, 512, "std", 0.8, 3),
    "g600":           (10, "mixed", 600, 2600, 81, False, 512, "gap", 1.6666666, 0),
    "rows1023":       (11, "mixed", 23, 1023, 81, False, 512, "gap", 0.8, 0),
    "rows1024":       (12, "mixed", 24, 1024, 81, True, 512, "std", 1.6666666, 3),
    "rows1025":       (13, "mixed", 25, 1025, 81, False, 512, "gap", 1.6666666, 0),
    "rows4100":       (14, "mixed", 40, 4100, 81, False, 512, "gap", 0.8, 3),
    "c1231":          (15, "mixed", 40, 700, 1231, False, 256, "std", 0.8, 3),
}


def crowd_rows(kind, G):
    if kind in ("crowd_only", "no_fg", "empty"):
        return list(range(G))
    return [1] + list(range(50, G - 1, 97))


def dup_groups(kind, G):
    """Groups of identical ground-truth rows (the first row is the original)."""
    if kind != "mixed":
        return []
    groups = [(0, 2)]
    if G >= 9:
        groups.append((3, 4, 5))
    if G >= 300:
        groups.append((255, 256))                                    # either side of the 256-box tile of roi_assign_kernel
    if G >= 600:
        groups.append((510, 511, 512))
    return groups


def _random_boxes(rng, n, lo, hi, x_max):
    w = np.exp(rng.uniform(np.log(lo), np.log(hi), n)); h = np.exp(rng.uniform(np.log(lo), np.log(hi), n))
    x1 = rng.uniform(0, x_max - w); y1 = rng.uniform(0, IM_H - 1 - h)
    return np.stack([x1, y1, x1 + w, y1 + h], 1).astype(np.float32)


def _jitter(rng, boxes, n, sigma):
    src = rng.randint(0, boxes.shape[0], n)
    wh = boxes[src, 2:] - boxes[src, :2] + 1
    p = boxes[src] + (rng.standard_normal((n, 4)) * np.concatenate([wh, wh], 1) * sigma).astype(np.float32)
    p[:, 0::2] = np.clip(p[:, 0::2], 0, IM_W - 1); p[:, 1::2] = np.clip(p[:, 1::2], 0, IM_H - 1)
    p[:, 2:] = np.maximum(p[:, 2:], p[:, :2])
    return p.astype(np.float32)


def roster(seed, kind, G, num_classes):
    """Ground truth of one image: boxes (G, 4) float32, gt_classes (G,) int32 in [1, num_classes), is_crowd (G,) int32."""
    rng = np.random.RandomState(seed)
    boxes = _random_boxes(rng, G, 24, 400, RESERVED_X - 1)
    classes = rng.randint(1, num_classes, G).astype(np.int32)
    crowd = np.zeros(G, np.int32)
    crowd[crowd_rows(kind, G)] = 1
    boxes[crowd_rows(kind, G)[0]] = CROWD_BOX
    if kind == "mixed":
        boxes[G - 1] = EDGE_BOX
        crowd[G - 1] = 0
    for grp in dup_groups(kind, G):
        boxes[list(grp)] = boxes[grp[0]]
        classes[list(grp)] = rng.choice(np.arange(1, num_classes), len(grp), replace=False)
    return boxes, classes, crowd


def proposals(seed, kind, gt, n):
    """n proposals (unscaled image coordinates) for the ground truth `gt`."""
    rng = np.random.RandomState(seed + 1000)
    if n == 0:
        return np.zeros((0, 4), np.float32)
    if kind == "mixed":
        fixed = [np.asarray(EDGE_PROPOSALS, np.float32)]
        fixed += [gt[grp[0]][None] for grp in dup_groups(kind, gt.shape[0])]            # equal to an identical-gt group
        fixed = np.concatenate(fixed)
        m = n - fixed.shape[0]
        crowd = np.asarray([CROWD_BOX], np.float32)
        parts = [fixed, _jitter(rng, crowd, m // 8, 0.06), _jitter(rng, gt, m // 2, 0.12)]
        parts.append(_random_boxes(rng, n - sum(p.shape[0] for p in parts), 8, 500, IM_W))
        p = np.concatenate(parts)
        return p[rng.permutation(n)]
    # the other kinds keep drawing until n proposals pass their filter
    out, have = [], 0
    while have < n:
        cand = np.concatenate([_jitter(rng, gt, 4 * n, 0.1), _random_boxes(rng, 4 * n, 8, 500, IM_W)])
        cand = cand[rng.permutation(cand.shape[0])]
        mo = bbox_overlaps(cand, gt).max(axis=1)
        keep = {"crowd_only": np.ones(mo.shape, bool), "no_fg": mo < 0.5, "no_bg": mo >= 0.6,
                "empty": (mo == 0) | ((mo >= 0.5) & (mo < 0.6))}[kind]
        if kind == "empty":                                          # both sorts, not only the easy one
            keep &= (mo > 0) | (rng.uniform(size=mo.shape) < 0.2)
        out.append(cand[keep]); have += int(keep.sum())
    return np.concatenate(out)[:n]


def image_case(name):
    """(gt_boxes, gt_classes, is_crowd, proposals, cfg dict) of a per-image case."""
    seed, kind, G, rows, num_classes, agnostic, batch, setting, im_scale, batch_idx = CASES[name]
    gt, classes, crowd = roster(seed, kind, G, num_classes)
    props = proposals(seed, kind, gt, rows - G)
    fg, hi, lo = SETTINGS[setting]
    cfg = dict(NUM_CLASSES=num_classes, CLS_AGNOSTIC_BBOX_REG=agnostic, BATCH_SIZE_PER_IM=batch, FG_FRACTION=0.25, FG_THRESH=fg,
               BG_THRESH_HI=hi, BG_THRESH_LO=lo, BBOX_REG_WEIGHTS=BBOX_REG_WEIGHTS, im_scale=np.float32(im_scale),
               batch_idx=batch_idx)
    return gt, classes, crowd, props, cfg


# Training branch of CollectAndDistributeFpnRpnProposalsOp: two images, RPN levels 2-6, RoI levels 2-5
TRAIN_SCALES = (1.6666666, 0.8)
TRAIN_IM_INFO = ((800.0, 1333.0), (640.0, 1066.0))
TRAIN_G = (9, 12)
TRAIN_PROPOSALS = 700
TRAIN_POST_NMS_TOP_N = 1000
TRAIN_CFG = dict(BATCH_SIZE_PER_IM=128, FG_FRACTION=0.25, FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.0, NUM_CLASSES=81,
                 BBOX_REG_WEIGHTS=BBOX_REG_WEIGHTS, CLS_AGNOSTIC_BBOX_REG=False)
TRAIN_MASK = dict(MASK_ON=True, MRCNN_RESOLUTION=14, CLS_SPECIFIC_MASK=True)
TRAIN_KEYPOINTS = dict(KEYPOINTS_ON=True, HEATMAP_SIZE=56, NUM_KEYPOINTS=17, IMS_PER_BATCH=2)


def train_rosters():
    """Per image (gt boxes, gt_classes, is_crowd, proposals in image coordinates) of the training-branch cases."""
    out = []
    for i, G in enumerate(TRAIN_G):
        gt, classes, crowd = roster(40 + i, "mixed", G, TRAIN_CFG["NUM_CLASSES"])
        out.append((gt, classes, crowd, proposals(40 + i, "mixed", gt, TRAIN_PROPOSALS)))
    return out


def train_rpn_inputs():
    """The RPN outputs of the training-branch cases: rpn_rois_fpn2..6 (scaled, with the image index) and unique scores."""
    rng = np.random.RandomState(17)
    props = np.concatenate([np.hstack([np.full((p.shape[0], 1), i, np.float32), p * np.float32(s)]).astype(np.float32)
                            for i, ((_, _, _, p), s) in enumerate(zip(train_rosters(), TRAIN_SCALES))])
    props = props[rng.permutation(props.shape[0])]
    scores = ((rng.permutation(props.shape[0]) + 0.5) / props.shape[0]).astype(np.float32)
    bounds = np.linspace(0, props.shape[0], 6).astype(int)
    return ([props[bounds[l]:bounds[l + 1]] for l in range(5)], [scores[bounds[l]:bounds[l + 1]].reshape(-1, 1) for l in range(5)])


def train_im_info():
    return np.asarray([[h, w, s] for (h, w), s in zip(TRAIN_IM_INFO, TRAIN_SCALES)], np.float32)
