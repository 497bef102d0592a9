"""Golden Mask R-CNN training mask targets (add_mask_rcnn_blobs), produced by the UNMODIFIED reference code on the CPU.

    python oracle/make_reflib.py                  # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_masks.py      # writes tests/golden/mask_targets.npz

roi_data.mask_rcnn.add_mask_rcnn_blobs runs as it is, with the reference's polys_to_boxes, polys_to_mask_wrt_box and cython
bbox_overlaps.  pycocotools is not installed: utils.segms' `mask_util` is replaced, from outside, by oracle/masks.py's
frPyObjects / decode, the step-by-step restatement of pycocotools' rleFrPoly + decode.  So these goldens pin the reference's
host logic around the rasteriser and the restatement of the rasteriser, not pycocotools' binary itself.

Single-image cases (key prefix "<case>/"): M = 14 and 28, class-specific on and off, an image with no fg.  Their objects cover
multi-polygon objects, crowd objects and a class-0 object (both skipped), two objects with the same tight box (a tied IoU:
the first wins), duplicate vertices (degenerate edges), RoIs narrower than 1 px, polygons reaching outside the RoI and to
negative normalised coordinates, and an fg RoI with zero IoU to every polygon box (it takes object 0, far away).
"train/": CollectAndDistributeFpnRpnProposalsOp.forward in training mode with MODEL.MASK_ON, two images, the npr.choice
draws recorded.
"""
import os
import sys
import types

import numpy as np
import scipy.sparse

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import masks as OM  # noqa: E402
from oracle import refmodel  # noqa: E402

NUM_CLASSES = 81


def star(rng, cx, cy, rx, ry, k):
    a = np.sort(rng.uniform(0, 2 * np.pi, k))
    r = rng.uniform(0.4, 1.0, k)
    return [float(v) for xy in zip(cx + rx * r * np.cos(a), cy + ry * r * np.sin(a)) for v in xy]


def image_case(seed, n_fg=24, n_bg=12):
    """One image: objects (segms, gt_classes, is_crowd), sampled boxes and labels with fg and bg rows interleaved."""
    rng = np.random.RandomState(seed)
    segms, classes, crowd = [], [], []

    def add(polys, cls=None, is_crowd=0):
        segms.append(polys); classes.append(int(rng.randint(1, NUM_CLASSES)) if cls is None else cls); crowd.append(is_crowd)
    add([star(rng, 900, 700, 60, 40, 12)])                                   # object 0: far from most RoIs
    add([star(rng, 150, 120, 50, 40, 9), star(rng, 260, 150, 30, 30, 7)])   # two polygons
    add({"counts": "crowd", "size": [600, 800]}, is_crowd=1)                 # crowd: an RLE, never rasterised
    add([star(rng, 400, 300, 80, 50, 20)], cls=0)                            # class 0: skipped
    tri = [500.0, 100.0, 600.0, 100.0, 550.0, 180.0]
    add([tri])                                                               # objects 4 and 5 have the same tight box (500, 100, 600, 180)
    add([[500.0, 100.0, 600.0, 100.0, 600.0, 180.0, 500.0, 180.0]])
    dup = star(rng, 300, 450, 70, 60, 10)
    dup = dup[:4] + dup[2:4] + dup[2:4] + dup[4:]                            # a vertex repeated three times
    add([dup, [250.0, 400.0, 250.0, 400.0, 262.5, 410.1, 250.0, 420.0]])
    for k in range(5):
        add([star(rng, rng.uniform(50, 750), rng.uniform(50, 550), rng.uniform(10, 90), rng.uniform(10, 90),
                  int(rng.randint(3, 40))) for _ in range(int(rng.randint(1, 4)))])
    boxes = OM.polys_to_boxes([s if isinstance(s, list) else [[0, 0, 1, 0, 1, 1]] for s in segms])
    boxes[2] = (100, 300, 220, 420)                                          # the crowd box
    rows = []
    for i in range(n_fg):
        o = int(rng.choice([1, 4, 6, 7, 8, 9, 10, 11]))
        b = boxes[o] + rng.standard_normal(4).astype(np.float32) * np.float32(12)
        rows.append(b)
    specials = [boxes[4].copy(),                                             # exactly the tied box
                np.asarray([110, 310, 200, 400], np.float32),                # on the crowd box: best non-crowd IoU is 0
                np.asarray([300.2, 440.0, 300.6, 470.0], np.float32),        # narrower than 1 px
                np.asarray([130.0, 100.0, 130.3, 100.4], np.float32),        # narrower than 1 px both ways
                np.asarray([270.0, 420.0, 320.0, 470.0], np.float32),        # part of object 6: polygons reach outside
                np.asarray([700.0, 10.0, 780.0, 60.0], np.float32)]          # zero IoU to every polygon box
    rows[:len(specials)] = specials[:n_fg]
    for i in range(n_bg):
        x, y = rng.uniform(0, 700), rng.uniform(0, 500)
        rows.append(np.asarray([x, y, x + rng.uniform(5, 100), y + rng.uniform(5, 100)], np.float32))
    sampled = np.stack(rows).astype(np.float32)
    labels = np.concatenate([rng.randint(1, NUM_CLASSES, n_fg), np.zeros(n_bg, int)]).astype(np.int32)
    perm = rng.permutation(labels.size)
    return segms, np.asarray(classes, np.int32), np.asarray(crowd, np.int32), sampled[perm], labels[perm]


def pack(segms):
    """Object / polygon tables of every object (crowd RLEs as zero polygons) for storage."""
    poly_begin, coord_begin, coords = [0], [0], []
    for s in segms:
        for p in (s if isinstance(s, list) else []):
            coords += list(p); coord_begin.append(len(coords))
        poly_begin.append(len(coord_begin) - 1)
    return np.asarray(poly_begin, np.int64), np.asarray(coord_begin, np.int64), np.asarray(coords, np.float64)


def main(out_path):
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import utils.segms as segm_utils
    segm_utils.mask_util = types.SimpleNamespace(frPyObjects=OM.frPyObjects, decode=OM.decode)
    import roi_data.mask_rcnn as ref_mask
    gold = {}
    cases = [("m14_cls", 1, 14, True, 24), ("m28_agn", 2, 28, False, 24), ("m28_cls", 3, 28, True, 40), ("nofg", 4, 14, True, 0)]
    for name, seed, M, cls_specific, n_fg in cases:
        segms, classes, crowd, sampled, labels = image_case(seed, n_fg=n_fg)
        cfg.MODEL.NUM_CLASSES = NUM_CLASSES; cfg.MRCNN.RESOLUTION = M; cfg.MRCNN.CLS_SPECIFIC_MASK = cls_specific
        roidb = dict(segms=segms, gt_classes=classes, is_crowd=crowd)
        blobs = dict(labels_int32=labels.copy())
        im_scale = np.float32(1.25)
        ref_mask.add_mask_rcnn_blobs(blobs, sampled.copy(), roidb, im_scale, 1)
        pb, cb, co = pack(segms)
        g = name + "/"
        gold.update({g + "cfg": np.asarray([M, int(cls_specific), NUM_CLASSES], np.int64), g + "im_scale": np.asarray(im_scale),
                     g + "gt_classes": classes, g + "is_crowd": crowd, g + "poly_begin": pb, g + "coord_begin": cb, g + "coords": co,
                     g + "sampled_boxes": sampled, g + "labels_int32": labels})
        for k in ("mask_rois", "roi_has_mask_int32", "masks_int32"):
            gold[g + k] = np.asarray(blobs[k])
        print(name, {k: (np.asarray(blobs[k]).shape, np.asarray(blobs[k]).dtype) for k in ("mask_rois", "roi_has_mask_int32", "masks_int32")})
    gold.update(training_branch(cfg))
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


def training_branch(cfg):
    """The reference's CollectAndDistributeFpnRpnProposalsOp.forward in TRAINING mode with MODEL.MASK_ON: proposals of two
    images spread over five RPN levels, the labels / targets and the mask blobs with their FPN distribution."""
    import numpy.random as npr
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden_targets import make_case
    import modeling.collect_and_distribute_fpn_rpn_proposals as CD
    import roi_data.fast_rcnn as FR
    cfg.FPN.FPN_ON = True; cfg.FPN.MULTILEVEL_ROIS = True; cfg.FPN.MULTILEVEL_RPN = True
    cfg.MODEL.NUM_CLASSES = NUM_CLASSES; cfg.MODEL.MASK_ON = True; cfg.MODEL.KEYPOINTS_ON = False
    cfg.MODEL.CLS_AGNOSTIC_BBOX_REG = False; cfg.MRCNN.RESOLUTION = 14; cfg.MRCNN.CLS_SPECIFIC_MASK = True
    cfg.TRAIN.BATCH_SIZE_PER_IM = 128; cfg.TRAIN.RPN_POST_NMS_TOP_N = 600
    out = {}
    scales = np.asarray([1.5, 1.25], np.float32)
    im_info = torch.from_numpy(np.stack([[800, 1216, scales[0]], [768, 1333, scales[1]]]).astype(np.float32))
    rng = np.random.RandomState(13)
    roidb, all_props = [], []
    for i in range(2):
        gt, gt_classes, prop = make_case(30 + i, 6 + i, 500, NUM_CLASSES, im_w=800.0, im_h=520.0)
        n_gt = gt.shape[0]
        segms = []
        for b in gt:                                                         # one or two polygons inside each box
            cx, cy, rx, ry = (b[0] + b[2]) / 2, (b[1] + b[3]) / 2, (b[2] - b[0]) / 2, (b[3] - b[1]) / 2
            segms.append([star(rng, cx, cy, rx, ry, int(rng.randint(3, 30))) for _ in range(int(rng.randint(1, 3)))])
        gt_overlaps = np.zeros((n_gt, NUM_CLASSES), np.float32); gt_overlaps[np.arange(n_gt), gt_classes] = 1.0
        roidb.append(dict(boxes=gt.copy(), gt_classes=gt_classes.copy(), seg_areas=np.zeros(n_gt, np.float32),
                          gt_overlaps=scipy.sparse.csr_matrix(gt_overlaps), is_crowd=np.zeros(n_gt, bool),
                          box_to_gt_ind_map=np.arange(n_gt, dtype=np.int32), segms=segms))
        all_props.append(np.hstack([np.full((prop.shape[0], 1), i, np.float32), prop * scales[i]]).astype(np.float32))
        pb, cb, co = pack(segms)
        out.update({"train/gt_%d" % i: gt, "train/gt_classes_%d" % i: gt_classes, "train/poly_begin_%d" % i: pb,
                    "train/coord_begin_%d" % i: cb, "train/coords_%d" % i: co})
    props = np.concatenate(all_props)
    props = props[rng.permutation(props.shape[0])]
    scores = ((rng.permutation(props.shape[0]) + 0.5) / props.shape[0]).astype(np.float32)
    bounds = np.linspace(0, props.shape[0], 6).astype(int)
    roi_inputs = [props[bounds[l]:bounds[l + 1]] for l in range(5)]
    score_inputs = [scores[bounds[l]:bounds[l + 1]].reshape(-1, 1) for l in range(5)]
    picks = []
    orig_choice = npr.choice

    def recording_choice(a, size=None, replace=True, p=None):
        sel = orig_choice(a, size=size, replace=replace, p=p)
        pos = {int(v): i for i, v in enumerate(np.asarray(a))}
        picks.append(np.asarray([pos[int(v)] for v in np.atleast_1d(sel)], np.int64))
        return sel
    op = CD.CollectAndDistributeFpnRpnProposalsOp()
    op.train()
    npr.seed(5)
    FR.npr.choice = recording_choice
    try:
        blobs = op.forward(roi_inputs + score_inputs, roidb, im_info)
    finally:
        FR.npr.choice = orig_choice
    assert len(picks) == 4
    for l in range(5):
        out["train/rpn_rois_%d" % l] = roi_inputs[l]; out["train/rpn_probs_%d" % l] = score_inputs[l]
    for i in range(2):
        out["train/fg_choice_%d" % i] = picks[2 * i]; out["train/bg_choice_%d" % i] = picks[2 * i + 1]
    out["train/im_info"] = im_info.numpy()
    for k, v in blobs.items():
        out["train/blob_" + k] = np.asarray(v)
    print("training branch blobs:", {k: np.asarray(v).shape for k, v in blobs.items()})
    return out


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "mask_targets.npz"))
