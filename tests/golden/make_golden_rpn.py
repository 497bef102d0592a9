"""Golden vectors for the RPN anchor labels and targets (add_rpn_blobs), produced by the UNMODIFIED reference code.

Runs on the CPU and needs a checkout of the reference (found by oracle/refpath.py, $DETECTRON_REFERENCE first):

    python tests/golden/make_golden_rpn.py          # writes tests/golden/rpn.npz

roi_data.rpn.add_rpn_blobs runs as it is, with the reference's generate_anchors, get_field_of_anchors, cython_bbox (the .pyx
built by make_golden_proposals.build_cython) and bbox_transform_inv.  From outside, numpy.random.choice and
numpy.random.randint are wrapped only to RECORD the positions they picked, and _get_rpn_blobs only to mark where each image's
draw begins, so that the device path can be driven with the same draw.  TRAIN.MAX_SIZE is small so the file stays small.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_proposals as MG  # noqa: E402


def entry(h, w, boxes, classes, crowd):
    return dict(height=h, width=w, boxes=np.asarray(boxes, np.float32), gt_classes=np.asarray(classes, np.int32),
                is_crowd=np.asarray(crowd, bool), seg_areas=np.zeros(len(boxes), np.float32),
                box_to_gt_ind_map=np.arange(len(boxes), dtype=np.int32), flipped=False)


def cases():
    rng = np.random.RandomState(7)

    def rand_boxes(n, w, h):
        x1 = rng.uniform(0, w * 0.8, n); y1 = rng.uniform(0, h * 0.8, n)
        bw = rng.uniform(12, w * 0.5, n); bh = rng.uniform(12, h * 0.5, n)
        return np.stack([x1, y1, np.minimum(x1 + bw, w - 1), np.minimum(y1 + bh, h - 1)], 1).astype(np.float32)
    fpn = dict(FPN_ON=True, MULTILEVEL_RPN=True)
    one = dict(FPN_ON=False, MULTILEVEL_RPN=False)
    out = []
    # FPN P2-P6, two images at different scales; crowd and class-0 boxes to filter out; a 44 x 36 box aligned to the P2 grid
    # (x1, y1 = 2 mod 4), so the 4 x 2 square P2 anchors inside it tie for its maximum IoU, 0.646 < RPN_POSITIVE_OVERLAP
    b0 = np.concatenate([rand_boxes(6, 300, 200), [[42, 62, 85, 97], [10, 10, 150, 120], [5, 5, 60, 60]]]).astype(np.float32)
    b1 = rand_boxes(5, 100, 150)
    out.append(("fpn2", fpn, dict(MAX_SIZE=320), [1.0, 1.6],
                [entry(200, 300, b0, [3, 1, 7, 2, 2, 5, 1, 9, 0], [0, 0, 0, 0, 0, 0, 0, 1, 0]), entry(150, 100, b1, [1, 2, 0, 4, 1], [0] * 5)]))
    # a small image with tiny boxes: their best IoU is < 0.3, so the tied anchors are fg AND bg candidates, and with few bg
    # candidates the bg draw relabels some of them 0 while they keep their targets
    tiny = [[20, 20, 22, 22], [60, 30, 63, 33], [40, 70, 42, 71], [10, 50, 70, 90]]
    out.append(("tiny", fpn, dict(MAX_SIZE=128), [1.0], [entry(96, 96, tiny, [1, 1, 1, 2], [0, 0, 0, 0])]))
    # every anchor kept (straddle -1) and a box far outside every anchor: its column maximum is 0, so every anchor is a fg
    # candidate and the fg subsample (> 128) runs
    far = np.concatenate([rand_boxes(3, 200, 160), [[2000, 2000, 2010, 2012]]]).astype(np.float32)
    out.append(("zero", fpn, dict(MAX_SIZE=256, RPN_STRADDLE_THRESH=-1), [1.25], [entry(160, 200, far, [1, 1, 1, 1], [0] * 4)]))
    # single-level RPN (RPN.STRIDE / RPN.SIZES), two images, straddle 0 and a non-default minibatch
    out.append(("single", one, dict(MAX_SIZE=320, RPN_BATCH_SIZE_PER_IM=128), [1.5, 0.8],
                [entry(180, 200, rand_boxes(4, 200, 180), [1, 2, 3, 1], [0, 1, 0, 0]), entry(300, 400, rand_boxes(3, 400, 300), [1, 1, 1], [0] * 3)]))
    # fewer bg candidates than the minibatch wants: no label 0 at all
    out.append(("fewbg", one, dict(MAX_SIZE=192, RPN_BATCH_SIZE_PER_IM=16384, RPN_STRADDLE_THRESH=-1), [1.0],
                [entry(150, 180, rand_boxes(5, 180, 150), [1] * 5, [0] * 5)]))
    return out


def main():
    tmp = tempfile.mkdtemp(prefix="ref_cython_")
    MG.build_cython(tmp)
    cfg = MG.import_reference(tmp)[0]
    import numpy.random as npr
    import roi_data.data_utils as DU
    import roi_data.rpn as RPN
    cfg.RPN.SIZES = (32, 64, 128)
    orig = (npr.choice, npr.randint, RPN._get_rpn_blobs)
    store = {}
    for name, fpn, train, scales, roidb in cases():
        for k, v in fpn.items():
            setattr(cfg.FPN, k, v)
        saved = {k: getattr(cfg.TRAIN, k) for k in train}
        for k, v in train.items():
            setattr(cfg.TRAIN, k, v)
        DU._threadlocal_foa.cache = {}          # get_field_of_anchors memoises per (stride, sizes, ratios), not per MAX_SIZE
        draws = []

        def rec_blobs(*a, **k):
            draws.append([np.zeros(0, np.int64), np.zeros(0, np.int64)])
            return orig[2](*a, **k)

        def rec_choice(a, size=None, replace=True, p=None):
            sel = orig[0](a, size=size, replace=replace, p=p)
            draws[-1][0] = np.searchsorted(np.asarray(a), sel).astype(np.int64)     # a = the ascending fg_inds
            return sel

        def rec_randint(low, high=None, size=None, dtype=int):
            sel = orig[1](low, high, size, dtype)
            draws[-1][1] = np.asarray(sel, np.int64).reshape(-1)
            return sel
        npr.seed(len(name))
        npr.choice, npr.randint, RPN._get_rpn_blobs = rec_choice, rec_randint, rec_blobs
        try:
            names = RPN.get_rpn_blob_names(True)
            blobs = {k: [] for k in names}
            RPN.add_rpn_blobs(blobs, scales, [dict(e) for e in roidb])
        finally:
            npr.choice, npr.randint, RPN._get_rpn_blobs = orig
        for k, v in saved.items():
            setattr(cfg.TRAIN, k, v)
        assert len(draws) == len(roidb)
        p = name + "/"
        store[p + "cfg"] = np.asarray([int(fpn["FPN_ON"]), train.get("MAX_SIZE"), train.get("RPN_STRADDLE_THRESH", 0),
                                       train.get("RPN_BATCH_SIZE_PER_IM", 256)], np.int64)
        store[p + "scales"] = np.asarray(scales, np.float64)
        for i, e in enumerate(roidb):
            for k in ("boxes", "gt_classes", "is_crowd"):
                store[p + "%s_%d" % (k, i)] = e[k]
            store[p + "hw_%d" % i] = np.asarray([e["height"], e["width"]], np.int64)
            store[p + "fg_disable_%d" % i], store[p + "bg_enable_%d" % i] = draws[i]
        for k in names:
            if k != "roidb":
                store[p + "blob_" + k] = np.asarray(blobs[k])
        lab = [np.asarray(blobs[k]) for k in names if k.startswith("rpn_labels")]
        print(name, "images", len(roidb), "disable", [d[0].size for d in draws], "enable", [d[1].size for d in draws],
              "fg", sum(int((x == 1).sum()) for x in lab), "bg", sum(int((x == 0).sum()) for x in lab))
    # the reference's cell anchors at the FPN and single-level shapes (pins roi_data/rpn.py's generate_anchors)
    import modeling.generate_anchors as GA
    for i, (stride, sizes) in enumerate([(4, (32.,)), (8, (64.,)), (64, (512.,)), (16, (32, 64, 128)), (16, (64, 128, 256, 512)),
                                         (8, (17, 33))]):
        store["anchors/%d/stride" % i] = np.asarray(stride, np.float64)
        store["anchors/%d/sizes" % i] = np.asarray(sizes, np.float64)
        store["anchors/%d/ratios" % i] = np.asarray((0.25, 0.7, 1, 1.5, 3) if i == 5 else (0.5, 1, 2), np.float64)
        store["anchors/%d/out" % i] = GA.generate_anchors(stride, sizes, tuple(store["anchors/%d/ratios" % i]))
    np.savez_compressed(os.path.join(HERE, "rpn.npz"), **store)
    print("wrote", os.path.join(HERE, "rpn.npz"), os.path.getsize(os.path.join(HERE, "rpn.npz")), "bytes")


if __name__ == "__main__":
    main()
