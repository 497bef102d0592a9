"""Fast R-CNN training targets on the roidb the reference builds: crowd objects, identical ground-truth boxes, overlaps at the
thresholds, minibatches without fg, without bg or empty, 300 and 600 gt boxes, 1 023 - 4 100 roidb rows and 1 231 classes.

CPU: the numpy oracle (oracle/targets.py) against the blobs of the UNMODIFIED reference functions
(tests/golden/fast_rcnn_roidb.npz, make_golden_fast_rcnn_roidb.py), bit for bit, and what the golden cases hold.
GPU: roi_data/fast_rcnn.py against the same goldens per image, CollectAndDistributeFpnRpnProposalsOp's training branch
(Fast R-CNN, MASK_ON and KEYPOINTS_ON) against the reference op, the device against the oracle on seeded rosters at the same
sizes, and the device-side draw.  Bit-exact except dw / dh of the regression targets, which agree within 2e-6 relative (CUDA
logf vs numpy's SIMD float32 log)."""
import os

import numpy as np
import pytest
import torch

from oracle import targets as OT
from tests import fast_rcnn_roidb_cases as C

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "fast_rcnn_roidb.npz"))
CASES = list(C.CASES)
BLOBS = ("labels_int32", "rois", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights")
CALLS = {"frcn": {}, "mask": C.TRAIN_MASK, "kp": C.TRAIN_KEYPOINTS}


def case(name):
    g = name + "/"
    gt, classes, crowd, props = GOLD[g + "gt"], GOLD[g + "gt_classes"], GOLD[g + "is_crowd"], GOLD[g + "prop"]
    return dict(gt=gt, classes=classes, crowd=crowd, boxes=np.concatenate([gt, props]).astype(np.float32), cfg=C.image_case(name)[4],
                fg_choice=GOLD[g + "fg_choice"], bg_choice=GOLD[g + "bg_choice"])


def oracle_blobs(p, fg_choice, bg_choice):
    t = p["cfg"]
    return OT.sample_rois(p["boxes"], p["gt"], p["classes"], t["im_scale"], t["batch_idx"], t["NUM_CLASSES"], fg_choice, bg_choice,
                          batch_size_per_im=t["BATCH_SIZE_PER_IM"], fg_fraction=t["FG_FRACTION"], fg_thresh=t["FG_THRESH"],
                          bg_thresh_hi=t["BG_THRESH_HI"], bg_thresh_lo=t["BG_THRESH_LO"], bbox_reg_weights=t["BBOX_REG_WEIGHTS"],
                          cls_agnostic_bbox_reg=t["CLS_AGNOSTIC_BBOX_REG"], is_crowd=p["crowd"])


def assert_targets_close(got, ref):
    assert got.shape == ref.shape and got.dtype == ref.dtype
    assert np.array_equal(got == 0, ref == 0)
    np.testing.assert_allclose(got, ref, rtol=2e-6, atol=1e-7)                # dw, dh: CUDA logf (1 ulp) vs numpy's float32 log
    cols = np.arange(got.shape[1]) % 4 < 2                                    # dx, dy: no transcendental -> exact
    assert np.array_equal(got[:, cols], ref[:, cols])


def assert_blobs_equal(got, ref):
    for k in BLOBS:
        if k == "bbox_targets":
            assert_targets_close(got[k], ref[k])
        else:
            assert got[k].dtype == ref[k].dtype and got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_golden_inputs_are_the_case_builders(name):
    gt, classes, crowd, props, _ = C.image_case(name)
    for k, v in (("gt", gt), ("gt_classes", classes), ("is_crowd", crowd), ("prop", props)):
        assert np.array_equal(GOLD[name + "/" + k], v), k


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_roidb(name):
    p = case(name)
    mo, am, mc = OT.assign_rois(p["boxes"], p["gt"], p["classes"], p["crowd"])
    assert np.array_equal(mo, GOLD[name + "/max_overlaps"])
    assert np.array_equal(am, GOLD[name + "/box_to_gt"])
    assert np.array_equal(mc, GOLD[name + "/max_classes"])
    b = oracle_blobs(p, p["fg_choice"], p["bg_choice"])
    for k in BLOBS:
        ref = GOLD[name + "/" + k]
        assert b[k].dtype == ref.dtype and b[k].shape == ref.shape and np.array_equal(b[k], ref), k


def test_golden_cases_hold_what_they_test():
    """The reference's roidb for the special rows, and the minibatch shapes the case names promise."""
    p = case("mixed_std")
    G = p["gt"].shape[0]
    mo, mc, am = GOLD["mixed_std/max_overlaps"], GOLD["mixed_std/max_classes"], GOLD["mixed_std/box_to_gt"]
    assert (mo[:G][p["crowd"] == 1] == -1).all() and (mc[:G][p["crowd"] == 1] == 0).all()          # crowd rows: -1, class 0
    assert np.array_equal(am[:G], np.arange(G))                                                     # gt rows map to themselves
    assert mc[2] == p["classes"][2] != p["classes"][0]                                             # row 2 == row 0, own class
    props = p["boxes"][G:]
    edge = {tuple(e): G + int(np.where((props == np.float32(e)).all(1))[0][0]) for e in C.EDGE_PROPOSALS}
    assert mo[edge[C.EDGE_PROPOSALS[0]]] == np.float32(0.5) and mo[edge[C.EDGE_PROPOSALS[3]]] == np.float32(0.6)
    assert mo[edge[C.EDGE_PROPOSALS[4]]] == np.float32(0.1) and mo[edge[C.EDGE_PROPOSALS[6]]] == 0
    assert 0 < mo[edge[C.EDGE_PROPOSALS[1]]] < np.float32(0.5) and mo[edge[C.EDGE_PROPOSALS[5]]] > 0
    crowd_fg = (mo[G:] >= 0.5) & (mc[G:] == p["classes"][1]) & (am[G:] == 1)
    assert crowd_fg.any()                                                   # proposals on the crowd box: fg, the crowd's class
    dup = (props == p["gt"][0]).all(1)
    assert dup.any() and (am[G:][dup] == 0).all()                           # a proposal equal to rows 0 and 2: the first
    for name, G in (("g300", 300), ("g600", 600)):
        q = case(name)
        same = np.where((q["boxes"][G:] == q["gt"][255]).all(1))[0]
        assert same.size and (GOLD[name + "/box_to_gt"][G + same] == 255).all()
        assert GOLD[name + "/max_classes"][256] == q["classes"][256] != q["classes"][255]
    q = case("g600")
    same = np.where((q["boxes"][600:] == q["gt"][510]).all(1))[0]
    assert same.size and (GOLD["g600/box_to_gt"][600 + same] == 510).all()
    n = {name: (GOLD[name + "/fg_choice"].size, GOLD[name + "/bg_choice"].size) for name in CASES}
    assert n["few_fg"][0] < int(round(0.25 * C.CASES["few_fg"][6])) and n["few_fg"][0] > 0
    assert n["no_fg"][0] == 0 and n["no_fg"][1] > 0 and n["no_bg"][1] == 0 and n["no_bg"][0] > 0
    for name in ("empty_gap", "empty_no_props"):
        assert GOLD[name + "/labels_int32"].shape == (0,) and GOLD[name + "/bbox_targets"].shape == (0, 4 * 81)
        assert GOLD[name + "/rois"].shape == (0, 5)
    assert GOLD["crowd_only_std/labels_int32"][:n["crowd_only_std"][0]].tolist() == [GOLD["crowd_only_std/gt_classes"][0]] * 16
    assert GOLD["c1231/bbox_targets"].shape[1] == 4924 and GOLD["mixed_agnostic/bbox_targets"].shape[1] == 8
    assert {C.CASES[k][3] for k in CASES} >= {1023, 1024, 1025, 4100}
    for call in CALLS:                                                      # the training branch samples no crowd row either
        lab = GOLD["train/%s/blob_labels_int32" % call]
        assert lab.size == 256 and (lab > 0).any()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def device_blobs(p, fg_choice=None, bg_choice=None):
    from detectron.pytorch_b200.roi_data import fast_rcnn as FR
    t = p["cfg"]
    b = FR.sample_rois(dev(p["boxes"]), dev(p["gt"]), dev(p["classes"]), float(t["im_scale"]), t["batch_idx"], t["NUM_CLASSES"],
                       batch_size_per_im=t["BATCH_SIZE_PER_IM"], fg_fraction=t["FG_FRACTION"], fg_thresh=t["FG_THRESH"],
                       bg_thresh_hi=t["BG_THRESH_HI"], bg_thresh_lo=t["BG_THRESH_LO"], bbox_reg_weights=t["BBOX_REG_WEIGHTS"],
                       cls_agnostic_bbox_reg=t["CLS_AGNOSTIC_BBOX_REG"], fg_choice=fg_choice, bg_choice=bg_choice, is_crowd=p["crowd"])
    return {k: v.cpu().numpy() for k, v in b.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_assignment_vs_reference_roidb(name):
    from detectron.pytorch_b200.roi_data import fast_rcnn as FR
    p = case(name)
    mo, am, mc = FR.roidb_assignment(dev(p["boxes"]), dev(p["gt"]), dev(p["classes"]), dev(p["crowd"]))
    assert np.array_equal(mo.cpu().numpy(), GOLD[name + "/max_overlaps"])
    assert np.array_equal(am.cpu().numpy(), GOLD[name + "/box_to_gt"])
    assert np.array_equal(mc.cpu().numpy(), GOLD[name + "/max_classes"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_sample_rois_vs_reference_blobs(name):
    p = case(name)
    b = device_blobs(p, p["fg_choice"], p["bg_choice"])
    assert_blobs_equal(b, {k: GOLD[name + "/" + k] for k in BLOBS})


def unpack_segms(pb, cb, co, crowd):
    segms = []
    for o in range(pb.size - 1):
        if crowd[o]:
            segms.append({"counts": "crowd", "size": [600, 800]})
        else:
            segms.append([co[cb[q]:cb[q + 1]].tolist() for q in range(pb[o], pb[o + 1])])
    return segms


@pytest.mark.gpu
@pytest.mark.parametrize("call", list(CALLS))
def test_training_branch_vs_reference_op(call):
    """CollectAndDistributeFpnRpnProposalsOp.forward in training mode on two images with crowd objects and identical gt boxes:
    every blob of the reference op -- labels / targets, FPN rois and restore index, mask or keypoint blobs -- with its draws."""
    from detectron.pytorch_b200.modeling.collect_and_distribute_fpn_rpn_proposals import CollectAndDistributeFpnRpnProposalsOp
    g = {k[len("train/"):]: GOLD[k] for k in GOLD.files if k.startswith("train/")}
    inputs = [dev(g["rpn_rois_%d" % l]) for l in range(5)] + [dev(g["rpn_probs_%d" % l]) for l in range(5)]
    roidb = []
    for i in range(2):
        crowd = g["is_crowd_%d" % i]
        roidb.append(dict(boxes=g["gt_%d" % i], gt_classes=g["gt_classes_%d" % i], is_crowd=crowd, gt_keypoints=g["gt_keypoints_%d" % i],
                          segms=unpack_segms(g["poly_begin_%d" % i], g["coord_begin_%d" % i], g["coords_%d" % i], crowd)))
    pre = call + "/"
    choices = [(g[pre + "fg_choice_%d" % i], g[pre + "bg_choice_%d" % i], g.get(pre + "kp_choice_%d" % i)) for i in range(2)]
    op = CollectAndDistributeFpnRpnProposalsOp(rpn_min_level=2, rpn_max_level=6, roi_min_level=2, roi_max_level=5,
                                               post_nms_topN=C.TRAIN_POST_NMS_TOP_N)
    op.train()
    blobs = op(inputs, roidb, g["im_info"], choices=choices, train=dict(C.TRAIN_CFG, **CALLS[call]))
    ref_keys = sorted(k[len(pre + "blob_"):] for k in g if k.startswith(pre + "blob_"))
    assert sorted(k for k in blobs if k != "counts") == ref_keys
    for k in ref_keys:
        got, ref = blobs[k], g[pre + "blob_" + k]
        got = got.cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
        if k == "bbox_targets":
            assert_targets_close(got, ref)
        else:
            assert got.dtype == ref.dtype and got.shape == ref.shape and np.array_equal(got, ref), k


SEEDED = {"g300": (300, 1500, 81, "std"), "g600": (600, 2400, 81, "gap"), "rows1023": (23, 1023, 81, "gap"),
          "rows1024": (24, 1024, 81, "std"), "rows1025": (25, 1025, 81, "gap"), "rows4100": (41, 4100, 81, "gap"),
          "c1231": (40, 700, 1231, "std"), "c1231_agnostic": (40, 700, 1231, "gap")}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SEEDED))
@pytest.mark.parametrize("seed", [101, 202])
def test_device_vs_oracle_seeded(name, seed):
    """Fresh rosters at the golden sizes, the draw from a seeded numpy RandomState, every blob against the oracle."""
    G, rows, ncls, setting = SEEDED[name]
    gt, classes, crowd = C.roster(seed, "mixed", G, ncls)
    props = C.proposals(seed, "mixed", gt, rows - G)
    fg, hi, lo = C.SETTINGS[setting]
    cfg = dict(NUM_CLASSES=ncls, CLS_AGNOSTIC_BBOX_REG=name.endswith("agnostic"), BATCH_SIZE_PER_IM=512, FG_FRACTION=0.25,
               FG_THRESH=fg, BG_THRESH_HI=hi, BG_THRESH_LO=lo, BBOX_REG_WEIGHTS=C.BBOX_REG_WEIGHTS, im_scale=np.float32(0.8), batch_idx=3)
    p = dict(gt=gt, classes=classes, crowd=crowd, boxes=np.concatenate([gt, props]).astype(np.float32), cfg=cfg)
    mo = OT.assign_rois(p["boxes"], gt, classes, crowd)[0]
    nf = int((mo >= np.float32(fg)).sum()); nb = int(((mo < np.float32(hi)) & (mo >= np.float32(lo))).sum())
    rng = np.random.RandomState(seed)
    n_fg = min(128, nf)
    fg_c = rng.permutation(nf)[:n_fg]; bg_c = rng.permutation(nb)[:min(512 - n_fg, nb)]
    got = device_blobs(p, fg_c, bg_c)
    ref = oracle_blobs(p, fg_c, bg_c)
    assert np.array_equal(got["keep_inds"], ref["keep_inds"])
    assert_blobs_equal(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixed_std", "few_fg", "crowd_only_std", "g600", "rows4100"])
def test_device_draw_skips_crowd_rows_and_keeps_each_gt_label(name):
    """Without host choices the minibatch is a torch.randperm draw on the device: it never takes a crowd row, every sampled
    ground-truth row -- identical boxes included -- carries its own class, and the blobs are the oracle's for that draw."""
    p = case(name)
    G = p["gt"].shape[0]
    t = p["cfg"]
    mo = OT.assign_rois(p["boxes"], p["gt"], p["classes"], p["crowd"])[0]
    fg_inds = np.where(mo >= np.float32(t["FG_THRESH"]))[0]
    bg_inds = np.where((mo < np.float32(t["BG_THRESH_HI"])) & (mo >= np.float32(t["BG_THRESH_LO"])))[0]
    torch.manual_seed(0)
    for _ in range(3):
        b = device_blobs(p)
        keep = b["keep_inds"].astype(np.int64)
        n_fg = min(int(round(t["FG_FRACTION"] * t["BATCH_SIZE_PER_IM"])), fg_inds.size)
        assert len(set(keep.tolist())) == keep.size
        gt_rows = keep[keep < G]
        assert not p["crowd"][gt_rows].any()
        pos = np.where(keep[:n_fg] < G)[0]
        assert np.array_equal(b["labels_int32"][pos], p["classes"][keep[pos]])
        ref = oracle_blobs(p, np.searchsorted(fg_inds, keep[:n_fg]), np.searchsorted(bg_inds, keep[n_fg:]))
        assert np.array_equal(b["keep_inds"], ref["keep_inds"])
        assert_blobs_equal(b, ref)
    if name == "few_fg":                                                    # every fg row is taken: all non-crowd gt rows
        assert set(np.where(p["crowd"] == 0)[0]) <= set(keep[:n_fg].tolist())
