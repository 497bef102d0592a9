"""C4 training blobs (GenerateProposalLabelsOp) and the batched RoI sampler shared with the FPN training branch.

Goldens: tests/golden/proposal_labels.npz from the unmodified reference op (tests/golden/make_golden_proposal_labels.py)."""
import os
import warnings

import numpy as np
import pytest

from oracle import targets as OT
from tests import fast_rcnn_roidb_cases as C

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "proposal_labels.npz"))
CASES = {"two": {}, "agnostic": dict(CLS_AGNOSTIC_BBOX_REG=True), "sparse": {}, "mask": C.TRAIN_MASK, "kp": C.TRAIN_KEYPOINTS}
FRCN = ("labels_int32", "rois", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights")


def case(name):
    g = {k[len(name) + 1:]: GOLD[k] for k in GOLD.files if k.startswith(name + "/")}
    return g, int(g["num_images"]), dict(C.TRAIN_CFG, **CASES[name])


def assert_targets_close(got, ref):
    """dx, dy bit-exact; dw, dh (logf) within 2e-6 relative."""
    assert got.shape == ref.shape and got.dtype == ref.dtype
    g, r = got.reshape(got.shape[0], -1, 4), ref.reshape(ref.shape[0], -1, 4)
    assert np.array_equal(g[..., :2], r[..., :2])
    np.testing.assert_allclose(g[..., 2:], r[..., 2:], rtol=2e-6, atol=0)


def oracle_blobs(name):
    """oracle/targets.sample_rois per image on the roidb that add_proposals builds, concatenated as add_fast_rcnn_blobs does."""
    g, N, t = case(name)
    rr, scales = g["rpn_rois"], g["im_info"][:, 2]
    per = []
    for i in range(N):
        gt, cl, cr = g["gt_%d" % i], g["gt_classes_%d" % i], g["is_crowd_%d" % i]
        props = rr[np.where(rr[:, 0] == i)[0], 1:] * (1. / scales[i])
        boxes = np.concatenate([gt, props.astype(np.float32)])
        per.append(OT.sample_rois(boxes, gt, cl, scales[i], i, t["NUM_CLASSES"], g["fg_choice_%d" % i], g["bg_choice_%d" % i],
                                  t["BATCH_SIZE_PER_IM"], t["FG_FRACTION"], t["FG_THRESH"], t["BG_THRESH_HI"], t["BG_THRESH_LO"],
                                  t["BBOX_REG_WEIGHTS"], t["CLS_AGNOSTIC_BBOX_REG"], cr))
    return {k: np.concatenate([b[k] for b in per]) for k in FRCN}, g


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_op(name):
    got, g = oracle_blobs(name)
    for k in FRCN:
        if k == "bbox_targets":
            assert_targets_close(got[k], g["blob_" + k])
        else:
            assert got[k].dtype == g["blob_" + k].dtype and np.array_equal(got[k], g["blob_" + k]), k


def test_goldens_hold_what_they_test():
    g, N, _ = case("sparse")
    assert N == 4
    counts = [int((g["rpn_rois"][:, 0] == i).sum()) for i in range(N)]
    assert counts[3] == 0 and min(counts[:3]) > 0                              # an image without proposals
    assert g["fg_choice_1"].size == 0 and g["is_crowd_1"].all()                # an image without fg
    rr = GOLD["two/rpn_rois"][:, 0]
    assert (np.diff(rr) != 0).sum() > 100                                      # the two images' proposals are interleaved
    assert GOLD["two/is_crowd_0"].any() or GOLD["two/is_crowd_1"].any()
    assert GOLD["mask/blob_masks_int32"].shape[1] == 81 * 14 * 14
    assert "kp/blob_keypoint_rois" in GOLD.files


# ---- GPU ----------------------------------------------------------------------------------------------------------------

def _roidb(g, N):
    from tests.test_fast_rcnn_roidb import unpack_segms
    out = []
    for i in range(N):
        crowd = g["is_crowd_%d" % i]
        out.append(dict(boxes=g["gt_%d" % i], gt_classes=g["gt_classes_%d" % i], is_crowd=crowd, gt_keypoints=g["gt_keypoints_%d" % i],
                        segms=unpack_segms(g["poly_begin_%d" % i], g["coord_begin_%d" % i], g["coords_%d" % i], crowd)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("tensor_input", [False, True])
def test_op_vs_reference_op(name, tensor_input):
    import torch
    from detectron.pytorch_b200.modeling.generate_proposal_labels import GenerateProposalLabelsOp
    g, N, t = case(name)
    choices = [(g["fg_choice_%d" % i], g["bg_choice_%d" % i], g.get("kp_choice_%d" % i)) for i in range(N)]
    rr = torch.from_numpy(g["rpn_rois"]).cuda() if tensor_input else g["rpn_rois"]
    roidb = _roidb(g, N)
    before = {k: np.copy(v) for k, v in roidb[0].items() if isinstance(v, np.ndarray)}
    blobs = GenerateProposalLabelsOp(train=t)(rr, roidb, g["im_info"], choices=choices)
    ref_keys = [k[len("blob_"):] for k in g if k.startswith("blob_")]
    assert sorted(blobs) == sorted(ref_keys)
    for k in ref_keys:
        got, ref = blobs[k], g["blob_" + k]
        assert got.is_cuda, k
        got = got.cpu().numpy()
        if k == "bbox_targets":
            assert_targets_close(got, ref)
        else:
            assert got.dtype == ref.dtype and got.shape == ref.shape and np.array_equal(got, ref), k
    assert all(np.array_equal(roidb[0][k], v) for k, v in before.items()) and "max_overlaps" not in roidb[0]


def _minibatch(seed, N, props_per_image=2000):
    """Seeded images (gt with crowd objects and duplicates, proposals around them); image 1 has no proposal and, when N > 2,
    image 2 only crowd ground truth."""
    rng = np.random.RandomState(seed)
    ims = []
    for i in range(N):
        gt, cl, cr = C.roster(seed * 100 + i, "mixed", int(rng.randint(3, 40)), 81)
        props = C.proposals(seed * 100 + i, "mixed", gt, props_per_image) if i != 1 else np.zeros((0, 4), np.float32)
        if i == 2 and N > 2:
            cr = np.ones_like(cr)
        ims.append((gt.astype(np.float32), cl.astype(np.int32), cr.astype(bool), props.astype(np.float32), float(rng.uniform(0.5, 2.0))))
    return ims


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 8, 16])
def test_batched_sampler_equals_per_image_sample_rois(N):
    import torch
    from detectron.pytorch_b200.roi_data import fast_rcnn as FR
    ims = _minibatch(N, N)
    dev = torch.device("cuda")
    t = dict(C.TRAIN_CFG, BATCH_SIZE_PER_IM=512)
    rng = np.random.RandomState(7 + N)
    merged, choices, per = [], [], []
    for i, (gt, cl, cr, props, s) in enumerate(ims):
        boxes = np.concatenate([gt, props])
        mo = OT.assign_rois(boxes, gt, cl, cr)[0]
        nf_all = int((mo >= 0.5).sum()); nb_all = int(((mo < 0.5) & (mo >= 0.0)).sum())
        nf = min(128, nf_all); nb = min(512 - nf, nb_all)
        fc = rng.permutation(nf_all)[:nf] if nf_all else np.zeros(0, np.int64)
        bc = rng.permutation(nb_all)[:nb] if nb_all else np.zeros(0, np.int64)
        choices.append((fc, bc)); merged.append(boxes)
        b = FR.sample_rois(torch.from_numpy(boxes).to(dev), torch.from_numpy(gt).to(dev) if len(gt) else None, torch.from_numpy(cl).to(dev),
                           s, i, 81, 512, 0.25, 0.5, 0.5, 0.0, (10.0, 10.0, 5.0, 5.0), False, fc, bc, is_crowd=cr)
        per.append(b)
    box_off = np.concatenate([[0], np.cumsum([m.shape[0] for m in merged])])
    gt_off = np.concatenate([[0], np.cumsum([im[0].shape[0] for im in ims])])
    blobs, info = FR.sample_rois_batched(
        torch.from_numpy(np.concatenate(merged)).to(dev), torch.from_numpy(box_off).to(dev),
        torch.from_numpy(np.concatenate([im[0] for im in ims])).to(dev), torch.from_numpy(np.concatenate([im[1] for im in ims])).to(dev),
        torch.from_numpy(gt_off).to(dev), torch.tensor([im[4] for im in ims], dtype=torch.float32, device=dev), 81, 512, 0.25, 0.5, 0.5,
        0.0, (10.0, 10.0, 5.0, 5.0), False, choices=choices,
        is_crowd=torch.from_numpy(np.concatenate([im[2] for im in ims]).astype(np.int32)).to(dev))
    for k in FRCN:
        ref = torch.cat([b[k] for b in per]).cpu().numpy()
        assert np.array_equal(blobs[k].cpu().numpy(), ref), k
    for i in range(N):
        assert np.array_equal(info["keep_inds"][i].cpu().numpy(), per[i]["keep_inds"].cpu().numpy())
        assert info["num_fg"][i] == min(128, choices[i][0].size)
    assert list(info["box_begin"]) == list(box_off)


@pytest.mark.gpu
def test_device_draw_gives_a_valid_minibatch():
    import torch
    from detectron.pytorch_b200.modeling.generate_proposal_labels import GenerateProposalLabelsOp
    g, N, t = case("sparse")
    torch.manual_seed(0)
    blobs = GenerateProposalLabelsOp(train=t)(g["rpn_rois"], _roidb(g, N), g["im_info"])
    ref = {k: g["blob_" + k] for k in FRCN}
    lab, rois = blobs["labels_int32"].cpu().numpy(), blobs["rois"].cpu().numpy()
    assert lab.shape == ref["labels_int32"].shape                              # same per-image sizes as the reference's draw
    for i in range(N):
        mine, theirs = rois[:, 0] == i, ref["rois"][:, 0] == i
        assert mine.sum() == theirs.sum() and (lab[mine] > 0).sum() == (ref["labels_int32"][theirs] > 0).sum()
        fg = lab[mine] > 0
        assert not np.any(fg[1:] & ~fg[:-1])                                   # each image's fg rows first, then its bg rows
    inside = blobs["bbox_inside_weights"].cpu().numpy()
    assert np.array_equal(inside.reshape(len(lab), -1, 4).sum(axis=(1, 2)), np.where(lab > 0, 4.0, 0.0).astype(np.float32))


def _sync_count(fn):
    import torch
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(x.message) for x in w)


@pytest.mark.gpu
def test_host_reads_do_not_grow_with_the_number_of_images():
    import torch
    from detectron.pytorch_b200.modeling.collect_and_distribute_fpn_rpn_proposals import CollectAndDistributeFpnRpnProposalsOp
    from detectron.pytorch_b200.modeling.generate_proposal_labels import GenerateProposalLabelsOp
    t = dict(C.TRAIN_CFG)
    c4, fpn = {}, {}
    for N in (2, 16):
        ims = _minibatch(3, N, 500)
        rr = np.concatenate([np.hstack([np.full((im[3].shape[0], 1), i, np.float32), im[3] * np.float32(im[4])])
                             for i, im in enumerate(ims)]).astype(np.float32)
        rr = torch.from_numpy(rr[np.random.RandomState(N).permutation(rr.shape[0])]).cuda()
        roidb = [dict(boxes=im[0], gt_classes=im[1], is_crowd=im[2]) for im in ims]
        im_info = np.asarray([[1000.0, 1000.0, im[4]] for im in ims], np.float32)
        op = GenerateProposalLabelsOp(train=t)
        op(rr, roidb, im_info)                                                 # warm up
        c4[N] = _sync_count(lambda: op(rr, roidb, im_info))
        scores = torch.rand(rr.shape[0], 1, device="cuda")
        inputs = [rr] + [rr[:0]] * 4 + [scores] + [scores[:0]] * 4
        cd = CollectAndDistributeFpnRpnProposalsOp(post_nms_topN=rr.shape[0])
        cd.train()
        cd(inputs, roidb, im_info, train=t)
        fpn[N] = _sync_count(lambda: cd(inputs, roidb, im_info, train=t))
    assert c4[16] <= c4[2] and fpn[16] <= fpn[2], (c4, fpn)
    assert c4[2] >= 1
