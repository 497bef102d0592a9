"""Keypoint R-CNN training targets (add_keypoint_rcnn_blobs, lib/roi_data/keypoint_rcnn.py:33-96) on the device.

CPU: the numpy oracle (oracle/keypoint_targets.py) against the blobs of the UNMODIFIED reference functions
(tests/golden/keypoint_targets.npz, make_golden_keypoint_targets.py), the reference quirks the goldens hold, the C ABI's
argument checks and the keypoint loss with an INT_MIN weight-0 target.
GPU: the device blobs against the same goldens (bit-exact), against the oracle at COCO scale and on randomised degenerate
boxes, the training branch of CollectAndDistributeFpnRpnProposalsOp with KEYPOINTS_ON (alone, with MASK_ON, and off), the
launch count, the device draw, the errors and the keypoint loss."""
import ctypes
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import _lib
from detectron.pytorch_b200.modeling.keypoint_rcnn_heads import keypoint_losses
from detectron.pytorch_b200.roi_data import keypoint_rcnn as KR
from oracle import keypoint_targets as OK

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "keypoint_targets.npz"))
CASES = ["hs56_k17", "hs56_k17_sub", "hs64_k5", "fg0", "nocand"]
EINVAL = -1
INT_MIN = -2 ** 31
BLOBS = ("keypoint_rois", "keypoint_locations_int32", "keypoint_weights")
CROWD_ROW, DUP_ROWS, ZERO_WIDTH_ROW = 5, (6, 7), 8                      # rows of the golden images' ground truth


def case(c):
    g = c + "/"
    HS, K, fg = [int(v) for v in GOLD[g + "cfg"]]
    entry = dict(boxes=GOLD[g + "boxes"], max_overlaps=GOLD[g + "max_overlaps"], box_to_gt_ind_map=GOLD[g + "box_to_gt_ind_map"],
                 gt_classes=GOLD[g + "gt_classes"], gt_keypoints=GOLD[g + "gt_keypoints"])
    return dict(HS=HS, K=K, fg=fg, fg_thresh=float(GOLD[g + "fg_thresh"]), entry=entry, im_scale=GOLD[g + "im_scale"].item(),
                choice=GOLD[g + "choice"] if g + "choice" in GOLD.files else None)


def oracle_blobs(p):
    blobs = {}
    cand = OK.add_keypoint_rcnn_blobs(blobs, p["entry"], p["fg"], p["im_scale"], 1, p["HS"], p["fg_thresh"], p["choice"])
    valid = OK.finalize_keypoint_minibatch(blobs, True, 2, 64, 0.25, p["K"])
    return blobs, cand, valid


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES)
def test_oracle_matches_reference_blobs(c):
    blobs, _, valid = oracle_blobs(case(c))
    for k in BLOBS + ("keypoint_loss_normalizer",):
        ref = GOLD[c + "/" + k]
        assert blobs[k].dtype == ref.dtype and blobs[k].shape == ref.shape and np.array_equal(blobs[k], ref), k
    assert valid == bool(GOLD[c + "/valid"])


def test_golden_cases_hold_the_reference_quirks():
    p = case("hs56_k17")
    HS, K = p["HS"], p["K"]
    _, cand, _ = oracle_blobs(p)
    loc = GOLD["hs56_k17/keypoint_locations_int32"].reshape(-1, K)
    w = GOLD["hs56_k17/keypoint_weights"].reshape(-1, K)
    row = {int(b): i for i, b in enumerate(cand)}
    # box 0 (its own gt row): keypoint 1 on x2 and keypoint 3 on y2 land in the last column / row, keypoint 4 on (x2, y2) in
    # the last cell; keypoints 6 and 7 just outside have weight 0
    r0 = loc[row[0]]
    assert r0[1] % HS == HS - 1 and r0[3] // HS == HS - 1 and r0[4] == HS * HS - 1 and r0[0] % HS == 0 and r0[2] // HS == 0
    assert w[row[0], 6] == 0 and w[row[0], 7] == 0
    # INT_MIN only with weight 0, and it appears (the zero-width gt box); the keypoint on x1 == x2 is in the last column
    assert (loc == INT_MIN).any() and (w[loc == INT_MIN] == 0).all()
    zw = loc[row[ZERO_WIDTH_ROW]]
    assert zw[0] % HS == HS - 1 and w[row[ZERO_WIDTH_ROW], 0] == 1 and zw[1] == INT_MIN
    # the crowd row is never a candidate; the duplicated gt boxes keep their own keypoints
    assert CROWD_ROW not in row
    assert all(d in row for d in DUP_ROWS)
    kp = p["entry"]["gt_keypoints"]
    box = p["entry"]["boxes"][list(DUP_ROWS)]
    own, _ = OK.heatmap_labels(kp[list(DUP_ROWS)], box, HS)
    assert np.array_equal(loc[[row[d] for d in DUP_ROWS]], own) and not np.array_equal(own[0], own[1])
    # FG_THRESH 0: proposals without overlap (map -1) are candidates through the last person, and get all -1 keypoints
    q = case("fg0")
    _, cand0, _ = oracle_blobs(q)
    neg = np.where(q["entry"]["box_to_gt_ind_map"][cand0] < 0)[0]
    assert neg.size > 0
    assert (GOLD["fg0/keypoint_weights"].reshape(-1, K)[neg] == 0).all()
    # the subsampled case took the recorded draw; the image without a visible keypoint has empty blobs
    assert GOLD["hs56_k17_sub/keypoint_rois"].shape[0] == 16 and GOLD["hs56_k17_sub/choice"].size == 16
    assert GOLD["nocand/keypoint_rois"].shape == (0, 5) and not bool(GOLD["nocand/valid"])


def test_abi_argument_errors_return_einval():
    lib = _lib.load()
    fake = 256                                                            # never dereferenced: every call fails its checks first
    t2 = (ctypes.c_int * 2)(0, 1)
    fl = (ctypes.c_float * 1)(1.0)

    def cand(boxes=fake, mo=fake, m=fake, N=1, bb=t2, gi=fake, gb=t2, kp=fake, pb=t2, K=17, c=fake, n=fake):
        return lib.b200_keypoint_candidates(boxes, mo, m, N, bb, gi, gb, kp, pb, K, 0.5, c, n, None)

    def emit(boxes=fake, m=fake, N=1, bb=t2, gi=fake, gb=t2, kp=fake, pb=t2, K=17, HS=56, c=fake, n=fake, pk=fake, rb=t2, sc=fl, bi=fl,
             rois=fake, loc=fake, w=fake):
        return lib.b200_keypoint_targets(boxes, m, N, bb, gi, gb, kp, pb, K, HS, c, n, pk, rb, sc, bi, rois, loc, w, None)
    for kw in (dict(boxes=None), dict(mo=None), dict(m=None), dict(gi=None), dict(kp=None), dict(c=None), dict(n=None), dict(bb=None),
               dict(N=0), dict(N=65), dict(K=0), dict(K=65), dict(bb=(ctypes.c_int * 2)(1, 1)), dict(gb=(ctypes.c_int * 3)(0, 2, 1), N=2)):
        assert cand(**kw) == EINVAL, kw
    for kw in (dict(boxes=None), dict(pk=None), dict(rois=None), dict(loc=None), dict(w=None), dict(rb=None), dict(sc=None), dict(HS=0),
               dict(HS=4097), dict(K=0), dict(K=65), dict(N=0), dict(rb=(ctypes.c_int * 2)(0, 2)),     # more RoIs than boxes
               dict(rb=(ctypes.c_int * 2)(1, 1)), dict(pb=(ctypes.c_int * 2)(0, -1))):
        assert emit(**kw) == EINVAL, kw


def _loss_reference(pred, loc, w, HS, normalizer=None):
    """keypoint_rcnn_heads.py:91-122 in float64 over the entries with weight > 0."""
    x = pred.reshape(-1, HS * HS).astype(np.float64)
    on = np.where(w > 0)[0]
    lse = np.log(np.exp(x[on] - x[on].max(1, keepdims=True)).sum(1)) + x[on].max(1)
    ce = lse - x[on, loc[on].astype(np.int64)]
    loss = (ce * w[on]).sum() / w.sum()
    return loss * (1.0 if normalizer is None else float(normalizer))


def test_keypoint_loss_masks_weight_zero_targets_on_cpu():
    """A target of INT_MIN (or any out-of-range value) with weight 0 must not reach cross_entropy: on the CPU a wrong
    implementation raises instead of asserting on a device."""
    rng = np.random.RandomState(0)
    HS, R, K = 8, 5, 3
    pred = rng.standard_normal((R, K, HS, HS)).astype(np.float32)
    loc = rng.randint(0, HS * HS, R * K).astype(np.int32)
    w = (rng.rand(R * K) < 0.6).astype(np.float32)
    loc[w == 0] = INT_MIN
    loc[np.where(w == 0)[0][:1]] = HS * HS + 7
    got = keypoint_losses(torch.from_numpy(pred), torch.from_numpy(loc), torch.from_numpy(w))
    assert abs(float(got) - _loss_reference(pred, loc, w, HS)) <= 1e-6 * abs(_loss_reference(pred, loc, w, HS))
    norm = np.float32(0.37)
    got = keypoint_losses(torch.from_numpy(pred), loc, w, norm, loss_weight=4.0, normalize_by_visible_keypoints=False)
    ref = _loss_reference(pred, loc, w, HS, norm) * 4.0
    assert abs(float(got) - ref) <= 1e-6 * abs(ref)


def test_cpu_tensors_are_rejected():
    p = case("hs56_k17")
    entry = dict(p["entry"], boxes=torch.from_numpy(p["entry"]["boxes"]))
    with pytest.raises(NotImplementedError):
        KR.add_keypoint_rcnn_blobs({}, entry, 64, None, 1.0, 0, heatmap_size=56, num_keypoints=17)
    with pytest.raises(NotImplementedError):
        KR.finalize_keypoint_minibatch(dict(keypoint_weights=torch.zeros(3)), True, num_keypoints=17)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def run_device(c):
    p = case(c)
    blobs = {}
    KR.add_keypoint_rcnn_blobs(blobs, p["entry"], p["fg"], None, p["im_scale"], 1, choice=p["choice"], heatmap_size=p["HS"],
                               num_keypoints=p["K"], fg_thresh=p["fg_thresh"])
    valid = KR.finalize_keypoint_minibatch(blobs, True, num_keypoints=p["K"])
    return blobs, valid


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_device_matches_reference_blobs(c):
    blobs, valid = run_device(c)
    for k in BLOBS + ("keypoint_loss_normalizer",):
        ref = GOLD[c + "/" + k]
        got = blobs[k]
        assert got.is_cuda and tuple(got.shape) == ref.shape, k
        got = got.cpu().numpy()
        assert got.dtype == ref.dtype and np.array_equal(got, ref), k
    assert bool(valid) == bool(GOLD[c + "/valid"])


@pytest.mark.gpu
def test_device_reads_cfg():
    class C:
        pass
    cfg = C(); cfg.KRCNN = C(); cfg.TRAIN = C()
    cfg.KRCNN.HEATMAP_SIZE = 64; cfg.KRCNN.NUM_KEYPOINTS = 5; cfg.TRAIN.FG_THRESH = 0.5
    p = case("hs64_k5")
    blobs = {}
    KR.add_keypoint_rcnn_blobs(blobs, p["entry"], p["fg"], None, p["im_scale"], 1, cfg=cfg)
    assert np.array_equal(blobs["keypoint_locations_int32"].cpu().numpy(), GOLD["hs64_k5/keypoint_locations_int32"])


@pytest.mark.gpu
def test_heatmap_labels_function_matches_oracle():
    from detectron.pytorch_b200.utils.keypoints import keypoints_to_heatmap_labels
    rng = np.random.RandomState(3)
    R, K, HS = 300, 17, 56
    x1, y1 = rng.uniform(0, 500, R), rng.uniform(0, 500, R)
    rois = np.stack([x1, y1, x1 + rng.choice([0, 0.5, 1, 30, 200], R), y1 + rng.choice([0, 0.25, 1, 40, 150], R)], 1).astype(np.float32)
    kp = np.stack([rng.randint(-5, 750, (R, K)), rng.randint(-5, 700, (R, K)), rng.randint(-1, 3, (R, K))], 1).astype(np.int32)
    edge = rng.rand(R, K) < 0.3
    kp[:, 0][edge] = np.floor(rois[:, 2:3].repeat(K, 1))[edge].astype(np.int32)
    heats, weights = keypoints_to_heatmap_labels(kp, rois, heatmap_size=HS)
    ref_h, ref_w = OK.heatmap_labels(kp, rois, HS)
    assert np.array_equal(heats.cpu().numpy(), ref_h) and np.array_equal(weights.cpu().numpy(), ref_w)


def coco_image(rng, n_person=20, n_prop=2000, h=800, w=1333, K=17, degenerate=False):
    """A merged roidb entry: n_person gt rows (self map, overlap 1) and n_prop proposals assigned to them by IoU (the
    reference's merge), keypoints inside the boxes with some on their edges."""
    x1, y1 = rng.uniform(0, w - 60, n_person), rng.uniform(0, h - 60, n_person)
    bw = rng.uniform(0, 1, n_person) if degenerate else rng.uniform(30, 400, n_person)
    bh = rng.uniform(0, 1, n_person) if degenerate else rng.uniform(60, 500, n_person)
    gt = np.stack([x1, y1, x1 + bw, y1 + bh], 1).astype(np.float32)
    if degenerate:
        gt[::3, 2] = gt[::3, 0]; gt[1::3, 3] = gt[1::3, 1]                # zero width / zero height
        gt = np.round(gt * 2) / 2
    kp = np.zeros((n_person, 3, K), np.int32)
    for i, b in enumerate(gt):
        kp[i, 0] = rng.randint(int(np.floor(b[0])) - 2, int(np.ceil(b[2])) + 3, K)
        kp[i, 1] = rng.randint(int(np.floor(b[1])) - 2, int(np.ceil(b[3])) + 3, K)
        kp[i, 2] = rng.choice([0, 1, 2], K, p=[0.3, 0.2, 0.5])
        on = rng.rand(K) < 0.3
        kp[i, 0][on] = rng.choice([int(np.floor(b[0])), int(np.ceil(b[2])), int(b[0]), int(b[2])], on.sum())
    src = rng.randint(0, n_person, n_prop)
    wh = np.maximum(gt[src, 2:] - gt[src, :2], 1.0)
    props = (gt[src] + rng.standard_normal((n_prop, 4)) * np.concatenate([wh, wh], 1) * 0.2).astype(np.float32)
    if degenerate:
        props[::4, 2] = props[::4, 0]
    props[:, 2:] = np.maximum(props[:, 2:], props[:, :2])
    from oracle.targets import bbox_overlaps                             # the cython_bbox restatement
    ov = bbox_overlaps(props, gt)
    am, mx = ov.argmax(1), ov.max(1).astype(np.float32)
    m = np.where(mx > 0, am, -1).astype(np.int32)
    boxes = np.concatenate([gt, props]).astype(np.float32)
    return dict(boxes=boxes, max_overlaps=np.concatenate([np.ones(n_person, np.float32), mx]),
                box_to_gt_ind_map=np.concatenate([np.arange(n_person, dtype=np.int32), m]), gt_classes=np.ones(n_person, np.int32),
                gt_keypoints=kp)


def _batched_vs_oracle(entries, fg, HS, K, fg_thresh, seed):
    rng = np.random.RandomState(seed)
    choices, ref = [], []
    for n, e in enumerate(entries):
        gt_inds = np.where(e["gt_classes"] > 0)[0]
        c = OK.candidates(e["boxes"], e["max_overlaps"], e["box_to_gt_ind_map"], gt_inds, e["gt_keypoints"], fg_thresh)
        choice = rng.choice(c.size, fg, replace=False) if c.size > fg else None
        choices.append(choice)
        bl = {}
        OK.add_keypoint_rcnn_blobs(bl, e, fg, 1.5, n, HS, fg_thresh, choice)
        ref.append(bl)
    box_begin = np.concatenate([[0], np.cumsum([e["boxes"].shape[0] for e in entries])])
    cat = lambda k: np.concatenate([e[k] for e in entries])             # noqa: E731
    out = KR.keypoint_rcnn_blobs(torch.from_numpy(cat("boxes")).cuda(), box_begin, torch.from_numpy(cat("max_overlaps")).cuda(),
                                 torch.from_numpy(cat("box_to_gt_ind_map")).cuda(), entries, [1.5] * len(entries), fg, HS, K, fg_thresh,
                                 choices=choices)
    for k in BLOBS:
        assert np.array_equal(out[k].cpu().numpy(), np.concatenate([r[k] for r in ref])), k
    return choices


@pytest.mark.gpu
def test_device_matches_oracle_at_coco_scale():
    """2 images of 800 x 1333, 2000 proposals and 20 persons each, BATCH_SIZE_PER_IM 512 (128 fg per image): the draw happens."""
    rng = np.random.RandomState(0)
    choices = _batched_vs_oracle([coco_image(rng), coco_image(rng)], 128, 56, 17, 0.5, 1)
    assert all(c is not None for c in choices)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(6))
def test_device_matches_oracle_on_degenerate_boxes(seed):
    """Boxes 0 to 1 px wide / high (a third of zero width, a third of zero height), keypoints on their edges, FG_THRESH 0 on
    odd seeds."""
    rng = np.random.RandomState(100 + seed)
    entries = [coco_image(rng, n_person=12, n_prop=400, degenerate=True) for _ in range(1 + seed % 3)]
    _batched_vs_oracle(entries, 64, [56, 64, 7][seed % 3], 17, 0.0 if seed % 2 else 0.5, seed)


def train_inputs():
    g = {k[len("train/"):]: GOLD[k] for k in GOLD.files if k.startswith("train/")}
    inputs = [torch.from_numpy(g["rpn_rois_%d" % l]).cuda() for l in range(5)] + [torch.from_numpy(g["rpn_probs_%d" % l]).cuda()
                                                                                  for l in range(5)]
    roidb = []
    for i in range(2):
        n = g["gt_%d" % i].shape[0]
        roidb.append(dict(boxes=g["gt_%d" % i], gt_classes=np.ones(n, np.int32), is_crowd=np.zeros(n, bool),
                          gt_keypoints=g["gt_keypoints_%d" % i]))
    train = dict(BATCH_SIZE_PER_IM=128, FG_FRACTION=0.25, FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.0, NUM_CLASSES=2,
                 BBOX_REG_WEIGHTS=(10.0, 10.0, 5.0, 5.0), CLS_AGNOSTIC_BBOX_REG=False)
    kp = dict(KEYPOINTS_ON=True, HEATMAP_SIZE=56, NUM_KEYPOINTS=17, IMS_PER_BATCH=2)
    choices = [(g["fg_choice_%d" % i], g["bg_choice_%d" % i], g.get("kp_choice_%d" % i)) for i in range(2)]
    return g, inputs, roidb, train, kp, choices


def _op():
    from detectron.pytorch_b200.modeling.collect_and_distribute_fpn_rpn_proposals import CollectAndDistributeFpnRpnProposalsOp
    op = CollectAndDistributeFpnRpnProposalsOp(rpn_min_level=2, rpn_max_level=6, roi_min_level=2, roi_max_level=5, post_nms_topN=600)
    op.train()
    return op


def _same(a, b):
    a = a.cpu().numpy() if torch.is_tensor(a) else a
    b = b.cpu().numpy() if torch.is_tensor(b) else b
    return np.array_equal(a, b) and (not hasattr(a, "dtype") or a.dtype == np.asarray(b).dtype)


@pytest.mark.gpu
def test_collect_and_distribute_training_branch_with_keypoints_vs_reference_op():
    g, inputs, roidb, train, kp, choices = train_inputs()
    op = _op()
    blobs = op(inputs, roidb, g["im_info"], choices=choices, train=dict(train, **kp))
    ref_keys = sorted(k[len("blob_"):] for k in g if k.startswith("blob_"))
    assert sorted(k for k in blobs if k != "counts") == ref_keys
    for k in ref_keys:
        got, ref = blobs[k].cpu().numpy(), g["blob_" + k]
        assert got.shape == ref.shape, k
        if k == "bbox_targets":
            np.testing.assert_allclose(got, ref, rtol=2e-6, atol=1e-7)
        else:
            assert got.dtype == ref.dtype and np.array_equal(got, ref), k
    # KEYPOINTS_ON off: today's keys and values, with two-entry choices
    plain = op(inputs, roidb, g["im_info"], choices=[c[:2] for c in choices], train=train)
    assert not any(k.startswith("keypoint") for k in plain)
    assert sorted(plain) == sorted(k for k in blobs if not k.startswith("keypoint"))
    for k, v in plain.items():
        assert _same(blobs[k], v), k
    off = op(inputs, roidb, g["im_info"], choices=[c[:2] for c in choices], train=dict(train, KEYPOINTS_ON=False))
    assert sorted(off) == sorted(plain) and all(_same(off[k], plain[k]) for k in plain)


@pytest.mark.gpu
def test_mask_and_keypoints_together_are_the_union():
    g, inputs, roidb, train, kp, choices = train_inputs()
    for e in roidb:                                                      # one triangle inside each person box
        e["segms"] = [[[float(b[0]), float(b[1]), float(b[2]), float(b[1]), float(b[0]), float(b[3])]] for b in e["boxes"]]
    mask = dict(MASK_ON=True, MRCNN_RESOLUTION=14, CLS_SPECIFIC_MASK=True)
    op = _op()
    m = op(inputs, roidb, g["im_info"], choices=choices, train=dict(train, **mask))
    k = op(inputs, roidb, g["im_info"], choices=choices, train=dict(train, **kp))
    both = op(inputs, roidb, g["im_info"], choices=choices, train=dict(train, **mask, **kp))
    assert sorted(both) == sorted(set(m) | set(k))
    for key, v in list(m.items()) + list(k.items()):
        assert _same(both[key], v), key


@pytest.mark.gpu
def test_one_call_makes_a_fixed_number_of_launches():
    """Candidates + emit: 2 launches whatever the number of images, boxes or persons (also with no candidate at all)."""
    for c in CASES:
        p = case(c)
        torch.cuda.synchronize()
        before = _lib.launch_count()
        KR.add_keypoint_rcnn_blobs({}, p["entry"], p["fg"], None, p["im_scale"], 1, choice=p["choice"], heatmap_size=p["HS"],
                                   num_keypoints=p["K"], fg_thresh=p["fg_thresh"])
        torch.cuda.synchronize()
        assert _lib.launch_count() - before == 2, c
    rng = np.random.RandomState(7)
    for n_img, n_person in ((1, 3), (2, 20), (5, 40)):
        entries = [coco_image(rng, n_person=n_person, n_prop=300 * n_img) for _ in range(n_img)]
        box_begin = np.concatenate([[0], np.cumsum([e["boxes"].shape[0] for e in entries])])
        torch.cuda.synchronize()
        before = _lib.launch_count()
        KR.keypoint_rcnn_blobs(np.concatenate([e["boxes"] for e in entries]), box_begin,
                               np.concatenate([e["max_overlaps"] for e in entries]),
                               np.concatenate([e["box_to_gt_ind_map"] for e in entries]), entries, [1.0] * n_img, 32, 56, 17)
        torch.cuda.synchronize()
        assert _lib.launch_count() - before == 2, (n_img, n_person)


@pytest.mark.gpu
def test_device_draw_gives_a_valid_minibatch():
    rng = np.random.RandomState(11)
    e = coco_image(rng)
    gt_inds = np.arange(20)
    cand = OK.candidates(e["boxes"], e["max_overlaps"], e["box_to_gt_ind_map"], gt_inds, e["gt_keypoints"], 0.5)
    boxes = e["boxes"][cand] * np.float32(1.5)
    for fg in (64, cand.size + 10):
        out = KR.keypoint_rcnn_blobs(e["boxes"], [0, e["boxes"].shape[0]], e["max_overlaps"], e["box_to_gt_ind_map"], [e], [1.5], fg, 56, 17)
        rois = out["keypoint_rois"].cpu().numpy()[:, 1:]
        assert rois.shape[0] == min(fg, cand.size)
        pos = [int(np.where((boxes == r).all(1))[0][0]) for r in rois]
        assert len(set(pos)) == len(pos)
        if fg > cand.size:
            assert pos == sorted(pos) == list(range(cand.size))


@pytest.mark.gpu
def test_errors():
    p = case("hs56_k17")
    e = p["entry"]
    with pytest.raises(ValueError):                                           # K is not NUM_KEYPOINTS
        KR.add_keypoint_rcnn_blobs({}, e, 64, None, 1.0, 0, heatmap_size=56, num_keypoints=5)
    bad = dict(e, box_to_gt_ind_map=np.where(np.arange(e["boxes"].shape[0]) == 20, 9, e["box_to_gt_ind_map"]).astype(np.int32))
    with pytest.raises(ValueError):                                           # numpy's IndexError: 9 persons, index 9
        KR.add_keypoint_rcnn_blobs({}, bad, 64, None, 1.0, 0, heatmap_size=56, num_keypoints=17)
    bad = dict(e, box_to_gt_ind_map=np.where(np.arange(e["boxes"].shape[0]) == 20, -10, e["box_to_gt_ind_map"]).astype(np.int32))
    with pytest.raises(ValueError):
        KR.add_keypoint_rcnn_blobs({}, bad, 64, None, 1.0, 0, heatmap_size=56, num_keypoints=17)
    with pytest.raises(ValueError):                                           # HEATMAP_SIZE beyond 4096
        KR.add_keypoint_rcnn_blobs({}, e, 64, None, 1.0, 0, heatmap_size=4097, num_keypoints=17)
    with pytest.raises(ValueError):                                           # a draw of the wrong size
        KR.add_keypoint_rcnn_blobs({}, e, 16, None, 1.0, 0, choice=np.arange(15), heatmap_size=56, num_keypoints=17)
    with pytest.raises(ValueError):                                           # a draw outside the candidate list
        KR.add_keypoint_rcnn_blobs({}, e, 16, None, 1.0, 0, choice=np.arange(16) + 10 ** 6, heatmap_size=56, num_keypoints=17)
    with pytest.raises(ValueError):
        KR.add_keypoint_rcnn_blobs({}, e, 64, None, 1.0, 0)                   # no configuration
    with pytest.raises(NotImplementedError):
        KR.add_keypoint_rcnn_blobs({}, dict(e, max_overlaps=torch.from_numpy(e["max_overlaps"])), 64, None, 1.0, 0, heatmap_size=56,
                                   num_keypoints=17)


@pytest.mark.gpu
@pytest.mark.parametrize("by_visible", [True, False])
def test_keypoint_loss_on_device_blob_matches_reference_formula(by_visible):
    blobs, _ = run_device("hs56_k17")
    loc, w = blobs["keypoint_locations_int32"], blobs["keypoint_weights"]
    R, K, HS = blobs["keypoint_rois"].size(0), 17, 56
    torch.manual_seed(0)
    pred = torch.randn((R, K, HS, HS), device="cuda")
    norm = blobs["keypoint_loss_normalizer"]
    got = keypoint_losses(pred, loc, w, None if by_visible else norm, heatmap_size=HS)
    on = w.cpu().numpy()
    assert set(np.unique(on)) <= {0.0, 1.0} and (loc.cpu().numpy()[on > 0] < HS * HS).all()
    ref = _loss_reference(pred.cpu().numpy(), loc.cpu().numpy(), on, HS, None if by_visible else GOLD["hs56_k17/keypoint_loss_normalizer"])
    assert abs(float(got) - ref) <= 1e-6 * abs(ref)
