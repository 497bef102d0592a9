"""Mask R-CNN training mask targets (add_mask_rcnn_blobs, lib/roi_data/mask_rcnn.py:34-122) on the device.

CPU: the numpy oracle (oracle/masks.py) against the blobs of the UNMODIFIED reference function (tests/golden/mask_targets.npz,
make_golden_masks.py), the rasteriser's hand-derived answers and its agreement with point-in-polygon away from the edges, the
polygon packer's rejections and the C ABI's argument checks.
GPU: the device blobs against the same goldens (bit-exact), against the oracle at COCO scale and on randomised polygons, the
training branch of CollectAndDistributeFpnRpnProposalsOp with MASK_ON, the launch count, the errors and the mask loss."""
import ctypes
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import _lib, ops
from detectron.pytorch_b200.roi_data import mask_rcnn as MR
from oracle import masks as OM

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "mask_targets.npz"))
CASES = ["m14_cls", "m28_agn", "m28_cls", "nofg"]
EINVAL = -1
BLOBS = ("mask_rois", "roi_has_mask_int32", "masks_int32")


def unpack(pb, cb, co, crowd):
    segms = []
    for o in range(pb.size - 1):
        if crowd[o]:
            segms.append({"counts": "crowd", "size": [600, 800]})
            continue
        segms.append([co[cb[p]:cb[p + 1]].tolist() for p in range(pb[o], pb[o + 1])])
    return segms


def case(c):
    g = c + "/"
    M, cls_specific, K = [int(v) for v in GOLD[g + "cfg"]]
    crowd = GOLD[g + "is_crowd"]
    roidb = dict(gt_classes=GOLD[g + "gt_classes"], is_crowd=crowd,
                 segms=unpack(GOLD[g + "poly_begin"], GOLD[g + "coord_begin"], GOLD[g + "coords"], crowd))
    return dict(M=M, cls_specific=bool(cls_specific), K=K, roidb=roidb, im_scale=GOLD[g + "im_scale"].item(),
                sampled=GOLD[g + "sampled_boxes"], labels=GOLD[g + "labels_int32"])


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES)
def test_oracle_matches_reference_blobs(c):
    p = case(c)
    blobs = OM.add_mask_rcnn_blobs(dict(labels_int32=p["labels"]), p["sampled"], p["roidb"], p["im_scale"], 1, M=p["M"],
                                   cls_specific=p["cls_specific"], num_classes=p["K"])
    for k in BLOBS:
        ref = GOLD[c + "/" + k]
        assert blobs[k].dtype == ref.dtype and np.array_equal(blobs[k], ref), k


def test_golden_cases_hold_the_reference_quirks():
    """The tied box takes the first object (the triangle, not the rectangle), the RoI with zero IoU everywhere takes object 0
    (far away: an empty mask), the no-fg image has one all -1 row and roi_has_mask[0] = 1."""
    p = case("m28_agn")
    fg = np.where(p["labels"] > 0)[0]
    masks = GOLD["m28_agn/masks_int32"].reshape(-1, 28, 28)
    tied = [i for i, r in enumerate(p["sampled"][fg]) if np.array_equal(r, OM.polys_to_boxes([p["roidb"]["segms"][4]])[0])]
    assert tied and 0 < masks[tied[0]].sum() < 28 * 28
    assert np.array_equal(masks[tied[0]], OM.polys_to_mask_wrt_box(p["roidb"]["segms"][4], p["sampled"][fg][tied[0]], 28))
    far = [i for i, r in enumerate(p["sampled"][fg]) if np.array_equal(r, np.asarray([700, 10, 780, 60], np.float32))]
    assert far and masks[far[0]].sum() == 0
    assert GOLD["nofg/masks_int32"].shape[0] == 1 and (GOLD["nofg/masks_int32"] == -1).all()
    assert GOLD["nofg/roi_has_mask_int32"][0] == 1 and GOLD["nofg/roi_has_mask_int32"][1:].sum() == 0


def raster(poly, M=8):
    return OM.decode(OM.frPyObjects([np.asarray(poly, np.float64)], M, M))[:, :, 0]


def test_rasteriser_known_answers():
    M = 8
    # the full square fills every pixel only because column c's bottom toggle and column c + 1's top toggle coincide
    assert raster([0, 0, M, 0, M, M, 0, M]).all()
    half = np.zeros((M, M), np.uint8); half[:, :4] = 1
    assert np.array_equal(raster([0, 0, 4, 0, 4, M, 0, M]), half)
    tri = np.array([[1 if x + y < 7 else 0 for x in range(M)] for y in range(M)], np.uint8)
    assert np.array_equal(raster([0, 0, M, 0, 0, M]), tri)
    assert raster([20, 20, 30, 20, 30, 30]).sum() == 0                    # entirely outside
    assert raster([-5, -5, -1, -5, -1, 30]).sum() == 0
    # x = -0.15: 5x + .5 = -0.25 truncates to 0 (floor would give -1): the same mask as x = 0
    assert np.array_equal(raster([-0.15, 0, 4, 0, 4, M, -0.15, M]), half)
    u, _ = OM.upsampled_walk([-0.15, 0, 4, 0, 4, 8])
    assert u[0] == 0


def _point_in_polygon(px, py, poly):
    xs, ys = poly[0::2], poly[1::2]
    inside = np.zeros(px.shape, bool)
    for j in range(xs.size):
        x0, y0, x1, y1 = xs[j], ys[j], xs[(j + 1) % xs.size], ys[(j + 1) % xs.size]
        cross = (y0 > py) != (y1 > py)
        with np.errstate(divide="ignore", invalid="ignore"):
            xint = x0 + (py - y0) * (x1 - x0) / (y1 - y0)
        inside ^= cross & (px < xint)
    return inside


def _edge_distance(px, py, poly):
    xs, ys = poly[0::2], poly[1::2]
    d = np.full(px.shape, np.inf)
    for j in range(xs.size):
        x0, y0, x1, y1 = xs[j], ys[j], xs[(j + 1) % xs.size], ys[(j + 1) % xs.size]
        dx, dy = x1 - x0, y1 - y0
        L = dx * dx + dy * dy
        t = np.clip(((px - x0) * dx + (py - y0) * dy) / L, 0, 1) if L > 0 else np.zeros(px.shape)
        d = np.minimum(d, np.hypot(px - x0 - t * dx, py - y0 - t * dy))
    return d


@pytest.mark.parametrize("seed", range(6))
def test_rasteriser_agrees_with_point_in_polygon_away_from_edges(seed):
    """Pixel (x, y) covers the centre (x + .5, y + .5); every pixel whose centre is more than 0.25 px from every edge is inside
    iff its centre is.  One upsampling step is 0.2 px, but the vertices and the interpolated rows are each rounded to that
    grid, and the two roundings together reach 0.206 px in these cases."""
    rng = np.random.RandomState(seed)
    M = int(rng.choice([14, 28, 40]))
    ys, xs = np.mgrid[0:M, 0:M]
    px, py = xs + .5, ys + .5
    for _ in range(20):
        k = int(rng.randint(3, 30))
        poly = rng.uniform(-0.3 * M, 1.3 * M, 2 * k).astype(np.float32).astype(np.float64)
        got = raster(poly, M).astype(bool)
        far = _edge_distance(px, py, poly) > 0.25
        assert np.array_equal(got[far], _point_in_polygon(px, py, poly)[far])


def test_packer_rejects_bad_polygons():
    ok = [[0, 0, 10, 0, 10, 10]]
    assert ops.pack_polygons([[ok]])[3].dtype == np.float32
    for bad in ([[0, 0, 10, 0]], [[0, 0, 10, 0, 10]], [[0, 0, 10, 0, 10, 10, 5]], [[0, 0, np.nan, 0, 10, 10]],
                [[0, 0, np.inf, 0, 10, 10]], [[0, 0, 2 ** 20 + 1, 0, 10, 10]], [], {"counts": "x", "size": [1, 1]}):
        with pytest.raises(ValueError):
            ops.pack_polygons([[ok, bad]])
    ob, pb, cb, co = ops.pack_polygons([[ok, [ok[0], [1, 1, 2, 2, 3, 1]]], [], [ok]])
    assert ob.tolist() == [0, 2, 2, 3] and pb.tolist() == [0, 1, 3, 4] and cb.tolist() == [0, 6, 12, 18, 24]


def test_abi_argument_errors_return_einval():
    lib = _lib.load()
    fake = 256                                                            # never dereferenced: every call fails its checks first
    ob = (ctypes.c_int * 2)(0, 1)

    def call(rois=fake, img=fake, cls=fake, R=1, N=1, ob=ob, P=1, pb=fake, C=6, cb=fake, co=fake, M=14, K=81, boxes=fake, out=fake):
        return lib.b200_mask_targets(rois, img, cls, R, N, ob, P, pb, C, cb, co, M, K, boxes, out, None)
    assert call(rois=None) == EINVAL
    assert call(cls=None) == EINVAL
    assert call(ob=None) == EINVAL
    assert call(co=None) == EINVAL
    assert call(out=None) == EINVAL
    assert call(R=0) == EINVAL
    assert call(N=0) == EINVAL
    assert call(N=65) == EINVAL
    assert call(M=0) == EINVAL
    assert call(M=65) == EINVAL
    assert call(K=-1) == EINVAL
    assert call(C=5) == EINVAL                                            # an odd coordinate count
    assert call(ob=(ctypes.c_int * 2)(1, 1)) == EINVAL
    assert call(ob=(ctypes.c_int * 3)(0, 2, 1), N=2) == EINVAL            # decreasing table
    assert call(P=0) == EINVAL                                            # an object without polygons
    assert call(out=fake + 4) == EINVAL                                   # a row of 81 * 196 needs 16-byte aligned masks
    assert call(rois=fake + 4) == EINVAL


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def run_device(c):
    p = case(c)
    blobs = dict(labels_int32=torch.from_numpy(p["labels"]).cuda())
    MR.add_mask_rcnn_blobs(blobs, torch.from_numpy(p["sampled"]).cuda(), p["roidb"], p["im_scale"], 1, resolution=p["M"],
                           cls_specific_mask=p["cls_specific"], num_classes=p["K"])
    return blobs


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_device_matches_reference_blobs(c):
    blobs = run_device(c)
    for k in BLOBS:
        ref = GOLD[c + "/" + k]
        got = blobs[k]
        assert got.is_cuda and tuple(got.shape) == ref.shape, k
        got = got.cpu().numpy()
        assert got.dtype == ref.dtype and np.array_equal(got, ref), k


@pytest.mark.gpu
def test_device_reads_cfg():
    class C:
        pass
    cfg = C(); cfg.MRCNN = C(); cfg.MODEL = C()
    cfg.MRCNN.RESOLUTION = 28; cfg.MRCNN.CLS_SPECIFIC_MASK = True; cfg.MODEL.NUM_CLASSES = 81
    p = case("m28_cls")
    blobs = dict(labels_int32=torch.from_numpy(p["labels"]).cuda())
    MR.add_mask_rcnn_blobs(blobs, torch.from_numpy(p["sampled"]).cuda(), p["roidb"], p["im_scale"], 1, cfg=cfg)
    assert np.array_equal(blobs["masks_int32"].cpu().numpy(), GOLD["m28_cls/masks_int32"])


def train_inputs():
    g = {k[len("train/"):]: GOLD[k] for k in GOLD.files if k.startswith("train/")}
    inputs = [torch.from_numpy(g["rpn_rois_%d" % l]).cuda() for l in range(5)] + [torch.from_numpy(g["rpn_probs_%d" % l]).cuda()
                                                                                  for l in range(5)]
    roidb = []
    for i in range(2):
        n = g["gt_%d" % i].shape[0]
        roidb.append(dict(boxes=g["gt_%d" % i], gt_classes=g["gt_classes_%d" % i], is_crowd=np.zeros(n, bool),
                          segms=unpack(g["poly_begin_%d" % i], g["coord_begin_%d" % i], g["coords_%d" % i], np.zeros(n, bool))))
    train = dict(BATCH_SIZE_PER_IM=128, FG_FRACTION=0.25, FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.0, NUM_CLASSES=81,
                 BBOX_REG_WEIGHTS=(10.0, 10.0, 5.0, 5.0), CLS_AGNOSTIC_BBOX_REG=False)
    choices = [(g["fg_choice_%d" % i], g["bg_choice_%d" % i]) for i in range(2)]
    return g, inputs, roidb, train, choices


@pytest.mark.gpu
def test_collect_and_distribute_training_branch_with_masks_vs_reference_op():
    from detectron.pytorch_b200.modeling.collect_and_distribute_fpn_rpn_proposals import CollectAndDistributeFpnRpnProposalsOp
    g, inputs, roidb, train, choices = train_inputs()
    op = CollectAndDistributeFpnRpnProposalsOp(rpn_min_level=2, rpn_max_level=6, roi_min_level=2, roi_max_level=5, post_nms_topN=600)
    op.train()
    plain = op(inputs, roidb, g["im_info"], choices=choices, train=train)
    blobs = op(inputs, roidb, g["im_info"], choices=choices, train=dict(train, MASK_ON=True, MRCNN_RESOLUTION=14, CLS_SPECIFIC_MASK=True))
    ref_keys = sorted(k[len("blob_"):] for k in g if k.startswith("blob_"))
    assert sorted(k for k in blobs if k != "counts") == ref_keys
    for k in ref_keys:
        got, ref = blobs[k].cpu().numpy(), g["blob_" + k]
        if k == "bbox_targets":
            np.testing.assert_allclose(got, ref, rtol=2e-6, atol=1e-7)
        else:
            assert got.dtype == ref.dtype and np.array_equal(got, ref), k
    for k, v in plain.items():                                               # every key of the plain branch is unchanged
        assert np.array_equal(blobs[k].cpu().numpy() if torch.is_tensor(v) else blobs[k], v.cpu().numpy() if torch.is_tensor(v) else v), k
    assert not any(k.startswith("mask") for k in plain)
    assert not any(k.startswith("mask") for k in op(inputs, roidb, g["im_info"], choices=choices, train=dict(train, MASK_ON=False)))


def coco_image(rng, n_obj=20, h=800, w=1333, n_fg=128):
    segms, boxes = [], []
    for _ in range(n_obj):
        cx, cy = rng.uniform(0, w), rng.uniform(0, h)
        rx, ry = rng.uniform(10, 250), rng.uniform(10, 250)
        polys = []
        for _ in range(int(rng.randint(1, 4))):
            k = int(rng.randint(20, 201))
            a = np.sort(rng.uniform(0, 2 * np.pi, k)); r = rng.uniform(0.3, 1.0, k)
            ox, oy = rng.uniform(-0.5, 0.5) * rx, rng.uniform(-0.5, 0.5) * ry
            polys.append(np.stack([cx + ox + rx * r * np.cos(a), cy + oy + ry * r * np.sin(a)], 1).ravel().tolist())
        segms.append(polys)
    pb = OM.polys_to_boxes(segms)
    src = rng.randint(0, n_obj, n_fg)
    sampled = (pb[src] + rng.standard_normal((n_fg, 4)).astype(np.float32) * np.float32(15)).astype(np.float32)
    sampled[:, 2:] = np.maximum(sampled[:, 2:], sampled[:, :2])
    classes = rng.randint(1, 81, n_obj).astype(np.int32)
    return dict(segms=segms, gt_classes=classes, is_crowd=np.zeros(n_obj, bool)), sampled, rng.randint(1, 81, n_fg).astype(np.int32)


def coco_step(seed=0):
    rng = np.random.RandomState(seed)
    return [coco_image(rng) for _ in range(2)]


@pytest.mark.gpu
def test_device_matches_oracle_at_coco_scale():
    """2 images of 800 x 1333, 128 fg RoIs each, 20 objects of 1-3 polygons of 20-200 vertices, M = 28, 81 classes."""
    step = coco_step()
    labels, rois, boxes, roidb, ref = [], [], [], [], []
    for n, (entry, sampled, lab) in enumerate(step):
        bl = OM.add_mask_rcnn_blobs(dict(labels_int32=lab), sampled, entry, 1.5, n, M=28, cls_specific=True, num_classes=81)
        ref.append(bl)
        labels.append(torch.from_numpy(lab).cuda()); boxes.append(torch.from_numpy(sampled).cuda())
        rois.append(torch.from_numpy(bl["mask_rois"]).cuda()); roidb.append(entry)
    out = MR.mask_rcnn_blobs(labels, rois, boxes, [l.numel() for l in labels], roidb, 28, True, 81)
    for k in BLOBS:
        assert np.array_equal(out[k].cpu().numpy(), np.concatenate([r[k] for r in ref])), k


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_rasteriser_stress_vs_oracle(seed):
    """Random polygons through the device rasteriser (class-agnostic, one object per RoI): shallow / steep and flipped edges,
    vertices on 0.1 and 0.5 multiples, duplicates, negative and far-outside coordinates, RoIs narrower than 1 px."""
    rng = np.random.RandomState(100 + seed)
    M = [7, 14, 28, 64][seed]
    segms, rois = [], []
    for i in range(300):
        mode = i % 5
        polys = []
        for _ in range(int(rng.randint(1, 4))):
            k = int(rng.randint(3, 40))
            if mode == 0:
                p = rng.uniform(0, 100, 2 * k)
            elif mode == 1:
                p = np.round(rng.uniform(-20, 120, 2 * k) * 10) / 10
            elif mode == 2:
                p = np.round(rng.uniform(-20, 120, 2 * k) * 2) / 2
            elif mode == 3:
                p = rng.uniform(-5000, 5000, 2 * k)
            else:
                p = rng.uniform(40, 60, 2 * k)
            if rng.rand() < 0.3:
                j = int(rng.randint(0, k - 1)); p[2 * j + 2:2 * j + 4] = p[2 * j:2 * j + 2]
            polys.append(p.astype(np.float32).tolist())
        segms.append(polys)
        x0, y0 = rng.uniform(-10, 90), rng.uniform(-10, 90)
        wd, ht = (rng.uniform(0.1, 0.9), rng.uniform(0.1, 0.9)) if i % 7 == 0 else (rng.uniform(1, 80), rng.uniform(1, 80))
        rois.append([x0, y0, x0 + wd, y0 + ht])
    rois = np.asarray(rois, np.float32)
    # one image per RoI would exceed 64 images: RoI i sees only object i through a single-object "image" of its own, so run in
    # chunks of 64 images
    got = []
    for s in range(0, len(segms), 64):
        part = segms[s:s + 64]
        got.append(ops.mask_targets_raw(torch.from_numpy(rois[s:s + 64]).cuda(), list(range(len(part))),
                                        torch.ones(len(part), dtype=torch.int32, device="cuda"), ops.pack_polygons([[o] for o in part]), M,
                                        0).cpu().numpy())
    got = np.concatenate(got).reshape(-1, M, M)
    for i, polys in enumerate(segms):
        assert np.array_equal(got[i], OM.polys_to_mask_wrt_box(polys, rois[i], M)), i


@pytest.mark.gpu
def test_one_call_makes_a_fixed_number_of_launches():
    """Boxes + targets: 2 launches whatever the number of images, RoIs, objects or vertices."""
    for c in CASES:
        p = case(c)
        blobs = dict(labels_int32=torch.from_numpy(p["labels"]).cuda())
        sampled = torch.from_numpy(p["sampled"]).cuda()
        torch.cuda.synchronize()
        before = _lib.launch_count()
        fg = np.where(p["labels"] > 0)[0]
        nf = fg.size
        order = torch.from_numpy(fg if nf else np.where(p["labels"] == 0)[0][:1]).cuda()
        MR.mask_rcnn_blobs([blobs["labels_int32"][order]], [torch.zeros((order.numel(), 5), device="cuda")], [sampled[order]], [nf],
                           [p["roidb"]], p["M"], p["cls_specific"], p["K"])
        torch.cuda.synchronize()
        assert _lib.launch_count() - before == 2, c
    step = coco_step(1)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    MR.mask_rcnn_blobs([torch.from_numpy(l).cuda() for _, _, l in step], [torch.zeros((128, 5), device="cuda")] * 2,
                       [torch.from_numpy(s).cuda() for _, s, _ in step], [128, 128], [e for e, _, _ in step], 28, True, 81)
    torch.cuda.synchronize()
    assert _lib.launch_count() - before == 2


@pytest.mark.gpu
def test_errors():
    p = case("m14_cls")
    lab = torch.from_numpy(p["labels"]).cuda()
    sampled = torch.from_numpy(p["sampled"]).cuda()
    no_poly = dict(p["roidb"], is_crowd=np.ones_like(p["roidb"]["is_crowd"]))
    with pytest.raises(ValueError):                                           # fg RoIs, no non-crowd polygon
        MR.add_mask_rcnn_blobs(dict(labels_int32=lab), sampled, no_poly, 1.0, 0, num_classes=81)
    with pytest.raises(ValueError):                                           # no RoI at all
        MR.add_mask_rcnn_blobs(dict(labels_int32=lab[:0]), sampled[:0], p["roidb"], 1.0, 0, num_classes=81)
    with pytest.raises(NotImplementedError):
        MR.add_mask_rcnn_blobs(dict(labels_int32=lab.cpu()), sampled.cpu(), p["roidb"], 1.0, 0, num_classes=81)
    bad = dict(p["roidb"], segms=[[[0, 0, 1, 1]]] * len(p["roidb"]["segms"]))
    with pytest.raises(ValueError):                                           # a 4-value "polygon"
        MR.add_mask_rcnn_blobs(dict(labels_int32=lab), sampled, bad, 1.0, 0, num_classes=81)
    with pytest.raises(ValueError):                                           # M beyond 64
        MR.add_mask_rcnn_blobs(dict(labels_int32=lab), sampled, p["roidb"], 1.0, 0, resolution=65, num_classes=81)


@pytest.mark.gpu
def test_mask_loss_on_device_blob_matches_reference_formula():
    from detectron.pytorch_b200.modeling.mask_rcnn_heads import mask_rcnn_losses
    blobs = run_device("m28_cls")
    masks = blobs["masks_int32"]
    torch.manual_seed(0)
    pred = torch.randn((masks.size(0), 81, 28, 28), device="cuda")
    got = mask_rcnn_losses(pred, masks, weight_loss_mask=0.5)
    # the reference's formula (mask_rcnn_heads.py:90-99) on the numpy blob, in float64
    gt = GOLD["m28_cls/masks_int32"].astype("float32").astype(np.float64)
    x = pred.cpu().numpy().reshape(masks.size(0), -1).astype(np.float64)
    w = (gt > -1).astype(np.float64)
    bce = np.maximum(x, 0) - x * gt + np.log1p(np.exp(-np.abs(x)))
    ref = (bce * w).sum() / w.sum() * 0.5
    assert abs(float(got) - ref) <= 1e-5 * abs(ref)
