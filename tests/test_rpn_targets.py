"""RPN anchor labels and box-regression targets (add_rpn_blobs, lib/roi_data/rpn.py:40-261) on the device.

CPU: the numpy oracle against the blobs of the UNMODIFIED reference function (tests/golden/rpn.npz, make_golden_rpn.py), the
package's cell anchors against the reference's generate_anchors, and the C ABI's argument checks.
GPU: the device blobs against the same goldens with the recorded draws (labels and weights bit-exact; targets dx / dy exact,
dw / dh within 2e-6 relative: CUDA logf vs numpy's float32 log), against the oracle at COCO scale, the device draw, the launch
count and the errors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import _lib
from detectron.pytorch_b200.roi_data import rpn as RPN
from oracle import rpn as OR
from oracle.targets import bbox_overlaps

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "rpn.npz"))
CASES = ["fpn2", "tiny", "zero", "single", "fewbg"]
EINVAL = -1
SINGLE_SIZES = (32, 64, 128)                                   # RPN.SIZES of the golden single-level cases


def case_params(c):
    fpn, max_size, straddle, batch = [int(v) for v in GOLD[c + "/cfg"]]
    return dict(multilevel_rpn=bool(fpn), max_size=max_size, straddle_thresh=straddle, batch_size_per_im=batch, rpn_sizes=SINGLE_SIZES)


def case_inputs(c):
    scales = GOLD[c + "/scales"].tolist()
    roidb, choices, i = [], [], 0
    while (c + "/boxes_%d" % i) in GOLD:
        h, w = [int(v) for v in GOLD[c + "/hw_%d" % i]]
        roidb.append(dict(height=h, width=w, boxes=GOLD[c + "/boxes_%d" % i], gt_classes=GOLD[c + "/gt_classes_%d" % i],
                          is_crowd=GOLD[c + "/is_crowd_%d" % i]))
        choices.append((GOLD[c + "/fg_disable_%d" % i], GOLD[c + "/bg_enable_%d" % i]))
        i += 1
    return scales, roidb, choices


def blob_names(c):
    return [k[len(c) + 6:] for k in GOLD.files if k.startswith(c + "/blob_")]


def oracle_params(p):
    return dict(straddle_thresh=p["straddle_thresh"], batch_size_per_im=p["batch_size_per_im"])


def assert_targets_close(got, ref):
    """(N, 4A, F, F) targets: dx / dy exact, dw / dh within 2e-6 relative, zeros where the reference has zeros."""
    N, C, F, _ = ref.shape
    got = got.reshape(N, C // 4, 4, F, F); ref = ref.reshape(N, C // 4, 4, F, F)
    assert np.array_equal(got == 0, ref == 0)
    assert np.array_equal(got[:, :, :2], ref[:, :, :2])
    np.testing.assert_allclose(got, ref, rtol=2e-6, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES)
def test_oracle_matches_reference_blobs(c):
    p = case_params(c)
    scales, roidb, choices = case_inputs(c)
    blobs, draws, _ = OR.add_rpn_blobs(scales, roidb, RPN.anchor_levels(**p), choices=choices, **oracle_params(p))
    for k in blob_names(c):
        ref = GOLD[c + "/blob_" + k]
        assert blobs[k].dtype == ref.dtype and np.array_equal(blobs[k], ref), k
    for (d, e), (gd, ge) in zip(draws, choices):
        assert np.array_equal(d, gd) and np.array_equal(e, ge)


def test_golden_cases_hold_the_reference_quirks():
    """The cases pin what they are meant to: several anchors tied at a column maximum below RPN_POSITIVE_OVERLAP, fg anchors
    relabelled 0 by the bg draw that keep their targets, the fg subsample, and a minibatch with no label 0."""
    lab = GOLD["tiny/blob_rpn_labels_int32_wide_fpn2"]
    tg = GOLD["tiny/blob_rpn_bbox_targets_wide_fpn2"]
    N, A, F, _ = lab.shape
    kept = (tg.reshape(N, A, 4, F, F) != 0).any(axis=2)
    assert ((lab == 0) & kept).any()
    assert GOLD["zero/fg_disable_0"].size > 0
    assert not any((GOLD[k] == 0).any() for k in GOLD.files if k.startswith("fewbg/blob_rpn_labels"))
    assert GOLD["fewbg/bg_enable_0"].size == 0
    box = np.asarray([[42, 62, 85, 97]], np.float32)
    lv = [l for l in RPN.anchor_levels(**case_params("fpn2")) if l[0] == 2][0]
    ov = bbox_overlaps(OR.field_of_anchors(lv[1], lv[2], lv[3]), box)[:, 0]
    assert (ov == ov.max()).sum() == 8 and ov.max() < np.float32(0.7)


@pytest.mark.parametrize("i", range(6))
def test_cell_anchors_match_reference(i):
    g = "anchors/%d/" % i
    out = RPN.generate_anchors(float(GOLD[g + "stride"]), tuple(GOLD[g + "sizes"]), tuple(GOLD[g + "ratios"]))
    assert out.dtype == np.float64 and np.array_equal(out, GOLD[g + "out"])


@pytest.mark.parametrize("c", CASES)
def test_blob_names_match_reference(c):
    names = RPN.get_rpn_blob_names(True, **case_params(c))
    assert names[:2] == ["im_info", "roidb"] and sorted(names[2:] + ["im_info"]) == sorted(blob_names(c))


def _tables(L=1, F=(8,), A=(1,)):
    Fa = (ctypes.c_int * L)(*F); Aa = (ctypes.c_int * L)(*A)
    S = (ctypes.c_double * L)(*([16.0] * L)); C = (ctypes.c_double * (4 * sum(A)))(*([0.0, 0.0, 15.0, 15.0] * sum(A)))
    return Fa, Aa, S, C


def test_abi_argument_errors_return_einval():
    lib = _lib.load()
    F, A, S, C = _tables()
    im = (ctypes.c_double * 2)(64.0, 64.0)
    gb = (ctypes.c_int * 2)(0, 1)
    fake = 256                                                            # never dereferenced: every call fails its checks first
    assert lib.b200_rpn_targets_workspace_bytes(1, F, A, 1, 1) > 0
    assert lib.b200_rpn_targets_workspace_bytes(0, F, A, 1, 1) == 0
    assert lib.b200_rpn_targets_workspace_bytes(1, F, A, 65, 1) == 0

    def labels(L=1, F=F, A=A, S=S, C=C, N=1, im=im, gb=gb, gt=fake, counts=fake):
        return lib.b200_rpn_labels(L, F, A, S, C, N, im, gb, gt, 0.0, 0.7, 0.3, counts, fake, 1 << 30, None)
    assert labels(L=0) == EINVAL
    assert labels(L=9) == EINVAL
    assert labels(N=0) == EINVAL
    assert labels(N=65) == EINVAL
    assert labels(gt=None) == EINVAL
    assert labels(counts=None) == EINVAL
    assert labels(F=None) == EINVAL
    assert labels(C=None) == EINVAL
    assert labels(im=None) == EINVAL
    assert labels(gb=(ctypes.c_int * 2)(0, 0)) == EINVAL                 # an image without ground truth
    assert labels(gb=(ctypes.c_int * 2)(1, 2)) == EINVAL
    F0, A0, _, _ = _tables(F=(0,))
    assert labels(F=F0) == EINVAL
    _, A33, _, C33 = _tables(A=(33,))
    assert labels(A=A33, C=C33) == EINVAL                                  # more than 32 cell anchors
    assert lib.b200_rpn_labels(1, F, A, S, C, 1, im, gb, fake, 0.0, 0.7, 0.3, fake, None, 0, None) == -2     # no workspace
    d0 = (ctypes.c_int * 2)(0, 0)
    ptrs = (ctypes.c_void_p * 1)(fake)

    def emit(dis_b=d0, en_b=d0, dis=fake, en=fake, outs=ptrs, counts=fake):
        return lib.b200_rpn_emit(1, F, A, S, C, 1, im, gb, fake, 0.0, counts, dis, dis_b, en, en_b, fake, 1 << 30, outs, outs, outs, outs,
                                 None)
    assert emit(counts=None) == EINVAL
    assert emit(dis_b=None) == EINVAL
    assert emit(dis_b=(ctypes.c_int * 2)(0, 3), dis=None) == EINVAL       # draws but no draw buffer
    assert emit(en_b=(ctypes.c_int * 2)(2, 1)) == EINVAL                  # decreasing table
    assert emit(outs=(ctypes.c_void_p * 1)(None)) == EINVAL
    assert emit(outs=(ctypes.c_void_p * 1)(fake + 4)) == EINVAL           # F * F % 4 == 0 needs 16-byte aligned blobs


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def run_device(c, choices):
    p = case_params(c)
    scales, roidb, _ = case_inputs(c)
    names = RPN.get_rpn_blob_names(True, **p)
    blobs = {k: [] for k in names}
    assert RPN.add_rpn_blobs(blobs, scales, roidb, choices=choices, **p) is True
    return blobs, roidb


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_device_matches_reference_blobs(c):
    _, _, choices = case_inputs(c)
    blobs, roidb = run_device(c, choices)
    for k in blob_names(c):
        ref = GOLD[c + "/blob_" + k]
        got = blobs[k]
        if k == "im_info":
            assert isinstance(got, np.ndarray) and got.dtype == ref.dtype and np.array_equal(got, ref)
            continue
        assert got.is_cuda and tuple(got.shape) == ref.shape, k
        got = got.cpu().numpy()
        assert got.dtype == ref.dtype, k
        if "targets" in k:
            assert_targets_close(got, ref)
        else:
            assert np.array_equal(got, ref), k
    assert [sorted(e) for e in blobs["roidb"]] == [sorted(k for k in ("boxes", "gt_classes", "is_crowd") if k in e) for e in roidb]


def coco_image(seed, G, h, w):
    rng = np.random.RandomState(seed)
    cx, cy = rng.uniform(0, w, G), rng.uniform(0, h, G)
    bw, bh = np.exp(rng.uniform(np.log(4), np.log(w * 0.7), G)), np.exp(rng.uniform(np.log(4), np.log(h * 0.7), G))
    boxes = np.stack([np.clip(cx - bw / 2, 0, w - 1), np.clip(cy - bh / 2, 0, h - 1), np.clip(cx + bw / 2, 0, w - 1),
                      np.clip(cy + bh / 2, 0, h - 1)], 1).astype(np.float32)
    classes = rng.randint(0, 81, G).astype(np.int32)
    classes[0] = 1
    crowd = rng.uniform(size=G) < 0.05
    crowd[0] = False
    return dict(height=h, width=w, boxes=boxes, gt_classes=classes, is_crowd=crowd)


@pytest.mark.gpu
def test_device_matches_oracle_at_coco_scale():
    """TRAIN.MAX_SIZE 1333, FPN P2-P6 (451 143 anchors per image), two images with 100 and 7 ground-truth boxes, the oracle's
    numpy draw injected."""
    p = dict(multilevel_rpn=True, max_size=1333)
    roidb = [coco_image(1, 100, 480, 640), coco_image(2, 7, 427, 640)]
    scales = [800 / 480.0, 1.8]
    ref, draws, counts = OR.add_rpn_blobs(scales, roidb, RPN.anchor_levels(**p), rng=np.random.RandomState(3))
    assert sum(d.size for d, _ in draws) > 0 and all(e.size > 0 for _, e in draws)
    blobs = {}
    RPN.add_rpn_blobs(blobs, scales, roidb, choices=draws, **p)
    assert np.array_equal(blobs["im_info"], ref["im_info"])
    for k, v in ref.items():
        if k == "im_info":
            continue
        got = blobs[k].cpu().numpy()
        if "targets" in k:
            assert_targets_close(got, v)
        else:
            assert np.array_equal(got, v), k


def candidates(c):
    """Per image of golden case c: (fg candidate mask, bg candidate mask) over the concatenated anchors, from the oracle's IoU."""
    p = case_params(c)
    levels = RPN.anchor_levels(**p)
    scales, roidb, _ = case_inputs(c)
    anchors = np.concatenate([OR.field_of_anchors(F, s, a) for _, F, s, a in levels])
    out = []
    for e, sc in zip(roidb, scales):
        keep = (e["gt_classes"] > 0) & (e["is_crowd"] == 0)
        ov = bbox_overlaps(anchors, e["boxes"][keep] * sc)
        h, w = np.round(e["height"] * sc), np.round(e["width"] * sc)
        inside = (anchors[:, 0] >= 0) & (anchors[:, 1] >= 0) & (anchors[:, 2] < w) & (anchors[:, 3] < h)
        mx = ov.max(axis=1)
        colmax = ov[inside].max(axis=0)
        fg = inside & (((ov == colmax).any(axis=1)) | (mx >= np.float32(0.7)))
        out.append((fg, inside & (mx < np.float32(0.3))))
    return levels, out


def flat(blob, levels, key, n):
    """Image n's blob `key` of every level in the reference's concatenated anchor order (level, h, w, a); (T,) or (T, 4)."""
    parts = []
    for lvl, F, _, a in levels:
        A = a.shape[0]
        t = blob[key + "_fpn%d" % lvl].cpu().numpy()[n]
        parts.append(t.transpose(1, 2, 0).reshape(F * F * A, -1) if "labels" in key else
                     t.reshape(A, 4, F, F).transpose(2, 3, 0, 1).reshape(F * F * A, 4))
    return np.concatenate(parts).squeeze()


@pytest.mark.gpu
def test_device_draw_gives_a_valid_minibatch():
    torch.manual_seed(0)
    c = "fpn2"
    blobs, _ = run_device(c, None)
    levels, cands = candidates(c)
    for n, (fg, bg) in enumerate(cands):
        lab = flat(blobs, levels, "rpn_labels_int32_wide", n)
        inside = flat(blobs, levels, "rpn_bbox_inside_weights_wide", n)
        outside = flat(blobs, levels, "rpn_bbox_outside_weights_wide", n)
        tg = flat(blobs, levels, "rpn_bbox_targets_wide", n)
        assert (lab == 1).sum() <= 128 and (lab >= 0).sum() <= 256
        assert fg[lab == 1].all() and bg[lab == 0].all()
        assert (lab[~(fg | bg)] == -1).all()
        if bg.sum() > 256 - min(fg.sum(), 128):
            assert (lab == 0).sum() > 0
        ne = int((lab >= 0).sum())
        assert np.array_equal(outside, np.where((lab >= 0)[:, None], np.float32(1.0 / ne), np.float32(0)) * np.ones((1, 4), np.float32))
        assert np.array_equal(inside, np.repeat((lab == 1)[:, None], 4, axis=1).astype(np.float32))
        assert ((tg != 0).any(axis=1) <= fg).all() and (tg[lab == 1] != 0).any(axis=1).all()


@pytest.mark.gpu
def test_one_call_makes_a_fixed_number_of_launches():
    """memset + 3 kernels to label, 3 to draw and emit, whatever the number of images and levels."""
    for c in ("fpn2", "single", "tiny"):
        _, _, choices = case_inputs(c)
        torch.cuda.synchronize()
        before = _lib.launch_count()
        run_device(c, choices)
        torch.cuda.synchronize()
        assert _lib.launch_count() - before == 7, c


@pytest.mark.gpu
def test_errors():
    p = case_params("fpn2")
    scales, roidb, choices = case_inputs("fpn2")
    bad = [dict(e) for e in roidb]
    bad[1]["gt_classes"] = np.zeros_like(bad[1]["gt_classes"])             # nothing eligible
    with pytest.raises(ValueError):
        RPN.add_rpn_blobs({}, scales, bad, **p)
    bad = [dict(e) for e in roidb]
    bad[0]["is_crowd"] = np.ones_like(bad[0]["is_crowd"])
    with pytest.raises(ValueError):
        RPN.add_rpn_blobs({}, scales, bad, **p)
    small = [dict(roidb[0], height=8, width=8)]                              # no anchor fits inside an 8 x 8 image
    with pytest.raises(ValueError):
        RPN.add_rpn_blobs({}, scales[:1], small, **p)
    with pytest.raises(ValueError):                                          # a draw of the wrong size
        RPN.add_rpn_blobs({}, scales, roidb, choices=[(c[0], c[1][:-1]) for c in choices], **p)
    with pytest.raises(ValueError):                                          # a position outside the candidate list
        RPN.add_rpn_blobs({}, scales, roidb, choices=[(c[0], c[1] + 10 ** 6) for c in choices], **p)
    gt = torch.from_numpy(roidb[0]["boxes"][:3])
    with pytest.raises(NotImplementedError):
        RPN.rpn_targets([gt], np.array([[200.0, 300.0, 1.0]]), **p)
    with pytest.raises(ValueError):
        RPN.rpn_targets([gt.cuda()[:0]], np.array([[200.0, 300.0, 1.0]]), **p)
