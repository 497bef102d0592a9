"""Test-time augmentation of the mask and keypoint heads (im_detect_mask_aug / im_detect_keypoints_aug, lib/core/test.py:365-729)
and the width-relative aspect-ratio resize (aspect_ratio_rel, lib/utils/image.py:27-32).

CPU: oracle/test_aug.py's running combine against the combined outputs of the UNMODIFIED reference (tests/golden/test_aug.npz,
make_golden_test_aug.py), the oracle resize against cv2.resize itself (IPP off), the package's host rois / FPN blobs against
the reference's, and the keypoint flip permutation against the reference's flip_heatmaps.
GPU: the package's functions driven by the same record / replay model make the same calls with the same blobs and return the
golden results; the kernels equal the oracle at COCO sizes; aspect_ratio_rel on the device equals the oracle; the combined
masks and heatmaps go into segm_results / keypoint_results as CUDA tensors.

LOGIT_AVG is compared within LOGIT_ULPS ulps: the device rounds log and exp once from double, numpy's SIMD float32 log / exp are
not correctly rounded.  The logit of a float32 y in [1e-20, 1) is at most 46.06 in magnitude, so one ulp of difference in a
transform's logit moves the logit mean m by up to 46.06 * 2^-23 (2^-23 the float32 epsilon), and the sigmoid carries an error
dm in m into a relative error of at most dm in the result: 4 rounding ulps plus 4 * 46.06 ulps for two such differences."""
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200.core import test as T
from detectron.pytorch_b200.utils import boxes as box_utils
from detectron.pytorch_b200.utils import keypoints as kp_utils
from oracle import test_aug as O
from tests import tta_cases as cases

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "test_aug.npz"))
LOGIT_ULPS = 4 + 4 * 47
NAMES = sorted(cases.CASES)


def _ulps(a, b):
    a = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(a - b)


def _assert_matches(got, want, heur):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32
    if heur == "LOGIT_AVG":
        assert np.array_equal(np.isnan(got), np.isnan(want))
        fin = ~np.isnan(want)
        ulps = _ulps(got[fin], want[fin]).max(initial=0)
        assert ulps <= LOGIT_ULPS, "LOGIT_AVG differs from numpy by %d ulps" % ulps
    else:
        nan = np.isnan(want)                                                      # NaN payloads are not compared
        assert np.array_equal(np.isnan(got), nan)
        assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))   # bit for bit, signed zeros included


def _case_outputs(case):
    ts = cases.transforms(case)
    C = cases.head_channels(case)
    outs = [cases.head_output(case["seed"], i, (case["R"], C, case["M"], case["M"])) for i in range(len(ts))]
    perm = kp_utils.flip_permutation(C) if case["kind"] == "keypoints" else None
    b = cases.boxes(case["seed"], case["R"])
    includes = [T._size_dep_include(b, ds, us, cases.AREA_TH) if case["size_dep"] else None for (_, ds, us, _, _, _) in ts]
    return outs, [t[0] for t in ts], [perm if t[0] else None for t in ts], includes


def _params(case):
    return T._aug_params(None, dict(num_classes=case["num_classes"], resolution=case["M"], cls_specific_mask=case["cls_specific"],
                                    num_keypoints=case["J"], heatmap_size=case["M"], test_scale=case["test_scale"],
                                    test_max_size=case["test_max_size"], multilevel_rois=case["fpn"],
                                    mask_aug={k.lower(): v for k, v in cases.aug_cfg(case).items() if k != "ENABLED"},
                                    kps_aug={k.lower(): v for k, v in cases.aug_cfg(case).items() if k != "ENABLED"},
                                    fpn_on=case["fpn"], coarsest_stride=32))


def _golden_rois(name, i):
    prefix = "%s/h%d/" % (name, i)
    return {k[len(prefix):]: GOLD[k] for k in GOLD.files if k.startswith(prefix)}


# ---------------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", NAMES)
def test_oracle_combine_matches_reference(name):
    case = cases.CASES[name]
    outs, hflips, perms, includes = _case_outputs(case)
    _assert_matches(O.combine(outs, case["heur"], hflips, perms, includes), GOLD[name + "/out"], case["heur"])


def test_golden_cases_cover_the_edges():
    outs = [GOLD[n + "/out"] for n in NAMES]
    assert any(np.any(np.signbit(o) & (o == 0)) for o in outs)                   # a -0.0 survives (SOFT_MAX / HM_MAX)
    assert any(np.any(o == 1.0) for o in outs) and any(np.any(o == 0.0) for o in outs)
    kinds = {(cases.CASES[n]["kind"], cases.CASES[n]["heur"], cases.CASES[n]["aug"]) for n in NAMES}
    for heur in ("SOFT_AVG", "SOFT_MAX", "LOGIT_AVG"):
        assert {("mask", heur, a) for a in ("hflip", "scales", "ratios")} <= kinds
    size_dep = [n for n in NAMES if cases.CASES[n]["size_dep"]]
    for n in size_dep:
        areas = box_utils_areas(cases.boxes(cases.CASES[n]["seed"], cases.CASES[n]["R"]))
        assert (areas < cases.AREA_TH).any() and (areas >= cases.AREA_TH).any()
    assert {cases.CASES[n]["R"] for n in NAMES} >= {1} and any(cases.CASES[n]["M"] % 2 for n in NAMES)


def box_utils_areas(b):
    return (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)


@pytest.mark.parametrize("name", NAMES)
def test_host_rois_and_fpn_blobs_match_reference(name):
    """The rois blob and the FPN level blobs of every head call, from the package's host code, equal the reference's."""
    case = cases.CASES[name]
    p = _params(case)
    from detectron.pytorch_b200.utils.blob import get_target_scale
    im_h, im_w = cases.IM_H, cases.IM_W
    b = cases.boxes(case["seed"], case["R"])
    key = "mask_rois" if case["kind"] == "mask" else "keypoint_rois"
    for i, (hflip, _, _, scale, max_size, ar) in enumerate(cases.transforms(case)):
        bx, w = b, im_w
        if ar is not None:
            bx, w = box_utils.aspect_ratio(bx, ar), int(round(ar * im_w))
        if hflip:
            bx = box_utils.flip_boxes(bx, w)
        s, m = (case["test_scale"], case["test_max_size"]) if scale is None else (scale, max_size)
        im_scale = get_target_scale(min(im_h, w), max(im_h, w), s, m)
        got = T._head_inputs(key, bx, im_scale, p)
        want = _golden_rois(name, i)
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), (i, k)


def test_keypoint_flip_permutation_matches_reference():
    coded = GOLD["flip_heatmaps/in"]
    perm = kp_utils.flip_permutation()
    assert np.array_equal(coded[:, perm][..., ::-1], GOLD["flip_heatmaps/out"])
    assert np.array_equal(O.transformed(coded, True, perm), GOLD["flip_heatmaps/out"])


def test_oracle_resize_matches_cv2_ipp_off():
    cv2 = pytest.importorskip("cv2")
    ipp = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        rng = np.random.RandomState(3)
        n = 0
        for _ in range(120):
            h, w = rng.randint(1, 70), rng.randint(1, 130)
            ar = rng.uniform(0.3, 2.5) if n % 4 else 1.0
            W = int(round(ar * w))
            if W < 1:
                continue
            im = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
            assert np.array_equal(O.resize_width_u8(im, W), cv2.resize(im, dsize=(W, h))), (h, w, W)
            n += 1
    finally:
        cv2.ipp.setUseIPP(ipp)


def test_abi_validates_arguments_without_gpu():
    from detectron.pytorch_b200 import _lib
    lib, EINVAL = _lib.load(), -1
    assert lib.b200_tta_combine(None, 16, 1, 1, 4, None, None, 1, 0, 0, None) == EINVAL
    assert lib.b200_tta_combine(16, 16, 1, 1, 4, None, None, 3, 0, 0, None) == EINVAL           # op neither start nor fold
    assert lib.b200_tta_combine(16, 16, 1, 1, 4, None, None, 1, 0, 3, None) == EINVAL           # unknown heuristic
    assert lib.b200_tta_combine(16, 16, 1, 0, 4, None, None, 1, 0, 0, None) == EINVAL
    assert lib.b200_tta_finish(16, 1, 1, 4, None, 0, 0, None) == EINVAL                         # no count
    assert lib.b200_tta_finish(None, 1, 1, 4, None, 1, 0, None) == EINVAL
    assert lib.b200_resize_width_u8(16, 8, 4, 4, 0, 16, None) == EINVAL                         # empty output
    assert lib.b200_resize_width_u8(16, 11, 4, 4, 4, 16, None) == EINVAL                        # pitch < 3 w
    assert lib.b200_resize_width_u8(None, 12, 4, 4, 4, 16, None) == EINVAL


def test_reference_errors_are_kept():
    with pytest.raises(AssertionError):
        T.im_detect_mask_aug(None, None, np.zeros((1, 4), np.float32), 1.0, None, mask_aug=dict(scale_size_dep=True))
    with pytest.raises(NotImplementedError):
        T.im_detect_mask_aug(None, None, np.zeros((1, 4), np.float32), 1.0, None, mask_aug=dict(heur="HM_AVG"))
    with pytest.raises(NotImplementedError):
        T.im_detect_keypoints_aug(None, None, np.zeros((1, 4), np.float32), 1.0, None, kps_aug=dict(heur="LOGIT_AVG"))


# ---------------------------------------------------------------------------------------------------------------------- GPU
def _cuda_model(case):
    return cases.ReplayModel(case, to_numpy=lambda t: t.detach().cpu().numpy(), wrap=lambda a: torch.from_numpy(a).cuda())


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_aug_matches_reference(name):
    case = cases.CASES[name]
    p = _params(case)
    model = _cuda_model(case)
    im = cases.image(case["seed"])
    b = cases.boxes(case["seed"], case["R"])
    blobs, im_scale = T.get_blobs(im, None, case["test_scale"], case["test_max_size"], fpn_on=case["fpn"], coarsest_stride=32)
    blob_conv = model.convbody_net(blobs["data"])
    fn = T.im_detect_mask_aug if case["kind"] == "mask" else T.im_detect_keypoints_aug
    out = fn(model, im, b, im_scale, blob_conv, **{k: v for k, v in p.items()})
    assert out.is_cuda
    assert list(model.calls) == [str(c) for c in GOLD[name + "/calls"]]
    for i, got in enumerate(model.rois):
        want = _golden_rois(name, i)
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), (i, k)
    _assert_matches(out.cpu().numpy(), GOLD[name + "/out"], case["heur"])


@pytest.mark.gpu
def test_device_combine_matches_numpy_at_mask_tta_size():
    """The X-152 mask TTA roster: 18 transforms of 100 x 81 x 28 x 28, every heuristic, against numpy's own reduction."""
    from detectron.pytorch_b200 import ops
    rng = np.random.RandomState(0)
    shape = (100, 81, 28, 28)
    outs = [rng.uniform(0, 1, shape).astype(np.float32) for _ in range(18)]
    for o in outs[::3]:
        o.reshape(-1)[::101] = 1.0
        o.reshape(-1)[::103] = np.nan
        o.reshape(-1)[::107] = -0.0
    hflips = [i % 2 == 1 for i in range(18)]
    dev = [torch.from_numpy(o).cuda() for o in outs]
    stacked = [o[..., ::-1] if hf else o for o, hf in zip(outs, hflips)]
    want = {"SOFT_AVG": np.mean(stacked, axis=0), "SOFT_MAX": np.amax(stacked, axis=0)}
    with np.errstate(divide="ignore", invalid="ignore"):
        want["LOGIT_AVG"] = (1.0 / (1.0 + np.exp(-np.mean([O.logit(y) for y in stacked], axis=0)))).astype(np.float32)
    for heur, w in want.items():
        acc = torch.empty(shape, dtype=torch.float32, device="cuda")
        for i, (d, hf) in enumerate(zip(dev, hflips)):
            ops.tta_combine_raw(d, acc, ops.TTA_HEURISTICS[heur], op=ops.TTA_START if i == 0 else ops.TTA_FOLD, hflip=hf)
        ops.tta_finish_raw(acc, ops.TTA_HEURISTICS[heur], count=18)
        _assert_matches(acc.cpu().numpy(), w, heur)


@pytest.mark.gpu
def test_device_size_dependent_keypoint_combine_matches_oracle():
    """100 x 17 x 56 x 56 heatmaps over 10 transforms with per-object selection and the keypoint flip."""
    rng = np.random.RandomState(1)
    R, shape = 100, (100, 17, 56, 56)
    b = rng.uniform(0, 400, (R, 2)).astype(np.float32)
    side = rng.uniform(10, 400, (R, 1)).astype(np.float32)
    bx = np.hstack([b, b + side]).astype(np.float32)
    flags = [(False, False, False), (True, False, False), (False, True, False), (True, True, False), (False, False, True),
             (True, False, True), (False, True, False), (False, False, True), (False, False, False), (True, False, False)]
    outs = [rng.standard_normal(shape).astype(np.float32) for _ in flags]
    perm = kp_utils.flip_permutation()
    incl = [T._size_dep_include(bx, ds, us, 180 ** 2) for _, ds, us in flags]
    assert any(not i.all() for i in incl)
    for heur in ("HM_AVG", "HM_MAX"):
        comb = T._RunningCombine(heur)
        for o, (hf, _, _), inc in zip(outs, flags, incl):
            comb.add(torch.from_numpy(o).cuda(), hflip=hf, perm=perm if hf else None, include=inc)
        got = comb.result().cpu().numpy()
        want = O.combine(outs, heur, [f[0] for f in flags], [perm if f[0] else None for f in flags], incl)
        _assert_matches(got, want, heur)
        # and the public combine_heatmaps_size_dep on already-flipped heatmaps
        flipped = [O.transformed(o, hf, perm if hf else None).copy() for o, (hf, _, _) in zip(outs, flags)]
        got2 = T.combine_heatmaps_size_dep([torch.from_numpy(f).cuda() for f in flipped], [f[1] for f in flags], [f[2] for f in flags],
                                           bx, heur, kps_aug=dict(area_th=180 ** 2))
        _assert_matches(got2.cpu().numpy(), want, heur)


@pytest.mark.gpu
def test_device_flip_heatmaps_and_odd_resolution():
    rng = np.random.RandomState(2)
    hm = rng.standard_normal((3, 17, 9, 9)).astype(np.float32)
    got = kp_utils.flip_heatmaps(torch.from_numpy(hm).cuda()).cpu().numpy()
    assert np.array_equal(got, O.transformed(hm, True, kp_utils.flip_permutation()))


@pytest.mark.gpu
def test_device_aspect_ratio_rel_matches_oracle():
    from detectron.pytorch_b200.utils.image import aspect_ratio_rel
    rng = np.random.RandomState(4)
    shapes = [(1, 1), (1, 7), (5, 1), (33, 47), (64, 96), (480, 640), (800, 1333)]
    ratios = [0.5, 0.75, 1.0, 1.3, 2.0, 0.5 / 0.7, 1.0 / 3]
    for h, w in shapes:
        im = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        for ar in ratios:
            W = int(round(ar * w))
            if W < 1:
                continue
            got = aspect_ratio_rel(im, ar)
            assert got.is_cuda and tuple(got.shape) == (h, W, 3)
            assert np.array_equal(got.cpu().numpy(), O.resize_width_u8(im, W)), (h, w, ar)
            # a CUDA input, and a strided one, give the same bytes
            assert torch.equal(aspect_ratio_rel(torch.from_numpy(im).cuda(), ar), got)
    wide = rng.randint(0, 256, (20, 50, 3)).astype(np.uint8)
    view = torch.from_numpy(wide).cuda()[:, 5:37]
    assert np.array_equal(aspect_ratio_rel(view, 1.5).cpu().numpy(), O.resize_width_u8(wide[:, 5:37], 48))


@pytest.mark.gpu
def test_combined_outputs_chain_into_segm_and_keypoint_results():
    """The CUDA results go straight into segm_results / keypoint_results and give what their numpy copies give."""
    for name in ("mask_soft_avg_scales", "kps_hm_avg_size_dep"):
        case = cases.CASES[name]
        p = _params(case)
        model = _cuda_model(case)
        im = cases.image(case["seed"])
        b = cases.boxes(case["seed"], case["R"])
        blobs, im_scale = T.get_blobs(im, None, case["test_scale"], case["test_max_size"], fpn_on=case["fpn"], coarsest_stride=32)
        fn = T.im_detect_mask_aug if case["kind"] == "mask" else T.im_detect_keypoints_aug
        out = fn(model, im, b, im_scale, model.convbody_net(blobs["data"]), **p)
        assert out.is_cuda
        R = case["R"]
        if case["kind"] == "mask":
            K = case["num_classes"]
            dets = np.hstack([b, np.linspace(0.9, 0.5, R, dtype=np.float32)[:, None]])
            cls_boxes = [[]] + [dets[j::K - 1] for j in range(K - 1)]
            order = np.concatenate([np.arange(R)[j::K - 1] for j in range(K - 1)])
            ref_boxes = np.vstack([c for c in cls_boxes[1:]])[:, :4]
            masks = out[torch.from_numpy(order).cuda()]
            got = T.segm_results(cls_boxes, masks, ref_boxes, cases.IM_H, cases.IM_W, num_classes=K, resolution=case["M"])
            want = T.segm_results(cls_boxes, masks.cpu().numpy(), ref_boxes, cases.IM_H, cases.IM_W, num_classes=K, resolution=case["M"])
            assert got == want and sum(len(s) for s in got) == R
        else:
            cls_boxes = [[], np.hstack([b, np.ones((R, 1), np.float32)])]
            got = T.keypoint_results(cls_boxes, out, b, num_classes=2)
            want = T.keypoint_results(cls_boxes, out.cpu().numpy(), b, num_classes=2)
            assert len(got[1]) == R and all(np.array_equal(g, w) for g, w in zip(got[1], want[1]))
