"""The box head's decode and test-time augmentation (im_detect_bbox / im_detect_bbox_aug, lib/core/test.py:127-362), the
reference's im_detect_all through install_reference_aliases(bbox=True, test_aug=True), and NMS at union size.

CPU: oracle/detect_bbox.py replays the golden model calls and equals the UNMODIFIED reference's results bit for bit
(tests/golden/detect_bbox.npz, make_golden_bbox.py); the package's host rois / FPN / im_info blobs and call order equal the
reference's; the ABI rejects bad arguments.
GPU: the package's functions driven by the same record / replay model make the same calls with the same blobs and return the
golden results; the decode equals the oracle at the X-152 load; the reference's im_detect_all with the aliases returns the
golden cls_boxes; one class of 14 000 and 18 000 candidates goes through box_results_with_nms_and_limit.

Pass bar for boxes: scores are compared bit for bit; boxes are >= 99.9 % bit-equal and every coordinate lies within one
float32 ulp of the largest coordinate magnitude in the comparison.  Derivation: the decode's only operation that is not
correctly rounded on both sides is the float64 exp (CUDA's and numpy's may differ in the last double bit).  That moves
exp(dw) * w by a relative 2^-52, and the sum `ctr -/+ 0.5 * pred_w (- 1)` by far less than half a float32 ulp of the result,
so the float32 rounding can change by at most one ulp of the coordinate, which is at most one ulp of the largest one.  The
clip, flip and aspect inverse are single correctly rounded float32 (or float64) operations on both sides and cannot widen a
one-ulp difference beyond one ulp of the largest coordinate."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import ops
from detectron.pytorch_b200.core import test as T
from detectron.pytorch_b200.utils import boxes as box_utils
from detectron.pytorch_b200.utils.blob import get_target_scale
from oracle import detect_bbox as O
from oracle import detections as OD
from tests import bbox_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "detect_bbox.npz"))
NAMES = sorted(cases.CASES)


def _blobs(name, i):
    prefix = "%s/c%d/" % (name, i)
    return {k[len(prefix):]: GOLD[k] for k in GOLD.files if k.startswith(prefix)}


def _want_boxes(name):
    """The reference's boxes as float32: without BBOX_REG under FASTER_RCNN its boxes stay float64 (rois / im_scale, flipped and
    aspect-scaled in float64); the package returns float32 throughout, rounded once from the same float64 values."""
    return GOLD[name + "/boxes"].astype(np.float32, copy=False)


def _assert_boxes(got, want, what=""):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype == np.float32, (what, got.shape, want.shape, got.dtype)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    if not want.size:
        return
    g, w = got[~nan], want[~nan]
    assert np.array_equal(np.isinf(g), np.isinf(w)), what
    fin = np.isfinite(w)
    equal = np.mean(g.view(np.uint32) == w.view(np.uint32))
    assert equal >= 0.999, "%s: %.5f of the coordinates bit-equal" % (what, equal)
    if fin.any():
        ulp = np.spacing(np.abs(w[fin]).max())
        assert np.abs(g[fin].astype(np.float64) - w[fin]).max() <= ulp, what


def _transform_inputs(case, t):
    """(image h, w, im_scale, the proposals the model sees or None) of transform t = (hflip, scale, max_size, ar)."""
    hflip, scale, max_size, ar = t
    h, w = cases.IM_H, cases.IM_W
    props = None if case["faster"] else cases.proposals(case["seed"], case["R"])
    if ar is not None:
        w = int(round(ar * w))
        props = None if props is None else box_utils.aspect_ratio(props, ar)
    if hflip and props is not None:
        props = box_utils.flip_boxes(props, w)
    return h, w, get_target_scale(min(h, w), max(h, w), scale, max_size), props


def _dedup(rois, dedup):
    if not dedup:
        return np.arange(rois.shape[0]), np.arange(rois.shape[0])
    hashes = np.round(rois * (1. / 16.)).dot(np.array([1, 1e3, 1e6, 1e9, 1e12]))
    _, index, inv = np.unique(hashes, return_index=True, return_inverse=True)
    return index, inv.reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    """The oracle decode of every golden model call, combined by the case's heuristics, equals the reference bit for bit."""
    case = cases.CASES[name]
    ts = cases.transforms(case)
    assert len(GOLD[name + "/calls"]) == len(ts)
    scores_ts, boxes_ts = [], []
    for i, t in enumerate(ts):
        h, w, im_scale, props = _transform_inputs(case, t)
        blobs = _blobs(name, i)
        Hp, Wp = int(blobs["im_info"][0, 0]), int(blobs["im_info"][0, 1])
        if case["faster"]:
            R = case["R"]
        else:
            index, inv = _dedup(T._get_rois_blob(props, im_scale), case["dedup"])
            R = len(index)
        rois, scores, deltas = cases.head_outputs(case["seed"], i, R, case["K"], Hp, Wp, case["agnostic"], case["nonfinite"])
        kw = dict(bbox_reg=case["bbox_reg"], agnostic=case["agnostic"], flip_width=w if t[0] else None,
                  ar_inv=1.0 / t[3] if t[3] is not None else 1.0)
        if case["faster"]:
            boxes = O.decode(rois, deltas, case["K"], h, w, im_scale=im_scale, **kw)
        else:
            boxes = O.decode(props[index], deltas, case["K"], h, w, **kw)[inv]
            scores = scores[inv]
        scores_ts.append(scores)
        boxes_ts.append(boxes)
    got_s = O.combine(scores_ts, case["heur"], scores_ts[-1]) if case["aug"] != "none" else scores_ts[-1]
    got_b = O.combine(boxes_ts, case["coord_heur"], boxes_ts[-1]) if case["aug"] != "none" else boxes_ts[-1]
    want_s, want_b = GOLD[name + "/scores"], _want_boxes(name)
    assert got_s.shape == want_s.shape and np.array_equal(got_s.view(np.uint32), want_s.view(np.uint32))
    nan = np.isnan(want_b)
    assert got_b.dtype == want_b.dtype == np.float32 and np.array_equal(np.isnan(got_b), nan)
    assert np.array_equal(got_b[~nan].view(np.uint32), want_b[~nan].view(np.uint32))


def test_golden_cases_cover_the_edges():
    boxes = [GOLD[n + "/boxes"] for n in NAMES]
    assert any(np.isnan(b).any() for b in boxes)                                   # NaN deltas give NaN coordinates
    assert {cases.CASES[n]["R"] for n in NAMES} >= {0, 1} and any(GOLD[n + "/boxes"].shape[0] == 0 for n in NAMES)
    assert any(b.size and (b == 0).any() for b in boxes)                           # clipped at the border
    assert {(c["faster"], c["fpn"]) for c in cases.CASES.values()} == {(a, b) for a in (False, True) for b in (False, True)}
    assert {c["heur"] for c in cases.CASES.values()} == {"UNION", "AVG", "ID"}
    capped = cases._AUGS["x152"]["SCALES"][-1]
    assert get_target_scale(cases.IM_H, cases.IM_W, capped, 150) < float(capped) / cases.IM_H     # a scale capped by MAX_SIZE
    assert any(n + "/cls_boxes" in GOLD.files and GOLD[n + "/cls_boxes"].shape[0] > 0 for n in NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_host_blobs_match_reference(name):
    """im_info and the rois / FPN level blobs of every model call, from the package's host code, equal the reference's, and
    the calls come in the reference's order with the reference's data blob shapes."""
    case = cases.CASES[name]
    p = T._aug_params(None, cases.params(case))
    for i, t in enumerate(cases.transforms(case)):
        h, w, im_scale, props = _transform_inputs(case, t)
        want = _blobs(name, i)
        oh, ow = ops.resized_size(h, w, im_scale)
        if case["fpn"]:
            oh, ow = int(np.ceil(oh / 32.) * 32), int(np.ceil(ow / 32.) * 32)
        call = str(GOLD[name + "/calls"][i])
        assert call.startswith("data 1x3x%dx%d " % (oh, ow)), (i, call)
        assert np.array_equal(np.hstack((oh, ow, im_scale))[np.newaxis, :].astype(np.float32), want["im_info"])
        got = {}
        if props is not None:
            got["rois"] = T._get_rois_blob(props, im_scale)
            index, _ = _dedup(got["rois"], case["dedup"])
            got["rois"] = got["rois"][index, :]
            if case["fpn"]:
                T._add_multilevel_rois_for_test(got, "rois", p)
        assert call.split(" ")[3:] == [",".join(sorted(got))]
        assert sorted(got) == sorted(k for k in want if k != "im_info")
        for k in got:
            assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), (i, k)


def test_abi_validates_arguments_without_gpu():
    from detectron.pytorch_b200 import _lib
    lib, EINVAL = _lib.load(), -1
    w = ops._host_array(ctypes.c_float, (10., 10., 5., 5.))
    args = dict(boxes=16, box_stride=5, box_col=1, im_scale=1.0, deltas=16, delta_stride=24, agnostic=0, R=4, K=6, bbox_reg=1, weights=w,
                clip=4.1, im_h=10, im_w=10, flip=0, ar_inv=1.0, out=16, stream=None)

    def call(**kw):
        a = dict(args, **kw)
        return lib.b200_bbox_decode(*a.values())
    assert call(K=0) == EINVAL
    assert call(R=-1) == EINVAL
    assert call(box_stride=4) == EINVAL                     # rois need 5 columns from column 1
    assert call(im_scale=-1.0) == EINVAL
    assert call(delta_stride=20) == EINVAL                  # 4K columns of deltas
    assert call(weights=None) == EINVAL
    assert call(im_w=0) == EINVAL
    assert call(boxes=None) == EINVAL
    assert call(deltas=None) == EINVAL
    assert call(out=8) == EINVAL                            # a misaligned output
    assert call(R=0, boxes=None, out=None) == 0              # nothing to do, no launch


def test_reference_errors_are_kept():
    b = np.zeros((1, 4), np.float32)
    with pytest.raises(AssertionError):
        T.im_detect_bbox_aug(None, None, b, bbox_aug=dict(scale_size_dep=True))
    with pytest.raises(AssertionError):
        T.im_detect_bbox_aug(None, None, b, bbox_aug=dict(score_heur="UNION", coord_heur="AVG"))
    with pytest.raises(AssertionError):
        T.im_detect_bbox_aug(None, None, b, bbox_aug=dict(score_heur="AVG", coord_heur="UNION"))
    with pytest.raises(AssertionError):
        T.im_detect_bbox_aug(None, None, None, faster_rcnn=True, bbox_aug=dict(score_heur="AVG", coord_heur="AVG"))
    with pytest.raises(NotImplementedError):
        T.im_detect_bbox_aug(None, None, b, bbox_aug=dict(score_heur="MAX", coord_heur="AVG"))
    with pytest.raises(NotImplementedError):
        T.im_detect_bbox_aug(None, None, b, bbox_aug=dict(score_heur="AVG", coord_heur="MEDIAN"))
    with pytest.raises(NotImplementedError):
        T.im_detect_bbox(None, None, 600, 1000, b, bbox_normalize_targets_precomputed=True)


# ---------------------------------------------------------------------------------------------------------------------- GPU
def _run_package(name, rois_numpy=False):
    case = cases.CASES[name]
    wrap = (lambda a: torch.from_numpy(a).cuda()) if not rois_numpy else (lambda a: a if a.shape[-1] == 5 else torch.from_numpy(a).cuda())
    model = cases.ReplayModel(case, to_numpy=lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else t, wrap=wrap)
    im = cases.image(case["seed"])
    props = None if case["faster"] else cases.proposals(case["seed"], case["R"])
    if case["aug"] != "none":
        out = T.im_detect_bbox_aug(model, im, props, **cases.params(case))
    else:
        out = T.im_detect_bbox(model, im, 72, 200, props, **cases.params(case))
    return model, out


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_matches_reference(name):
    model, (scores, boxes, im_scale, blob_conv) = _run_package(name)
    assert scores.is_cuda and boxes.is_cuda
    assert list(model.calls) == [str(c) for c in GOLD[name + "/calls"]]
    for i, got in enumerate(model.blobs):
        want = _blobs(name, i)
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), (i, k)
    assert im_scale == float(GOLD[name + "/im_scale"].reshape(-1)[0]) and blob_conv == ("blob_conv", len(model.calls) - 1)
    s = scores.cpu().numpy()
    assert s.dtype == np.float32 and np.array_equal(s.view(np.uint32), GOLD[name + "/scores"].view(np.uint32))
    _assert_boxes(boxes.cpu().numpy(), _want_boxes(name), name)


@pytest.mark.gpu
def test_model_rois_may_be_numpy():
    for name in ("c4_faster_x152", "faster_r1"):
        _, (scores, boxes, _, _) = _run_package(name, rois_numpy=True)
        _assert_boxes(boxes.cpu().numpy(), _want_boxes(name), name)


@pytest.mark.gpu
def test_device_decode_matches_oracle_at_x152_size():
    """18 transforms of 1000 rois x 81 classes (the X-152 roster), flipped, aspect-scaled and class-agnostic variants, with
    deltas above the clip and non-finite ones; each transform and their union against the oracle."""
    rng = np.random.RandomState(0)
    R, K, H, W = 1000, 81, 800, 1201
    got, want = [], []
    for t in range(18):
        rois = np.zeros((R, 5), np.float32)
        xy = rng.uniform(-50, 1300, (R, 2))
        rois[:, 1:3] = xy
        rois[:, 3:5] = xy + rng.uniform(1, 600, (R, 2))
        deltas = (rng.standard_normal((R, 4 * K)) * 0.5).astype(np.float32)
        flat = deltas.reshape(-1)
        flat[rng.randint(0, flat.size, 3000)] = rng.choice(np.array([5.0, 40.0, -40.0, np.nan, np.inf, -np.inf], np.float32), 3000)
        im_scale = rng.choice([0.5, 1.0 / 1.4, 1.2, 1.6])
        kw = dict(flip_width=W if t % 2 else None, ar_inv=(1.0 / 0.75) if t % 6 == 5 else 1.0, agnostic=t == 17)
        dev = ops.bbox_decode_raw(torch.from_numpy(rois).cuda(), torch.from_numpy(deltas).cuda(), K, H, W, im_scale=im_scale, **kw)
        got.append(dev)
        want.append(O.decode(rois, deltas, K, H, W, im_scale=im_scale, **kw))
        _assert_boxes(dev.cpu().numpy(), want[-1], "transform %d" % t)
    _assert_boxes(torch.cat(got).cpu().numpy(), np.vstack(want), "union")
    # proposals, no regression
    props = rng.uniform(0, 900, (R, 4)).astype(np.float32)
    dev = ops.bbox_decode_raw(torch.from_numpy(props).cuda(), None, K, H, W, bbox_reg=False, flip_width=W, ar_inv=1.0 / 1.3)
    assert np.array_equal(dev.cpu().numpy(), O.decode(props, None, K, H, W, bbox_reg=False, flip_width=W, ar_inv=1.0 / 1.3))


_ALIAS_SCRIPT = r"""
import sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
from oracle import refmodel
from tests import bbox_cases as cases
cfg = refmodel.setup(use_b200_ops=False)
import core.test as ref_test
import detectron.pytorch_b200 as pkg
installed = pkg.install_reference_aliases(bbox=True, test_aug=True)
assert "core.test.im_detect_bbox_aug" in installed and "core.test.box_results_with_nms_and_limit" in installed
out = {}
for name in sys.argv[3:]:
    case = cases.CASES[name]
    cases.configure(cfg, case)
    model = cases.ReplayModel(case, to_numpy=lambda t: t.detach().cpu().numpy() if torch.is_tensor(t) else t,
                              wrap=lambda a: torch.from_numpy(a).cuda())
    props = None if case["faster"] else cases.proposals(case["seed"], case["R"])
    cls_boxes, _, _ = ref_test.im_detect_all(model, cases.image(case["seed"]), props)
    out[name + "/cls_boxes"] = np.vstack([np.asarray(b, np.float32).reshape(-1, 5) for b in cls_boxes[1:]])
    out[name + "/cls_counts"] = np.array([len(b) for b in cls_boxes[1:]])
    # the detections chain into the device mask paste: one RLE per detection
    masks = torch.rand((out[name + "/cls_boxes"].shape[0], case["K"], 14, 14), device="cuda")
    segms = ref_test.segm_results(cls_boxes, masks, out[name + "/cls_boxes"][:, :4], cases.IM_H, cases.IM_W)
    assert [len(s) for s in segms[1:]] == list(out[name + "/cls_counts"])
np.savez(sys.argv[2], **out)
"""


@pytest.mark.gpu
def test_reference_im_detect_all_with_aliases(tmp_path):
    """install_reference_aliases(bbox=True, test_aug=True) inside the reference's own process: its unmodified im_detect_all
    returns the golden cls_boxes.  Runs in a subprocess so the reference's modules never enter this test session."""
    from oracle import refmodel
    if not refmodel.available():
        pytest.skip("no reference core.test to alias (oracle/_ref/reflib is built only where a checkout is present)")
    names = [n for n in NAMES if cases.CASES[n]["im_detect_all"]]
    out = str(tmp_path / "alias.npz")
    subprocess.check_call([sys.executable, "-c", _ALIAS_SCRIPT, ROOT, out] + names, cwd=str(tmp_path))
    r = np.load(out)
    for n in names:
        counts = GOLD[n + "/cls_counts"]
        assert np.array_equal(r[n + "/cls_counts"], counts), n
        # each class's rows as a set: DEDUP_BOXES maps duplicate proposals to identical rows, and which of two identical rows
        # NMS keeps (so where it sits in the class's ascending order) is the reference's unstable argsort's choice
        got, want = r[n + "/cls_boxes"], GOLD[n + "/cls_boxes"]
        for a, b in zip(np.cumsum(counts) - counts, np.cumsum(counts)):
            g, w = got[a:b][np.lexsort(got[a:b].T[::-1])], want[a:b][np.lexsort(want[a:b].T[::-1])]
            _assert_boxes(g[:, :4], w[:, :4], n)
            assert np.array_equal(g[:, 4], w[:, 4]), n


@pytest.mark.gpu
@pytest.mark.parametrize("n", [14000, 18000])
def test_one_class_at_union_size(n):
    """One class with more candidates than the pipelined NMS scan reaches (13 888 rows) goes through
    box_results_with_nms_and_limit and equals oracle/detections.py; soft-NMS and box voting take the same class."""
    rng = np.random.RandomState(n)
    K = 3
    centres = rng.uniform(0, 1000, (n, 2))
    side = rng.uniform(20, 120, (n, 1))
    b = np.hstack([centres - side / 2, centres + side / 2]).astype(np.float32)
    boxes = np.tile(b, (1, K))
    scores = np.zeros((n, K), np.float32)
    scores[:, 1] = rng.uniform(0.06, 1.0, n).astype(np.float32)
    scores[: n // 100, 2] = 0.5
    kw = dict(num_classes=K, detections_per_im=0)
    _, _, got = T.box_results_with_nms_and_limit(torch.from_numpy(scores).cuda(), torch.from_numpy(boxes).cuda(), **kw)
    want = OD.box_results_with_nms_and_limit(scores, boxes, K, detections_per_im=0)
    assert got[1].shape[0] > 100
    for j in (1, 2):
        assert np.array_equal(got[j], want[j]), j
    soft = T.box_results_with_nms_and_limit(scores, boxes, soft_nms=True, **kw)[2]
    assert 0 < soft[1].shape[0] <= n and np.all(np.isfinite(soft[1]))
    voted = T.box_results_with_nms_and_limit(scores, boxes, bbox_vote=True, **kw)[2]
    assert np.array_equal(voted[1][:, 4], got[1][:, 4])
    np.testing.assert_allclose(voted[1], OD.box_voting(want[1], np.hstack([b, scores[:, 1:2]]), 0.8), rtol=1e-5, atol=2e-3)
