"""SURVEY.md 8f N3, Keypoint R-CNN: the test-time keypoint extraction and OKS NMS of keypoint_results
(lib/core/test.py:850-866, lib/utils/keypoints.py:103-157, 225-266) on the device, against golden keypoints of the
REFERENCE'S OWN function run unmodified on the seeded inputs of tests/keypoint_cases.py (tests/golden/make_golden_keypoints.py
-> keypoints.npz, identical with cv2's IPP on and off) and against oracle/keypoints.py.

x, y and logit follow cv2's float32 INTER_CUBIC and numpy's coordinate arithmetic, so they must match bit for bit; prob
is a sum of exponentials that numpy accumulates pairwise in float32 and the device in double, so it gets a tolerance."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import keypoints as O
from tests import keypoint_cases as cases

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "keypoints.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROB_RTOL_ORACLE = 1e-6
PROB_RTOL_DEVICE = 2e-5


def _case(k):
    seed, D, min_size, nms_oks = cases.KEYPOINT_CASES[k]
    cls_boxes, maps, ref_boxes = cases.keypoint_case(seed, D, min_size, nms_oks)
    return (D, min_size, nms_oks), cls_boxes, maps, ref_boxes


def _check_xy(mine, gold, rtol, what):
    assert mine.shape == gold.shape and mine.dtype == np.float32, what
    assert np.array_equal(mine[:, :3], gold[:, :3]), "%s: x / y / logit differ at %s" % (what, np.argwhere(mine[:, :3] != gold[:, :3])[:5])
    np.testing.assert_allclose(mine[:, 3], gold[:, 3], rtol=rtol, atol=0, err_msg=what)


# ------------------------------------------------------------------------------------------------ CPU: the oracle itself
def test_oracle_resize_matches_cv2_inter_cubic():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(11)
    old = cv2.ipp.useIPP()
    n = 0
    try:
        for ipp, channels in ((False, (1, 3, 4, 5, 17)), (True, (5, 17))):
            cv2.ipp.setUseIPP(ipp)
            for t in range(44 if ipp else 48):
                for K in channels:
                    H, W = (56, 56) if t % 3 else (int(rng.randint(1, 60)), int(rng.randint(1, 60)))
                    src = (rng.standard_normal((H, W, K)) * 3).astype(np.float32)
                    kind = t % 6
                    if kind == 0:
                        w, h = 1, int(rng.randint(1, 900))
                    elif kind == 1:
                        w, h = int(rng.randint(1, 900)), 1
                    elif kind == 2:
                        w, h = int(rng.randint(1, W + 1)), int(rng.randint(1, H + 1))              # downscale
                    elif kind == 3 and t % 12 == 3:
                        w, h = W, H                                                              # a copy
                    else:
                        w, h = int(rng.randint(1, 1400)), int(rng.randint(1, 900))
                    a = cv2.resize(src[:, :, 0] if K == 1 else src, (w, h), interpolation=cv2.INTER_CUBIC).reshape(h, w, K)
                    assert np.array_equal(a, O.resize_cubic(src, w, h)), (ipp, K, H, W, w, h)
                    n += 1
    finally:
        cv2.ipp.setUseIPP(old)
    assert n >= 300


def test_oracle_matches_the_reference():
    g = np.load(GOLDEN)
    for k in range(len(cases.KEYPOINT_CASES)):
        (D, min_size, nms_oks), cls_boxes, maps, ref_boxes = _case(k)
        xy = O.heatmaps_to_keypoints(maps, ref_boxes, min_size)
        _check_xy(xy, g["c%d_xy" % k], PROB_RTOL_ORACLE, "case %d" % k)
        if nms_oks:
            keep = O.nms_oks(xy, ref_boxes, 0.3)
            assert keep == g["c%d_keep" % k].tolist()
            assert np.array_equal(cls_boxes[1][keep], g["c%d_boxes" % k])
        else:
            assert np.array_equal(cls_boxes[1], g["c%d_boxes" % k])


def test_cases_cover_the_edge_shapes():
    sizes, min_sizes = [], set()
    for k in range(len(cases.KEYPOINT_CASES)):
        (D, min_size, nms_oks), cls_boxes, maps, ref_boxes = _case(k)
        assert maps.shape == (D, 17, 56, 56) and ref_boxes.shape == (D, 4) and cls_boxes[1].shape == (D, 5)
        c = maps[0, cases.CONSTANT_CHANNEL]
        assert not maps[0, cases.ZERO_CHANNEL].any() and c[0, 0] != 0 and np.all(c == c[0, 0])
        w, h, mw, mh = O.map_sizes(ref_boxes, min_size)
        sizes.append((ref_boxes[:, 2] - ref_boxes[:, 0], ref_boxes[:, 3] - ref_boxes[:, 1], mw, mh, min_size))
        min_sizes.add(min_size)
        if nms_oks:
            scores = O.oks_scores(O.heatmaps_to_keypoints(maps, ref_boxes, min_size))
            assert len(np.unique(scores)) == D                                        # no ties in the greedy order
    assert min_sizes == {1, 64}
    bw = np.concatenate([s[0] for s in sizes]); bh = np.concatenate([s[1] for s in sizes])
    assert np.any(bw < 1) and np.any(bh < 1)                                          # clamped to one pixel
    assert np.any(bw != np.round(bw))                                                 # fractional
    assert any(np.any((s[2] == 56) & (s[3] == 56)) for s in sizes if s[4] < 56)       # a copy
    assert any(np.any((s[2] >= cases.KP_IM_W - 1) & (s[3] >= cases.KP_IM_H - 1)) for s in sizes)   # the whole image
    assert any(np.any(s[2] == 64) for s in sizes if s[4] == 64)                       # raised to the minimum


def test_device_summation_orders_equal_numpy():
    """nms_oks_kernel restates np.mean of 17 float32 logits and the float64 sum of 17 OKS terms as numpy's pairwise sum:
    eight accumulators a[j] + a[8 + j], a fixed tree, then a[16]."""
    rng = np.random.RandomState(4)

    def pairwise17(a):
        r = [a[:, j] + a[:, 8 + j] for j in range(8)]
        return (((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))) + a[:, 16]

    x32 = (rng.standard_normal((20000, 17)) * rng.uniform(0.1, 100, (20000, 1))).astype(np.float32)
    assert np.array_equal(np.mean(x32, axis=1), (pairwise17(x32).astype(np.float64) / 17).astype(np.float32))
    x64 = rng.rand(20000, 17)
    assert np.array_equal(np.sum(x64, axis=1) / 17, pairwise17(x64) / 17)


def test_keypoint_entry_points_validate_without_gpu():
    from detectron.pytorch_b200 import _lib
    lib = _lib.load()
    EINVAL = -1
    p = ctypes.c_void_p(256)                                  # never dereferenced: every call below fails validation
    assert lib.b200_heatmaps_to_keypoints(p, p, -1, 17, 56, 0, p, None) == EINVAL
    assert lib.b200_heatmaps_to_keypoints(p, p, 3, 0, 56, 0, p, None) == EINVAL                # no keypoint
    assert lib.b200_heatmaps_to_keypoints(p, p, 3, 17, 0, 0, p, None) == EINVAL
    assert lib.b200_heatmaps_to_keypoints(p, p, 3, 17, 65, 0, p, None) == EINVAL               # M > 64
    assert lib.b200_heatmaps_to_keypoints(p, p, 3, 17, 56, 16385, p, None) == EINVAL           # min_size too large
    assert lib.b200_heatmaps_to_keypoints(p, p, 1 << 27, 17, 56, 0, p, None) == EINVAL         # D * K >= 2^31
    assert lib.b200_heatmaps_to_keypoints(None, p, 3, 17, 56, 0, p, None) == EINVAL
    assert lib.b200_heatmaps_to_keypoints(p, p, 3, 17, 56, 0, None, None) == EINVAL
    assert lib.b200_heatmaps_to_keypoints(None, None, 0, 17, 56, 0, None, None) == 0          # nothing to do
    assert lib.b200_nms_oks(p, p, 3, 16, 0.3, p, p, None) == EINVAL                             # OKS needs the 17 COCO keypoints
    assert lib.b200_nms_oks(p, p, 4097, 17, 0.3, p, p, None) == EINVAL
    assert lib.b200_nms_oks(p, p, -1, 17, 0.3, p, p, None) == EINVAL
    assert lib.b200_nms_oks(p, p, 3, 17, 0.3, p, None, None) == EINVAL
    assert lib.b200_nms_oks(None, None, 0, 17, 0.3, None, None, None) == 0


def test_keypoint_results_host_checks_without_gpu():
    from detectron.pytorch_b200.core.test import keypoint_results
    from detectron.pytorch_b200.utils.keypoints import nms_oks
    cls_boxes = [np.zeros((0, 5), np.float32), np.zeros((0, 5), np.float32)]
    out = keypoint_results(cls_boxes, np.zeros((0, 17, 56, 56), np.float32), np.zeros((0, 4), np.float32), nms_oks=True)
    assert out == [[], []] and cls_boxes[1].shape == (0, 5)
    assert keypoint_results(cls_boxes, np.zeros((0, 17, 56, 56), np.float32), np.zeros((0, 4), np.float32), num_classes=3) == [[], [], []]
    with pytest.raises(ValueError):
        keypoint_results(cls_boxes, np.zeros((2, 17, 56, 56), np.float32), np.zeros((3, 4), np.float32))
    with pytest.raises(ValueError):
        keypoint_results(cls_boxes, np.zeros((2, 16, 56, 56), np.float32), np.zeros((2, 4), np.float32))
    assert nms_oks(np.zeros((0, 4, 17), np.float32), np.zeros((0, 4), np.float32), 0.3) == []


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_keypoints_match_the_reference_on_the_device():
    import torch
    from detectron.pytorch_b200 import ops
    g = np.load(GOLDEN)
    for k in range(len(cases.KEYPOINT_CASES)):
        (D, min_size, nms_oks), cls_boxes, maps, ref_boxes = _case(k)
        B = torch.from_numpy(ref_boxes).cuda()
        xy = ops.heatmaps_to_keypoints_raw(torch.from_numpy(maps).cuda(), B, min_size)
        _check_xy(xy.cpu().numpy(), g["c%d_xy" % k], PROB_RTOL_DEVICE, "case %d" % k)
        if nms_oks:
            keep, num = ops.nms_oks_raw(xy, B, 0.3)
            assert keep[:int(num.item())].cpu().tolist() == g["c%d_keep" % k].tolist()


@pytest.mark.gpu
def test_keypoint_results_numpy_and_cuda_inputs_agree():
    import torch
    from detectron.pytorch_b200.core.test import keypoint_results
    from detectron.pytorch_b200.utils import keypoints as U
    g = np.load(GOLDEN)
    for k in range(len(cases.KEYPOINT_CASES)):
        (D, min_size, nms_oks), cls_boxes, maps, ref_boxes = _case(k)
        kw = dict(num_classes=cases.KP_NUM_CLASSES, num_keypoints=17, inference_min_size=min_size, nms_oks=nms_oks)
        boxes_in = [cls_boxes[0], cls_boxes[1].copy()]
        a = keypoint_results(boxes_in, maps, ref_boxes, **kw)                                    # numpy, like the reference
        assert np.array_equal(boxes_in[1], g["c%d_boxes" % k])                                  # filtered in place (NMS_OKS)
        boxes_dev = [cls_boxes[0], cls_boxes[1].copy()]
        b = keypoint_results(boxes_dev, torch.from_numpy(maps).cuda(), torch.from_numpy(ref_boxes).cuda(), **kw)   # head's tensor
        nc = torch.from_numpy(np.ascontiguousarray(maps.transpose(0, 1, 3, 2))).cuda().transpose(2, 3)           # non-contiguous
        assert not nc.is_contiguous()
        c = keypoint_results([cls_boxes[0], cls_boxes[1].copy()], nc, ref_boxes, **kw)
        assert len(a) == len(b) == len(c) == 2 and a[0] == b[0] == c[0] == []
        assert np.array_equal(boxes_dev[1], boxes_in[1])
        keep = g["c%d_keep" % k] if nms_oks else np.arange(D)
        gold = g["c%d_xy" % k][keep]
        assert len(a[1]) == len(keep)
        for r in (a, b, c):
            assert all(x.shape == (4, 17) and x.dtype == np.float32 for x in r[1])
            assert np.array_equal(np.stack(r[1]), np.stack(a[1]))
        _check_xy(np.stack(a[1]), gold, PROB_RTOL_DEVICE, "case %d" % k)
        # the utils.keypoints front door, numpy and CUDA input
        xy = U.heatmaps_to_keypoints(maps, ref_boxes, min_size)
        assert np.array_equal(xy, U.heatmaps_to_keypoints(torch.from_numpy(maps).cuda(), ref_boxes, min_size))
        if nms_oks:
            assert U.nms_oks(xy, ref_boxes, 0.3) == U.nms_oks(torch.from_numpy(xy).cuda(), torch.from_numpy(ref_boxes).cuda(), 0.3) \
                == g["c%d_keep" % k].tolist()


@pytest.mark.gpu
def test_keypoint_edge_cases_on_the_device():
    import torch
    from detectron.pytorch_b200 import _lib, ops
    rng = np.random.RandomState(9)
    # min_size 0 (the reference's default) and 1 give the same result; a few channels other than 17
    (D, _, _), _, maps, ref_boxes = _case(2)
    M, B = torch.from_numpy(maps).cuda(), torch.from_numpy(ref_boxes).cuda()
    assert torch.equal(ops.heatmaps_to_keypoints_raw(M, B, 0), ops.heatmaps_to_keypoints_raw(M, B, 1))
    for K, Mh in ((1, 56), (3, 28), (5, 64), (18, 7)):
        mk = (rng.standard_normal((9, K, Mh, Mh)) * 2).astype(np.float32)
        bx = ref_boxes[:9]
        xy = ops.heatmaps_to_keypoints_raw(torch.from_numpy(mk).cuda(), torch.from_numpy(bx).cuda(), 0).cpu().numpy()
        _check_xy(xy, O.heatmaps_to_keypoints(mk, bx, 0), PROB_RTOL_DEVICE, "K = %d, M = %d" % (K, Mh))
    # zero detections
    z = ops.heatmaps_to_keypoints_raw(torch.zeros((0, 17, 56, 56), device="cuda"), torch.zeros((0, 4), device="cuda"))
    assert z.shape == (0, 4, 17)
    keep, num = ops.nms_oks_raw(z, torch.zeros((0, 4), device="cuda"), 0.3)
    assert keep.numel() == 0 and num.item() == 0
    # equal scores: the higher index first; an identical detection is suppressed, a far one kept
    xy = np.zeros((4, 4, 17), np.float32)
    xy[:, 0], xy[:, 1], xy[:, 2] = 100.0, 50.0, 1.0
    xy[3, 0] += 500.0
    rois = np.tile(np.array([[80, 20, 180, 260]], np.float32), (4, 1))
    keep, num = ops.nms_oks_raw(torch.from_numpy(xy).cuda(), torch.from_numpy(rois).cuda(), 0.3)
    assert keep[:int(num.item())].cpu().tolist() == [3, 2] == O.nms_oks(xy, rois, 0.3)
    with pytest.raises(RuntimeError):
        ops.nms_oks_raw(torch.zeros((2, 4, 16), device="cuda"), torch.zeros((2, 4), device="cuda"), 0.3)
    # one launch per image whatever the number of detections
    def launches(n):
        mk = torch.from_numpy(np.repeat(maps[:1], n, 0)).cuda()
        bx = torch.from_numpy(np.repeat(ref_boxes[1:2], n, 0)).cuda()
        n0 = _lib.launch_count()
        ops.heatmaps_to_keypoints_raw(mk, bx)
        return _lib.launch_count() - n0
    assert launches(1) == launches(100) == 1


_ALIAS_SCRIPT = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from oracle import refmodel
from tests import keypoint_cases as cases
cfg = refmodel.setup(use_b200_ops=False)
import core.test as ref_test
import detectron.pytorch_b200 as pkg
assert "core.test.keypoint_results" in pkg.install_reference_aliases(keypoints=True)
seed, D, min_size, nms_oks = cases.KEYPOINT_CASES[int(sys.argv[2])]
cfg.MODEL.NUM_CLASSES = cases.KP_NUM_CLASSES
cfg.KRCNN.NUM_KEYPOINTS = 17
cfg.KRCNN.INFERENCE_MIN_SIZE = 0                    # the reference's default: raises in cv2 4.13 unaliased
cfg.KRCNN.NMS_OKS = nms_oks
cls_boxes, maps, ref_boxes = cases.keypoint_case(seed, D, min_size, nms_oks)
cls_keyps = ref_test.keypoint_results(cls_boxes, maps, ref_boxes)
np.savez(sys.argv[3], xy=np.stack(cls_keyps[1]), boxes=cls_boxes[1])
"""


@pytest.mark.gpu
def test_reference_alias(tmp_path):
    """install_reference_aliases(keypoints=True) inside the reference's own process: its core.test.keypoint_results then
    returns the golden keypoints.  Runs in a subprocess so the reference's modules never enter this test session."""
    from oracle import refmodel
    if not refmodel.available():
        pytest.skip("no reference core.test to alias (oracle/_ref/reflib is built only where a checkout is present)")
    g = np.load(GOLDEN)
    k = 4                                                # the NMS_OKS case
    out = str(tmp_path / "alias.npz")
    subprocess.check_call([sys.executable, "-c", _ALIAS_SCRIPT, ROOT, str(k), out], cwd=str(tmp_path))
    r = np.load(out)
    assert np.array_equal(r["boxes"], g["c%d_boxes" % k])
    _check_xy(r["xy"], g["c%d_xy" % k][g["c%d_keep" % k]], PROB_RTOL_DEVICE, "alias")
