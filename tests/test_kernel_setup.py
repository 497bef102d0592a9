"""Per-device kernel setup: raising a kernel's dynamic shared-memory limit and reading the SM count.

CPU part (no marker): every translation unit goes through smem_opt_in / device_sm_count (api.cu), which keep one table per
(kernel, device) under one lock and only ever raise a limit; no other file sets the attribute or queries the SM count itself.

GPU part (`-m gpu`): each kernel whose shared-memory request depends on the call runs at its smaller request, then its larger
one, then the smaller one again, in one process.  The limit is raised when a call first needs more and is never lowered, so
every call launches; each result is checked the way the rest of the suite checks that op.
"""
import glob
import os

import numpy as np
import pytest

from detectron.pytorch_b200 import synthetic as S
from oracle import cpu as O

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "detectron", "pytorch_b200", "csrc")
GRAD_TOL = dict(rtol=1e-5, atol=1e-5)


def test_kernel_setup_lives_in_api_cu():
    offenders = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu*"))):
        if os.path.basename(path) == "api.cu":
            continue
        with open(path) as f:
            text = f.read()
        offenders += ["%s: %s" % (os.path.basename(path), name) for name in ("cudaFuncSetAttribute", "cudaDevAttrMultiProcessorCount")
                      if name in text]
    assert not offenders, "use smem_opt_in / device_sm_count (api.cu): %s" % offenders


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
def test_nms_resolver_limit_rises_and_stays():
    """2 000 boxes ask the resolver for 66 576 B, 6 000 boxes for 195 536 B."""
    from detectron.pytorch_b200.model.nms.nms_gpu import nms_gpu
    for n in (2000, 6000, 2000):
        b = S.make_nms_boxes(n)
        k = nms_gpu(dev(b), 0.7).cpu().numpy().reshape(-1)
        assert np.array_equal(k, O.nms_cuda(b, 0.7)), n


@pytest.mark.gpu
def test_roi_align_backward_nhwc_limit_rises_and_stays(lib_option):
    """The NHWC scatter backward at P 7, C 256 (50 960 B of shared memory) and at P 14, C 128 (103 488 B), against the
    scalar-atomic kernel."""
    from detectron.pytorch_b200 import _lib, ops
    s, sr = 1.0 / 8, 2
    small, large = ((1, 256, 30, 40), 7), ((1, 128, 30, 40), 14)
    for shape, P in (small, large, small):
        r = np.concatenate([S.make_rois(48, shape, s, seed=2), S.make_edge_rois(shape, s)]).astype(np.float32)
        dy = np.random.RandomState(3).standard_normal((r.shape[0], shape[1], P, P)).astype(np.float32)
        lib_option("B200_ROI_ALIGN_BWD_PATH", "nhwc")
        before = _lib.launch_count()
        dx = ops.roi_align_backward(dev(dy), dev(r), shape, P, P, s, sr).cpu().numpy()
        assert _lib.launch_count() - before == 2, "the NHWC backward (scatter + transpose) did not run at %s, P %d" % (shape, P)
        lib_option("B200_ROI_ALIGN_BWD_PATH", "generic")
        ref = ops.roi_align_backward(dev(dy), dev(r), shape, P, P, s, sr).cpu().numpy()
        np.testing.assert_allclose(dx, ref, **GRAD_TOL)
        assert np.count_nonzero(ref) > 0


@pytest.mark.gpu
def test_roi_crop_backward_limit_rises_and_stays():
    """The NHWC scatter backward of RoICrop at 7 x 7 (50 960 B of shared memory) and 13 x 13 (175 760 B) crops of 256
    channels, against the fp64 oracle."""
    from detectron.pytorch_b200 import _lib, ops
    from tests import legacy_pool_crop_cases as LC
    for o in (7, 13, 7):
        c = dict(shape=(1, 256, 20, 24), R=32, oh=o, ow=o, grid="random")
        img, grid, go = LC.crop_case(c)
        before = _lib.launch_count()
        gi, gg = ops.roi_crop_backward(dev(go), dev(grid), c["shape"])
        assert _lib.launch_count() - before == 2, "the NHWC RoICrop backward did not run at %d x %d" % (o, o)
        ref = O.roi_crop_backward(go, grid, c["shape"], acc64=True)
        np.testing.assert_allclose(gi.cpu().numpy(), ref, **GRAD_TOL)
        assert np.count_nonzero(ref) > 0


@pytest.mark.gpu
def test_coco_match_limit_rises_and_stays():
    """COCO box AP with up to 7 and with 1 300 ground-truth objects of one category in one image: coco_match asks for
    A x T x max_gt = 4 x 10 x 1 300 = 52 000 B of shared memory at the larger one."""
    from tests import coco_eval_cases as CC
    from tests.test_coco_eval import _assert_same, _device_eval
    small = CC.make_set(0, masks=False)
    large = CC.make_set(1, n_images=3, n_cats=2, gt_per_image=1300, dets_per_image=40, masks=False)
    for ds, ab, asg, ak in (small, large, small):
        ora = CC.oracle_eval(ds, CC.results(ds, ab, asg, ak, "bbox"), "bbox")
        _assert_same(_device_eval(ds, ab, asg, ak, "bbox"), ora)
