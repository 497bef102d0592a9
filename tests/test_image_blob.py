"""The network's input image blob (get_image_blob, lib/utils/blob.py:37-148; _get_image_blob, lib/roi_data/minibatch.py:47-79)
on the device.

CPU: oracle/blob.py against cv2.resize itself (IPP off) on seeded shapes and scales, against the blobs of the UNMODIFIED
reference functions (tests/golden/image_blob.npz, make_golden_image_blob.py, IPP off), the host arithmetic against the
same goldens, and the C ABI's argument checks.
GPU: the device blob against the IPP-off goldens and the oracle bit for bit (COCO sizes in one mixed call), against the
IPP-on goldens no further than IPP-off cv2 is, and the call's contract: full overwrite of `out`, CUDA or host input, one
launch per call, N images in one call equal to N calls, and back-to-back calls that each keep their own staged images."""
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import _lib, ops
from detectron.pytorch_b200.core import test as T
from detectron.pytorch_b200.roi_data import minibatch as MB
from detectron.pytorch_b200.utils import blob as B
from oracle import blob as O
from tests import image_blob_cases as cases

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "image_blob.npz"))
MEANS = O.DEFAULT_PIXEL_MEANS
EINVAL = -1
MAX_SHAPE_CASES = ([(17, 23)], [(32, 64)], [(33, 65), (100, 7), (1, 1)], [(800, 1067), (800, 1201), (750, 1333)])
TARGET_SCALE_CASES = ((480, 640, 800, 1333), (427, 640, 800, 1333), (600, 1000, 800, 1333), (500, 833, 800, 1333),
                      (2, 5, 2, 5), (4, 10, 2, 5), (4, 9, 2, 4), (1200, 1600, 600, 1000), (333, 1333, 800, 1333))


def _stride(fpn):
    return 32 if fpn else None


def _train_oracle(name, seed, shapes, scales, max_size, fpn):
    inds = GOLD["train/%s/scale_inds" % name]
    return O.minibatch_image_blob(cases.train_images(seed, shapes), [f for _, _, f in shapes], scales, inds, max_size, MEANS, _stride(fpn))


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def _cv2_resize_cases(rng, n):
    """(H, W, fx, flipped): exact 2x on odd sides, 1-px sides, rint half-to-even sizes, upscales to 800 / 1333, random."""
    out = []
    for t in range(n):
        k = t % 8
        if k == 0:
            H, W, fx = 2 * int(rng.randint(1, 40)) + 1, 2 * int(rng.randint(1, 40)) + int(rng.randint(2)), 0.5
        elif k == 1:
            H, W = (1, int(rng.randint(1, 80))) if rng.randint(2) else (int(rng.randint(1, 80)), 1)
            fx = float(rng.choice([0.5, 2.0, 3.0, 1.0 / 3, float(rng.uniform(0.4, 9))]))
        elif k == 2:
            H, W = 2 * int(rng.randint(1, 40)) + 1, 2 * int(rng.randint(1, 40)) + 1      # h * .5 and w * .5 end in .5
            fx = 0.5 if rng.randint(2) else 1.5 if rng.randint(2) else 2.5
        elif k == 3 and t < 40:
            H, W = int(rng.randint(24, 64)), int(rng.randint(24, 64))
            fx = B.get_target_scale(min(H, W), max(H, W), 800, 1333)
        elif k == 4:
            H, W = int(rng.randint(2, 90)), int(rng.randint(2, 90))
            fx = float(rng.choice([1.0, 1.02, 0.99, 1.0 / 3, 0.25, 2.0 / 3]))         # near 1: cv2 copies an unchanged size
        else:
            H, W = int(rng.randint(1, 90)), int(rng.randint(1, 90))
            fx = float(rng.uniform(0.05, 1.0) if k % 2 else rng.uniform(1.0, 6.0))
        out.append((H, W, fx, bool(rng.randint(2))))
    return out


def test_oracle_matches_cv2_ipp_off():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(11)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    compared, raised = 0, 0
    try:
        for H, W, fx, flipped in _cv2_resize_cases(rng, 420):
            im = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
            x = (im[:, ::-1, :] if flipped else im).astype(np.float32)
            x -= MEANS
            try:
                ref = cv2.resize(x, None, None, fx=fx, fy=fx, interpolation=cv2.INTER_LINEAR)
            except cv2.error:
                with pytest.raises(ValueError):
                    O.prep_image(im, fx, flipped, MEANS)
                with pytest.raises(ValueError):
                    ops.resized_size(H, W, fx)
                raised += 1
                continue
            got = O.prep_image(im, fx, flipped, MEANS)
            assert ref.shape == got.shape == ops.resized_size(H, W, fx) + (3,), (H, W, fx)
            assert np.array_equal(ref, got), (H, W, fx, flipped)
            compared += 1
    finally:
        cv2.ipp.setUseIPP(old)
    assert compared >= 300 and raised > 0
    print("oracle == cv2 (IPP off) on %d cases; %d zero-size cases raise like cv2" % (compared, raised))


def test_mean_table_is_numpys_subtraction():
    v = np.arange(256, dtype=np.uint8)
    im = np.stack([v, v, v], axis=1)[None].astype(np.float32)
    im -= MEANS
    assert np.array_equal(ops.pixel_mean_table(MEANS), im[0].T)
    assert np.array_equal(ops.pixel_mean_table(MEANS), O.mean_table(MEANS))
    f32 = (np.arange(256, dtype=np.float32)[:, None] - MEANS.reshape(1, 3).astype(np.float32)).T
    assert (ops.pixel_mean_table(MEANS) != f32).mean() > 0.3          # a float32 subtraction would not be exact


@pytest.mark.parametrize("c", cases.TEST_CASES, ids=[c[0] for c in cases.TEST_CASES])
def test_oracle_matches_reference_get_image_blob(c):
    name, seed, H, W, scale, max_size, fpn = c
    blob, im_scale, im_info = O.get_image_blob(cases.image(seed, H, W), scale, max_size, MEANS, _stride(fpn))
    g = "test/%s/ipp0/" % name
    assert blob.dtype == GOLD[g + "blob"].dtype and np.array_equal(blob, GOLD[g + "blob"])
    assert im_scale == GOLD[g + "im_scale"]
    assert im_info.dtype == np.float32 and np.array_equal(im_info, GOLD[g + "im_info"])


@pytest.mark.parametrize("c", cases.TRAIN_CASES, ids=[c[0] for c in cases.TRAIN_CASES])
def test_oracle_matches_reference_minibatch_blob(c):
    name, seed, shapes, scales, max_size, fpn, _ = c
    blob, im_scales = _train_oracle(name, seed, shapes, scales, max_size, fpn)
    g = "train/%s/ipp0/" % name
    assert np.array_equal(blob, GOLD[g + "blob"])
    assert np.array_equal(np.asarray(im_scales), GOLD[g + "im_scales"])


def test_host_arithmetic_matches_reference():
    for k, shapes in enumerate(MAX_SHAPE_CASES):
        for fpn in (0, 1):
            got = B.get_max_shape(shapes, fpn_on=bool(fpn), coarsest_stride=32)
            assert np.array_equal(got, GOLD["max_shape/%d/fpn%d" % (k, fpn)]), (shapes, fpn)
    assert np.array_equal(np.array([B.get_target_scale(*c) for c in TARGET_SCALE_CASES]), GOLD["target_scale"])
    for name, seed, H, W, scale, max_size, fpn in cases.TEST_CASES:
        g = "test/%s/ipp0/" % name
        s = B.get_target_scale(min(H, W), max(H, W), scale, max_size)
        assert s == GOLD[g + "im_scale"]
        oh, ow = ops.resized_size(H, W, s)
        b = GOLD[g + "blob"]
        hp, wp = B.get_max_shape([(oh, ow)], fpn_on=fpn, coarsest_stride=32)
        assert b.shape == (1, 3, hp, wp)
        assert np.any(b[0, :, oh - 1, ow - 1] != 0)                              # the last resized pixel is inside the blob
        assert not b[0, :, oh:, :].any() and not b[0, :, :, ow:].any()           # everything past it is padding


def test_golden_cases_cover_the_edges():
    kinds = set()
    for name, seed, H, W, scale, max_size, fpn in cases.TEST_CASES:
        s = B.get_target_scale(min(H, W), max(H, W), scale, max_size)
        oh, ow = ops.resized_size(H, W, s)
        kinds.add("up" if s > 1 else "down" if s < 1 else "same")
        if s != float(scale) / min(H, W):
            kinds.add("cap")
        if 1.0 / s == 2.0:
            kinds.add("area_odd" if 2 * oh > H or 2 * ow > W else "area_even")
        if (H * s) % 1 == 0.5 and oh % 2 == 0 and oh < H * s:
            kinds.add("half_even_down")
        if min(H, W) == 1:
            kinds.add("1px")
        if not fpn and ow % 4:
            kinds.add("scalar_stores")
    assert kinds >= {"up", "down", "same", "cap", "area_odd", "area_even", "half_even_down", "1px", "scalar_stores"}, kinds
    assert any(len(c[2]) > 1 and len(set((h, w) for h, w, _ in c[2])) > 1 for c in cases.TRAIN_CASES)
    assert any(f for c in cases.TRAIN_CASES for _, _, f in c[2])


def test_ipp_on_goldens_differ_from_ipp_off():
    """The IPP-on goldens are a different arithmetic: record how far (the GPU test bounds the device by it)."""
    worst = 0.0
    for name, *_ in cases.TEST_CASES:
        a, b = GOLD["test/%s/ipp0/blob" % name], GOLD["test/%s/ipp1/blob" % name]
        assert a.shape == b.shape
        worst = max(worst, float(np.abs(a.astype(np.float64) - b).max()))
    print("max |IPP on - IPP off| over the test-time goldens: %g" % worst)


def test_abi_validates_arguments_without_gpu():
    lib = _lib.load()
    assert lib.b200_image_blob(None, None, 1, None, 32, 32, None, None) == EINVAL
    assert lib.b200_image_blob(8, 8, 0, 8, 32, 32, 16, None) == EINVAL                 # no image
    assert lib.b200_image_blob(8, 8, 65536, 8, 32, 32, 16, None) == EINVAL             # beyond the grid's y extent
    assert lib.b200_image_blob(8, 8, 1, 8, 0, 32, 16, None) == EINVAL
    assert lib.b200_image_blob(8, 8, 1, 8, 1 << 16, 1 << 15, 16, None) == EINVAL       # blob plane of 2^31 elements


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("c", cases.TEST_CASES, ids=[c[0] for c in cases.TEST_CASES])
def test_device_get_image_blob_matches_reference(c):
    name, seed, H, W, scale, max_size, fpn = c
    blob, im_scale, im_info = B.get_image_blob(cases.image(seed, H, W), scale, max_size, fpn_on=fpn, coarsest_stride=32)
    assert blob.is_cuda and blob.dtype == torch.float32
    off, on = GOLD["test/%s/ipp0/blob" % name], GOLD["test/%s/ipp1/blob" % name]
    got = blob.cpu().numpy()
    assert np.array_equal(got, off)
    assert isinstance(im_scale, float) and im_scale == GOLD["test/%s/ipp0/im_scale" % name]
    assert im_info.dtype == np.float32 and np.array_equal(im_info, GOLD["test/%s/ipp0/im_info" % name])
    # IPP on: the device is never further from it than cv2 with IPP off is
    d_dev, d_off = np.abs(got.astype(np.float64) - on).max(), np.abs(off.astype(np.float64) - on).max()
    print("%s: max |device - IPP on| = %g, max |IPP off - IPP on| = %g" % (name, d_dev, d_off))
    assert d_dev <= d_off


@pytest.mark.gpu
@pytest.mark.parametrize("c", cases.TRAIN_CASES, ids=[c[0] for c in cases.TRAIN_CASES])
def test_device_minibatch_blob_matches_reference(c):
    name, seed, shapes, scales, max_size, fpn, draw_seed = c
    roidb = [{"flipped": f} for _, _, f in shapes]
    ims = cases.train_images(seed, shapes)
    kw = dict(scales=scales, max_size=max_size, fpn_on=fpn, coarsest_stride=32)
    blob, im_scales = MB.get_image_blob(roidb, ims, GOLD["train/%s/scale_inds" % name], **kw)
    assert np.array_equal(blob.cpu().numpy(), GOLD["train/%s/ipp0/blob" % name])
    assert im_scales == GOLD["train/%s/ipp0/im_scales" % name].tolist()
    np.random.seed(draw_seed)                                              # the reference's own draw
    blob2, im_scales2 = MB.get_image_blob(roidb, ims, **kw)
    assert im_scales2 == im_scales and torch.equal(blob2, blob)
    on = GOLD["train/%s/ipp1/blob" % name]
    assert np.abs(blob.cpu().numpy().astype(np.float64) - on).max() <= np.abs(GOLD["train/%s/ipp0/blob" % name].astype(np.float64) - on).max()


def _coco_batch():
    rng = np.random.RandomState(5)
    shapes = [(480, 640), (640, 480), (1200, 1600), (333, 500)]
    ims = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    scales = [B.get_target_scale(min(h, w), max(h, w), 800, 1333) for h, w in shapes]
    scales[2] = 0.5                                                         # the 2x INTER_AREA path
    return ims, scales, [False, False, False, True]


@pytest.mark.gpu
def test_device_matches_oracle_at_coco_scale():
    ims, scales, flipped = _coco_batch()
    blob, sizes = ops.image_blob_raw(ims, scales, flipped, MEANS, 32)
    ref = O.im_list_to_blob([O.prep_image(im, s, f, MEANS) for im, s, f in zip(ims, scales, flipped)], 32)
    assert tuple(blob.shape) == ref.shape == (4, 3, 1088, 1216)
    assert sizes == [(800, 1067), (1067, 800), (600, 800), (800, 1201)]
    got = blob.cpu().numpy()
    for i in range(4):
        assert np.array_equal(got[i], ref[i]), i


@pytest.mark.gpu
def test_out_is_fully_overwritten_and_host_and_cuda_inputs_agree():
    ims, scales, flipped = _coco_batch()
    ref, _ = ops.image_blob_raw(ims, scales, flipped, MEANS, 32)
    out = torch.full_like(ref, float("nan"))
    got, _ = ops.image_blob_raw([torch.from_numpy(im).cuda() for im in ims], scales, flipped, MEANS, 32, out=out)
    assert got.data_ptr() == out.data_ptr()
    assert not torch.isnan(out).any() and torch.equal(out, ref)
    # a non-multiple-of-4 blob width (FPN off) takes the scalar stores; padding is still written
    out = torch.full((2, 3, 800, 1201), float("nan"), device="cuda")
    got, _ = ops.image_blob_raw([ims[0], ims[3]], [scales[0], scales[3]], [False, True], MEANS, None, out=out)
    assert not torch.isnan(out).any()
    assert not out[0, :, :, 1067:].any()
    # a pitched CUDA view (a crop of a wider image) is read in place
    wide = torch.from_numpy(np.concatenate([ims[0], ims[0][:, :37]], axis=1)).cuda()
    got, _ = ops.image_blob_raw([wide[:, :640]], [scales[0]], [False], MEANS, 32)
    assert tuple(got.shape) == (1, 3, 800, 1088) and torch.equal(got[0], ref[0, :, :800, :1088])


@pytest.mark.gpu
def test_one_call_equals_single_calls_and_makes_one_launch():
    ims, scales, flipped = _coco_batch()
    ops.image_blob_raw(ims[:1], scales[:1], flipped[:1], MEANS, 32)        # warm: library loaded
    n0 = _lib.launch_count()
    blob, sizes = ops.image_blob_raw(ims, scales, flipped, MEANS, 32)
    assert _lib.launch_count() - n0 == 1
    for i in range(4):
        one, s1 = ops.image_blob_raw([ims[i]], [scales[i]], [flipped[i]], MEANS, None)
        h, w = sizes[i]
        assert s1 == [sizes[i]] and torch.equal(one[0], blob[i, :, :h, :w])


@pytest.mark.gpu
def test_back_to_back_calls_keep_their_own_images():
    """Host images are staged in pinned memory and copied asynchronously; calls queued without a synchronisation in between
    must each see their own images (the staging buffer is not reused before its copy has run)."""
    rng = np.random.RandomState(9)
    ims = [rng.randint(0, 256, (300 + 7 * k, 400 - 5 * k, 3)).astype(np.uint8) for k in range(12)]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)                                       # keep the stream busy while the host moves on
        blobs = [ops.image_blob_raw([im], [0.75], [k % 2 == 1], MEANS, 32)[0] for k, im in enumerate(ims)]
    torch.cuda.synchronize()
    for k, im in enumerate(ims):
        ref = O.im_list_to_blob([O.prep_image(im, 0.75, k % 2 == 1, MEANS)], 32)
        assert np.array_equal(blobs[k].cpu().numpy(), ref), k


@pytest.mark.gpu
def test_get_blobs_projects_rois_like_the_reference():
    ims, _, _ = _coco_batch()
    rois = np.random.RandomState(2).uniform(0, 600, (50, 4)).astype(np.float32)
    blobs, im_scale = T.get_blobs(ims[0], rois, 800, 1333, fpn_on=True, coarsest_stride=32)
    assert im_scale == 800 / 480.
    assert np.array_equal(blobs["im_info"], np.array([[800, 1088, im_scale]], np.float32))
    ref = np.hstack((np.zeros((50, 1)), rois.astype(np.float64) * im_scale)).astype(np.float32)
    assert blobs["rois"].dtype == np.float32 and np.array_equal(blobs["rois"], ref)
    assert tuple(blobs["data"].shape) == (1, 3, 800, 1088)
    assert T.get_blobs(ims[0], None, 800, 1333)[0].keys() == {"data", "im_info"}


@pytest.mark.gpu
def test_errors():
    im = np.zeros((5, 7, 3), np.uint8)
    with pytest.raises(ValueError):
        ops.image_blob_raw([im], [0.05], [False], MEANS, 32)               # rint(0.25) = 0 rows: cv2 raises
    with pytest.raises(ValueError):
        ops.image_blob_raw([im[:, :, :2]], [1.0], [False], MEANS, 32)
    with pytest.raises(ValueError):
        ops.image_blob_raw([im.astype(np.float32)], [1.0], [False], MEANS, 32)
    with pytest.raises(ValueError):
        ops.image_blob_raw([im], [1.0], [False], MEANS, 32, out=torch.empty((1, 3, 32, 33), device="cuda"))
