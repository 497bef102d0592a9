"""SURVEY.md 8f N3, Mask R-CNN: the test-time mask paste + COCO RLE of segm_results (lib/core/test.py:793-847) on the device,
against golden run-length encodings of the REFERENCE'S OWN function run unmodified on the seeded inputs of tests/segm_cases.py
(tests/golden/make_golden_segms.py -> segms.npz, recorded with cv2's IPP resize off and on) and against oracle/segms.py.

The device follows cv2's IPP-off arithmetic, so it must match the IPP-off golden bit for bit.  IPP's float resize differs
from it by ~1e-6, so against the IPP-on golden a pixel may differ only where the oracle's interpolated value lies within
TOL of the threshold."""
import ctypes
import os

import numpy as np
import pytest

from oracle import segms as O
from tests import segm_cases as cases

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "segms.npz")
THRESH = 0.5
TOL = 4e-6


def _mask_class(cls_boxes, cls_specific):
    return np.concatenate([[j if cls_specific else 0] * len(cls_boxes[j]) for j in range(1, len(cls_boxes))]).astype(np.int32)


def _oracle(k):
    seed, im_h, im_w, M, cs = cases.SEGM_CASES[k]
    cls_boxes, masks, ref_boxes = cases.segm_case(seed, im_h, im_w, M, cs)
    mc = _mask_class(cls_boxes, cs)
    counts, strings, interp = O.segm_rles(masks, mc, ref_boxes, im_h, im_w, THRESH)
    return (im_h, im_w, M, cs), cls_boxes, masks, ref_boxes, mc, counts, strings, interp


def _golden(g, k, ipp):
    c, o = g["c%d_ipp%d_counts" % (k, ipp)], g["c%d_ipp%d_offs" % (k, ipp)]
    return [c[o[d]:o[d + 1]] for d in range(len(o) - 1)]


def _near_threshold_only(a, b, win, vals):
    """Pixels where full-image masks a and b differ: all inside the window and within TOL of the threshold.  Returns their number."""
    ys, xs = np.nonzero(a != b)
    if len(ys) == 0:
        return 0
    y0, y1, x0, x1 = win
    assert np.all((ys >= y0) & (ys < y1) & (xs >= x0) & (xs < x1)), "a pixel outside the box differs"
    v = vals[ys - y0, xs - x0]
    assert np.all(np.abs(v.astype(np.float64) - THRESH) <= TOL), "a pixel differs away from the threshold: %s" % v
    return len(ys)


# ------------------------------------------------------------------------------------------------ CPU: the oracle itself
def test_oracle_resize_matches_cv2_ipp_off():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(7)
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        n = 0
        for t in range(360):
            S = (30, 16, 7, 12, 3)[t % 5]
            src = rng.rand(S, S).astype(np.float32)
            kind = t % 6
            if kind == 0:
                w, h = S // 2, S // 2                              # cv2's 2x INTER_AREA path (when S is even)
            elif kind == 1:
                w, h = 1, int(rng.randint(1, 400))
            elif kind == 2:
                w, h = int(rng.randint(1, 400)), 1
            elif kind == 3:
                w, h = int(rng.randint(1, S + 1)), int(rng.randint(1, S + 1))       # downscale
            else:
                w, h = int(rng.randint(1, 400)), int(rng.randint(1, 400))
            a = cv2.resize(src, (w, h)).reshape(h, w)
            assert np.array_equal(a, O.resize(src, w, h)), (S, w, h)
            n += 1
        assert n >= 300
    finally:
        cv2.ipp.setUseIPP(old)


def test_oracle_counts_match_the_reference():
    """Bit for bit against the reference run with IPP off (2x INTER_AREA detections included); with IPP on, only pixels
    within TOL of the threshold may differ."""
    g = np.load(GOLDEN)
    near = 0
    for k in range(len(cases.SEGM_CASES)):
        (im_h, im_w, M, cs), _, _, ref_boxes, _, counts, _, interp = _oracle(k)
        off, on = _golden(g, k, 0), _golden(g, k, 1)
        assert len(off) == len(counts) == ref_boxes.shape[0]
        for d in range(len(counts)):
            assert np.array_equal(off[d], counts[d]), (k, d)
            if not np.array_equal(on[d], counts[d]):
                near += _near_threshold_only(O.decode_counts(on[d], im_h, im_w), O.decode_counts(counts[d], im_h, im_w), *interp[d])
    print("pixels differing from the IPP-on reference, all within %g of the threshold: %d" % (TOL, near))


def test_cases_cover_the_edge_shapes():
    for seed, im_h, im_w, M, cs in cases.SEGM_CASES:
        cls_boxes, masks, ref_boxes = cases.segm_case(seed, im_h, im_w, M, cs)
        ib = O.expand_boxes_int(ref_boxes, M)
        w, h = ib[:, 2] - ib[:, 0] + 1, ib[:, 3] - ib[:, 1] + 1
        assert np.any((2 * w == M + 2) & (2 * h == M + 2))                         # 2x INTER_AREA
        assert np.any(np.maximum(w, 1) == 1) or np.any(np.maximum(h, 1) == 1)       # collapsed side
        assert np.any((ib[:, 1] <= 0) & (ib[:, 3] >= im_h - 1))                    # spans the image height
        for side in (ib[:, 0] < 0, ib[:, 1] < 0, ib[:, 2] > im_w - 1, ib[:, 3] > im_h - 1):
            assert np.any(side)                                                   # sticks out on every side
        assert any(len(cls_boxes[j]) == 0 for j in range(1, len(cls_boxes)))


def test_rle_string_round_trips():
    rng = np.random.RandomState(3)
    for t in range(200):
        n = int(rng.randint(1, 60))
        counts = rng.randint(0, (1 << int(rng.randint(1, 22))) + 1, n).astype(np.int64)
        counts[1:][counts[1:] == 0] = 1                      # only the first run may be empty
        s = O.rle_string(counts)
        assert all(48 <= ch < 48 + 64 for ch in s)
        assert np.array_equal(O.rle_from_string(s, (1, int(counts.sum()))), counts)
    im = (rng.rand(37, 23) > 0.6).astype(np.uint8)
    c = O.rle_counts(im)
    assert np.array_equal(O.decode_counts(c, 37, 23), im)
    assert O.rle_counts(np.ones((2, 3), np.uint8)).tolist() == [0, 6]
    try:
        from pycocotools import mask as mask_util
    except ImportError:
        return
    for t in range(20):
        im = np.asfortranarray((rng.rand(31, 47) > rng.rand()).astype(np.uint8)[:, :, None])
        rle = mask_util.encode(im)[0]
        assert rle["counts"] == O.rle_string(O.rle_counts(im[:, :, 0]))


def test_segm_entry_points_validate_without_gpu():
    from detectron.pytorch_b200 import _lib
    lib = _lib.load()
    EINVAL, EWS = -1, -2
    # workspace: one 20-byte scan state per thread (256 per detection), 256-byte aligned -- host arithmetic
    assert lib.b200_segm_workspace_bytes(100) == 100 * 256 * 20
    assert lib.b200_segm_workspace_bytes(1) == 5120 and lib.b200_segm_workspace_bytes(0) == 0
    f = ctypes.c_float(0.5)
    p = ctypes.c_void_p(256)                                  # never dereferenced: every call below fails validation
    assert lib.b200_segm_rle_sizes(p, p, p, 3, 81, 28, 800, 0, f, p, p, 1 << 20, None) == EINVAL          # im_w = 0
    assert lib.b200_segm_rle_sizes(p, p, p, 3, 81, 65, 800, 1333, f, p, p, 1 << 20, None) == EINVAL       # M > 64
    assert lib.b200_segm_rle_sizes(p, p, p, 3, 0, 28, 800, 1333, f, p, p, 1 << 20, None) == EINVAL        # no channel
    assert lib.b200_segm_rle_sizes(p, p, p, -1, 81, 28, 800, 1333, f, p, p, 1 << 20, None) == EINVAL
    assert lib.b200_segm_rle_sizes(p, p, p, 3, 81, 28, 20000, 20000, f, p, p, 1 << 20, None) == EINVAL    # >= 2^28 pixels
    assert lib.b200_segm_rle_sizes(None, p, p, 3, 81, 28, 800, 1333, f, p, p, 1 << 20, None) == EINVAL
    assert lib.b200_segm_rle_sizes(p, p, p, 3, 81, 28, 800, 1333, f, p, p, 3 * 5120 - 1, None) == EWS
    assert lib.b200_segm_rle_sizes(p, p, p, 3, 81, 28, 800, 1333, f, p, None, 0, None) == EWS
    assert lib.b200_segm_rle_sizes(None, None, None, 0, 81, 28, 800, 1333, f, None, None, 0, None) == 0    # nothing to do
    assert lib.b200_segm_rle_emit(p, p, p, 3, 81, 28, 800, 1333, f, p, p, 1 << 20, p, None, p, p, None) == EINVAL
    assert lib.b200_segm_rle_emit(p, p, p, 3, 81, 28, 800, 1333, f, p, p, 100, p, p, p, p, None) == EWS
    assert lib.b200_paste_masks(p, p, p, 70000, 81, 28, 800, 1333, f, p, None) == EINVAL                 # D > 65535
    assert lib.b200_paste_masks(p, p, None, 3, 81, 28, 800, 1333, f, p, None) == EINVAL


def test_segm_results_host_checks_without_gpu():
    from detectron.pytorch_b200.core.test import segm_results
    cls_boxes = [np.zeros((0, 5), np.float32) for _ in range(4)]
    out = segm_results(cls_boxes, np.zeros((0, 4, 14, 14), np.float32), np.zeros((0, 4), np.float32), 10, 12, num_classes=4)
    assert out == [[], [], [], []]
    cls_boxes[2] = np.ones((3, 5), np.float32)
    with pytest.raises(ValueError):
        segm_results(cls_boxes, np.zeros((2, 4, 14, 14), np.float32), np.zeros((3, 4), np.float32), 10, 12, num_classes=4)


# ------------------------------------------------------------------------------------------------ GPU
def _decode_all(counts, co, h, w):
    return [O.decode_counts(counts[co[d]:co[d + 1]], h, w) for d in range(len(co) - 1)]


@pytest.mark.gpu
def test_segm_rle_matches_the_reference_on_the_device():
    import torch
    from detectron.pytorch_b200 import ops
    g = np.load(GOLDEN)
    near = 0
    for k in range(len(cases.SEGM_CASES)):
        (im_h, im_w, M, cs), _, masks, ref_boxes, mc, counts, strings, interp = _oracle(k)
        Mk = torch.from_numpy(masks).cuda(); B = torch.from_numpy(ref_boxes).cuda(); C = torch.from_numpy(mc).cuda()
        cnt, co, st, so = ops.segm_rle_raw(Mk, C, B, im_h, im_w, THRESH)
        dense = ops.paste_masks(Mk, C, B, im_h, im_w, THRESH).cpu().numpy()
        cnt, co, st, so = cnt.cpu().numpy(), co.cpu().numpy(), st.cpu().numpy().tobytes(), so.cpu().numpy()
        off, on = _golden(g, k, 0), _golden(g, k, 1)
        D = ref_boxes.shape[0]
        assert co.shape == (D + 1,) and so.shape == (D + 1,) and co[-1] == cnt.size and so[-1] == len(st)
        for d in range(D):
            mine = cnt[co[d]:co[d + 1]]
            assert np.array_equal(mine, off[d]), (k, d)                                 # bit for bit, IPP off
            assert st[so[d]:so[d + 1]] == strings[d], (k, d)                            # same strings as the oracle
            im = O.decode_counts(mine, im_h, im_w)
            assert np.array_equal(dense[d], im), (k, d)                                 # paste_masks == decoded RLE
            if not np.array_equal(on[d], mine):
                near += _near_threshold_only(O.decode_counts(on[d], im_h, im_w), im, *interp[d])
    print("pixels differing from the IPP-on reference, all within %g of the threshold: %d" % (TOL, near))


@pytest.mark.gpu
def test_segm_results_matches_the_reference_structure_and_inputs():
    import torch
    from detectron.pytorch_b200.core.test import segm_results
    g = np.load(GOLDEN)
    for k in (0, 1):
        (im_h, im_w, M, cs), cls_boxes, masks, ref_boxes, mc, counts, strings, _ = _oracle(k)
        K = len(cls_boxes)
        kw = dict(num_classes=K, resolution=M, cls_specific_mask=cs, thresh_binarize=THRESH)
        a = segm_results(cls_boxes, masks, ref_boxes, im_h, im_w, **kw)                                 # numpy, like the reference
        flat = torch.from_numpy(masks.reshape(masks.shape[0], -1)).cuda()
        b = segm_results(cls_boxes, flat, torch.from_numpy(ref_boxes).cuda(), im_h, im_w, **kw)         # mask head's tensor
        nc = torch.from_numpy(np.ascontiguousarray(masks.transpose(0, 1, 3, 2))).cuda().transpose(2, 3)   # non-contiguous
        assert not nc.is_contiguous()
        c = segm_results(cls_boxes, nc, ref_boxes, im_h, im_w, **kw)
        assert a == b == c
        assert len(a) == K and a[0] == []
        d = 0
        off = _golden(g, k, 0)
        for j in range(1, K):
            assert len(a[j]) == len(cls_boxes[j])
            for r in a[j]:
                assert r["size"] == [im_h, im_w] and isinstance(r["counts"], str)
                assert r["counts"].encode() == strings[d]
                assert np.array_equal(O.rle_from_string(r["counts"].encode(), (im_h, im_w)), off[d])
                d += 1
        assert d == masks.shape[0]


@pytest.mark.gpu
def test_segm_edge_cases_on_the_device():
    import torch
    from detectron.pytorch_b200 import _lib, ops
    from detectron.pytorch_b200.core.test import segm_results
    im_h, im_w, M = 57, 83, 14
    rng = np.random.RandomState(5)
    masks = rng.rand(6, 1, M, M).astype(np.float32)
    boxes = np.array([[-200, -100, -120, -20],                    # wholly outside (above left)
                      [im_w + 40, 3, im_w + 90, 30],              # wholly outside (right)
                      [3, im_h + 5, 30, im_h + 60],               # wholly outside (below)
                      [0, 0, im_w - 1, im_h - 1],                 # the whole image: runs wrap from column to column
                      [np.nan, 0, 10, 10], [0, -np.inf, np.inf, 20]], np.float32)
    mc = np.zeros(6, np.int32)
    cnt, co, st, so = ops.segm_rle_raw(torch.from_numpy(masks).cuda(), torch.from_numpy(mc).cuda(), torch.from_numpy(boxes).cuda(),
                                       im_h, im_w, THRESH)
    cnt, co, st, so = cnt.cpu().numpy(), co.cpu().numpy(), st.cpu().numpy().tobytes(), so.cpu().numpy()
    for d in range(3):
        assert cnt[co[d]:co[d + 1]].tolist() == [im_h * im_w]
        assert st[so[d]:so[d + 1]] == O.rle_string([im_h * im_w])
    oc, os_, _ = O.segm_rles(masks[3:4], mc[3:4], boxes[3:4], im_h, im_w, THRESH)
    assert np.array_equal(cnt[co[3]:co[4]], oc[0]) and st[so[3]:so[4]] == os_[0]
    for d in (4, 5):                                              # non-finite: unspecified, but a valid RLE
        assert cnt[co[d]:co[d + 1]].sum() == im_h * im_w
    # zero detections and empty classes
    z = ops.segm_rle_raw(torch.zeros((0, 1, M, M), device="cuda"), torch.zeros((0,), dtype=torch.int32, device="cuda"),
                         torch.zeros((0, 4), device="cuda"), im_h, im_w, THRESH)
    assert z[0].numel() == 0 and z[1].tolist() == [0] and z[2].numel() == 0 and z[3].tolist() == [0]
    assert ops.paste_masks(torch.zeros((0, 1, M, M), device="cuda"), torch.zeros((0,), dtype=torch.int32, device="cuda"),
                           torch.zeros((0, 4), device="cuda"), im_h, im_w, THRESH).shape == (0, im_h, im_w)
    cls_boxes = [np.zeros((0, 5), np.float32), np.zeros((0, 5), np.float32),
                 np.concatenate([boxes[3:4], [[0.9]]], 1).astype(np.float32), np.zeros((0, 5), np.float32)]
    r = segm_results(cls_boxes, masks[3:4], boxes[3:4], im_h, im_w, num_classes=4, resolution=M, cls_specific_mask=False)
    assert r[0] == [] and r[1] == [] and r[3] == [] and len(r[2]) == 1 and r[2][0]["counts"] == os_[0].decode()
    # launches per call do not grow with the number of detections
    def launches(D):
        mk = torch.from_numpy(np.repeat(masks[3:4], D, 0)).cuda()
        bx = torch.from_numpy(np.repeat(boxes[3:4], D, 0)).cuda()
        n0 = _lib.launch_count()
        ops.segm_rle_raw(mk, torch.zeros((D,), dtype=torch.int32, device="cuda"), bx, im_h, im_w, THRESH)
        return _lib.launch_count() - n0
    assert launches(1) == launches(97) == 2
