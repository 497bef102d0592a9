"""Golden input image blobs, produced by the UNMODIFIED reference functions on the CPU: get_image_blob, prep_im_for_blob,
im_list_to_blob, get_max_shape and get_target_scale (lib/utils/blob.py:37-148) with FPN on and off, and the training
_get_image_blob (lib/roi_data/minibatch.py:47-79).

    python oracle/make_reflib.py                       # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_image_blob.py      # writes tests/golden/image_blob.npz

The inputs are tests/image_blob_cases.py.  minibatch's `cv2` is replaced, from outside, by a namespace whose imread returns
the seeded image named by the roidb entry; the resize is the real cv2.resize.  The scale draw (np.random.randint) runs under
np.random.seed(case seed) and is recorded.  Every case is recorded twice, with cv2's IPP on and off:
  "test/<name>/ipp<0|1>/blob|im_scale|im_info", "train/<name>/ipp<0|1>/blob|im_scales", "train/<name>/scale_inds",
  "max_shape/<k>/fpn<0|1>" for the shape lists of MAX_SHAPE_CASES, "target_scale" for TARGET_SCALE_CASES.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402
from tests import image_blob_cases as cases  # noqa: E402

MAX_SHAPE_CASES = ([(17, 23)], [(32, 64)], [(33, 65), (100, 7), (1, 1)], [(800, 1067), (800, 1201), (750, 1333)])
# (im_size_min, im_size_max, target_size, max_size): the cap's np.round(.5) boundary both ways, and COCO shapes
TARGET_SCALE_CASES = ((480, 640, 800, 1333), (427, 640, 800, 1333), (600, 1000, 800, 1333), (500, 833, 800, 1333),
                      (2, 5, 2, 5), (4, 10, 2, 5), (4, 9, 2, 4), (1200, 1600, 600, 1000), (333, 1333, 800, 1333))


def main(out_path):
    import cv2
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import utils.blob as ref_blob
    import roi_data.minibatch as ref_mb
    images = {}
    ref_mb.cv2 = types.SimpleNamespace(imread=lambda path: images[path].copy())
    gold = {}
    for ipp in (0, 1):
        cv2.ipp.setUseIPP(bool(ipp))
        for name, seed, H, W, scale, max_size, fpn in cases.TEST_CASES:
            cfg.FPN.FPN_ON = fpn
            blob, im_scale, im_info = ref_blob.get_image_blob(cases.image(seed, H, W), scale, max_size)
            g = "test/%s/ipp%d/" % (name, ipp)
            gold[g + "blob"], gold[g + "im_scale"], gold[g + "im_info"] = blob, np.float64(im_scale), im_info
        for name, seed, shapes, scales, max_size, fpn, draw_seed in cases.TRAIN_CASES:
            cfg.FPN.FPN_ON = fpn
            cfg.TRAIN.SCALES = scales
            cfg.TRAIN.MAX_SIZE = max_size
            roidb = []
            for k, (im, (H, W, flipped)) in enumerate(zip(cases.train_images(seed, shapes), shapes)):
                images["%s_%d" % (name, k)] = im
                roidb.append({"image": "%s_%d" % (name, k), "flipped": flipped})
            np.random.seed(draw_seed)
            blob, im_scales = ref_mb._get_image_blob(roidb)
            np.random.seed(draw_seed)
            gold["train/%s/scale_inds" % name] = np.random.randint(0, high=len(scales), size=len(roidb))
            g = "train/%s/ipp%d/" % (name, ipp)
            gold[g + "blob"], gold[g + "im_scales"] = blob, np.asarray(im_scales, np.float64)
    cv2.ipp.setUseIPP(True)
    for k, shapes in enumerate(MAX_SHAPE_CASES):
        for fpn in (0, 1):
            cfg.FPN.FPN_ON = bool(fpn)
            gold["max_shape/%d/fpn%d" % (k, fpn)] = np.asarray(ref_blob.get_max_shape(shapes))
    gold["target_scale"] = np.array([ref_blob.get_target_scale(*c) for c in TARGET_SCALE_CASES], np.float64)
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "image_blob.npz"))
