"""Golden vectors for test-time augmentation of the mask and keypoint heads, produced by the UNMODIFIED reference functions
core.test.im_detect_mask_aug / im_detect_keypoints_aug on the CPU with cv2's IPP off.

    python oracle/make_reflib.py                       # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_test_aug.py        # writes tests/golden/test_aug.npz

The model is tests/tta_cases.py's record / replay stand-in: its head outputs are generated from (seed, call index), so only
what the reference did with them is stored, per case <name>:
  <name>/calls      the model calls in order ("conv <shape> <sha256 of the data blob>", "<head> <input keys> conv<i>");
  <name>/h<i>/<key> every rois / FPN blob of head call i, in full (a few rows each);
  <name>/out        the combined result.
Shims applied from outside, for today's numpy / torch and a CPU-only run: np.float / np.int (refmodel), torch.Tensor.cuda as
the identity.  KPS_AUG.SCALE_SIZE_DEP cases: the reference's combine_heatmaps_size_dep compares `box_utils.boxes_area(boxes)`
with AREA_TH, but this version of boxes_area returns (areas, negative indices), which raises TypeError; the generator hands
core.test a boxes_area that returns the areas alone (the contract the selection was written against) and changes nothing else.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402
from tests import tta_cases as cases  # noqa: E402


def main(out_path):
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    import cv2
    import torch
    cv2.ipp.setUseIPP(False)
    torch.Tensor.cuda = lambda self, *a, **k: self
    cfg = refmodel.setup(use_b200_ops=False)
    import core.test as ref_test
    ref_boxes = ref_test.box_utils
    proxy = types.ModuleType("box_utils_areas_only")
    proxy.__dict__.update(ref_boxes.__dict__)
    proxy.boxes_area = lambda b: ref_boxes.boxes_area(b)[0]
    gold = {}
    for name, case in sorted(cases.CASES.items()):
        cases.configure(cfg, case)
        ref_test.box_utils = proxy if case["size_dep"] else ref_boxes
        im = cases.image(case["seed"])
        boxes = cases.boxes(case["seed"], case["R"])
        model = cases.ReplayModel(case, to_numpy=lambda t: t.numpy() if torch.is_tensor(t) else t, wrap=torch.from_numpy)
        # the identity transform's backbone call, as im_detect_bbox makes it before the augmentation
        inputs, im_scale = ref_test._get_blobs(im, None, cfg.TEST.SCALE, cfg.TEST.MAX_SIZE)
        blob_conv = model.convbody_net(torch.from_numpy(inputs["data"]))
        if case["kind"] == "mask":
            out = ref_test.im_detect_mask_aug(model, im, boxes, im_scale, blob_conv)
        else:
            out = ref_test.im_detect_keypoints_aug(model, im, boxes, im_scale, blob_conv)
        out = np.asarray(out)
        assert out.dtype == np.float32 and out.shape == (case["R"], cases.head_channels(case), case["M"], case["M"]), (name, out.shape, out.dtype)
        gold[name + "/calls"] = np.array(model.calls)
        for i, blobs in enumerate(model.rois):
            for k, v in blobs.items():
                gold["%s/h%d/%s" % (name, i, k)] = v
        gold[name + "/out"] = out
    ref_test.box_utils = ref_boxes
    # the keypoint flip of the reference (lib/utils/keypoints.py:90-100) on channel-coded heatmaps: channel c holds c
    import utils.keypoints as ref_kp
    coded = np.broadcast_to(np.arange(17, dtype=np.float32)[None, :, None, None] * 4 + np.arange(4, dtype=np.float32)[None, None, None, :],
                            (1, 17, 1, 4)).copy()
    gold["flip_heatmaps/in"] = coded
    gold["flip_heatmaps/out"] = ref_kp.flip_heatmaps(coded)
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "test_aug.npz"))
