"""Golden vectors for the RPN proposal layer (SURVEY.md 8f N1), produced by the UNMODIFIED reference code.

Runs on the CPU and needs a checkout of the reference (found by oracle/refpath.py, $DETECTRON_REFERENCE first):

    python tests/golden/make_golden_proposals.py          # writes tests/golden/proposals.npz

How the reference is made importable without touching it (SURVEY.md 8c):
  * utils.cython_nms / utils.cython_bbox: the reference's own .pyx files, copied to a temp dir, built with the
    installed Cython after the 3-token dtype patch (np.int_t -> np.intp_t, np.int -> np.intp) that numpy 2 needs;
  * torch._six, dataloader.numpy_type_map, collections.Sequence/Mapping, np.float/int/bool: removed APIs aliased
    from outside, exactly the list SURVEY.md 8c verified.
The op itself -- GenerateProposalsOp.forward, proposals_for_one_image, bbox_transform, clip_tiled_boxes,
_filter_boxes, generate_anchors, cython_nms.nms -- is the reference's code, run on CPU.
"""
import collections
import collections.abc
import os
import shutil
import subprocess
import sys
import tempfile
import types

import numpy as np
import numpy.ma  # noqa: F401  (imported before import_reference aliases np.bool, which numpy.ma's own import trips over)
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.refpath import reference_dir  # noqa: E402

REF = os.path.join(reference_dir() or "", "lib")


def build_cython(tmp):
    for f in ("cython_nms.pyx", "cython_bbox.pyx"):
        shutil.copy(os.path.join(REF, "utils", f), tmp)
    p = os.path.join(tmp, "cython_nms.pyx")
    s = open(p).read().replace("np.int_t", "np.intp_t")
    import re
    s = re.sub(r"np\.int\b", "np.intp", s)
    open(p, "w").write(s)
    open(os.path.join(tmp, "setup.py"), "w").write(
        "from setuptools import setup, Extension\nfrom Cython.Build import cythonize\nimport numpy as np\n"
        "setup(ext_modules=cythonize([Extension('cython_nms', ['cython_nms.pyx'], include_dirs=[np.get_include()]),\n"
        "                             Extension('cython_bbox', ['cython_bbox.pyx'], include_dirs=[np.get_include()])], language_level=2))\n")
    subprocess.check_call([sys.executable, "setup.py", "build_ext", "--inplace"], cwd=tmp, stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)


def import_reference(tmp):
    sys.path.insert(0, tmp)
    import cython_bbox
    import cython_nms
    sys.modules["utils.cython_bbox"] = cython_bbox
    sys.modules["utils.cython_nms"] = cython_nms
    six = types.ModuleType("torch._six"); six.string_classes = (str, bytes); six.int_classes = (int,)
    sys.modules["torch._six"] = six
    import torch.utils.data.dataloader as dl
    if not hasattr(dl, "numpy_type_map"):
        dl.numpy_type_map = {}
    collections.Sequence = collections.abc.Sequence; collections.Mapping = collections.abc.Mapping
    np.float = float; np.int = int; np.bool = bool
    sys.path.insert(0, REF)
    from core.config import cfg
    import modeling.generate_anchors as ga
    import modeling.generate_proposals as gp
    import utils.fpn as fpn_utils
    return cfg, ga, gp, cython_nms, fpn_utils


def make_inputs(seed, N, A, H, W):
    rng = np.random.RandomState(seed)
    scores = rng.permutation(N * A * H * W).astype(np.float32).reshape(N, A, H, W)
    scores = (scores + np.float32(0.5)) / np.float32(N * A * H * W)                     # unique values in (0, 1): no ties
    deltas = (rng.standard_normal((N, 4 * A, H, W)) * 0.3).astype(np.float32)
    deltas[:, 2::4][:, :, ::7, ::5] = 5.0                                                # dw beyond BBOX_XFORM_CLIP
    return scores, deltas


def main():
    tmp = tempfile.mkdtemp(prefix="ref_cython_")
    build_cython(tmp)
    cfg, ga, gp, cython_nms, fpn_utils = import_reference(tmp)
    cases = {
        # name: (training, N, H, W, stride, anchor sizes, pre, post, thresh, min_size, im_info)
        "fpn_p5_train": (True, 2, 25, 42, 32, (256,), 600, 100, 0.7, 0, [[800, 1333, 1.6], [768, 1024, 1.2]]),
        "c4_test": (False, 1, 38, 50, 16, (32, 64, 128, 256, 512), 500, 50, 0.7, 0, [[600, 800, 1.5]]),
        "min_size": (False, 1, 20, 30, 16, (32, 64), 400, 80, 0.5, 16, [[320, 480, 2.0]]),
        "all_candidates": (True, 1, 6, 9, 32, (64, 128), -1, -1, 0.7, 0, [[192, 288, 1.0]]),
    }
    out = {}
    for name, (training, N, H, W, stride, sizes, pre, post, thresh, min_size, im_info) in cases.items():
        key = "TRAIN" if training else "TEST"
        cfg[key].RPN_PRE_NMS_TOP_N = pre; cfg[key].RPN_POST_NMS_TOP_N = post
        cfg[key].RPN_NMS_THRESH = thresh; cfg[key].RPN_MIN_SIZE = min_size
        anchors = ga.generate_anchors(stride=stride, sizes=sizes, aspect_ratios=(0.5, 1, 2))
        A = anchors.shape[0]
        scores, deltas = make_inputs(len(name), N, A, H, W)
        op = gp.GenerateProposalsOp(anchors, 1.0 / stride)
        op.train(training)
        rois, probs = op(torch.from_numpy(scores), torch.from_numpy(deltas), torch.tensor(im_info, dtype=torch.float32))
        out[name + "/scores"] = scores; out[name + "/deltas"] = deltas
        out[name + "/im_info"] = np.asarray(im_info, dtype=np.float32); out[name + "/anchors"] = anchors
        out[name + "/params"] = np.asarray([stride, pre, post, thresh, min_size], dtype=np.float64)
        out[name + "/rois"] = rois.astype(np.float32); out[name + "/probs"] = probs.astype(np.float32)
        print(name, "A =", A, "rois", rois.shape)
    # cases from tests/proposal_cases.py on which the reference is deterministic: NaN / inf deltas and NaN scores kept out of the
    # top k, dw / dh at the float32 neighbours of BBOX_XFORM_CLIP, and an FPN P2 level with unique sigmoid-shaped scores (the
    # tests regenerate their inputs from the case seed: only a sha256 of them is stored)
    from tests import proposal_cases as PC
    for name in PC.GOLDEN:
        scores, deltas, im_info, anchors, stride, pre, post, thresh, min_size, training = PC.golden_inputs(name)
        key = "TRAIN" if training else "TEST"
        cfg[key].RPN_PRE_NMS_TOP_N = pre; cfg[key].RPN_POST_NMS_TOP_N = post
        cfg[key].RPN_NMS_THRESH = thresh; cfg[key].RPN_MIN_SIZE = min_size
        op = gp.GenerateProposalsOp(anchors, 1.0 / stride)
        op.train(training)
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")                                          # NaN / inf arithmetic
            rois, probs = op(torch.from_numpy(scores.copy()), torch.from_numpy(deltas.copy()), torch.from_numpy(im_info.copy()))
        out[name + "/input_sha256"] = np.array(PC.sha256(scores, deltas))
        out[name + "/im_info"] = im_info; out[name + "/anchors"] = anchors
        out[name + "/params"] = np.asarray([stride, pre, post, thresh, min_size], dtype=np.float64)
        out[name + "/rois"] = rois.astype(np.float32); out[name + "/probs"] = probs.astype(np.float32)
        print(name, "A =", anchors.shape[0], "rois", rois.shape)
    # the live CPU NMS of the reference on the NMS oracle's own cases (pins oracle_nms_cython)
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from detectron.pytorch_b200 import synthetic as S
    for n in (1, 65, 1000, 3000):
        b = S.make_nms_boxes(n, seed=n)
        out["cython_nms/%d/keep" % n] = np.asarray(cython_nms.nms(b, np.float32(0.7)), dtype=np.int64)
    # FPN level assignment by the reference's own utils.fpn.map_rois_to_fpn_levels (pins oracle/fpn.py)
    for seed, (k_min, k_max) in enumerate([(2, 5), (2, 6), (3, 4)]):
        r = S.make_rois(400, (2, 8, 200, 336), 1.0 / 4, seed=seed)[:, 1:5].astype(np.float32)
        r[:7] = [[0, 0, 223, 223], [0, 0, 222.99, 223], [10, 10, 9, 9], [5, 5, 4, 30], [0, 0, 111, 111], [0, 0, 447, 447], [0, 0, 2000, 2000]]
        out["fpn_levels/%d/rois" % seed] = r
        out["fpn_levels/%d/k" % seed] = np.asarray([k_min, k_max])
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out["fpn_levels/%d/lvls" % seed] = fpn_utils.map_rois_to_fpn_levels(r.copy(), k_min, k_max)
    np.savez_compressed(os.path.join(HERE, "proposals.npz"), **out)
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
