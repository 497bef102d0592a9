"""Seeded inputs of the test-time augmentation tests (im_detect_mask_aug / im_detect_keypoints_aug, lib/core/test.py:404-729)
-- inputs only; the expected model calls and combined outputs come from tests/golden/test_aug.npz (make_golden_test_aug.py,
the unmodified reference on the CPU).

The model is a record / replay stand-in with the reference's `model.module.convbody_net / mask_net / keypoint_net` surface:
it records every `data` blob it receives (shape and SHA-256 of its float32 bytes), every rois / FPN blob in full and the call
order, and answers each head call with an output generated from (case seed, head call index) by numpy, so the outputs need
not be stored.  The outputs hold exact 0 and 1, values on both sides of 0.5, maxima tied across transforms and signed zeros
that differ from transform to transform."""
import hashlib

import numpy as np

IM_H, IM_W = 64, 96

# name -> configuration.  kind "mask" / "keypoints"; aug: which transforms (hflip, scales, aspect ratios); R rows, M resolution
_BASE = dict(test_scale=64, test_max_size=200, fpn=False, cls_specific=True, num_classes=4, R=5, M=14, size_dep=False, J=17)
_AUGS = {
    "hflip": dict(h_flip=True, scales=(), scale_h_flip=False, aspect_ratios=(), aspect_ratio_h_flip=False),
    "scales": dict(h_flip=False, scales=(48, 80), scale_h_flip=True, aspect_ratios=(), aspect_ratio_h_flip=False),
    "ratios": dict(h_flip=False, scales=(), scale_h_flip=False, aspect_ratios=(0.75, 1.3), aspect_ratio_h_flip=True),
    "all": dict(h_flip=True, scales=(48, 80), scale_h_flip=True, aspect_ratios=(0.75,), aspect_ratio_h_flip=True),
}


def _cases():
    cases = {}
    for heur in ("SOFT_AVG", "SOFT_MAX", "LOGIT_AVG"):
        for aug in ("hflip", "scales", "ratios"):
            cases["mask_%s_%s" % (heur.lower(), aug)] = dict(_BASE, kind="mask", heur=heur, aug=aug)
    for heur in ("HM_AVG", "HM_MAX"):
        for aug in ("hflip", "scales", "ratios"):
            cases["kps_%s_%s" % (heur.lower(), aug)] = dict(_BASE, kind="keypoints", heur=heur, aug=aug, M=8)
        cases["kps_%s_size_dep" % heur.lower()] = dict(_BASE, kind="keypoints", heur=heur, aug="all", M=8, size_dep=True, R=6)
    cases["mask_agnostic_fpn"] = dict(_BASE, kind="mask", heur="SOFT_AVG", aug="all", cls_specific=False, fpn=True)
    cases["mask_fpn_logit"] = dict(_BASE, kind="mask", heur="LOGIT_AVG", aug="all", fpn=True, M=12)
    cases["mask_r1_odd"] = dict(_BASE, kind="mask", heur="SOFT_MAX", aug="all", R=1, M=7)
    cases["kps_r1_fpn_odd"] = dict(_BASE, kind="keypoints", heur="HM_AVG", aug="all", R=1, M=9, fpn=True)
    for i, name in enumerate(sorted(cases)):
        cases[name]["seed"] = i
    return cases


CASES = _cases()
AREA_TH = 30 ** 2         # KPS_AUG.AREA_TH of the size-dependent cases: the boxes below lie on both sides of it


def image(seed):
    rng = np.random.RandomState(500 + seed)
    ramp = (np.arange(IM_H)[:, None, None] * 5 + np.arange(IM_W)[None, :, None] * 3 + np.array([0, 85, 170])) % 256
    return (ramp + rng.randint(-40, 41, (IM_H, IM_W, 3))).clip(0, 255).astype(np.uint8)


def boxes(seed, R):
    """(R, 4) float32 detections in image coordinates, small and large (areas on both sides of AREA_TH), some at the border."""
    rng = np.random.RandomState(700 + seed)
    x1 = rng.uniform(0, IM_W * 0.6, R)
    y1 = rng.uniform(0, IM_H * 0.6, R)
    side = np.where(np.arange(R) % 2 == 0, rng.uniform(8, 20, R), rng.uniform(34, 60, R))
    b = np.stack([x1, y1, np.minimum(x1 + side * rng.uniform(0.8, 1.25, R), IM_W - 1), np.minimum(y1 + side, IM_H - 1)], axis=1)
    b[0, 0] = 0.0
    return b.astype(np.float32)


def head_output(seed, call, shape):
    """The stand-in head's output of head call `call` (0, 1, ...) of a case, float32 of `shape` (R, C, M, M)."""
    rng = np.random.RandomState(10000 * (seed + 1) + call)
    out = rng.uniform(0, 1, shape).astype(np.float32)
    flat = out.reshape(-1)
    n = flat.size
    pos = np.arange(n)
    flat[pos % 11 == 0] = 0.0
    flat[pos % 13 == 0] = 1.0
    flat[pos % 17 == 0] = np.float32(0.5) + np.float32(call % 3 - 1) * np.float32(2 ** -24)
    flat[pos % 19 == 0] = 0.75                                            # tied across every transform
    flat[pos % 23 == 0] = -0.0 if call % 2 else 0.0                        # +0.0 and -0.0 in alternate transforms
    flat[pos % 29 == 0] = -0.0
    return out


def aug_cfg(case):
    """The TEST.MASK_AUG / TEST.KPS_AUG values of a case (upper-case keys, as in the reference's config)."""
    a = _AUGS[case["aug"]]
    return dict(ENABLED=True, HEUR=case["heur"], H_FLIP=a["h_flip"], SCALES=a["scales"], MAX_SIZE=200, SCALE_H_FLIP=a["scale_h_flip"],
                SCALE_SIZE_DEP=case["size_dep"], AREA_TH=AREA_TH, ASPECT_RATIOS=a["aspect_ratios"],
                ASPECT_RATIO_H_FLIP=a["aspect_ratio_h_flip"])


def configure(cfg, case):
    """Set the reference-shaped `cfg` (an AttrDict tree) for a case."""
    cfg.MODEL.NUM_CLASSES = case["num_classes"]
    cfg.MRCNN.RESOLUTION = case["M"]
    cfg.MRCNN.CLS_SPECIFIC_MASK = case["cls_specific"]
    cfg.KRCNN.HEATMAP_SIZE = case["M"]
    cfg.KRCNN.NUM_KEYPOINTS = case["J"]
    cfg.TEST.SCALE = case["test_scale"]
    cfg.TEST.MAX_SIZE = case["test_max_size"]
    cfg.FPN.FPN_ON = case["fpn"]
    cfg.FPN.MULTILEVEL_ROIS = case["fpn"]
    cfg.FPN.COARSEST_STRIDE = 32
    cfg.FPN.ROI_MIN_LEVEL, cfg.FPN.ROI_MAX_LEVEL = 2, 5
    cfg.FPN.ROI_CANONICAL_SCALE, cfg.FPN.ROI_CANONICAL_LEVEL = 224, 4
    aug = aug_cfg(case)
    for key in ("MASK_AUG", "KPS_AUG"):
        for k, v in aug.items():
            getattr(cfg.TEST, key)[k] = v
    cfg.TEST.MASK_AUG.SCALE_SIZE_DEP = False
    cfg.TEST.MASK_AUG.ENABLED = case["kind"] == "mask"
    cfg.TEST.KPS_AUG.ENABLED = case["kind"] == "keypoints"


def head_channels(case):
    if case["kind"] == "keypoints":
        return case["J"]
    return case["num_classes"] if case["cls_specific"] else 1


class ReplayModel:
    """model.module.convbody_net(data=...) / mask_net(blob_conv, inputs) / keypoint_net(blob_conv, inputs), recording.
    `to_numpy` turns a blob (numpy or tensor) into numpy; `wrap` turns a generated output into what the head returns."""

    def __init__(self, case, to_numpy, wrap):
        self.case, self.to_numpy, self.wrap = case, to_numpy, wrap
        self.module = self
        self.calls = []              # "conv <shape> <sha256>" / "mask <keys>" / "keypoints <keys>"
        self.rois = []               # per head call: {key: array}
        self.heads = 0

    def convbody_net(self, data):
        d = np.ascontiguousarray(self.to_numpy(data), dtype=np.float32)
        self.calls.append("conv %s %s" % ("x".join(str(s) for s in d.shape), hashlib.sha256(d.tobytes()).hexdigest()))
        return ("blob_conv", len(self.calls) - 1)

    def _head(self, kind, blob_conv, inputs):
        assert blob_conv[0] == "blob_conv"
        self.calls.append("%s %s conv%d" % (kind, ",".join(sorted(inputs)), blob_conv[1]))
        self.rois.append({k: np.asarray(v).copy() for k, v in inputs.items()})
        R = inputs["mask_rois" if kind == "mask" else "keypoint_rois"].shape[0]
        out = head_output(self.case["seed"], self.heads, (R, head_channels(self.case), self.case["M"], self.case["M"]))
        self.heads += 1
        return self.wrap(out)

    def mask_net(self, blob_conv, inputs):
        return self._head("mask", blob_conv, inputs)

    def keypoint_net(self, blob_conv, inputs):
        return self._head("keypoints", blob_conv, inputs)


def transforms(case):
    """The reference's transforms of a case in order (lib/core/test.py:421-449, 586-617): per head call
    (hflip, downscaled, upscaled, scale or None, max_size, aspect_ratio or None)."""
    a, s = _AUGS[case["aug"]], case["test_scale"]
    t = [(False, False, False, None, None, None)]
    if a["h_flip"]:
        t.append((True, False, False, s, case["test_max_size"], None))
    for scale in a["scales"]:
        t.append((False, scale < s, scale > s, scale, 200, None))
        if a["scale_h_flip"]:
            t.append((True, scale < s, scale > s, scale, 200, None))
    for ar in a["aspect_ratios"]:
        t.append((False, False, False, s, case["test_max_size"], ar))
        if a["aspect_ratio_h_flip"]:
            t.append((True, False, False, s, case["test_max_size"], ar))
    return t
