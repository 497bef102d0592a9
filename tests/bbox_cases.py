"""Seeded inputs of the box head tests (im_detect_bbox / im_detect_bbox_aug / im_detect_all, lib/core/test.py:50-362) -- inputs
only; the expected model calls and results come from tests/golden/detect_bbox.npz (make_golden_bbox.py, the unmodified
reference on the CPU).

The model is a record / replay stand-in with the reference's `model(**inputs)` surface: it records the shape and SHA-256 of
every `data` blob, every im_info / rois / FPN blob in full and the call order, and answers call i of a case with rois (Faster
R-CNN: boxes in blob coordinates, some outside the image), cls_score, bbox_pred (values above BBOX_XFORM_CLIP, and NaN / +-inf
where the case asks) and blob_conv generated from (case seed, i) by numpy, so the outputs need not be stored."""
import hashlib

import numpy as np

IM_H, IM_W = 60, 91                     # an odd width: flip_boxes' `W - x - 1` is not symmetric about a pixel centre

_AUGS = {
    "none": None,
    # the X-152 transform list (H_FLIP, SCALES with SCALE_H_FLIP) at small sizes; scale 120 is capped by MAX_SIZE 150
    "x152": dict(H_FLIP=True, SCALES=(48, 96, 120), SCALE_H_FLIP=True, ASPECT_RATIOS=(), ASPECT_RATIO_H_FLIP=False),
    "ratios": dict(H_FLIP=True, SCALES=(), SCALE_H_FLIP=False, ASPECT_RATIOS=(0.75, 1.5), ASPECT_RATIO_H_FLIP=True),
}
_BASE = dict(fpn=False, faster=True, aug="none", heur="UNION", coord_heur=None, dedup=False, agnostic=False, bbox_reg=True, R=12,
             K=6, nonfinite=False, im_detect_all=False)


def _cases():
    c = {
        "c4_faster_plain": dict(im_detect_all=True),
        "c4_faster_x152": dict(aug="x152", nonfinite=True),
        "fpn_faster_x152": dict(fpn=True, aug="x152", im_detect_all=True),
        "fpn_faster_ratios_agnostic": dict(fpn=True, aug="ratios", agnostic=True),
        "c4_fast_union_dedup": dict(faster=False, aug="x152", dedup=True, nonfinite=True),
        "fpn_fast_union_dedup": dict(fpn=True, faster=False, aug="ratios", dedup=True, im_detect_all=True),
        "c4_fast_avg": dict(faster=False, aug="x152", heur="AVG", dedup=True),
        "fpn_fast_id": dict(fpn=True, faster=False, aug="ratios", heur="ID"),
        "c4_fast_avg_score_id_coord": dict(faster=False, aug="ratios", heur="AVG", coord_heur="ID"),
        "c4_fast_plain_dedup": dict(faster=False, dedup=True),
        "faster_noreg": dict(aug="ratios", bbox_reg=False),
        "fast_noreg_avg": dict(faster=False, aug="x152", heur="AVG", bbox_reg=False),
        "faster_r1": dict(aug="x152", R=1),
        "fast_r1_agnostic": dict(faster=False, aug="ratios", R=1, agnostic=True),
        "faster_r0": dict(aug="ratios", R=0),
    }
    out = {}
    for i, name in enumerate(sorted(c)):
        out[name] = dict(_BASE, **c[name])
        out[name]["seed"] = i
        if out[name]["coord_heur"] is None:
            out[name]["coord_heur"] = out[name]["heur"]
    return out


CASES = _cases()


def image(seed):
    rng = np.random.RandomState(900 + seed)
    ramp = (np.arange(IM_H)[:, None, None] * 7 + np.arange(IM_W)[None, :, None] * 2 + np.array([0, 85, 170])) % 256
    return (ramp + rng.randint(-40, 41, (IM_H, IM_W, 3))).clip(0, 255).astype(np.uint8)


def proposals(seed, R):
    """(R, 4) float32 proposals in image coordinates: some past the border, and exact and near duplicates for DEDUP_BOXES."""
    rng = np.random.RandomState(1900 + seed)
    x1 = rng.uniform(-8, IM_W * 0.7, R)
    y1 = rng.uniform(-8, IM_H * 0.7, R)
    b = np.stack([x1, y1, x1 + rng.uniform(4, 50, R), y1 + rng.uniform(4, 40, R)], axis=1).astype(np.float32)
    if R >= 6:
        b[3] = b[1]                                       # an exact duplicate
        b[5] = b[2] + np.float32(0.01)                    # the same box after DEDUP_BOXES' rounding
    return b


def head_outputs(seed, call, R, K, blob_h, blob_w, agnostic, nonfinite):
    """The stand-in model's rois (R, 5) in blob coordinates, cls_score (R, K) and bbox_pred (R, 4K, or 8 class-agnostic) of call
    `call` of a case, float32."""
    rng = np.random.RandomState(30000 * (seed + 1) + call)
    x1 = rng.uniform(-0.15 * blob_w, 0.8 * blob_w, R)
    y1 = rng.uniform(-0.15 * blob_h, 0.8 * blob_h, R)
    rois = np.stack([np.zeros(R), x1, y1, x1 + rng.uniform(2, 0.6 * blob_w, R), y1 + rng.uniform(2, 0.6 * blob_h, R)], axis=1)
    rois = rois.astype(np.float32)
    logits = rng.standard_normal((R, K)) * 2
    scores = (np.exp(logits) / np.exp(logits).sum(axis=1, keepdims=True)).astype(np.float32)
    C = 8 if agnostic else 4 * K
    deltas = (rng.standard_normal((R, C)) * 0.4).astype(np.float32)
    flat = deltas.reshape(-1)
    pos = np.arange(flat.size)
    flat[(pos % 4 >= 2) & (pos % 13 == 3)] = 6.5                 # dw / dh above BBOX_XFORM_CLIP = log(1000 / 16)
    flat[(pos % 4 >= 2) & (pos % 17 == 2)] = -30.0
    if nonfinite:
        flat[pos % 29 == 5] = np.nan
        flat[pos % 31 == 7] = np.inf
        flat[pos % 37 == 11] = -np.inf
    return rois, scores, deltas


def configure(cfg, case):
    """Set the reference-shaped `cfg` (an AttrDict tree) for a case."""
    cfg.MODEL.NUM_CLASSES = case["K"]
    cfg.MODEL.FASTER_RCNN = case["faster"]
    cfg.MODEL.CLS_AGNOSTIC_BBOX_REG = case["agnostic"]
    cfg.MODEL.BBOX_REG_WEIGHTS = (10., 10., 5., 5.)
    cfg.MODEL.MASK_ON = False
    cfg.MODEL.KEYPOINTS_ON = False
    cfg.TEST.BBOX_REG = case["bbox_reg"]
    cfg.DEDUP_BOXES = 1. / 16. if case["dedup"] else 0.
    cfg.TEST.SCALE = 72
    cfg.TEST.MAX_SIZE = 200
    cfg.TEST.SCORE_THRESH = 0.05
    cfg.TEST.NMS = 0.5
    cfg.TEST.DETECTIONS_PER_IM = 100
    cfg.TEST.SOFT_NMS.ENABLED = False
    cfg.TEST.BBOX_VOTE.ENABLED = False           # the reference's np.average raises on the clipped degenerate boxes here
    cfg.TEST.BBOX_VOTE.VOTE_TH = 0.8
    cfg.TEST.BBOX_VOTE.SCORING_METHOD = "ID"
    cfg.FPN.FPN_ON = case["fpn"]
    cfg.FPN.MULTILEVEL_ROIS = case["fpn"]
    cfg.FPN.COARSEST_STRIDE = 32
    cfg.FPN.ROI_MIN_LEVEL, cfg.FPN.ROI_MAX_LEVEL = 2, 5
    cfg.FPN.ROI_CANONICAL_SCALE, cfg.FPN.ROI_CANONICAL_LEVEL = 224, 4
    a = _AUGS[case["aug"]]
    cfg.TEST.BBOX_AUG.ENABLED = a is not None
    cfg.TEST.BBOX_AUG.SCORE_HEUR = case["heur"]
    cfg.TEST.BBOX_AUG.COORD_HEUR = case["coord_heur"]
    cfg.TEST.BBOX_AUG.MAX_SIZE = 150
    cfg.TEST.BBOX_AUG.SCALE_SIZE_DEP = False
    for k, v in (a or _AUGS["x152"]).items():
        cfg.TEST.BBOX_AUG[k] = v


def params(case):
    """The same configuration as keyword arguments of the package's core.test functions."""
    a = _AUGS[case["aug"]] or _AUGS["x152"]
    return dict(num_classes=case["K"], test_scale=72, test_max_size=200, multilevel_rois=case["fpn"], faster_rcnn=case["faster"],
                dedup_boxes=1. / 16. if case["dedup"] else 0., bbox_reg=case["bbox_reg"], cls_agnostic_bbox_reg=case["agnostic"],
                bbox_reg_weights=(10., 10., 5., 5.), fpn_on=case["fpn"], coarsest_stride=32,
                bbox_aug=dict(score_heur=case["heur"], coord_heur=case["coord_heur"], max_size=150,
                              **{k.lower(): v for k, v in a.items()}))


def _digest(d):
    d = np.ascontiguousarray(d, dtype=np.float32)
    return "%s %s" % ("x".join(str(s) for s in d.shape), hashlib.sha256(d.tobytes()).hexdigest())


class ReplayModel:
    """model(**inputs) of Generalized_RCNN at test time, recording.  `to_numpy` turns a blob (numpy or tensor) into numpy;
    `wrap` turns a generated output into what the model returns (a torch tensor, on the CPU or the device)."""

    def __init__(self, case, to_numpy, wrap):
        self.case, self.to_numpy, self.wrap = case, to_numpy, wrap
        self.calls = []              # "data <shape> <sha256> <input keys>"
        self.blobs = []              # per call: {key: array} of im_info and every rois blob
        self.outputs = []            # per call: (rois, cls_score, bbox_pred) as generated

    def __call__(self, data, im_info, **rois):
        d = self.to_numpy(data[0])
        self.calls.append("data %s %s" % (_digest(d), ",".join(sorted(rois))))
        blobs = {"im_info": np.asarray(self.to_numpy(im_info[0])).copy()}
        blobs.update({k: np.asarray(v).copy() for k, v in rois.items()})
        self.blobs.append(blobs)
        c = self.case
        R = rois["rois"].shape[0] if "rois" in rois else c["R"]
        out = head_outputs(c["seed"], len(self.calls) - 1, R, c["K"], d.shape[2], d.shape[3], c["agnostic"], c["nonfinite"])
        self.outputs.append(out)
        return {"rois": self.wrap(out[0]), "cls_score": self.wrap(out[1]), "bbox_pred": self.wrap(out[2]),
                "blob_conv": ("blob_conv", len(self.calls) - 1)}


def transforms(case):
    """The reference's transforms of a case in call order (lib/core/test.py:216-260): (hflip, scale, max_size, aspect_ratio)."""
    a = _AUGS[case["aug"]]
    t = []
    if a is not None:
        if a["H_FLIP"]:
            t.append((True, 72, 200, None))
        for s in a["SCALES"]:
            t.append((False, s, 150, None))
            if a["SCALE_H_FLIP"]:
                t.append((True, s, 150, None))
        for ar in a["ASPECT_RATIOS"]:
            t.append((False, 72, 200, ar))
            if a["ASPECT_RATIO_H_FLIP"]:
                t.append((True, 72, 200, ar))
    t.append((False, 72, 200, None))
    return t
