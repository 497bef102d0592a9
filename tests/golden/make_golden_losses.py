"""Golden RPN and Fast R-CNN losses and gradients, produced by the UNMODIFIED reference functions on the CPU.

    python oracle/make_reflib.py                 # the reference's Python tree under oracle/_ref/reflib (build() does it too)
    python tests/golden/make_golden_losses.py    # writes tests/golden/losses.npz

modeling.FPN.fpn_rpn_losses, modeling.rpn_heads.single_scale_rpn_losses and modeling.fast_rcnn_heads.fast_rcnn_losses run as they
are, with `cfg` set from outside and `Tensor.cuda` made the identity for the duration (fast_rcnn_losses moves its host blobs with
.cuda(device_id)).  Gradients are those of sum_l (gcoef[l, 0] * loss_cls_l + gcoef[l, 1] * loss_bbox_l) by autograd.

Cases (key prefix "<case>/"):
  fpn_sigmoid / fpn_softmax   FPN P2-P6, N = 2, A = 3, a 32 x 48 image with wide blobs for MAX_SIZE 64; every P6 label ignored
                              (sigmoid: loss 0, softmax: NaN)
  single_sigmoid / _softmax   single scale, N = 1, A = 15
  single_ignored              single scale sigmoid, every label ignored (NaN)
  tie                         single scale sigmoid whose box terms include |w_in * (p - t)| == beta exactly
  nonfinite_sigmoid / _softmax  NaN, +inf and -inf logits on ignored labels and box predictions under zero weights
  frcn_specific / frcn_agnostic  Fast R-CNN, R = 40, C = 6, bbox 4C / 8 columns; tied maximal logits, |i| == 1 ties
  frcn_nonfinite              a NaN cls_score row (NaN is maximal for the accuracy) and non-finite box predictions under zero
                              weights
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refmodel  # noqa: E402

RPN_BETA = np.float32(1.0 / 9.0)
NAMES = ("rpn_labels_int32_wide", "rpn_bbox_targets_wide", "rpn_bbox_inside_weights_wide", "rpn_bbox_outside_weights_wide")


def rpn_level(rng, N, A, h, w, Hw, Ww, softmax, ignore_all=False):
    """(cls_logits, bbox_pred, labels_wide, targets_wide, inside_wide, outside_wide) with labels -1 / 0 / 1 and the weights of
    add_rpn_blobs (inside 1 on positives, outside 1 / 256-ish on non-ignored)."""
    cls = (rng.standard_normal((N, (2 if softmax else 1) * A, h, w)) * 2).astype(np.float32)
    bbox = (rng.standard_normal((N, 4 * A, h, w)) * 0.3).astype(np.float32)
    lab = rng.choice([-1, -1, -1, 0, 0, 1], size=(N, A, Hw, Ww)).astype(np.int32)
    if ignore_all:
        lab[:] = -1
    tg = (rng.standard_normal((N, 4 * A, Hw, Ww)) * 0.3).astype(np.float32)
    pos = np.repeat(lab == 1, 4, axis=1)
    inside = pos.astype(np.float32)
    outside = np.repeat(lab >= 0, 4, axis=1).astype(np.float32) * np.float32(1.0 / 37)
    # a few elements where both weights are nonzero but the target far away (linear branch)
    tg[:, :, ::3, ::2] += 0.5
    return [cls, bbox, lab, tg, inside, outside]


def fpn_levels(rng, softmax):
    sizes = [(8, 12, 16, 16), (4, 6, 8, 8), (2, 3, 4, 4), (1, 2, 2, 2), (1, 1, 1, 1)]
    return [rpn_level(rng, 2, 3, h, w, Hw, Ww, softmax, ignore_all=(k == 4)) for k, (h, w, Hw, Ww) in enumerate(sizes)]


def put_nonfinite(lv, softmax):
    cls, bbox, lab, tg, inside, outside = lv
    h, w = cls.shape[2:]
    ign = np.argwhere(lab[:, :, :h, :w] == -1)[:6]
    for k, (n, a, y, x) in enumerate(ign):
        cls[n, a, y, x] = (np.nan, np.inf, -np.inf)[k % 3]
        if softmax and k >= 3:
            cls[n, cls.shape[1] // 2 + a, y, x] = (np.nan, np.inf, -np.inf)[k % 3]
    zero = np.argwhere((inside[:, :, :h, :w] == 0) & (outside[:, :, :h, :w] == 0))[:6]
    for k, (n, c, y, x) in enumerate(zero):
        bbox[n, c, y, x] = (np.nan, np.inf, -np.inf)[k % 3]


def put_ties(lv):
    cls, bbox, lab, tg, inside, outside = lv
    # |w_in * (p - t)| == beta exactly: t = 0, w_in = 1, p = +-beta (float32)
    for k in range(6):
        n, c, y, x = 0, k, 1, k
        tg[n, c, y, x] = 0.0
        inside[n, c, y, x] = 1.0
        outside[n, c, y, x] = np.float32(0.5)
        bbox[n, c, y, x] = RPN_BETA if k % 2 == 0 else -RPN_BETA


def frcn_case(rng, R, C, B, nonfinite=False):
    cls = rng.standard_normal((R, C)).astype(np.float32)
    cls[3, 1] = cls[3, 4] = cls[3].max() + 1                      # tied maxima: the first index wins
    labels = rng.randint(0, C, R).astype(np.int32)
    labels[3] = 4
    labels[5] = 0
    bbox = (rng.standard_normal((R, B)) * 0.8).astype(np.float32)
    tg = (rng.standard_normal((R, B)) * 0.8).astype(np.float32)
    inside = np.zeros((R, B), np.float32)
    outside = np.zeros((R, B), np.float32)
    for r in range(R):
        if labels[r] > 0:
            k = labels[r] if B == 4 * C else 1
            inside[r, 4 * k:4 * k + 4] = 1.0
            outside[r, 4 * k:4 * k + 4] = 1.0
    # |i| == 1 ties (beta = 1)
    r = int(np.argmax(labels > 0))
    k = labels[r] if B == 4 * C else 1
    tg[r, 4 * k:4 * k + 2] = 0.0
    bbox[r, 4 * k] = 1.0
    bbox[r, 4 * k + 1] = -1.0
    if nonfinite:
        cls[7, 2] = np.nan
        cls[8, :] = -np.inf
        cls[8, 3] = np.nan
        z = np.argwhere(inside == 0)[:6]
        for q, (rr, cc) in enumerate(z):
            bbox[rr, cc] = (np.nan, np.inf, -np.inf)[q % 3]
    return [cls, bbox, labels, tg, inside, outside]


def main(out_path):
    import torch
    assert refmodel.available(), "oracle/_ref/reflib not built (python oracle/make_reflib.py)"
    cfg = refmodel.setup(use_b200_ops=False)
    import modeling.FPN as FPN
    import modeling.fast_rcnn_heads as FH
    import modeling.rpn_heads as RH
    rng = np.random.RandomState(2024)
    cfg.FPN.RPN_MIN_LEVEL, cfg.FPN.RPN_MAX_LEVEL = 2, 6
    cfg.TRAIN.RPN_BATCH_SIZE_PER_IM, cfg.TRAIN.IMS_PER_BATCH = 16, 2
    gold = {}
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        cases = []
        for act in ("sigmoid", "softmax"):
            cases.append(("fpn_" + act, act, True, fpn_levels(rng, act == "softmax")))
        cases.append(("single_sigmoid", "sigmoid", False, [rpn_level(rng, 1, 15, 6, 9, 8, 10, False)]))
        cases.append(("single_softmax", "softmax", False, [rpn_level(rng, 1, 15, 6, 9, 8, 10, True)]))
        cases.append(("single_ignored", "sigmoid", False, [rpn_level(rng, 1, 15, 6, 9, 8, 10, False, ignore_all=True)]))
        tie = [rpn_level(rng, 1, 3, 5, 7, 6, 8, False)]
        put_ties(tie[0])
        cases.append(("tie", "sigmoid", False, tie))
        for act in ("sigmoid", "softmax"):
            lv = [rpn_level(rng, 1, 3, 5, 7, 6, 8, act == "softmax")]
            put_nonfinite(lv[0], act == "softmax")
            cases.append(("nonfinite_" + act, act, False, lv))
        for name, act, fpn, levels in cases:
            cfg.RPN.CLS_ACTIVATION = act
            cfg.FPN.FPN_ON = fpn
            L = len(levels)
            gcoef = np.stack([1.0 + 0.25 * np.arange(L), 0.5 + 0.125 * np.arange(L)], axis=1)
            preds = [(torch.from_numpy(lv[0].copy()).requires_grad_(True), torch.from_numpy(lv[1].copy()).requires_grad_(True))
                     for lv in levels]
            tgts = [[torch.from_numpy(x) for x in lv[2:]] for lv in levels]
            if fpn:
                kw = {}
                for l, ((c, b), t) in enumerate(zip(preds, tgts)):
                    s = str(2 + l)
                    kw["rpn_cls_logits_fpn" + s], kw["rpn_bbox_pred_fpn" + s] = c, b
                    for k, x in zip(NAMES, t):
                        kw[k + "_fpn" + s] = x
                lc, lb = FPN.fpn_rpn_losses(**kw)
            else:
                c, b = preds[0]
                lc, lb = RH.single_scale_rpn_losses(c, b, *tgts[0])
                lc, lb = [lc], [lb]
            total = sum(gcoef[l, 0] * lc[l] + gcoef[l, 1] * lb[l] for l in range(L))
            total.backward()
            g = name + "/"
            gold[g + "meta"] = np.asarray([L, int(act == "softmax"), int(fpn), 16 * 2 if fpn else 0], np.int64)
            gold[g + "gcoef"] = gcoef
            gold[g + "losses"] = np.asarray([[float(lc[l]), float(lb[l])] for l in range(L)], np.float32)
            for l, lv in enumerate(levels):
                for k, x in zip(("cls", "bbox", "labels", "targets", "inside", "outside"), lv):
                    gold[g + "%s_%d" % (k, l)] = x
                gold[g + "d_cls_%d" % l] = preds[l][0].grad.numpy()
                gold[g + "d_bbox_%d" % l] = preds[l][1].grad.numpy()
            print(name, gold[g + "losses"].tolist())
        for name, C, B, nf in (("frcn_specific", 6, 24, False), ("frcn_agnostic", 6, 8, False), ("frcn_nonfinite", 6, 24, True)):
            cls, bbox, labels, tg, inside, outside = frcn_case(rng, 40, C, B, nf)
            cs = torch.from_numpy(cls.copy()).requires_grad_(True)
            bp = torch.from_numpy(bbox.copy()).requires_grad_(True)
            loss_cls, loss_bbox, acc = FH.fast_rcnn_losses(cs, bp, labels, tg, inside, outside)
            gcoef = np.asarray([0.75, 1.5])
            (gcoef[0] * loss_cls + gcoef[1] * loss_bbox).backward()
            g = name + "/"
            gold[g + "gcoef"] = gcoef
            gold[g + "losses"] = np.asarray([float(loss_cls), float(loss_bbox), float(acc)], np.float32)
            for k, x in zip(("cls", "bbox", "labels", "targets", "inside", "outside"), (cls, bbox, labels, tg, inside, outside)):
                gold[g + k] = x
            gold[g + "d_cls"] = cs.grad.numpy()
            gold[g + "d_bbox"] = bp.grad.numpy()
            print(name, gold[g + "losses"].tolist())
    finally:
        torch.Tensor.cuda = cuda
    np.savez_compressed(out_path, **gold)
    print("golden written to", out_path, len(gold), "arrays,", os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "losses.npz"))
