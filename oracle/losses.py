"""Float64 numpy restatement of the RPN and Fast R-CNN training losses and their gradients (CHECKER ONLY; nothing under
detectron/ imports it).

  * smooth_l1            lib/utils/net.py:15-32 (beta: the float32 value torch compares and divides with)
  * rpn_sigmoid_cls      binary_cross_entropy_with_logits(x, float(label), weight = label >= 0, sum), rpn_heads.py:153-157
  * rpn_softmax_cls      cross_entropy over the pair (logit[n, a], logit[n, A + a]) with ignore_index = -1, rpn_heads.py:144-151
  * fast_rcnn_cls        cross_entropy averaged over the RoIs, fast_rcnn_heads.py:53
  * accuracy             argmax (first maximal index, NaN maximal) == label, averaged, fast_rcnn_heads.py:63-64

Each gradient follows the reference's autograd graph, so a NaN appears exactly where the reference's has one: smooth L1 through
pow's 2 * i and abs's sgn (sgn(NaN) = 0), BCE as (sigmoid(x) - y) * g * w, cross entropy as log_softmax's backward of
nll_loss's gradient (an ignored pair gets -exp(log_softmax) * 0).
"""
import numpy as np

RPN_BETA = float(np.float32(1.0 / 9.0))


def _f64(x):
    return np.asarray(x, dtype=np.float64)


def smooth_l1(p, t, wi, wo, beta, g=1.0):
    """(loss, d loss / d p * g): sum of wo * SmoothL1(wi * (p - t)) over every element, divided by p.shape[0]."""
    p, t, wi, wo = _f64(p), _f64(t), _f64(wi), _f64(wo)
    n = p.shape[0]
    with np.errstate(all="ignore"):
        i = wi * (p - t)
        a = np.abs(i)
        s = (a < beta).astype(np.float64)
        out = wo * (s * 0.5 * i * i / beta + (1 - s) * (a - 0.5 * beta))
        gn = g / n
        dterm = gn * wo
        sgn = (i > 0).astype(np.float64) - (i < 0).astype(np.float64)
        grad = ((dterm / beta) * (s * 0.5) * (2 * i) + dterm * (1 - s) * sgn) * wi
    return out.sum() / n, grad


def rpn_sigmoid_cls(x, labels):
    """(sum of the weighted BCE terms, count of labels >= 0, grad(divisor, g)) for logits x and labels of the same shape."""
    x, lab = _f64(x), np.asarray(labels)
    w = (lab >= 0).astype(np.float64)
    y = lab.astype(np.float64)
    with np.errstate(all="ignore"):
        logsig = np.minimum(x, 0.0) - np.log1p(np.exp(-np.abs(x)))
        terms = ((1 - y) * x - logsig) * w
        sig = 1.0 / (1.0 + np.exp(-x))

    def grad(divisor, g=1.0):
        with np.errstate(all="ignore"):
            return (sig - y) * (g / divisor) * w
    return terms.sum(), w.sum(), grad


def _pair_log_softmax(l0, l1):
    with np.errstate(all="ignore"):
        m = np.maximum(l0, l1)
        lse = np.log(np.exp(l0 - m) + np.exp(l1 - m))
        return l0 - m - lse, l1 - m - lse


def rpn_softmax_cls(x, labels):
    """x (N, 2A, h, w), labels (N, A, h, w) in {-1, 0, 1}: (sum of -log_softmax at the label over non-ignored pairs, their count,
    grad(divisor, g) of x)."""
    x, lab = _f64(x), np.asarray(labels)
    A = x.shape[1] // 2
    o0, o1 = _pair_log_softmax(x[:, :A], x[:, A:])
    keep = lab != -1
    with np.errstate(all="ignore"):
        picked = np.where(lab == 1, o1, o0)
        total = np.where(keep, -picked, 0.0).sum()
        bad = keep & (lab != 0) & (lab != 1)
        if bad.any():
            total = np.nan

    def grad(divisor, g=1.0):
        with np.errstate(all="ignore"):
            gw = g / divisor
            gs = np.where(keep, -gw, 0.0)
            d0 = np.where(lab == 0, -gw, 0.0) - np.exp(o0) * gs
            d1 = np.where(lab == 1, -gw, 0.0) - np.exp(o1) * gs
            d0[bad] = np.nan
            d1[bad] = np.nan
        return np.concatenate([d0, d1], axis=1)
    return total, keep.sum(), grad


def rpn_losses(levels, softmax, fixed_divisor=0.0, grad_coef=None):
    """levels: per level (cls_logits, bbox_pred, labels_wide, targets_wide, inside_wide, outside_wide) numpy arrays.  Returns
    (losses (L, 2) float64, [(d cls_logits, d bbox_pred)] for the upstream gradients grad_coef (L, 2), default ones)."""
    L = len(levels)
    gc = np.ones((L, 2)) if grad_coef is None else _f64(grad_coef).reshape(L, 2)
    losses, grads = np.zeros((L, 2)), []
    for l, (x, bp, lab, tg, wi, wo) in enumerate(levels):
        h, w = x.shape[2:]
        hb, wb = bp.shape[2:]
        lab = np.asarray(lab)[:, :, :h, :w]
        total, count, cgrad = (rpn_softmax_cls if softmax else rpn_sigmoid_cls)(x, lab)
        div = float(fixed_divisor) if (fixed_divisor > 0 and not softmax) else float(count)
        with np.errstate(all="ignore"):
            losses[l, 0] = np.float64(total) / div
        bl, bg = smooth_l1(bp, tg[:, :, :hb, :wb], wi[:, :, :hb, :wb], wo[:, :, :hb, :wb], RPN_BETA, gc[l, 1])
        losses[l, 1] = bl
        grads.append((cgrad(div, gc[l, 0]), bg))
    return losses, grads


def fast_rcnn_losses(cls_score, bbox_pred, labels, targets, inside, outside, grad_coef=(1.0, 1.0)):
    """(loss_cls, loss_bbox, accuracy_cls, d cls_score, d bbox_pred).  A label outside [0, C) gives NaN loss_cls and NaN rows of
    d cls_score, and counts as a miss."""
    x = _f64(cls_score)
    lab = np.asarray(labels).astype(np.int64).reshape(-1)
    R, C = x.shape
    valid = (lab >= 0) & (lab < C)
    t = np.where(valid, lab, 0)
    with np.errstate(all="ignore"):
        m = np.max(x, axis=1, keepdims=True)
        lsm = x - m - np.log(np.exp(x - m).sum(axis=1, keepdims=True))
        ce = -lsm[np.arange(R), t]
        ce[~valid] = np.nan
        loss_cls = ce.sum() / R
        gw = grad_coef[0] / R
        onehot = np.zeros_like(x)
        onehot[np.arange(R), t] = 1.0
        d_cls = (np.exp(lsm) - onehot) * gw
        d_cls[~valid] = np.nan
    nan = np.isnan(x)
    pred = np.argmax(np.where(nan.any(axis=1, keepdims=True), nan, x), axis=1)
    accuracy = float(np.mean(valid & (pred == lab)))
    loss_bbox, d_bbox = smooth_l1(bbox_pred, targets, inside, outside, 1.0, grad_coef[1])
    return loss_cls, loss_bbox, accuracy, d_cls, d_bbox
