"""Seeded inputs for the RPN proposal layer tests (top-k, decode, NMS, collect / distribute): score maps of the kinds an RPN
produces or can produce, deltas at the decode's edges, the shapes of a real pyramid and the reference's modes.  Nothing is
read from disk; every array is a function of its arguments.

Scores, (A, H, W) float32:
  unique      every value distinct, evenly spread in (0, 1) (what the older tests used)
  sigmoid     float32 sigmoid of N(-4, 6) logits plus a cluster of high logits around 13, where float32 has only a few dozen
              values below 1: the k-th score is tied and its ties straddle the cut
  saturated   more exact 1.0 values than k, the rest sigmoid
  all_equal   one value everywhere
  quantised   five distinct values
  nonfinite   sigmoid, with about 1 % NaN, a few +-inf, and a run of alternating -0.0 / +0.0
Deltas, (4A, H, W) float32: normal; dw / dh at the float32 neighbours of log(1000 / 16) (clip_edges); +-30 (large); +-inf (inf);
NaN in one channel (nan_dx, nan_dy, nan_dw, nan_dh).
"""
import hashlib

import numpy as np

from detectron.pytorch_b200.roi_data.rpn import generate_anchors

# (A, H, W): the FPN pyramid of an 800 x 1333 image (P2..P6, 3 aspect ratios), C4 (5 sizes x 3 ratios at stride 16), one cell
SHAPES = {"p2": (3, 200, 336), "p3": (3, 100, 168), "p4": (3, 50, 84), "p5": (3, 25, 42), "p6": (3, 13, 21), "c4": (15, 50, 84),
          "one": (1, 1, 1)}
FPN_LEVELS = (("p2", 2), ("p3", 3), ("p4", 4), ("p5", 5), ("p6", 6))
# two images of different sizes padded into one map
IM_INFO = np.array([[800, 1333, 1.6], [600, 1000, 1.2]], dtype=np.float32)
# the reference's RPN_PRE_NMS_TOP_N, RPN_POST_NMS_TOP_N, RPN_NMS_THRESH, RPN_MIN_SIZE for FPN (TRAIN / TEST) and C4 TRAIN
MODES = {"fpn_train": (2000, 2000, 0.7, 0), "fpn_test": (1000, 1000, 0.7, 0), "c4_train": (12000, 2000, 0.7, 0),
         "min_size": (1000, 1000, 0.7, 16)}
SCORE_KINDS = ("unique", "sigmoid", "saturated", "all_equal", "quantised", "nonfinite")
DELTA_KINDS = ("normal", "clip_edges", "large", "inf", "nan_dx", "nan_dy", "nan_dw", "nan_dh")
BBOX_XFORM_CLIP = np.float32(np.log(1000.0 / 16.0))
CLIP_NEIGHBOURS = np.array([np.nextafter(BBOX_XFORM_CLIP, np.float32(0)), BBOX_XFORM_CLIP,
                            np.nextafter(BBOX_XFORM_CLIP, np.float32(10))], dtype=np.float32)


def anchors_and_stride(shape_name):
    """Cell anchors and feature stride of a shape: FPN level l has one 2^(l+3)-pixel size at stride 2^l, C4 the five sizes at 16."""
    if shape_name == "c4":
        return generate_anchors(16, (32, 64, 128, 256, 512), (0.5, 1, 2)), 16
    if shape_name == "one":
        return generate_anchors(16, (32,), (1,)), 16
    lvl = dict(FPN_LEVELS)[shape_name]
    return generate_anchors(2 ** lvl, (2.0 ** (lvl + 3),), (0.5, 1, 2)), 2 ** lvl


def _sigmoid32(logits):
    return (1.0 / (1.0 + np.exp(-np.asarray(logits, np.float64)))).astype(np.float32)


def scores(kind, shape, k, seed):
    """(A, H, W) float32 score map of `kind`; k is the top-k the map is meant for (it sizes the tied clusters)."""
    A, H, W = shape
    n = A * H * W
    rng = np.random.RandomState(seed)
    if kind == "unique":
        x = ((rng.permutation(n) + 0.5) / n).astype(np.float32)
    elif kind == "all_equal":
        x = np.full(n, 0.5, np.float32)
    elif kind == "quantised":
        x = (rng.randint(0, 5, n) / 4.0).astype(np.float32)
    else:
        logits = rng.normal(-4.0, 6.0, n)
        hot = rng.permutation(n)[:min(n, k + k // 2 + 1)]
        if kind == "saturated":
            logits[hot] = rng.uniform(20.0, 40.0, hot.size)           # sigmoid rounds to exactly 1.0 in float32
        else:
            logits[hot] = rng.normal(13.0, 1.5, hot.size)             # a few dozen float32 values just below 1
        x = _sigmoid32(logits)
        if kind == "nonfinite":
            p = rng.permutation(n)
            nn = max(1, n // 100)
            x[p[:nn]] = np.nan
            x[p[nn:nn + 3]] = np.inf
            x[p[nn + 3:nn + 6]] = -np.inf
            z = np.sort(p[nn + 6:nn + 6 + max(2, n // 200)])          # zeros of both signs, alternating in (H, W, A) order
            x[z] = np.where(np.arange(z.size) % 2 == 0, np.float32(-0.0), np.float32(0.0))
        elif kind not in ("sigmoid", "saturated"):
            raise ValueError(kind)
    return np.ascontiguousarray(x.reshape(H, W, A).transpose(2, 0, 1))    # x enumerates (H, W, A), like the reference


def deltas(kind, shape, seed):
    """(4A, H, W) float32 box deltas of `kind`."""
    A, H, W = shape
    n = A * H * W
    rng = np.random.RandomState(seed + 1000)
    d = (rng.standard_normal((n, 4)) * 0.3).astype(np.float32)           # rows in (H, W, A) order, columns dx, dy, dw, dh
    some = rng.permutation(n)[:max(1, n // 50)]
    if kind == "clip_edges":
        third = rng.permutation(n)[:max(1, n // 3)]
        d[third, 2] = CLIP_NEIGHBOURS[rng.randint(0, 3, third.size)]
        d[third, 3] = CLIP_NEIGHBOURS[rng.randint(0, 3, third.size)]
    elif kind == "large":
        d[some] = rng.choice(np.array([-30.0, 30.0], np.float32), (some.size, 4))
    elif kind == "inf":
        d[some, rng.randint(0, 4, some.size)] = rng.choice(np.array([-np.inf, np.inf], np.float32), some.size)
    elif kind.startswith("nan_"):
        d[some, ("nan_dx", "nan_dy", "nan_dw", "nan_dh").index(kind)] = np.nan
    elif kind != "normal":
        raise ValueError(kind)
    return np.ascontiguousarray(d.reshape(H, W, A * 4).transpose(2, 0, 1))


def batch(score_kind, delta_kind, shape_name, k, seed, N=2):
    """(N, A, H, W) scores and (N, 4A, H, W) deltas, one seed per image."""
    shape = SHAPES[shape_name]
    s = np.stack([scores(score_kind, shape, k, seed + 7 * i) for i in range(N)])
    d = np.stack([deltas(delta_kind, shape, seed + 7 * i) for i in range(N)])
    return s, d


def stable_topk(x_ahw, k):
    """The rule b200_topk_batched follows: np.argsort(-x, kind="stable")[:k] of the (H, W, A)-flattened map, NaN last."""
    x = np.asarray(x_ahw, np.float32).transpose(1, 2, 0).reshape(-1)
    return np.argsort(-x, kind="stable")[:k]


def unique_sigmoid_scores(N, shape, seed):
    """(N, A, H, W) float32 scores shaped like sigmoid outputs (dense near 0 and 1) with every value distinct, so any correct
    top-k -- the reference's argpartition included -- gives one answer."""
    A, H, W = shape
    n = N * A * H * W
    rng = np.random.RandomState(seed)
    pool = np.unique(_sigmoid32(rng.normal(-3.0, 3.0, 3 * n)))
    pool = pool[(pool > 0) & (pool < 1)]
    assert pool.size >= n
    return rng.permutation(pool)[:n].reshape(N, A, H, W)


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(str(a.dtype).encode() + str(a.shape).encode())
        h.update(a.tobytes())
    return h.hexdigest()


# Reference golden cases on which the reference op is a function of its inputs (no tied scores anywhere a top-k or sort
# looks): tests/golden/make_golden_proposals.py runs the reference on them, tests/test_oracle_proposals.py and
# tests/test_proposal_layer.py compare against what it stored (the outputs, and only a sha256 of the inputs, which are
# regenerated from the case seed).  name: (training, N, shape, pre, post, thresh, min_size, im_info)
GOLDEN = {
    "nonfinite": (False, 2, "p4", 1000, 500, 0.7, 0, IM_INFO),
    "clip_edges": (True, 1, "c4", 3000, 500, 0.7, 0, IM_INFO[1:]),
    "fpn_p2_sigmoid": (True, 2, "p2", 2000, 2000, 0.7, 0, IM_INFO),
}


def golden_inputs(name):
    """(scores, deltas, im_info, anchors, stride, pre, post, thresh, min_size, training) of a golden case, from its seed."""
    training, N, shape_name, pre, post, thresh, min_size, im_info = GOLDEN[name]
    shape = SHAPES[shape_name]
    anchors, stride = anchors_and_stride(shape_name)
    seed = sum(map(ord, name))
    if name == "nonfinite":
        # unique finite scores, about 1 % NaN and one each of +-inf (pre < the finite count: no NaN is selected); deltas with
        # +-inf and NaN in each channel at separate places
        s = np.stack([scores("unique", shape, pre, seed + i) for i in range(N)])
        d = np.stack([deltas("inf", shape, seed + i) for i in range(N)])
        rng = np.random.RandomState(seed)
        for i in range(N):
            flat = s[i].reshape(-1)
            p = rng.permutation(flat.size)
            flat[p[:flat.size // 100]] = np.nan
            flat[p[-1]] = np.inf
            flat[p[-2]] = -np.inf
            dd = d[i].reshape(shape[0], 4, -1)
            for c in range(4):
                dd[:, c, rng.permutation(dd.shape[2])[:dd.shape[2] // 50]] = np.nan
    elif name == "clip_edges":
        s = np.stack([scores("unique", shape, pre, seed + i) for i in range(N)])
        d = np.stack([deltas("clip_edges", shape, seed + i) for i in range(N)])
    else:
        s = unique_sigmoid_scores(N, shape, seed)
        d = np.stack([deltas("normal", shape, seed + i) for i in range(N)])
    return s, d, np.asarray(im_info, np.float32), anchors, stride, pre, post, thresh, min_size, training
