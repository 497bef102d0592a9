"""Numpy restatement of the test-time augmentation kernels (detectron/pytorch_b200/csrc/test_aug.cu), for the CPU tests.

combine(outputs, heur, hflips, perms, includes): the running per-row fold of the transforms in order, as the device does it,
which must equal the reference's np.mean / np.amax (and logit mean) over the stacked transforms, with
combine_heatmaps_size_dep's per-row selection.  resize_width_u8(im, out_w): cv2.resize(im, (out_w, h)) of a uint8 image,
cv2's 8-bit fixed-point INTER_LINEAR (IPP off), restated.
"""
import numpy as np

HEURS = {"SOFT_AVG": 0, "HM_AVG": 0, "SOFT_MAX": 1, "HM_MAX": 1, "LOGIT_AVG": 2}


def logit(y):
    """The reference's float32 expression (lib/core/test.py:462-463)."""
    y = np.asarray(y, dtype=np.float32)
    return -1.0 * np.log((1.0 - y) / np.maximum(y, np.float32(1e-20)))


def np_max(acc, v):
    """np.maximum(acc, v) elementwise: NaN propagates, of two equal values the second is kept."""
    return np.where((acc > v) | np.isnan(acc), acc, v)


def transformed(out, hflip=False, perm=None):
    """The transform's output as read by the combine: out[:, perm][..., ::-1]."""
    out = np.asarray(out, dtype=np.float32)
    if perm is not None:
        out = out[:, np.asarray(perm)]
    return out[..., ::-1] if hflip else out


def combine(outputs, heur, hflips=None, perms=None, includes=None):
    """outputs: list of (R, C, M, M) float32 head outputs in transform order; hflips / perms per transform; includes per
    transform an (R,) bool array or None (all rows).  Returns the combined (R, C, M, M) float32."""
    h = HEURS[heur]
    T = len(outputs)
    hflips = hflips or [False] * T
    perms = perms or [None] * T
    includes = includes or [None] * T
    R = outputs[0].shape[0]
    acc = np.zeros(outputs[0].shape, np.float32)
    count = np.zeros((R,), np.int64)
    for out, hf, pm, inc in zip(outputs, hflips, perms, includes):
        v = transformed(out, hf, pm)
        if h == 2:
            v = logit(v)
        inc = np.ones((R,), bool) if inc is None else np.asarray(inc, bool)
        start = (inc & (count == 0))[:, None, None, None]
        folded = np_max(acc, v) if h == 1 else acc + v
        first = v if h == 1 else np.float32(0) + v
        acc = np.where(start, first, np.where(inc[:, None, None, None], folded, acc)).astype(np.float32)
        count += inc
    assert (count >= 1).all()
    if h == 1:
        return acc
    m = acc / count.astype(np.float32)[:, None, None, None]
    return m if h == 0 else (1.0 / (1.0 + np.exp(-m))).astype(np.float32)


def resize_width_u8(im, out_w):
    """cv2.resize(im, dsize=(out_w, h)) for a uint8 (h, w, 3) image, INTER_LINEAR, IPP off."""
    im = np.asarray(im)
    h, w = im.shape[:2]
    if out_w == w:
        return im.copy()
    scale_x = 1.0 / (float(out_w) / w)
    dx = np.arange(out_w, dtype=np.float64)
    fx = ((dx + 0.5) * scale_x - 0.5).astype(np.float32)
    sx = np.floor(fx).astype(np.int64)
    fx = (fx - sx.astype(np.float32)).astype(np.float32)
    lo = sx < 0
    fx[lo], sx[lo] = 0, 0
    hi = sx >= w - 1
    fx[hi], sx[hi] = 0, w - 1
    a0 = np.rint((np.float32(1) - fx) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(fx * np.float32(2048)).astype(np.int64)
    sx1 = np.minimum(sx + 1, w - 1)
    s = im[:, sx, :].astype(np.int64) * a0[None, :, None] + im[:, sx1, :].astype(np.int64) * a1[None, :, None]
    return np.clip((((s >> 4) * 2048) >> 16) + 2 >> 2, 0, 255).astype(np.uint8)
