"""TEST INFRASTRUCTURE: numpy restatement of the reference's keypoint extraction, heatmaps_to_keypoints
(lib/utils/keypoints.py:103-157), and of its OKS NMS, nms_oks / compute_oks (lib/utils/keypoints.py:225-266), as called by
keypoint_results (lib/core/test.py:850-866).  Nothing under detectron/ imports this module.

The resize is cv2's float32 INTER_CUBIC on the K-channel HWC heatmap, step by step:
  * per axis scale = 1 / (dst / src) in double, f = float((d + .5) * scale - .5), s = floor(f), f -= s; the four taps
    s - 1 .. s + 2 are clamped into [0, src - 1] and f is kept at the borders;
  * cv2's interpolateCubic coefficients in float32 with A = -0.75: c0 = ((A(x+1) - 5A)(x+1) + 8A)(x+1) - 4A,
    c1 = ((A+2)x - (A+3))x x + 1, c2 the same with 1 - x, c3 = ((1 - c0) - c1) - c2;
  * horizontal pass ((S0 a0 + S1 a1) + S2 a2) + S3 a3;
  * vertical pass over the flattened row of n = w * K floats (channel fastest): its first 4 * floor(n / 4) elements come
    from cv2's 4-lane vector loop, S0 b0 + (S1 b1 + (S2 b2 + S3 b3)), the rest from its scalar tail,
    ((S0 b0 + S1 b1) + S2 b2) + S3 b3;
  * a destination the size of the source is a copy.
Every product and sum is rounded on its own in float32 (numpy ufuncs never fuse).

Per detection, as numpy 2 (NEP 50) evaluates the reference: w = max(x2 - x1, 1) in float32, map_w = int(max(ceil(w),
min_size)) (int(ceil(w)) when min_size <= 0), corr = float32(w / map_w), first argmax in row-major order,
x = float32(float64(x_int + .5) * float64(corr) + float64(x1)), logit = map[y_int, x_int], prob = 1 / sum(exp(map - max)).
"""
import numpy as np

A = np.float32(-0.75)
# COCO keypoint sigmas (lib/utils/keypoints.py:239-241)
OKS_SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0


def cubic_coeffs(x):
    """cv2 interpolateCubic for float32 fractions x (any shape) -> (..., 4) float32."""
    x = np.asarray(x, dtype=np.float32)
    one = np.float32(1)
    xp = x + one
    c0 = ((A * xp - np.float32(5) * A) * xp + np.float32(8) * A) * xp - np.float32(4) * A
    c1 = ((A + np.float32(2)) * x - (A + np.float32(3))) * x * x + one
    y = one - x
    c2 = ((A + np.float32(2)) * y - (A + np.float32(3))) * y * y + one
    c3 = one - c0 - c1 - c2
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.float32)


def cubic_axis(dst, src):
    """(dst, 4) clamped source taps and (dst, 4) float32 coefficients of one axis."""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    f = (f - s).astype(np.float32)
    taps = np.clip(s.astype(np.int64)[:, None] + np.arange(-1, 3)[None, :], 0, src - 1)
    return taps, cubic_coeffs(f)


def resize_cubic(src, w, h):
    """cv2.resize(src, (w, h), interpolation=cv2.INTER_CUBIC) of a float32 (H, W) or (H, W, K) array (K <= 4 with IPP
    off; any K > 4)."""
    src = np.asarray(src, dtype=np.float32)
    squeeze = src.ndim == 2
    if squeeze:
        src = src[:, :, None]
    H, W, K = src.shape
    if (w, h) == (W, H):
        out = src.copy()
    else:
        tx, a = cubic_axis(w, W)
        ty, b = cubic_axis(h, H)
        S = src[:, tx, :]                                              # (H, w, 4, K)
        a = a[None, :, :, None]
        rows = ((S[:, :, 0] * a[:, :, 0] + S[:, :, 1] * a[:, :, 1]) + S[:, :, 2] * a[:, :, 2]) + S[:, :, 3] * a[:, :, 3]
        R = rows.reshape(H, w * K)[ty]                                 # (h, 4, n)
        B = b[:, :, None]
        p = [R[:, j] * B[:, j] for j in range(4)]
        out = ((p[0] + p[1]) + p[2]) + p[3]                            # scalar tail
        v = (w * K) & ~3                                               # cv2's 4-lane vector loop
        out[:, :v] = p[0][:, :v] + (p[1][:, :v] + (p[2][:, :v] + p[3][:, :v]))
        out = out.reshape(h, w, K)
    return out[:, :, 0] if squeeze else out


def map_sizes(rois, min_size=0):
    """float32 widths / heights (clamped to 1) and the int heatmap sizes of every detection."""
    r = np.asarray(rois, dtype=np.float32)
    w = np.maximum(r[:, 2] - r[:, 0], np.float32(1))
    h = np.maximum(r[:, 3] - r[:, 1], np.float32(1))
    if min_size > 0:
        mw = np.maximum(np.ceil(w), np.float32(min_size)).astype(np.int64)
        mh = np.maximum(np.ceil(h), np.float32(min_size)).astype(np.int64)
    else:
        mw, mh = np.ceil(w).astype(np.int64), np.ceil(h).astype(np.int64)
    return w, h, mw, mh


def heatmaps_to_keypoints(maps, rois, min_size=0):
    """maps float32 (D, K, M, M), rois (D, >= 4) -> xy_preds float32 (D, 4, K) = (x, y, logit, prob) per keypoint."""
    maps = np.asarray(maps, dtype=np.float32)
    r = np.asarray(rois, dtype=np.float32)
    D, K = maps.shape[:2]
    w, h, mw, mh = map_sizes(r, min_size)
    out = np.zeros((D, 4, K), np.float32)
    for i in range(D):
        cx = np.float32(w[i] / np.float32(mw[i]))
        cy = np.float32(h[i] / np.float32(mh[i]))
        # CHW, contiguous like the reference's roi_map.copy(): numpy then sums each channel pairwise
        m = np.ascontiguousarray(resize_cubic(maps[i].transpose(1, 2, 0), int(mw[i]), int(mh[i])).transpose(2, 0, 1)).reshape(K, -1)
        pos = m.argmax(axis=1)
        mx = m[np.arange(K), pos]
        xi, yi = pos % mw[i], pos // mw[i]
        out[i, 0] = ((xi + 0.5) * np.float64(cx) + np.float64(r[i, 0])).astype(np.float32)
        out[i, 1] = ((yi + 0.5) * np.float64(cy) + np.float64(r[i, 1])).astype(np.float32)
        out[i, 2] = mx
        out[i, 3] = np.float32(1) / np.exp(m - mx[:, None]).sum(axis=1)
    return out


def oks_scores(xy_preds):
    """float32 mean logit per detection, as np.mean computes it."""
    return np.mean(np.asarray(xy_preds, dtype=np.float32)[:, 2, :], axis=1)


def compute_oks(src_kp, src_roi, dst_kp, dst_roi):
    """OKS of one detection against others, in the reference's dtypes (float32 offsets and area, float64 after that)."""
    var = (OKS_SIGMAS * 2) ** 2
    area = (src_roi[2] - src_roi[0] + np.float32(1)) * (src_roi[3] - src_roi[1] + np.float32(1))
    dx = dst_kp[:, 0, :] - src_kp[0, :]
    dy = dst_kp[:, 1, :] - src_kp[1, :]
    e = (dx ** 2 + dy ** 2) / var / (area + np.spacing(1)) / 2
    return np.sum(np.exp(-e), axis=1) / e.shape[1]


def nms_oks(xy_preds, rois, thresh):
    """Greedy OKS NMS: kept indices in descending score order; equal scores: the higher index first."""
    kp = np.asarray(xy_preds, dtype=np.float32)
    r = np.asarray(rois, dtype=np.float32)
    scores = oks_scores(kp)
    order = np.lexsort((-np.arange(len(scores)), -scores.astype(np.float64)))
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(int(i))
        ovr = compute_oks(kp[i], r[i], kp[order[1:]], r[order[1:]])
        order = order[np.where(ovr <= thresh)[0] + 1]
    return keep
