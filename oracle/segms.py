"""TEST INFRASTRUCTURE: numpy restatement of the loop body of the reference's segm_results (lib/core/test.py:793-847) --
box expansion (lib/utils/boxes.py:233-249) and int32 truncation, cv2.resize(INTER_LINEAR) of the zero-padded float32 mask
with IPP off, the strict threshold, the paste into the full image, and the COCO RLE (pycocotools rleEncode + rleToString).
Nothing under detectron/ imports this module.

The resize is cv2's float32 INTER_LINEAR step by step: per axis scale = 1 / (dst / src) in double, f = float((d + .5) *
scale - .5), s = floor(f), f -= s.  On the x axis a position left of the first or right of the last source column is
clamped to it (f = 0); on the y axis f is kept and both row indices s, s + 1 are clipped into the source, so a border row
is r0 * (1 - f) + r0 * f, which is not always r0.  A horizontal pass, then a vertical pass; every product and sum rounded
separately in float32.  When both axes shrink by exactly 2, cv2 switches to INTER_AREA.  Its 4-lane (128-bit) vector
loop covers the first 4 * floor(w / 4) output columns of a row as ((a00 + a01) + (a10 + a11)) * 0.25; the remaining
columns go through its scalar loop, (((a00 + a01) + a10) + a11) * 0.25.
"""
import numpy as np


def expand_boxes_int(boxes, M):
    """float32 (D, 4) detections -> int32 (D, 4) pasting boxes, like segm_results (float32 arithmetic, truncation)."""
    b = np.asarray(boxes, dtype=np.float32)[:, :4]
    scale = np.float32((M + 2.0) / M)
    w_half = (b[:, 2] - b[:, 0]) * np.float32(.5)
    h_half = (b[:, 3] - b[:, 1]) * np.float32(.5)
    x_c = (b[:, 2] + b[:, 0]) * np.float32(.5)
    y_c = (b[:, 3] + b[:, 1]) * np.float32(.5)
    w_half = w_half * scale
    h_half = h_half * scale
    return np.stack([x_c - w_half, y_c - h_half, x_c + w_half, y_c + h_half], axis=1).astype(np.int32)


def _axis(dst, src, clamp):
    """Source taps and weights of one axis.  cv2 clamps the position on the x axis (clamp=True: weight 0 on the second
    tap); on the y axis it keeps the fraction and clips both row indices into the source."""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    f = (f - s).astype(np.float32)
    s = s.astype(np.int64)
    if clamp:
        lo = s < 0
        f[lo] = 0; s[lo] = 0
        hi = s >= src - 1
        f[hi] = 0; s[hi] = src - 1
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), (np.float32(1) - f).astype(np.float32), f


def resize(src, w, h):
    """cv2.resize(src, (w, h)) for a 2-D float32 array with IPP off."""
    src = np.asarray(src, dtype=np.float32)
    H, W = src.shape
    if 2 * w == W and 2 * h == H:
        a00, a01, a10, a11 = src[0::2, 0::2], src[0::2, 1::2], src[1::2, 0::2], src[1::2, 1::2]
        out = (((a00 + a01) + a10) + a11) * np.float32(0.25)
        v = w & ~3                              # columns of cv2's 4-lane vector loop, the rest is its scalar tail
        out[:, :v] = ((a00[:, :v] + a01[:, :v]) + (a10[:, :v] + a11[:, :v])) * np.float32(0.25)
        return out
    sx, sx1, a0, a1 = _axis(w, W, True)
    sy, sy1, b0, b1 = _axis(h, H, False)
    rows = src[:, sx] * a0 + src[:, sx1] * a1
    return rows[sy] * b0[:, None] + rows[sy1] * b1[:, None]


def paste_window(box, im_h, im_w):
    """(y0, y1, x0, x1) of the pasted region of an int32 box; empty when the box lies outside the image."""
    x0, x1 = max(int(box[0]), 0), min(int(box[2]) + 1, im_w)
    y0, y1 = max(int(box[1]), 0), min(int(box[3]) + 1, im_h)
    return y0, max(y1, y0), x0, max(x1, x0)


def segm_one(mask, box, im_h, im_w, thresh):
    """mask (M, M) float32, box int32 (4,) -> (uint8 full-image mask, window, interpolated float32 values in the window)."""
    M = mask.shape[0]
    padded = np.zeros((M + 2, M + 2), np.float32)
    padded[1:-1, 1:-1] = mask
    w = max(int(box[2]) - int(box[0]) + 1, 1)
    h = max(int(box[3]) - int(box[1]) + 1, 1)
    y0, y1, x0, x1 = paste_window(box, im_h, im_w)
    im = np.zeros((im_h, im_w), np.uint8)
    vals = np.zeros((y1 - y0, x1 - x0), np.float32)
    if y1 > y0 and x1 > x0:
        r = resize(padded, w, h)
        vals = r[y0 - box[1]:y1 - box[1], x0 - box[0]:x1 - box[0]]
        im[y0:y1, x0:x1] = vals > np.float32(thresh)
    return im, (y0, y1, x0, x1), vals


def rle_counts(im_mask):
    """Uncompressed COCO counts of a 2-D binary mask: column-major, starting with a run of zeros (pycocotools rleEncode)."""
    flat = np.asarray(im_mask, dtype=np.uint8).ravel(order="F")
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    if flat.size and flat[0]:
        change = np.concatenate([[0], change])
    bounds = np.concatenate([[0], change, [flat.size]])
    return np.diff(bounds).astype(np.uint32)


def rle_string(counts):
    """pycocotools rleToString: counts -> compressed ASCII bytes."""
    out = bytearray()
    cnts = [int(c) for c in counts]
    for i, c in enumerate(cnts):
        x = c - cnts[i - 2] if i > 2 else c
        more = True
        while more:
            ch = x & 0x1f
            x >>= 5
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(ch + 48)
    return bytes(out)


def rle_from_string(s, size):
    """Inverse of rle_string (pycocotools rleFrString), written independently of it for round trips."""
    cnts, p, data = [], 0, bytes(s)
    while p < len(data):
        x, k, more = 0, 0, True
        while more:
            c = data[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1; k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    assert sum(cnts) == size[0] * size[1]
    return np.asarray(cnts, dtype=np.int64)


def decode_counts(counts, im_h, im_w):
    """Uncompressed counts -> (im_h, im_w) uint8 mask."""
    vals = np.zeros(len(counts), np.uint8)
    vals[1::2] = 1
    return np.repeat(vals, np.asarray(counts, dtype=np.int64)).reshape((im_w, im_h)).T.copy()


def segm_rles(masks, mask_class, boxes, im_h, im_w, thresh):
    """Every detection of one image: masks (D, Kc, M, M), mask_class (D,) channel per detection, boxes float32 (D, 4).
    Returns (list of uncompressed counts, list of strings, list of (window, interpolated values))."""
    masks = np.asarray(masks, dtype=np.float32)
    M = masks.shape[-1]
    ib = expand_boxes_int(boxes, M)
    counts, strings, interp = [], [], []
    for d in range(masks.shape[0]):
        im, win, vals = segm_one(masks[d, int(mask_class[d])], ib[d], im_h, im_w, thresh)
        c = rle_counts(im)
        counts.append(c); strings.append(rle_string(c)); interp.append((win, vals))
    return counts, strings, interp
