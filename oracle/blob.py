"""TEST INFRASTRUCTURE: numpy restatement of the reference's input image blob (lib/utils/blob.py:37-148,
lib/roi_data/minibatch.py:47-79, lib/roi_data/loader.py:251-260) with cv2's resize taken step by step, IPP off.
Nothing under detectron/ imports this module.

- Mean subtraction: `im -= PIXEL_MEANS` on a float32 image with the float64 (1, 1, 3) means is float32(float64(v) - mean),
  so a uint8 image maps through a (3, 256) float32 table.
- cv2.resize(im, None, None, fx=s, fy=s, INTER_LINEAR): the output is rint(W * s) x rint(H * s) (half to even); a zero side
  raises.  An output as large as the input is a copy.  With 1 / s == 2.0 exactly cv2 takes its fast INTER_AREA path: for 3
  channels every element is (((a00 + a01) + a10) + a11) * .25 (its scalar loop; no vector prefix).  On an odd side the last
  output row or column has only the taps inside the image, averaged as (a + b) * .5 (cv2 sums them from 0 and divides by
  their count), and the corner of two odd sides is a00.
  Otherwise per axis scale = 1 / s in double, f = float((d + .5) * scale - .5), s0 = floor(f), f -= s0; on x a position left
  of the first or right of the last column is clamped to it (f = 0), on y f is kept and both row indices are clipped.  A
  horizontal pass S[s0] * (1 - f) + S[s0 + 1] * f, then a vertical one, every product and sum rounded in float32.
- A flipped roidb entry is im[:, ::-1, :] before the mean subtraction.
- Padding: with FPN on, every image of the call is zero-padded to ceil(max(h) / stride) * stride by the same for w.
"""
import numpy as np

DEFAULT_PIXEL_MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])        # lib/core/config.py


def mean_table(pixel_means):
    """(3, 256) float32: channel c of a pixel with value v after `im -= pixel_means`, as numpy computes it."""
    v = np.arange(256, dtype=np.float32).reshape(256, 1, 1)
    out = np.empty((256, 1, 3), np.float32)
    out[...] = v                                        # the image after astype(np.float32)
    out -= np.asarray(pixel_means)                      # numpy's own in-place subtraction
    return np.ascontiguousarray(out.reshape(256, 3).T)


def output_size(h, w, fx):
    """cv2's fx / fy sizing: (rint(h * fx), rint(w * fx)); a zero side raises ValueError where cv2 raises."""
    oh, ow = int(np.rint(h * float(fx))), int(np.rint(w * float(fx)))
    if oh <= 0 or ow <= 0:
        raise ValueError("cv2.resize of a %d x %d image at scale %r has an empty side" % (h, w, fx))
    return oh, ow


def is_area_2x(fx):
    return 1.0 / float(fx) == 2.0


def _axis(dst, src, scale, clamp):
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


def resize(im, fx):
    """cv2.resize(im, None, None, fx=fx, fy=fx, interpolation=cv2.INTER_LINEAR) of an (H, W, C) float32 image, IPP off."""
    im = np.asarray(im, dtype=np.float32)
    H, W = im.shape[:2]
    oh, ow = output_size(H, W, fx)
    if (oh, ow) == (H, W):
        return im.copy()
    if is_area_2x(fx):
        y1, x1 = np.minimum(2 * np.arange(oh) + 1, H - 1), np.minimum(2 * np.arange(ow) + 1, W - 1)
        r0, r1 = im[2 * np.arange(oh)], im[y1]
        a00, a01, a10, a11 = r0[:, 0::2][:, :ow], r0[:, x1], r1[:, 0::2][:, :ow], r1[:, x1]
        out = (((a00 + a01) + a10) + a11) * np.float32(0.25)
        # an odd last row / column: cv2 averages the taps inside the image, summed in row-major order from 0
        if 2 * ow > W:
            out[:, -1] = (a00[:, -1] + a10[:, -1]) * np.float32(0.5)
        if 2 * oh > H:
            out[-1] = (a00[-1] + a01[-1]) * np.float32(0.5)
        if 2 * ow > W and 2 * oh > H:
            out[-1, -1] = a00[-1, -1]
        return out
    scale = 1.0 / float(fx)
    sx, sx1, a0, a1 = _axis(ow, W, scale, True)
    sy, sy1, b0, b1 = _axis(oh, H, scale, False)
    rows = im[:, sx] * a0[None, :, None] + im[:, sx1] * a1[None, :, None]
    return rows[sy] * b0[:, None, None] + rows[sy1] * b1[:, None, None]


def prep_image(im, fx, flipped=False, pixel_means=DEFAULT_PIXEL_MEANS):
    """uint8 (H, W, 3) BGR -> the resized float32 (h, w, 3) image of prep_im_for_blob (flip first, like minibatch.py)."""
    im = np.asarray(im)
    if flipped:
        im = im[:, ::-1, :]
    tab = mean_table(pixel_means)
    f = np.stack([tab[c][im[:, :, c]] for c in range(3)], axis=2)
    return resize(f, fx)


def get_target_scale(im_size_min, im_size_max, target_size, max_size):
    im_scale = float(target_size) / float(im_size_min)
    if np.round(im_scale * im_size_max) > max_size:
        im_scale = float(max_size) / float(im_size_max)
    return im_scale


def get_max_shape(im_shapes, stride=None):
    """Largest (h, w); with an FPN stride rounded up to a multiple of it."""
    max_shape = np.array(im_shapes).max(axis=0)
    if stride:
        max_shape[0] = int(np.ceil(max_shape[0] / float(stride)) * float(stride))
        max_shape[1] = int(np.ceil(max_shape[1] / float(stride)) * float(stride))
    return max_shape


def im_list_to_blob(ims, stride=None):
    hp, wp = get_max_shape([im.shape[:2] for im in ims], stride)
    blob = np.zeros((len(ims), hp, wp, 3), np.float32)
    for i, im in enumerate(ims):
        blob[i, :im.shape[0], :im.shape[1], :] = im
    return np.ascontiguousarray(blob.transpose(0, 3, 1, 2))


def get_image_blob(im, target_scale, target_max_size, pixel_means=DEFAULT_PIXEL_MEANS, stride=None):
    """Test time: (blob (1, 3, Hp, Wp), im_scale, im_info (1, 3) float32 = (Hp, Wp, im_scale))."""
    h, w = np.asarray(im).shape[:2]
    s = get_target_scale(min(h, w), max(h, w), target_scale, target_max_size)
    blob = im_list_to_blob([prep_image(im, s, False, pixel_means)], stride)
    im_info = np.array([[blob.shape[2], blob.shape[3], s]], dtype=np.float32)
    return blob, s, im_info


def minibatch_image_blob(ims, flipped, scales, scale_inds, max_size, pixel_means=DEFAULT_PIXEL_MEANS, stride=None):
    """Training (_get_image_blob): image i at target scales[scale_inds[i]], capped at max_size -> (blob, im_scales)."""
    out, im_scales = [], []
    for im, fl, k in zip(ims, flipped, scale_inds):
        h, w = np.asarray(im).shape[:2]
        s = get_target_scale(min(h, w), max(h, w), scales[int(k)], max_size)
        out.append(prep_image(im, s, fl, pixel_means))
        im_scales.append(s)
    return im_list_to_blob(out, stride), im_scales
