"""The network's input image blob on the device, under the names of lib/utils/blob.py (reference).

The reference builds the `data` blob on the host: the decoded uint8 image becomes float32, loses PIXEL_MEANS, goes through
cv2.resize(fx = fy = im_scale, INTER_LINEAR), is zero-padded to a multiple of FPN.COARSEST_STRIDE and transposed to NCHW,
and the float blob (10.4 MB for a COCO image at 800 / 1333) is copied to the GPU.  Here the uint8 image is uploaded and one
launch writes the finished blob (ops.image_blob_raw), with the same values as the reference run with cv2's IPP off:
  * the mean subtraction is numpy's float32(float64(v) - mean);
  * the resized size is cv2's rint(h * im_scale) x rint(w * im_scale), and the interpolation is cv2's float32 arithmetic,
    including its fast INTER_AREA path for an exact 2x shrink.
With IPP on (cv2's default) the reference's own float resize differs from that by a few float32 ulps at 2x and up to ~1e-2 on
upscaled noise; the device follows IPP off.

Configuration (PIXEL_MEANS, FPN.FPN_ON, FPN.COARSEST_STRIDE) is read from `cfg` at call time, or passed as keywords
pixel_means, fpn_on, coarsest_stride.
"""
import numpy as np

from .. import ops

DEFAULT_PIXEL_MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])          # lib/core/config.py:942


def blob_params(cfg=None, **kw):
    if cfg is not None:
        p = dict(pixel_means=cfg.PIXEL_MEANS, fpn_on=bool(cfg.FPN.FPN_ON), coarsest_stride=int(cfg.FPN.COARSEST_STRIDE))
    else:
        p = dict(pixel_means=DEFAULT_PIXEL_MEANS, fpn_on=False, coarsest_stride=32)       # lib/core/config.py:683-693, 942
    p.update(kw)
    return p


def get_image_blob(im, target_scale, target_max_size, cfg=None, _hflip=False, **kw):
    """lib/utils/blob.py:37-60 on the device.  im: a decoded uint8 (H, W, 3) BGR image, a host array or a CUDA tensor.
    Returns (blob float32 CUDA (1, 3, Hp, Wp), im_scale float, im_info float32 numpy (1, 3) = (Hp, Wp, im_scale)).
    _hflip: the blob of im[:, ::-1, :], read mirrored by the blob kernel (the box head's flipped test-time transforms)."""
    p = blob_params(cfg, **kw)
    h, w = int(im.shape[0]), int(im.shape[1])
    im_scale = get_target_scale(min(h, w), max(h, w), target_scale, target_max_size)
    blob, _ = ops.image_blob_raw([im], [im_scale], [_hflip], p["pixel_means"], p["coarsest_stride"] if p["fpn_on"] else None)
    im_info = np.hstack((blob.shape[2], blob.shape[3], im_scale))[np.newaxis, :]
    return blob, im_scale, im_info.astype(np.float32)


def get_max_shape(im_shapes, cfg=None, **kw):
    """lib/utils/blob.py:88-98: the largest (h, w), rounded up to a multiple of FPN.COARSEST_STRIDE with FPN on."""
    p = blob_params(cfg, **kw)
    max_shape = np.array(im_shapes).max(axis=0)
    assert max_shape.size == 2
    if p["fpn_on"]:
        stride = float(p["coarsest_stride"])
        max_shape[0] = int(np.ceil(max_shape[0] / stride) * stride)
        max_shape[1] = int(np.ceil(max_shape[1] / stride) * stride)
    return max_shape


def get_target_scale(im_size_min, im_size_max, target_size, max_size):
    """lib/utils/blob.py:139-148: target_size / im_size_min, unless that makes the rounded long side exceed max_size."""
    im_scale = float(target_size) / float(im_size_min)
    if np.round(im_scale * im_size_max) > max_size:
        im_scale = float(max_size) / float(im_size_max)
    return im_scale
