"""Image transforms of the reference's lib/utils/image.py on the device.

`aspect_ratio_rel(im, aspect_ratio)` (:27-32) is the width-relative aspect-ratio change that test-time augmentation
(TEST.MASK_AUG / KPS_AUG.ASPECT_RATIOS) applies to the decoded uint8 image: cv2.resize(im, (int(round(ar * w)), h)), whose
INTER_LINEAR on uint8 is cv2's 8-bit fixed-point arithmetic.  Here one launch computes the same bytes (ops.resize_width_u8,
IPP off) and the result stays on the device, where it feeds the input blob (utils/blob.py) without another upload.
"""
from .. import ops


def aspect_ratio_rel(im, aspect_ratio):
    """im: a uint8 (h, w, 3) BGR image, a host array or a CUDA tensor.  Returns the uint8 CUDA tensor (h, round(ar * w), 3)."""
    im_h, im_w = int(im.shape[0]), int(im.shape[1])
    im_ar_w = int(round(aspect_ratio * im_w))
    return ops.resize_width_u8(im, im_ar_w)
