"""Image transforms of the reference's lib/utils/image.py on the device, and the image decode that feeds them.

`aspect_ratio_rel(im, aspect_ratio)` (:27-32) is the width-relative aspect-ratio change that test-time augmentation
(TEST.MASK_AUG / KPS_AUG.ASPECT_RATIOS) applies to the decoded uint8 image: cv2.resize(im, (int(round(ar * w)), h)), whose
INTER_LINEAR on uint8 is cv2's 8-bit fixed-point arithmetic.  Here one launch computes the same bytes (ops.resize_width_u8,
IPP off) and the result stays on the device, where it feeds the input blob (utils/blob.py) without another upload.

`imread(path)` / `imdecode(buffers)` replace cv2.imread (lib/roi_data/minibatch.py:58, lib/core/test_engine.py:252,
tools/infer_simple.py:144): the JPEG is decoded on the device (ops.jpeg_decode_raw) and the image is a CUDA uint8 (H, W, 3) BGR
tensor equal to cv2.imread's array bit for bit, EXIF orientation included.  A file the device decoder does not take
(progressive, arithmetic-coded, 12-bit, CMYK, other sampling factors; utils/jpeg.py names the reason) or whose entropy data does
not decode is decoded by cv2.imdecode on the host and uploaded, so the result is cv2's for every file.
"""
import numpy as np
import torch

from .. import ops
from . import jpeg as J


def aspect_ratio_rel(im, aspect_ratio):
    """im: a uint8 (h, w, 3) BGR image, a host array or a CUDA tensor.  Returns the uint8 CUDA tensor (h, round(ar * w), 3)."""
    im_h, im_w = int(im.shape[0]), int(im.shape[1])
    im_ar_w = int(round(aspect_ratio * im_w))
    return ops.resize_width_u8(im, im_ar_w)


def _host_decode(p):
    import cv2          # only for files the device decoder does not take
    im = cv2.imdecode(np.frombuffer(p.data, np.uint8), cv2.IMREAD_COLOR)
    if im is None:
        raise ValueError("cv2 could not decode the image (%s)" % (p.fallback or "entropy data"))
    return im


def imdecode(buffers, device=None):
    """Decode JPEG files -- each given as its bytes (bytes, bytearray, a uint8 numpy array) or as the utils/jpeg.parse result
    made in a loader worker (it pickles) -- into a list of uint8 CUDA (H, W, 3) BGR tensors equal to
    cv2.imdecode(buf, cv2.IMREAD_COLOR).  The device decodes the whole list in one launch sequence; the call then reads the
    per-image statuses back once (one synchronisation) to decode any file the device did not on the host.  Raises ValueError
    for a malformed header."""
    parsed = [b if isinstance(b, J.Parsed) else J.parse(b.tobytes() if isinstance(b, np.ndarray) else b) for b in buffers]
    if not parsed:
        return []
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    images, status = ops.jpeg_decode_raw(parsed, device=dev)
    st = status.cpu().numpy()
    for i in np.flatnonzero(st != ops.JPEG_DECODED):
        im = torch.from_numpy(_host_decode(parsed[i]))
        if images[i] is not None and tuple(images[i].shape) == tuple(im.shape):
            images[i].copy_(im)
        else:
            images[i] = im.to(dev)
    return images


def imread(path, device=None):
    """cv2.imread(path) (IMREAD_COLOR) decoded on the device: a uint8 CUDA (H, W, 3) BGR tensor.  Raises OSError when the file
    cannot be read, where cv2.imread returns None."""
    with open(path, "rb") as f:
        data = f.read()
    return imdecode([data], device)[0]
