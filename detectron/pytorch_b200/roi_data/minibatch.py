"""The training step's input image blob on the device: _get_image_blob of lib/roi_data/minibatch.py:47-79 (reference), with
the loader's padding to a common size (lib/roi_data/loader.py:251-260) folded in.

The reference builds one float blob per image in each loader worker and pads them together in collate_minibatch.  Here the
workers hand over the decoded uint8 images (CUDA cannot be used in a worker) and the main process builds the step's whole
blob in one launch (utils/blob.py, ops.image_blob_raw), with the reference's values under cv2's IPP off.
"""
import numpy as np

from .. import ops
from ..utils import blob as blob_utils


def get_image_blob(roidb, images, scale_inds=None, cfg=None, **kw):
    """_get_image_blob for all images of a step.  roidb: the entries (their 'flipped' flags are used); images: the decoded
    uint8 (H, W, 3) BGR images of those entries, unflipped, host arrays or CUDA tensors.  scale_inds: the indices into
    TRAIN.SCALES, or None to draw them with the reference's np.random.randint call (so a seeded loader draws the same ones).
    Configuration: `cfg` (TRAIN.SCALES, TRAIN.MAX_SIZE, PIXEL_MEANS, FPN.FPN_ON, FPN.COARSEST_STRIDE) or keywords scales,
    max_size, pixel_means, fpn_on, coarsest_stride.  Returns (blob float32 CUDA (N, 3, Hp, Wp), im_scales list of floats)."""
    p = blob_utils.blob_params(cfg, **{k: v for k, v in kw.items() if k not in ("scales", "max_size")})
    scales = tuple(kw["scales"]) if "scales" in kw else tuple(cfg.TRAIN.SCALES) if cfg is not None else (600,)
    max_size = kw["max_size"] if "max_size" in kw else cfg.TRAIN.MAX_SIZE if cfg is not None else 1000      # lib/core/config.py:45-48
    num_images = len(roidb)
    if len(images) != num_images:
        raise ValueError("get_image_blob: %d roidb entries, %d images" % (num_images, len(images)))
    if scale_inds is None:
        scale_inds = np.random.randint(0, high=len(scales), size=num_images)
    im_scales = []
    for i in range(num_images):
        h, w = int(images[i].shape[0]), int(images[i].shape[1])
        im_scales.append(blob_utils.get_target_scale(min(h, w), max(h, w), scales[int(scale_inds[i])], max_size))
    blob, _ = ops.image_blob_raw(list(images), im_scales, [bool(e["flipped"]) for e in roidb], p["pixel_means"],
                                 p["coarsest_stride"] if p["fpn_on"] else None)
    return blob, im_scales
