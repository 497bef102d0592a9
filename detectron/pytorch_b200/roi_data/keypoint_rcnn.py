"""Keypoint R-CNN training targets on the device (SURVEY.md 8f N4): add_keypoint_rcnn_blobs and finalize_keypoint_minibatch,
lib/roi_data/keypoint_rcnn.py:33-96 with lib/utils/keypoints.py:160-211.

The reference tests every merged box of every image against the 17 keypoints of its person in numpy, draws up to
fg_rois_per_image of the candidates and encodes one heatmap index and one weight per (RoI, keypoint).  Here all images of a
step go through one candidates launch, one host read of the N candidate counts (they size the draw), and one emit launch
(csrc/keypoint_targets.cu); the roidb's host arrays are uploaded once and the blobs come out as CUDA tensors.

Kept from the reference:
  * gt_inds[box_to_gt_ind_map] is numpy indexing: -1 (a proposal without overlap) selects the last person for the candidate
    test; a selected RoI whose map entry is negative gets keypoints of all -1, so weights 0 (only with FG_THRESH <= 0);
  * in the merged roidb a ground-truth row maps to itself with overlap 1 and a crowd row has overlap -1: a crowd row is never
    a candidate, and identical gt boxes keep their own people's keypoints;
  * np.random.choice draws only when there are more candidates than fg_rois_per_image; otherwise every candidate is taken in
    ascending order.  The draw is an input (`choice`: the positions it picked) or torch.randperm on the device;
  * the locations are the float32 heatmap labels after astype(int32): INT_MIN where the label is NaN (zero-width or
    zero-height boxes), always with weight 0;
  * keypoint_loss_normalizer = float32(sum of weights) / float32(IMS_PER_BATCH * BATCH_SIZE_PER_IM * FG_FRACTION *
    NUM_KEYPOINTS), the value numpy 2 gives.
Configuration (KRCNN.HEATMAP_SIZE, KRCNN.NUM_KEYPOINTS, TRAIN.*) is read from `cfg` at call time, or from keywords.
"""
import numpy as np
import torch

from .. import ops


def _config(cfg, heatmap_size, num_keypoints, fg_thresh):
    if cfg is not None:
        return int(cfg.KRCNN.HEATMAP_SIZE), int(cfg.KRCNN.NUM_KEYPOINTS), float(cfg.TRAIN.FG_THRESH)
    if heatmap_size is None or num_keypoints is None:
        raise ValueError("keypoint targets need heatmap_size and num_keypoints (or cfg=)")
    return int(heatmap_size), int(num_keypoints), 0.5 if fg_thresh is None else float(fg_thresh)


def _no_cpu_tensors(*xs):
    for x in xs:
        if torch.is_tensor(x) and not x.is_cuda:
            raise NotImplementedError("keypoint targets are computed on the device: pass CUDA tensors or host arrays, not CPU tensors")


def _keypoints(entry, K):
    kp = np.asarray(entry["gt_keypoints"])
    if kp.ndim != 3 or kp.shape[1] != 3 or kp.shape[2] != K:
        raise ValueError("gt_keypoints must be (G, 3, NUM_KEYPOINTS = %d), got %s" % (K, kp.shape))
    return kp


def keypoint_rcnn_blobs(boxes, box_begin, max_overlaps, box_to_gt_ind_map, roidb, im_scales, fg_rois_per_image, heatmap_size,
                        num_keypoints, fg_thresh=0.5, choices=None, batch_index=None):
    """The keypoint blobs of N images in one device call.  boxes (B, 4) unscaled, max_overlaps (B,), box_to_gt_ind_map (B,): the
    merged roidb's, image n's in rows box_begin[n] .. box_begin[n + 1] - 1, CUDA tensors or host arrays; roidb: per image
    the entry holding 'gt_classes' and 'gt_keypoints'; choices: per image the np.random.choice positions (used when the image
    has more candidates than fg_rois_per_image) or None (torch.randperm on the device).  Returns dict(keypoint_rois,
    keypoint_locations_int32, keypoint_weights), concatenated over images."""
    _no_cpu_tensors(boxes, max_overlaps, box_to_gt_ind_map)
    K, fg = int(num_keypoints), int(fg_rois_per_image)
    kps = [_keypoints(e, K) for e in roidb]
    gt_inds = [np.where(np.asarray(e["gt_classes"]).reshape(-1) > 0)[0] for e in roidb]
    dev = next((t.device for t in (boxes, max_overlaps, box_to_gt_ind_map) if torch.is_tensor(t)), None)
    dev = dev if dev is not None else torch.device("cuda", torch.cuda.current_device())

    def draw(counts):
        out = []
        for n, c in enumerate(counts):
            c = int(c)
            if c <= fg:
                out.append(None)                                        # no draw: every candidate, ascending
            elif choices is not None and choices[n] is not None:
                out.append(choices[n])
            else:
                out.append(torch.randperm(c, device=dev)[:fg])
        return out
    rois, loc, w, _ = ops.keypoint_targets_raw(boxes, box_begin, max_overlaps, box_to_gt_ind_map, gt_inds, kps, im_scales, fg, draw,
                                               heatmap_size, fg_thresh, batch_index, device=dev)
    return dict(keypoint_rois=rois, keypoint_locations_int32=loc, keypoint_weights=w)


def add_keypoint_rcnn_blobs(blobs, roidb, fg_rois_per_image, fg_inds, im_scale, batch_idx, cfg=None, choice=None, heatmap_size=None,
                            num_keypoints=None, fg_thresh=None):
    """The reference's signature for one image.  roidb = the merged entry: 'boxes' (unscaled), 'max_overlaps',
    'box_to_gt_ind_map', 'gt_classes', 'gt_keypoints' (G, 3, K) (host arrays or CUDA tensors).  fg_inds is accepted and unused,
    as in the reference.  choice: the np.random.choice positions into the candidate list (used only when there are more
    candidates than fg_rois_per_image), else a device draw.  Adds 'keypoint_rois' (R, 5) float32, 'keypoint_locations_int32'
    (R * K,) int32 and 'keypoint_weights' (R * K,) float32, all CUDA."""
    HS, K, thresh = _config(cfg, heatmap_size, num_keypoints, fg_thresh)
    boxes = roidb["boxes"]
    B = boxes.shape[0] if not torch.is_tensor(boxes) else boxes.size(0)
    out = keypoint_rcnn_blobs(boxes, [0, B], roidb["max_overlaps"], roidb["box_to_gt_ind_map"], [roidb], [im_scale], fg_rois_per_image,
                              HS, K, thresh, choices=[choice], batch_index=[batch_idx])
    blobs.update(out)


def finalize_keypoint_minibatch(blobs, valid, cfg=None, ims_per_batch=2, batch_size_per_im=64, fg_fraction=0.25, num_keypoints=None,
                                min_count=20):
    """After the images' blobs are concatenated: 'keypoint_loss_normalizer' as a 0-d float32 CUDA tensor, computed on the device.
    Returns the minibatch's validity (valid, weights not empty, more than min_count visible keypoints) as a 0-d CUDA bool
    tensor: nothing is read back here."""
    if cfg is not None:
        ims_per_batch, batch_size_per_im, fg_fraction = cfg.TRAIN.IMS_PER_BATCH, cfg.TRAIN.BATCH_SIZE_PER_IM, cfg.TRAIN.FG_FRACTION
        num_keypoints, min_count = cfg.KRCNN.NUM_KEYPOINTS, cfg.KRCNN.MIN_KEYPOINT_COUNT_FOR_VALID_MINIBATCH
    if num_keypoints is None:
        raise ValueError("finalize_keypoint_minibatch needs num_keypoints (or cfg=)")
    w = blobs["keypoint_weights"]
    _no_cpu_tensors(w)
    if not torch.is_tensor(w):
        raise NotImplementedError("keypoint_weights must be a CUDA tensor (from add_keypoint_rcnn_blobs)")
    visible = w.sum(dtype=torch.float32)                                # 0 / 1 weights: exact below 2^24
    # a tensor divisor: torch turns division by a host scalar into a multiplication by its reciprocal
    den = torch.full((), float(np.float32(ims_per_batch * batch_size_per_im * fg_fraction * num_keypoints)), dtype=torch.float32,
                     device=w.device)
    blobs["keypoint_loss_normalizer"] = visible / den
    ok = (visible > float(min_count)) & (w.numel() > 0)
    return ok & valid if torch.is_tensor(valid) else ok & bool(valid)
