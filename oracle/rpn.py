"""TEST INFRASTRUCTURE (CPU oracle, never imported by the product): numpy restatement of the reference's RPN anchor labels and
targets (lib/roi_data/rpn.py:40-261, lib/roi_data/data_utils.py:50-125), with the random draw as an input.

  field_of_anchors   data_utils.get_field_of_anchors: float64 cell anchors + shifts, cast to float32
  rpn_blobs          rpn._get_rpn_blobs for one image: inside test, IoU (oracle.targets.bbox_overlaps), tie rule, fg / bg
                     draw, targets for the fg set before the bg draw, weights, unmap, per-level (1, A, F, F) blobs
  add_rpn_blobs      rpn.add_rpn_blobs: ground-truth selection and scaling, im_info, concatenation over images

Levels are (level or None, field_size, stride, cell_anchors) tuples.  Pinned by tests/golden/rpn.npz, produced by the
UNMODIFIED reference function (tests/golden/make_golden_rpn.py).
"""
import numpy as np

from oracle.targets import bbox_overlaps, bbox_transform_inv

f32 = np.float32
NAMES = ("rpn_labels_int32_wide", "rpn_bbox_targets_wide", "rpn_bbox_inside_weights_wide", "rpn_bbox_outside_weights_wide")
_CHUNK = 65536


def field_of_anchors(F, stride, cell):
    shifts = np.arange(F) * stride
    sx, sy = np.meshgrid(shifts, shifts)
    s = np.stack([sx.ravel(), sy.ravel(), sx.ravel(), sy.ravel()], axis=1)
    return (np.asarray(cell)[None, :, :] + s[:, None, :]).reshape(-1, 4).astype(f32)


def _rows(anchors, gt, fn):
    """fn(overlap rows) for chunks of anchors: the (num_anchors, G) matrix is never held at once."""
    return [fn(bbox_overlaps(anchors[i:i + _CHUNK], gt)) for i in range(0, anchors.shape[0], _CHUNK)]


def rpn_blobs(im_h, im_w, levels, gt, fg_disable=None, bg_enable=None, rng=None, straddle_thresh=0, positive_overlap=0.7,
              negative_overlap=0.3, fg_fraction=0.5, batch_size_per_im=256):
    """One image.  The draw: fg_disable / bg_enable positions (into the ascending fg / bg candidate lists), or `rng` (a
    numpy RandomState drawing like npr.choice / npr.randint).  Returns (per-level dicts of (1, ...) blobs, (disable, enable)
    positions used, (#fg candidates, #bg candidates, #inside))."""
    gt = np.asarray(gt, f32)
    all_anchors = np.concatenate([field_of_anchors(F, s, c) for _, F, s, c in levels])
    total = all_anchors.shape[0]
    if straddle_thresh >= 0:
        inds_inside = np.where((all_anchors[:, 0] >= -straddle_thresh) & (all_anchors[:, 1] >= -straddle_thresh) &
                               (all_anchors[:, 2] < im_w + straddle_thresh) & (all_anchors[:, 3] < im_h + straddle_thresh))[0]
    else:
        inds_inside = np.arange(total)
    anchors = all_anchors[inds_inside]
    n_in = anchors.shape[0]
    if n_in == 0 or gt.shape[0] == 0:
        raise ValueError("no inside anchor or no ground truth")
    argmax = np.concatenate(_rows(anchors, gt, lambda o: o.argmax(axis=1)))
    colmax = np.max(np.stack(_rows(anchors, gt, lambda o: o.max(axis=0))), axis=0)
    row_max = np.concatenate(_rows(anchors, gt, lambda o: o.max(axis=1)))
    tie = np.concatenate(_rows(anchors, gt, lambda o: (o == colmax[None, :]).any(axis=1)))
    labels = np.full((n_in,), -1, np.int32)
    labels[tie] = 1
    labels[row_max >= f32(positive_overlap)] = 1
    num_fg = int(fg_fraction * batch_size_per_im)
    fg_inds = np.where(labels == 1)[0]
    nf = fg_inds.size
    bg_cand = np.where(row_max < f32(negative_overlap))[0]
    nb = bg_cand.size
    dis = np.zeros((0,), np.int64)
    if nf > num_fg:
        dis = np.asarray(fg_disable, np.int64) if rng is None else rng.permutation(nf)[:nf - num_fg]
        assert dis.size == nf - num_fg and np.unique(dis).size == dis.size
        labels[fg_inds[dis]] = -1
    fg_inds = np.where(labels == 1)[0]
    num_bg = batch_size_per_im - np.sum(labels == 1)
    en = np.zeros((0,), np.int64)
    if nb > num_bg:
        en = np.asarray(bg_enable, np.int64) if rng is None else rng.randint(nb, size=num_bg)
        assert en.size == num_bg
        labels[bg_cand[en]] = 0
    targets = np.zeros((n_in, 4), f32)
    targets[fg_inds] = bbox_transform_inv(anchors[fg_inds], gt[argmax[fg_inds]], (1.0, 1.0, 1.0, 1.0))
    inside = np.zeros((n_in, 4), f32)
    inside[labels == 1] = 1
    outside = np.zeros((n_in, 4), f32)
    outside[labels >= 0] = 1.0 / np.sum(labels >= 0)

    def unmap(v, fill):
        out = np.full((total,) + v.shape[1:], fill, v.dtype)
        out[inds_inside] = v
        return out
    full = (unmap(labels, -1), unmap(targets, 0), unmap(inside, 0), unmap(outside, 0))
    per_level, start = [], 0
    for _, F, _, c in levels:
        A = np.asarray(c).shape[0]
        end = start + F * F * A
        lab = full[0][start:end].reshape(1, F, F, A).transpose(0, 3, 1, 2)
        rest = [v[start:end].reshape(1, F, F, 4 * A).transpose(0, 3, 1, 2) for v in full[1:]]
        per_level.append(dict(zip(NAMES, [lab] + rest)))
        start = end
    return per_level, (dis, en), (nf, nb, n_in)


def add_rpn_blobs(im_scales, roidb, levels, choices=None, rng=None, **params):
    """The blobs of add_rpn_blobs for all images (numpy), the draws used and the per-image candidate counts."""
    blobs = {"im_info": []}
    draws, counts = [], []
    for i, entry in enumerate(roidb):
        scale = im_scales[i]
        im_h = np.round(entry["height"] * scale)
        im_w = np.round(entry["width"] * scale)
        keep = np.where((entry["gt_classes"] > 0) & (entry["is_crowd"] == 0))[0]
        gt = entry["boxes"][keep, :] * scale
        blobs["im_info"].append(np.array([[im_h, im_w, scale]], dtype=f32))
        dis, en = choices[i] if choices is not None else (None, None)
        per_level, used, cnt = rpn_blobs(im_h, im_w, levels, gt, dis, en, rng, **params)
        draws.append(used); counts.append(cnt)
        for (lvl, _, _, _), d in zip(levels, per_level):
            for k, v in d.items():
                blobs.setdefault(k if lvl is None else k + "_fpn" + str(lvl), []).append(v)
    return {k: np.concatenate(v) for k, v in blobs.items()}, draws, counts
