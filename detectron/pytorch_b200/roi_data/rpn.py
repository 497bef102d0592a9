"""RPN anchor labels and box-regression targets on the device: the training loader's add_rpn_blobs.

The reference builds these blobs on the host for every image of every step (lib/roi_data/rpn.py:40-261 with
lib/roi_data/data_utils.py:50-125): a field of anchors over every level, the anchor x ground-truth IoU matrix
(cython_bbox.bbox_overlaps), a sampled minibatch of RPN_BATCH_SIZE_PER_IM anchors, and four dense blobs per level that are
almost entirely -1 / 0 -- about 23.5 MB per 1333-pixel image at FPN P2-P6, copied host -> device afterwards.  Here the
ground truth goes to the GPU (a few hundred bytes) and the blobs are made there: csrc/rpn_targets.cu, one launch sequence
for all images and levels, one host read (the candidate counts, which size the random draw).

  * `get_rpn_blob_names`  lib/roi_data/rpn.py:13-37
  * `add_rpn_blobs`       lib/roi_data/rpn.py:40-112: same signature, blob names, `im_info` and minimal-`roidb` side effects;
                          the RPN blobs come out as CUDA tensors, concatenated over the images
  * `rpn_targets`         the same for ground truth that is already on the device
  * `generate_anchors`    lib/modeling/generate_anchors.py (the cell anchors, float64)

The random draw of the reference (`npr.choice(fg_inds, n, replace=False)`, `npr.randint(len(bg_inds), size=num_bg)`) is an
INPUT: pass `choices`, per image (positions into the ascending fg candidate list to disable, positions into the ascending bg
candidate list to enable), for a bit-identical minibatch, or leave it None for the same distribution drawn on the device
(torch.randperm / torch.randint).

Configuration: pass the reference's `cfg` (read at call time: FPN.FPN_ON / MULTILEVEL_RPN / RPN_MIN_LEVEL / RPN_MAX_LEVEL /
RPN_ANCHOR_START_SIZE / RPN_ASPECT_RATIOS / COARSEST_STRIDE, RPN.STRIDE / SIZES / ASPECT_RATIOS, TRAIN.MAX_SIZE /
RPN_STRADDLE_THRESH / RPN_POSITIVE_OVERLAP / RPN_NEGATIVE_OVERLAP / RPN_FG_FRACTION / RPN_BATCH_SIZE_PER_IM) or the same
values as keyword arguments (see `_DEFAULTS`, the reference's config defaults).
"""
import numpy as np
import torch

from .. import ops

_DEFAULTS = dict(multilevel_rpn=False, rpn_min_level=2, rpn_max_level=6, rpn_anchor_start_size=32, fpn_aspect_ratios=(0.5, 1, 2),
                 coarsest_stride=32, max_size=1000, rpn_stride=16, rpn_sizes=(64, 128, 256, 512), rpn_aspect_ratios=(0.5, 1, 2),
                 straddle_thresh=0, positive_overlap=0.7, negative_overlap=0.3, fg_fraction=0.5, batch_size_per_im=256)

_NAMES = ("rpn_labels_int32_wide", "rpn_bbox_targets_wide", "rpn_bbox_inside_weights_wide", "rpn_bbox_outside_weights_wide")


def _params(cfg, kw):
    p = dict(_DEFAULTS)
    if cfg is not None:
        f, r, t = cfg.FPN, cfg.RPN, cfg.TRAIN
        p.update(multilevel_rpn=bool(f.FPN_ON and f.MULTILEVEL_RPN), rpn_min_level=f.RPN_MIN_LEVEL, rpn_max_level=f.RPN_MAX_LEVEL,
                 rpn_anchor_start_size=f.RPN_ANCHOR_START_SIZE, fpn_aspect_ratios=f.RPN_ASPECT_RATIOS, coarsest_stride=f.COARSEST_STRIDE,
                 max_size=t.MAX_SIZE, rpn_stride=r.STRIDE, rpn_sizes=r.SIZES, rpn_aspect_ratios=r.ASPECT_RATIOS,
                 straddle_thresh=t.RPN_STRADDLE_THRESH, positive_overlap=t.RPN_POSITIVE_OVERLAP, negative_overlap=t.RPN_NEGATIVE_OVERLAP,
                 fg_fraction=t.RPN_FG_FRACTION, batch_size_per_im=t.RPN_BATCH_SIZE_PER_IM)
    unknown = set(kw) - set(_DEFAULTS)
    if unknown:
        raise TypeError("unknown RPN target parameters: %s" % sorted(unknown))
    p.update(kw)
    return p


def generate_anchors(stride=16, sizes=(32, 64, 128, 256, 512), aspect_ratios=(0.5, 1, 2)):
    """(len(aspect_ratios) * len(sizes), 4) float64 cell anchors, ratio-major.  The reference window is the stride x stride
    square at the origin; for aspect ratio r its width becomes round(sqrt(stride^2 / r)) and its height round(width * r), both
    about its centre; each such box is then scaled by size / stride about the same centre.  A box of width w around centre c
    spans c -+ (w - 1) / 2 (inclusive pixel convention)."""
    scales = np.asarray(sizes, dtype=np.float64) / stride
    ratios = np.asarray(aspect_ratios, dtype=np.float64)
    side = float(stride)                                             # width == height of the reference window (0, 0, side - 1, side - 1)
    ctr = 0.5 * (side - 1)
    rw = np.round(np.sqrt(side * side / ratios))
    rh = np.round(rw * ratios)
    out = []
    for w0, h0 in zip(rw, rh):
        # the ratio box's own width / height / centre, recomputed from its corners as the reference does
        x1, y1, x2, y2 = ctr - 0.5 * (w0 - 1), ctr - 0.5 * (h0 - 1), ctr + 0.5 * (w0 - 1), ctr + 0.5 * (h0 - 1)
        w, h = x2 - x1 + 1, y2 - y1 + 1
        cx, cy = x1 + 0.5 * (w - 1), y1 + 0.5 * (h - 1)
        ws, hs = w * scales, h * scales
        out.append(np.stack([cx - 0.5 * (ws - 1), cy - 0.5 * (hs - 1), cx + 0.5 * (ws - 1), cy + 0.5 * (hs - 1)], axis=1))
    return np.concatenate(out)


def anchor_levels(cfg=None, **kw):
    """[(level or None, field_size, stride, cell_anchors)] of the RPN: one per FPN level, or the single level
    (data_utils.get_field_of_anchors; the field spans FPN.COARSEST_STRIDE * ceil(TRAIN.MAX_SIZE / COARSEST_STRIDE) pixels)."""
    p = _params(cfg, kw)
    cs = p["coarsest_stride"]
    fpn_max = cs * np.ceil(p["max_size"] / float(cs))

    def field(stride):
        return int(np.ceil(fpn_max / float(stride)))
    if p["multilevel_rpn"]:
        k_min, k_max = p["rpn_min_level"], p["rpn_max_level"]
        out = []
        for lvl in range(k_min, k_max + 1):
            stride = 2.0 ** lvl
            sizes = (p["rpn_anchor_start_size"] * 2.0 ** (lvl - k_min),)
            out.append((lvl, field(stride), stride, generate_anchors(stride, sizes, p["fpn_aspect_ratios"])))
        return out
    stride = p["rpn_stride"]
    return [(None, field(stride), stride, generate_anchors(stride, p["rpn_sizes"], p["rpn_aspect_ratios"]))]


def get_rpn_blob_names(is_training=True, cfg=None, **kw):
    """Blob names of the RPN: im_info, and in training roidb plus the four target blobs (per FPN level with the multilevel RPN)."""
    names = ["im_info"]
    if is_training:
        names += ["roidb"]
        for lvl, _, _, _ in anchor_levels(cfg, **kw):
            names += [k if lvl is None else k + "_fpn" + str(lvl) for k in _NAMES]
    return names


def _device_draw(dev):
    def draw(n_dis, nf, n_en, nb):
        dis = torch.randperm(nf, device=dev)[:n_dis] if n_dis else torch.empty((0,), dtype=torch.int64, device=dev)
        en = torch.randint(nb, (n_en,), device=dev) if n_en else torch.empty((0,), dtype=torch.int64, device=dev)
        return dis, en
    return draw


def _host_choice(c, n, size, limit, unique):
    a = np.asarray([] if c is None else c, dtype=np.int64).reshape(-1)
    if a.size != size:
        raise ValueError("image %d: the draw has %d positions, the minibatch takes %d" % (n, a.size, size))
    if a.size and (a.min() < 0 or a.max() >= limit):
        raise ValueError("image %d: draw positions must lie in [0, %d)" % (n, limit))
    if unique and np.unique(a).size != a.size:
        raise ValueError("image %d: the fg draw is without replacement, positions repeat" % n)
    return a


def rpn_targets(gt_boxes_list, im_info, cfg=None, choices=None, **kw):
    """The RPN blobs of N images.  gt_boxes_list: N float32 CUDA (G_i, 4) tensors of scaled ground truth, each G_i >= 1;
    im_info: (N, >= 2) host rows (im_height, im_width, ...).  Returns {blob name: CUDA tensor} with the reference's names and
    (N, A, F, F) / (N, 4A, F, F) shapes."""
    p = _params(cfg, kw)
    N = len(gt_boxes_list)
    if N == 0:
        raise ValueError("rpn_targets needs at least one image")
    for i, g in enumerate(gt_boxes_list):
        ops._need_cuda_f32(g, "gt_boxes")
        if g.dim() != 2 or g.size(1) != 4:
            raise ValueError("gt_boxes must be (G, 4) = [x1, y1, x2, y2], got %s" % (tuple(g.shape),))
        if g.size(0) == 0:
            raise ValueError("image %d has no ground-truth box: the reference's _get_rpn_blobs has no labels for it" % i)
    im_info = im_info.cpu().numpy() if torch.is_tensor(im_info) else np.asarray(im_info)
    im_sizes = np.asarray(im_info, dtype=np.float64).reshape(N, -1)[:, :2]
    levels = anchor_levels(**p)
    dev = gt_boxes_list[0].device
    gt = torch.cat([g.to(dev) for g in gt_boxes_list]) if N > 1 else gt_boxes_list[0]
    num_fg = int(p["fg_fraction"] * p["batch_size_per_im"])
    if choices is not None and len(choices) != N:
        raise ValueError("choices has %d entries for %d images" % (len(choices), N))
    device_draw = _device_draw(dev)

    def draw(counts):
        picks = []
        for n, (nf, nb, ni) in enumerate(counts.tolist()):
            if ni == 0:
                raise ValueError("image %d has no anchor inside it: the reference's _get_rpn_blobs fails there" % n)
            n_dis = max(nf - num_fg, 0)
            num_bg = p["batch_size_per_im"] - (nf - n_dis)
            n_en = num_bg if nb > num_bg else 0
            if choices is None:
                picks.append(device_draw(n_dis, nf, n_en, nb))
            else:
                dis, en = choices[n]
                picks.append((_host_choice(dis, n, n_dis, nf, True), _host_choice(en, n, n_en, nb, False)))
        return picks
    outs = ops.rpn_targets_raw(gt, [g.size(0) for g in gt_boxes_list], im_sizes, [(F, s, c) for _, F, s, c in levels], draw,
                               straddle_thresh=p["straddle_thresh"], positive_overlap=p["positive_overlap"],
                               negative_overlap=p["negative_overlap"])
    blobs = {}
    for (lvl, _, _, _), tensors in zip(levels, outs):
        for k, t in zip(_NAMES, tensors):
            blobs[k if lvl is None else k + "_fpn" + str(lvl)] = t
    return blobs


def add_rpn_blobs(blobs, im_scales, roidb, cfg=None, choices=None, **kw):
    """lib/roi_data/rpn.py:40-112 on the device.  For each roidb entry: im_info row (round(height * scale), round(width *
    scale), scale), ground truth = boxes with gt_classes > 0 and is_crowd == 0, times the scale in float32.  Sets the RPN
    target blobs (CUDA tensors over all images), concatenates every list-valued blob like the reference, and stores the
    minimal roidb under 'roidb'.  Returns True."""
    dev = torch.device("cuda", torch.cuda.current_device())
    im_info, gts, counts = [], [], []
    for i, entry in enumerate(roidb):
        scale = float(im_scales[i])
        im_h = np.round(entry["height"] * scale)
        im_w = np.round(entry["width"] * scale)
        keep = np.where((np.asarray(entry["gt_classes"]) > 0) & (np.asarray(entry["is_crowd"]) == 0))[0]
        gts.append(np.asarray(entry["boxes"], dtype=np.float32)[keep, :] * np.float32(scale))      # float32 * Python float in numpy
        counts.append(keep.size)
        im_info.append(np.array([[im_h, im_w, scale]], dtype=np.float32))
    for i, c in enumerate(counts):
        if c == 0:
            raise ValueError("image %d has no ground-truth box with gt_classes > 0 and is_crowd == 0: the reference's "
                             "_get_rpn_blobs has no labels for it" % i)
    gt_all = torch.from_numpy(np.concatenate(gts).astype(np.float32)).to(dev)                    # one upload for the step
    gt_list = list(torch.split(gt_all, counts))
    rpn = rpn_targets(gt_list, np.concatenate(im_info), cfg=cfg, choices=choices, **kw)
    blobs.setdefault("im_info", [])
    blobs["im_info"].extend(im_info)
    blobs.update(rpn)
    for k, v in blobs.items():
        if isinstance(v, list) and len(v) > 0:
            blobs[k] = np.concatenate(v)
    valid_keys = ["has_visible_keypoints", "boxes", "segms", "seg_areas", "gt_classes", "gt_overlaps", "is_crowd", "box_to_gt_ind_map",
                  "gt_keypoints"]
    blobs["roidb"] = [{k: e[k] for k in valid_keys if k in e} for e in roidb]
    return True
