"""GPU-resident RPN proposal layer (SURVEY.md 8f N1).

Mirrors `GenerateProposalsOp` of lib/modeling/generate_proposals.py:12-168 (reference): same constructor
`(anchors, spatial_scale)`, same `forward(rpn_cls_prob, rpn_bbox_pred, im_info) -> (rois ndarray (R, 5), roi_probs
ndarray (R, 1))`.  The reference copies the score map, the deltas and im_info to the host (three blocking D2H copies,
generate_proposals.py:58-63), runs a 200 k-anchor numpy top-k, decode, clip, filter and the Cython NMS on one CPU
thread, and the caller copies the RoIs back.  Here everything up to the final result stays on the device:

    b200_topk_batched (radix select + in-CTA sort over every (level, image) score map of the step, read in place)  ->
    b200_proposal_decode (anchor rebuild + bbox_transform + clip + filter, one kernel)  ->  b200_nms_batched (bitmask +
    on-device scan)  ->  ONE D2H of the kept rows per image
(torch.sort remains only as the fallback for k > 16384 candidates per map.)

Configuration: the reference reads `cfg[TRAIN|TEST].RPN_{PRE,POST}_NMS_TOP_N, RPN_NMS_THRESH, RPN_MIN_SIZE` from its
global config at call time; pass that object as `cfg=` to do the same, or give the four values per mode as keyword
arguments (`train=dict(...)`, `test=dict(...)`); defaults are the reference's (lib/core/config.py:127-141, 200-214).

Documented differences (see oracle/proposals.py): the reference leaves the order of EQUAL scores unspecified (its
argpartition/argsort); here the pre-NMS candidates are exactly np.argsort(-scores, kind="stable")[:pre_nms_topN] of the
(H, W, A)-flattened map, on the device top-k and on the torch.sort fallback alike: equal scores -- also those that straddle the
cut -- are taken in ascending (h, w, a) index, NaN scores rank below every number (as numpy sorts them) and -0.0 ties with
+0.0.  A candidate whose decoded box has a NaN coordinate is dropped, as the reference's _filter_boxes drops it.  NaN scores
that do reach NMS (only when pre_nms_topN exceeds the number of finite scores) stay where the sort put them, last; the
reference's Cython NMS re-sorts and puts them first.  NMS suppresses at IoU > thresh with the CUDA kernel's rounding (the
reference's host NMS uses >=); results on the golden vectors are identical.  All images of a call -- and, through
generate_proposals_batched, all FPN levels of a step -- share ONE batched NMS launch pair and ONE host read.
"""
import numpy as np
import torch
from torch import nn

from detectron.pytorch_b200 import ops

_DEFAULTS = {
    "TRAIN": dict(RPN_PRE_NMS_TOP_N=12000, RPN_POST_NMS_TOP_N=2000, RPN_NMS_THRESH=0.7, RPN_MIN_SIZE=0),
    "TEST": dict(RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=1000, RPN_NMS_THRESH=0.7, RPN_MIN_SIZE=0),
}


class GenerateProposalsOp(nn.Module):
    def __init__(self, anchors, spatial_scale, cfg=None, train=None, test=None, return_tensors=False):
        super().__init__()
        self._return_tensors = bool(return_tensors)       # True: CUDA tensors out (for the on-device FPN chain), False: numpy like the reference
        self._anchors = np.asarray(anchors)
        self._num_anchors = self._anchors.shape[0]
        self._feat_stride = 1. / spatial_scale
        self._cfg = cfg
        self._params = {"TRAIN": dict(_DEFAULTS["TRAIN"], **(train or {})), "TEST": dict(_DEFAULTS["TEST"], **(test or {}))}
        self._anchors_dev = {}

    def _mode_params(self):
        key = 'TRAIN' if self.training else 'TEST'
        if self._cfg is not None:
            c = self._cfg[key]
            return c.RPN_PRE_NMS_TOP_N, c.RPN_POST_NMS_TOP_N, c.RPN_NMS_THRESH, c.RPN_MIN_SIZE
        p = self._params[key]
        return p["RPN_PRE_NMS_TOP_N"], p["RPN_POST_NMS_TOP_N"], p["RPN_NMS_THRESH"], p["RPN_MIN_SIZE"]

    def _anchors_on(self, device):
        key = str(device)
        if key not in self._anchors_dev:
            self._anchors_dev[key] = torch.from_numpy(np.ascontiguousarray(self._anchors, dtype=np.float32)).to(device)
        return self._anchors_dev[key]

    def forward(self, rpn_cls_prob, rpn_bbox_pred, im_info):
        """rpn_cls_prob (N, A, H, W), rpn_bbox_pred (N, 4A, H, W) CUDA fp32; im_info (N, 3) [height, width, scale] (any
        device).  Returns numpy arrays like the reference: rois (R, 5) [batch, x1, y1, x2, y2], roi_probs (R, 1)."""
        return generate_proposals_batched([self], [rpn_cls_prob], [rpn_bbox_pred], im_info)[0]

    def _decode_images(self, rpn_cls_prob, rpn_bbox_pred, info, ranked=None):
        """top-k + decode for every image of this level: list of (dets (k, 5), valid (k,)) CUDA tensors, nothing synchronised.
        ranked: per image (order, top_scores) already selected by the batched device top-k (generate_proposals_batched)."""
        if not rpn_cls_prob.is_cuda:
            raise NotImplementedError("GenerateProposalsOp (device path) needs CUDA tensors; the host path is the reference's own")
        A = rpn_cls_prob.size(1)
        if A != self._num_anchors or rpn_bbox_pred.size(1) != 4 * A:
            raise ValueError("score map has %d anchors per cell and the deltas %d channels, but the op was built with %d anchors"
                             % (A, rpn_bbox_pred.size(1), self._num_anchors))
        scores = rpn_cls_prob.detach().float()
        deltas = rpn_bbox_pred.detach().float().contiguous()
        pre, post, thresh, min_size = self._mode_params()
        return [self.proposals_for_one_image(info[i], deltas[i], scores[i], pre, post, thresh, min_size, run_nms=False,
                                             ranked=None if ranked is None else ranked[i])[:2]
                for i in range(scores.size(0))]

    def num_candidates(self, A, H, W):
        """How many candidates survive the pre-NMS top-k for an (A, H, W) score map in the current mode."""
        pre = self._mode_params()[0]
        total = A * H * W
        return total if (pre <= 0 or pre >= total) else int(pre)

    def proposals_for_one_image(self, im_info, bbox_deltas, scores, pre_nms_topN, post_nms_topN, nms_thresh, min_size, run_nms=True,
                                ranked=None):
        """Device part for one image: returns (dets (k, 5), valid (k), keep indices, number kept) as CUDA tensors."""
        A, H, W = scores.shape
        dev = scores.device
        total = A * H * W
        if ranked is not None:
            order, top_scores = ranked
        else:                                                                       # library fallback: k beyond the device top-k's 16384
            flat = scores.permute(1, 2, 0).reshape(-1)                              # (H, W, A) order, as the reference enumerates anchors
            order = _stable_descending_order(flat)
            if 0 < pre_nms_topN < total:
                order = order[:int(pre_nms_topN)]
            top_scores = flat[order]
        k = int(order.numel())
        dets = torch.empty((k, 5), dtype=torch.float32, device=dev)
        valid = torch.empty((k,), dtype=torch.int32, device=dev)
        min_size_scaled = float(np.float32(min_size) * np.float32(im_info[2]))
        top_scores = top_scores.contiguous()
        ops._launch("b200_proposal_decode", dev, bbox_deltas.data_ptr(), self._anchors_on(dev).data_ptr(), order.data_ptr(),
                    top_scores.data_ptr(), k, A, H, W, float(self._feat_stride), float(im_info[0]), float(im_info[1]), min_size_scaled,
                    dets.data_ptr(), valid.data_ptr())
        if run_nms and nms_thresh > 0 and k > 0:
            keep, num = ops.nms_raw(dets, float(nms_thresh))
            return dets, valid, keep, num
        return dets, valid, None, None


def _stable_descending_order(flat):
    """np.argsort(-flat, kind="stable") on the device: NaN after every number (torch.sort puts it first), NaNs and equal
    scores in ascending index, -0.0 equal to +0.0 -- the rule b200_topk_batched follows."""
    nan = torch.isnan(flat)
    key = torch.where(nan, torch.full_like(flat, float("-inf")), flat) + 0.0    # + 0.0 turns -0.0 into +0.0
    order = torch.sort(key, descending=True, stable=True).indices
    return order[torch.sort(nan[order].to(torch.uint8), stable=True).indices]  # NaNs to the end, keeping their index order


def generate_proposals_batched(op_list, cls_probs, bbox_preds, im_info):
    """All (level, image) proposal sets of one step with ONE batched NMS (b200_nms_batched: one mask launch over every
    problem's tiles, one scan CTA per problem) and ONE device-to-host read of the kept counts -- the reference runs them one
    after the other on the host (lib/modeling/FPN.py loops the levels, generate_proposals.py:91-99 the images).

    op_list[l] is the GenerateProposalsOp of level l; cls_probs[l] / bbox_preds[l] its (N, A, H, W) / (N, 4A, H, W) maps.
    Returns [(rois, roi_probs)] per level, exactly what op_list[l](cls_probs[l], bbox_preds[l], im_info) returns (numpy
    arrays, or CUDA tensors for ops built with return_tensors=True)."""
    info = im_info.detach().cpu().numpy().astype(np.float32) if torch.is_tensor(im_info) else np.asarray(im_info, np.float32)
    # ONE batched device top-k (b200_topk_batched) over every (level, image) score map whose k fits its limits
    ranked = [None] * len(op_list)
    problems = []
    for l, (op, p) in enumerate(zip(op_list, cls_probs)):
        if p.is_cuda and p.dim() == 4:
            k = op.num_candidates(p.size(1), p.size(2), p.size(3))
            if 0 < k <= ops.TOPK_MAX_K:
                problems.extend((l, i, k) for i in range(p.size(0)))
    for c0 in range(0, len(problems), ops.TOPK_MAX_PROBLEMS):
        chunk = problems[c0:c0 + ops.TOPK_MAX_PROBLEMS]
        maps = [cls_probs[l][i].detach().float() for l, i, _ in chunk]
        order, top = ops.topk_batched_raw(maps, [k for _, _, k in chunk])
        off = 0
        for l, i, k in chunk:
            if ranked[l] is None:
                ranked[l] = [None] * cls_probs[l].size(0)
            ranked[l][i] = (order[off:off + k], top[off:off + k])
            off += k
    per_level = [op._decode_images(p, d, info, ranked=r) for op, p, d, r in zip(op_list, cls_probs, bbox_preds, ranked)]
    params = [op._mode_params() for op in op_list]
    # problems that go through NMS, grouped by threshold (one batched call per distinct threshold; normally one)
    keep_of = {}
    by_thresh = {}
    for l, (imgs, (pre, post, thresh, min_size)) in enumerate(zip(per_level, params)):
        for i, (dets, valid) in enumerate(imgs):
            if thresh > 0 and dets.size(0) > 0:
                by_thresh.setdefault(float(thresh), []).append((l, i))
    for thresh, probs in by_thresh.items():
        for c0 in range(0, len(probs), 64):                                     # b200_nms_batched takes up to 64 problems
            chunk = probs[c0:c0 + 64]
            counts = [int(per_level[l][i][0].size(0)) for l, i in chunk]
            if max(counts) > 13000:                                             # beyond the pipelined scan: one call per problem
                for (l, i) in chunk:
                    keep, num = ops.nms_raw(per_level[l][i][0], thresh)
                    keep_of[(l, i)] = (keep, num, 0, 0)
                continue
            cat = torch.cat([per_level[l][i][0] for l, i in chunk], dim=0) if len(chunk) > 1 else per_level[chunk[0][0]][chunk[0][1]][0]
            keep, num = ops.nms_batched_raw(cat, counts, thresh)
            off = 0
            for j, (l, i) in enumerate(chunk):
                keep_of[(l, i)] = (keep, num, off, j)
                off += counts[j]
    # ONE host read of every kept count
    nums = {}
    if keep_of:
        keys = list(keep_of)
        stacked = torch.stack([keep_of[k][1][keep_of[k][3]] for k in keys]).cpu().numpy()
        nums = {k: int(v) for k, v in zip(keys, stacked)}
    out = []
    for l, (op, imgs, (pre, post, thresh, min_size)) in enumerate(zip(op_list, per_level, params)):
        rois = np.empty((0, 5), dtype=np.float32)
        probs = np.empty((0, 1), dtype=np.float32)
        t_rois, t_probs = [], []
        for i, (dets, valid) in enumerate(imgs):
            if (l, i) in keep_of:
                keep, _, off, _ = keep_of[(l, i)]
                k = keep[off:off + nums[(l, i)]].long()
            else:
                k = torch.arange(dets.size(0), device=dets.device)
            k = k[valid[k] != 0]
            if thresh > 0 and post > 0:
                k = k[:post]
            d = dets[k]
            if op._return_tensors:
                t_rois.append(torch.cat([torch.full((d.size(0), 1), float(i), device=d.device), d[:, :4]], dim=1))
                t_probs.append(d[:, 4:5])
                continue
            d = d.cpu().numpy()
            rois = np.append(rois, np.hstack((np.full((d.shape[0], 1), i, dtype=np.float32), d[:, :4])), axis=0)
            probs = np.append(probs, d[:, 4:5], axis=0)
        out.append((torch.cat(t_rois, dim=0), torch.cat(t_probs, dim=0)) if op._return_tensors else (rois, probs))
    return out
