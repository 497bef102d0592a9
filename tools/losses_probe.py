"""Fused RPN / Fast R-CNN losses (forward + backward) against the reference formulas run as torch ops on the same GPU tensors.

    python tools/losses_probe.py [--iters 200] [--out FILE]

The two are alternated call by call in one run and timed with CUDA events.  The torch path is the reference's own
modeling.FPN.fpn_rpn_losses / modeling.rpn_heads.single_scale_rpn_losses / modeling.fast_rcnn_heads.fast_rcnn_losses when
oracle/_ref/reflib exists (oracle/refmodel.py; its smooth_l1_loss shim makes the narrowed blobs contiguous first), and in
every case a restatement of the same formulas below (no copies).  Cases:
  fpn   2 images of 800 x 1344, P2-P6, A = 3, sigmoid, wide blobs for TRAIN.MAX_SIZE = 1333 (roi_data.rpn.rpn_targets)
  c4    the same images, single-scale RPN at stride 16, A = 15, sigmoid
  box   2 x 512 RoIs from roi_data.fast_rcnn.sample_rois, 81 classes, class-specific
Reports the median per-call time, the device activities of one call and the device time of the two fused loss kernels in
torch.profiler (a run of its own), the HBM floor of the RPN cases (72 B per anchor forward, 92 B backward, at 3.35 TB/s) and
the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM = 3.35e12


def smooth_l1_loss(bbox_pred, bbox_targets, bbox_inside_weights, bbox_outside_weights, beta=1.0):
    box_diff = bbox_pred - bbox_targets
    in_box_diff = bbox_inside_weights * box_diff
    abs_in_box_diff = torch.abs(in_box_diff)
    sign = (abs_in_box_diff < beta).detach().float()
    in_loss_box = sign * 0.5 * torch.pow(in_box_diff, 2) / beta + (1 - sign) * (abs_in_box_diff - (0.5 * beta))
    out = bbox_outside_weights * in_loss_box
    return out.reshape(-1).sum(0) / out.size(0)


def torch_rpn(levels, fpn, divisor):
    """The reference's per-level sigmoid RPN loss as torch ops (FPN.py:422-466 / rpn_heads.py:130-161)."""
    lc, lb = [], []
    for c, b, lab, tg, wi, wo in levels:
        h, w = c.shape[2:]
        lab = lab[:, :, :h, :w]
        weight = (lab >= 0).float()
        loss = F.binary_cross_entropy_with_logits(c, lab.float(), weight, reduction="sum")
        lc.append(loss / divisor if fpn else loss / weight.sum())
        lb.append(smooth_l1_loss(b, tg[:, :, :h, :w], wi[:, :, :h, :w], wo[:, :, :h, :w], beta=1 / 9))
    return (lc, lb) if fpn else (lc[0], lb[0])


def reference_paths():
    from oracle import refmodel
    if not refmodel.available():
        return None
    cfg = refmodel.setup(use_b200_ops=False)
    import modeling.FPN as RF
    import modeling.fast_rcnn_heads as RFH
    import modeling.rpn_heads as RR
    cfg.RPN.CLS_ACTIVATION = "sigmoid"
    cfg.FPN.RPN_MIN_LEVEL, cfg.FPN.RPN_MAX_LEVEL = 2, 6
    cfg.TRAIN.RPN_BATCH_SIZE_PER_IM, cfg.TRAIN.IMS_PER_BATCH = 256, 2
    return RF, RR, RFH


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def time_alternating(paths, iters, warmup=10):
    """paths: {name: fn() doing one forward + backward}.  Median ms per call of each, alternating the paths call by call."""
    for _ in range(warmup):
        for fn in paths.values():
            fn()
    torch.cuda.synchronize()
    ev = {k: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)] for k in paths}
    for i in range(iters):
        for k, fn in paths.items():
            ev[k][i][0].record()
            fn()
            ev[k][i][1].record()
    torch.cuda.synchronize()
    return {k: float(np.median([a.elapsed_time(b) for a, b in v])) for k, v in ev.items()}


def activities(fn, reps=20):
    """(device activities of one call, microseconds per call spent in this project's loss kernels) from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    cuda = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ours = sum(getattr(e, "device_time", 0.0) for e in cuda if "loss_forward_kernel" in e.name or "loss_backward_kernel" in e.name)
    return len(cuda) // reps, ours / reps


def rpn_case(kind, ref):
    from test_losses import _c4_step, _fpn_step
    from detectron.pytorch_b200.modeling import FPN, rpn_heads
    fpn = kind == "fpn"
    levels = _fpn_step(False, seed=0) if fpn else _c4_step(False, seed=1)
    preds = [(c.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)) for c, b, *_ in levels]
    tg = [lv[2:] for lv in levels]
    names = ("rpn_labels_int32_wide", "rpn_bbox_targets_wide", "rpn_bbox_inside_weights_wide", "rpn_bbox_outside_weights_wide")
    kw = {}
    for l, ((c, b), t) in enumerate(zip(preds, tg)):
        s = "_fpn%d" % (2 + l) if fpn else ""
        kw["rpn_cls_logits" + s], kw["rpn_bbox_pred" + s] = c, b
        kw.update({k + s: x for k, x in zip(names, t)})

    def run(losses_fn):
        def fn():
            for c, b in preds:
                c.grad = b.grad = None
            lc, lb = losses_fn()
            lc, lb = (lc, lb) if fpn else ([lc], [lb])
            sum(x.unsqueeze(0) for x in lc + lb).sum().backward()
        return fn
    paths = {"fused": run(lambda: FPN.fpn_rpn_losses(**kw) if fpn else rpn_heads.single_scale_rpn_losses(**kw)),
             "torch_restated": run(lambda: torch_rpn([p + tuple(t) for p, t in zip(preds, tg)], fpn, 512.0))}
    if ref is not None:
        RF, RR, _ = ref
        RF.cfg.FPN.FPN_ON = fpn
        paths["torch_reference"] = run(lambda: RF.fpn_rpn_losses(**kw) if fpn else RR.single_scale_rpn_losses(**kw))
    anchors = sum(c.numel() for c, _ in preds)
    return paths, dict(anchors=anchors, floor_fwd_us=72 * anchors / HBM * 1e6, floor_bwd_us=92 * anchors / HBM * 1e6)


def box_case(ref):
    from test_losses import _box_head
    from detectron.pytorch_b200.modeling import fast_rcnn_heads
    cls, bbox, b = _box_head(False, seed=3)
    cs, bp = cls.clone().requires_grad_(True), bbox.clone().requires_grad_(True)
    args = [b[k] for k in ("labels_int32", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights")]
    lab64 = args[0].long()

    def torch_box():
        loss_cls = F.cross_entropy(cs, lab64)
        loss_bbox = smooth_l1_loss(bp, *args[1:])
        acc = cs.max(dim=1)[1].type_as(lab64).eq(lab64).float().mean(dim=0)
        return loss_cls, loss_bbox, acc

    def run(losses_fn):
        def fn():
            cs.grad = bp.grad = None
            lc, lb, _ = losses_fn()
            (lc + lb).backward()
        return fn
    paths = {"fused": run(lambda: fast_rcnn_heads.fast_rcnn_losses(cs, bp, *args)), "torch_restated": run(torch_box)}
    if ref is not None:
        # the reference's fast_rcnn_losses takes host blobs; its upload is part of what it costs
        host = [a.cpu().numpy() for a in args]
        paths["torch_reference"] = run(lambda: ref[2].fast_rcnn_losses(cs, bp, *host))
    return paths, dict(rois=cs.shape[0], classes=cs.shape[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "losses_probe needs a GPU"
    torch.cuda.set_device(0)
    ref = reference_paths()
    result = dict(card=card(), reference_functions=ref is not None, cases={})
    for name in ("fpn", "c4", "box"):
        paths, info = rpn_case(name, ref) if name != "box" else box_case(ref)
        ms = time_alternating(paths, a.iters)
        acts = {k: activities(fn) for k, fn in paths.items()}
        info.update(ms_per_call=ms, device_activities={k: v[0] for k, v in acts.items()}, fused_kernel_us=acts["fused"][1])
        if "floor_fwd_us" in info:
            floor = info["floor_fwd_us"] + info["floor_bwd_us"]
            info["floor_fraction_of_call"] = floor / (ms["fused"] * 1e3)
            info["floor_fraction_of_kernels"] = floor / acts["fused"][1] if acts["fused"][1] else None
        result["cases"][name] = info
        print(name, json.dumps(info), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
