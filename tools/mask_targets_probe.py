"""Mask R-CNN training mask targets per step: device (roidb -> CUDA blobs, host packing included) vs the numpy oracle.

    python tools/mask_targets_probe.py [--steps 20] [--out DIR]

Two 800 x 1333 images, 128 fg RoIs each, 20 objects of 1-3 polygons with 20-200 vertices, M = 28, 81 classes (the COCO-scale
case of tests/test_mask_targets.py).  The Fast R-CNN blobs (labels, rois, sampled boxes) are already on the device, as
sample_rois leaves them.  Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from detectron.pytorch_b200 import _lib  # noqa: E402
from detectron.pytorch_b200.roi_data import mask_rcnn as MR  # noqa: E402
from oracle import masks as OM  # noqa: E402
from tests.test_mask_targets import coco_step  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--oracle-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the device path"
    step = coco_step(0)
    roidb = [e for e, _, _ in step]
    labels = [torch.from_numpy(l).cuda() for _, _, l in step]
    boxes = [torch.from_numpy(s).cuda() for _, s, _ in step]
    rois = [torch.cat([torch.full((s.size(0), 1), float(n), device="cuda"), s * 1.5], 1) for n, s in enumerate(boxes)]
    nf = [l.numel() for l in labels]

    def device_step():
        return MR.mask_rcnn_blobs(labels, rois, boxes, nf, roidb, 28, True, 81)
    for _ in range(3):
        device_step()
    torch.cuda.synchronize()
    times = []
    before = _lib.launch_count()
    for _ in range(a.steps):
        t0 = time.perf_counter()
        out = device_step()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    launches = (_lib.launch_count() - before) / a.steps
    # the kernels alone, CUDA events around the call with the host packing done beforehand
    from detectron.pytorch_b200 import ops
    packed = ops.pack_polygons([MR.mask_polygons(e) for e in roidb])
    sel = torch.cat(boxes).contiguous(); cls = torch.cat(labels)
    img = [0] * nf[0] + [1] * nf[1]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ktimes = []
    for _ in range(a.steps):
        ev[0].record()
        ops.mask_targets_raw(sel, img, cls, packed, 28, 81)
        ev[1].record()
        torch.cuda.synchronize()
        ktimes.append(ev[0].elapsed_time(ev[1]))
    otimes = []
    for _ in range(a.oracle_steps):
        t0 = time.perf_counter()
        ref = [OM.add_mask_rcnn_blobs(dict(labels_int32=l), s, e, 1.5, n, M=28, cls_specific=True, num_classes=81)
               for n, (e, s, l) in enumerate(step)]
        otimes.append(time.perf_counter() - t0)
    same = bool(np.array_equal(out["masks_int32"].cpu().numpy(), np.concatenate([r["masks_int32"] for r in ref])))
    res = dict(card=card(), images=2, fg_rois=sum(nf), M=28, num_classes=81, steps=a.steps,
               device_step_ms_median=1e3 * float(np.median(times)), device_call_ms_median=float(np.median(ktimes)),
               launches_per_step=launches, oracle_host_ms_median=1e3 * float(np.median(otimes)),
               blob_mb=out["masks_int32"].numel() * 4 / 1e6, matches_oracle=same)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "mask_targets_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
