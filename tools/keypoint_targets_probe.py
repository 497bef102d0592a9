"""Keypoint R-CNN training targets per step: device (roidb -> CUDA blobs, host packing and upload included) vs the numpy oracle
and, when oracle/_ref/reflib is present, the reference's own add_keypoint_rcnn_blobs.

    python tools/keypoint_targets_probe.py [--steps 20] [--out DIR]

Two 800 x 1333 images per step, 2 000 proposals and 20 persons of 17 keypoints each, HEATMAP_SIZE 56, BATCH_SIZE_PER_IM 512
(128 fg RoIs per image, so the draw happens): the COCO-scale case of tests/test_keypoint_targets.py, as numpy roidb entries.
Reports the median step time, the two launches alone with CUDA events, and the card's name and power limit read in the same run.
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
from detectron.pytorch_b200.roi_data import keypoint_rcnn as KR  # noqa: E402
from oracle import keypoint_targets as OK  # noqa: E402
from tests.test_keypoint_targets import coco_image  # noqa: E402

HS, K, FG = 56, 17, 128


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def reference_step(entries, choices):
    """The reference's add_keypoint_rcnn_blobs per image (numpy.random.choice replaced by the recorded positions)."""
    from oracle import refmodel
    if not refmodel.available():
        return None
    cfg = refmodel.setup(use_b200_ops=False)
    import roi_data.keypoint_rcnn as ref_kp
    cfg.KRCNN.HEATMAP_SIZE = HS; cfg.KRCNN.NUM_KEYPOINTS = K; cfg.TRAIN.FG_THRESH = 0.5
    orig = np.random.choice
    times = []
    try:
        for _ in range(3):
            t0 = time.perf_counter()
            for n, (e, c) in enumerate(zip(entries, choices)):
                np.random.choice = lambda a, size=None, replace=True, p=None, c=c: np.asarray(a)[c]
                ref_kp.add_keypoint_rcnn_blobs({}, e, FG, None, 1.5, n)
            times.append(time.perf_counter() - t0)
    finally:
        np.random.choice = orig
    return 1e3 * float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--oracle-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the device path"
    rng = np.random.RandomState(0)
    entries = [coco_image(rng), coco_image(rng)]
    choices = []
    for e in entries:
        c = OK.candidates(e["boxes"], e["max_overlaps"], e["box_to_gt_ind_map"], np.arange(20), e["gt_keypoints"], 0.5)
        choices.append(rng.choice(c.size, FG, replace=False) if c.size > FG else None)
    box_begin = np.concatenate([[0], np.cumsum([e["boxes"].shape[0] for e in entries])])
    cat = lambda k: np.concatenate([e[k] for e in entries])             # noqa: E731

    def device_step():                                                  # from the numpy roidb to the CUDA blobs
        return KR.keypoint_rcnn_blobs(cat("boxes"), box_begin, cat("max_overlaps"), cat("box_to_gt_ind_map"), entries, [1.5, 1.5], FG, HS,
                                      K, 0.5, choices=choices)
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
    # the two launches alone: library calls bracketed by CUDA events, inputs already on the device
    lib = _lib.load()
    boxes = torch.from_numpy(cat("boxes")).cuda(); mo = torch.from_numpy(cat("max_overlaps")).cuda()
    bm = torch.from_numpy(cat("box_to_gt_ind_map")).cuda()
    gi = torch.arange(40, dtype=torch.int32, device="cuda") % 20
    kp = torch.from_numpy(cat("gt_keypoints")).cuda()
    tab = lambda v: (__import__("ctypes").c_int * len(v))(*[int(x) for x in v])   # noqa: E731
    bb, gb, pb = tab(box_begin), tab([0, 20, 40]), tab([0, 20, 40])
    cand = torch.empty((int(box_begin[-1]),), dtype=torch.int32, device="cuda")
    counts = torch.empty((2,), dtype=torch.int32, device="cuda")
    picks = torch.cat([torch.from_numpy(np.asarray(c, np.int32)) for c in choices]).cuda()
    rb = tab([0, FG, 2 * FG])
    flt = lambda v: (__import__("ctypes").c_float * len(v))(*v)   # noqa: E731
    rois = torch.empty((2 * FG, 5), device="cuda"); loc = torch.empty((2 * FG * K,), dtype=torch.int32, device="cuda")
    w = torch.empty((2 * FG * K,), device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ktimes = []
    s = torch.cuda.current_stream().cuda_stream
    for _ in range(a.steps):
        ev[0].record()
        _lib.check(lib.b200_keypoint_candidates(boxes.data_ptr(), mo.data_ptr(), bm.data_ptr(), 2, bb, gi.data_ptr(), gb, kp.data_ptr(), pb,
                                                K, 0.5, cand.data_ptr(), counts.data_ptr(), s), "candidates")
        _lib.check(lib.b200_keypoint_targets(boxes.data_ptr(), bm.data_ptr(), 2, bb, gi.data_ptr(), gb, kp.data_ptr(), pb, K, HS,
                                             cand.data_ptr(), counts.data_ptr(), picks.data_ptr(), rb, flt([1.5, 1.5]), flt([0, 1]),
                                             rois.data_ptr(), loc.data_ptr(), w.data_ptr(), s), "targets")
        ev[1].record()
        torch.cuda.synchronize()
        ktimes.append(ev[0].elapsed_time(ev[1]))
    otimes = []
    for _ in range(a.oracle_steps):
        t0 = time.perf_counter()
        ref = []
        for n, (e, c) in enumerate(zip(entries, choices)):
            bl = {}
            OK.add_keypoint_rcnn_blobs(bl, e, FG, 1.5, n, HS, 0.5, c)
            ref.append(bl)
        otimes.append(time.perf_counter() - t0)
    same = all(np.array_equal(out[k].cpu().numpy(), np.concatenate([r[k] for r in ref]))
               for k in ("keypoint_rois", "keypoint_locations_int32", "keypoint_weights"))
    ref_ms = reference_step(entries, choices)
    res = dict(card=card(), images=2, proposals_per_image=2000, persons_per_image=20, fg_rois_per_image=FG, heatmap_size=HS, steps=a.steps,
               device_step_ms_median=1e3 * float(np.median(times)), launches_ms_median=float(np.median(ktimes)),
               launches_per_step=launches, oracle_host_ms_median=1e3 * float(np.median(otimes)),
               reference_host_ms_median=ref_ms if ref_ms is not None else "not measured", matches_oracle=bool(same))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "keypoint_targets_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
