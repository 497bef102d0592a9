"""Time proposal recall at COCO-minival scale: the device path against the numpy restatement of the reference's loop on the host.

    python tools/box_proposals_probe.py [--images 5000] [--repeats 3] [--oracle-images 5000]

The seeded synthetic roidb of tests/box_proposal_cases.scale_set: 5 000 images, 1 000 .. 2 000 proposals each jittered from the
ground truth, Poisson(7.3) gt boxes per image.  Timed, each the median of --repeats runs after one warm-up:
  * task_evaluation.evaluate_box_proposals end to end (packing, upload, one launch per chunk, copy-back, the host tail), host clock;
  * ops.box_proposal_match_raw on the whole packed set (8 work items per image: input checks, allocation, the kernel), CUDA events;
  * the numpy restatement (oracle/box_proposals.py) over the eight (area, limit) pairs, once, on --oracle-images images (scaled to
    the full set when fewer).
Checks the device's eight values against the restatement's when it ran on the whole set.  Prints one JSON line with the card's name
and power limit.  Never reads the reference.
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
from detectron.pytorch_b200 import ops  # noqa: E402
from detectron.pytorch_b200.datasets import json_dataset_evaluator as J  # noqa: E402
from detectron.pytorch_b200.datasets import task_evaluation as T  # noqa: E402
from oracle import box_proposals as O  # noqa: E402
from tests import box_proposal_cases as BC  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


class _Dataset:
    name = "synthetic_minival"


def end_to_end(roidb):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = T.evaluate_box_proposals(_Dataset(), roidb)
    return res, time.perf_counter() - t0


def kernel_ms(roidb, repeats):
    prop_box, prop_begin, gt_box, gt_area, gt_begin = J.pack_roidb(roidb)
    limits, areas = T._BOX_PROPOSAL_LIMITS, list(T._BOX_PROPOSAL_AREAS)
    ranges = [J.BOX_PROPOSAL_AREA_RANGES[a] for a in areas]
    cuda = lambda x: torch.from_numpy(x).cuda()  # noqa: E731
    args = (cuda(prop_box), cuda(prop_begin), cuda(gt_box), cuda(gt_area), cuda(gt_begin),
            cuda(J.effective_proposal_counts(np.diff(prop_begin), limits)), ranges, cuda(J.default_recall_thresholds()))
    ops.box_proposal_match_raw(*args)
    times = []
    for _ in range(repeats):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        ops.box_proposal_match_raw(*args)
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return float(np.median(times)), int(prop_box.shape[0]), int(gt_box.shape[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-images", type=int, default=5000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    roidb = BC.scale_set(n_images=args.images)
    out = {"card": card(), "images": len(roidb), "chunk_images": J.BOX_PROPOSAL_CHUNK_IMAGES}
    end_to_end(roidb)
    runs = [end_to_end(roidb) for _ in range(args.repeats)]
    res = runs[-1][0][_Dataset.name]["box_proposal"]
    out["device_end_to_end_s"] = float(np.median([r[1] for r in runs]))
    out["raw_call_whole_set_ms"], out["proposals"], out["gt_boxes"] = kernel_ms(roidb, args.repeats)
    sub = roidb[:args.oracle_images]
    t0 = time.perf_counter()
    want = {}
    for limit in T._BOX_PROPOSAL_LIMITS:
        for area, suffix in T._BOX_PROPOSAL_AREAS.items():
            want["AR{}@{:d}".format(suffix, limit)] = O.evaluate_box_proposals(sub, area=area, limit=limit)["ar"]
    out["oracle_images"] = len(sub)
    out["oracle_s"] = time.perf_counter() - t0
    out["oracle_s_scaled_to_set"] = out["oracle_s"] * len(roidb) / max(len(sub), 1)
    if len(sub) == len(roidb):
        out["equal"] = all(res[k] == v or (np.isnan(res[k]) and np.isnan(v)) for k, v in want.items())
    out["results"] = {k: float(v) for k, v in res.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
