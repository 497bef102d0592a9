"""Time COCO evaluation at COCO-val scale: the device evaluators against the numpy restatement of COCOeval on the host.

    python tools/coco_eval_probe.py [--images 5000] [--repeats 3] [--types bbox,segm,keypoints]

Boxes and masks: the seeded synthetic set of tests/coco_eval_cases.coco_scale_set: 5 000 images, 80 categories, about 7 objects
per image (1-3 polygons of 20-200 vertices, some crowd RLEs), 100 detections per image with masks pasted and encoded on the
device.  Keypoints: 5 000 images of about 7 persons each (some without visible keypoints) and 100 person detections per image
with 17 keypoints, scored by the box (KEYPOINT_CONFIDENCE 'bbox').
Each timing runs from all_boxes / all_segms / all_keyps in host memory to `stats`; the device path's median over --repeats runs after one
warm-up, the oracle's single run.  The oracle is oracle/cocoeval.py, not pycocotools' C / Cython path, whose time is not
measured here.  Checks that precision, recall, scores and stats are equal.  Prints one JSON line with the card's name and
power limit.
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
from detectron.pytorch_b200.datasets import json_dataset_evaluator as J  # noqa: E402
from detectron.pytorch_b200.datasets import coco_eval as DE  # noqa: E402
from tests import coco_eval_cases as CC  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def device(ds, ab, asg, ak, t):
    jd = J.load_json_dataset("coco_synthetic_val", ds)
    if t == "bbox":
        dets = J._box_results(jd, ab)
    elif t == "segm":
        dets = J._segm_results(jd, ab, asg)
    else:
        dets = J._keypoint_results(jd, ab, ak, "bbox")
    res = DE.evaluate(ds, dets, t)
    res.summarize(out=None)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--types", default="bbox,segm,keypoints")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    types = args.types.split(",")
    out = {"card": card(), "images": args.images}
    if "bbox" in types or "segm" in types:
        ds, ab, asg = CC.coco_scale_set(n_images=args.images)
        out.update(annotations=len(ds["annotations"]), detections=int(sum(len(d) for cls in ab for d in cls)))
    if "keypoints" in types:
        kds, kab, _, kak = CC.make_set(2025, n_images=args.images, n_cats=1, dets_per_image=100, size=(240, 480), keypoints=True,
                                       masks=False, vertices=(6, 12))
        out.update(kp_annotations=len(kds["annotations"]), kp_detections=int(sum(len(d) for cls in kab for d in cls)))
    for t in types:
        sets = (kds, kab, None, kak) if t == "keypoints" else (ds, ab, asg, None)
        device(*sets, t)
        times = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dev = device(*sets, t)
            times.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        ora = CC.oracle_eval(sets[0], CC.results(*sets, t), t)
        t_ora = time.perf_counter() - t0
        # keypoints: equal arrays are expected where no OKS lies within a few ulp of a threshold or of a rival (tests/)
        same = all(np.array_equal(dev.eval[k], ora.eval[k]) for k in ("precision", "recall", "scores")) and \
            np.array_equal(np.asarray(dev.stats), np.asarray(ora.stats))
        out[t] = {"device_s": float(np.median(times)), "oracle_s": t_ora, "equal": bool(same), "AP": float(dev.stats[0])}
        sys.stderr.write("%s %s\n" % (t, out[t])); sys.stderr.flush()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
