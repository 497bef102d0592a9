"""Time PASCAL VOC evaluation at VOC2007-test scale: the device path against the numpy restatement of voc_eval on the host.

    python tools/voc_eval_probe.py [--images 4952] [--repeats 3]

The seeded synthetic set of tests/voc_eval_cases.scale_set: 4 952 images, 20 classes, about 3 objects per image (some difficult),
100 detections per image, scores with ties.  The device path runs from all_boxes and the parsed annotations in host memory to the
APs under both rules (voc_eval.pack_all_boxes, Packed, upload, the matching kernels, curves); its stages are timed separately:
host packing (values, stable order, ground-truth CSR) by the host clock, upload + kernels + copy-back of the outcome bytes by the
host clock around a synchronise, and the kernels alone by CUDA events.  Each is the median of --repeats runs after one warm-up.
The oracle is oracle/voc_eval.py (restated writer lines, the per-detection loop, both AP rules), run once; the reference's own
voc_eval is not run here.  Checks that rec, prec and both APs are equal.  Prints one JSON line with the card's name and power limit.
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
from detectron.pytorch_b200.datasets import voc_eval as V  # noqa: E402
from oracle import voc_eval as O  # noqa: E402
from tests import voc_eval_cases as VC  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def device_run(classes, names, recs, ab):
    t0 = time.perf_counter()
    dets = V.pack_all_boxes(ab, list(range(1, len(classes))), len(names))
    packed = V.Packed(recs, names, classes[1:], *dets)
    t1 = time.perf_counter()
    pgb, gb, gd, dp, db, _keep = V.upload(packed)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    outcome = ops.voc_match_raw(pgb, gb, gd, dp, db, 0.5)
    end.record()
    outcome = outcome.cpu().numpy()
    t2 = time.perf_counter()
    res = {rule: V.curves(packed, outcome, rule) for rule in (True, False)}
    t3 = time.perf_counter()
    return res, {"pack_s": t1 - t0, "device_s": t2 - t1, "kernels_ms": start.elapsed_time(end), "curves_s": t3 - t2, "total_s": t3 - t0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4952)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a GPU"
    classes, names, recs, ab = VC.scale_set(n_images=args.images)
    out = {"card": card(), "images": len(names), "classes": len(classes) - 1,
           "objects": int(sum(len(v) for v in recs.values())), "detections": int(sum(len(a) for cls in ab for a in cls))}
    device_run(classes, names, recs, ab)
    runs = [device_run(classes, names, recs, ab) for _ in range(args.repeats)]
    res = runs[-1][0]
    for k in runs[0][1]:
        out[k] = float(np.median([r[1][k] for r in runs]))
    t0 = time.perf_counter()
    same = True
    for c, cls in enumerate(classes[1:], start=1):
        rec, prec, _ = O.voc_eval(O.writer_lines(ab, c, names), recs, names, cls)
        for rule in (True, False):
            r, p, a = res[rule][c - 1]
            same &= np.array_equal(r, rec, equal_nan=True) and np.array_equal(p, prec) and a == O.average_precision(rec, prec, rule)
    out["oracle_s"] = time.perf_counter() - t0
    out["equal"] = bool(same)
    out["mAP07"] = float(np.mean([x[2] for x in res[True]]))
    out["mAP"] = float(np.mean([x[2] for x in res[False]]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
