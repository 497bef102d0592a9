"""Time per image of the box head's decode, test-time combine and detection post-processing.

    python tools/bbox_probe.py [--images 10] [--out DIR]

Loads, with the head outputs synthetic and already on the device (81 classes, 1000 rois per transform, Faster R-CNN rois):
  x152   the X-152 box TTA (TEST.BBOX_AUG: H_FLIP, 8 SCALES with SCALE_H_FLIP, identity = 18 transforms), UNION;
  single one transform (TEST.BBOX_AUG off).
Two timings per image, alternated, both ending in the same device box_results_with_nms_and_limit:
  device  ops.bbox_decode_raw per transform (half of them flipped), torch.cat of scores and boxes;
  host    the reference's path: each transform's D2H copies of rois, cls_score and bbox_pred, the numpy decode / clip / flip
          (oracle/detect_bbox.py, the reference's lines), np.vstack, and the upload inside box_results_with_nms_and_limit.
Wall clock from a synchronise to the result.  One JSON line, with the GPU's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R, K, H, W, SCALE = 1000, 81, 800, 1201, 1.2
LOADS = {"x152": 18, "single": 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from detectron.pytorch_b200 import ops
    from detectron.pytorch_b200.core import test as T
    from oracle import detect_bbox as O
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    res = {}
    for name, n_t in LOADS.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        heads = []
        for t in range(n_t):
            xy = torch.rand((R, 2), generator=g, device="cuda") * 1200 * SCALE
            rois = torch.cat([torch.zeros((R, 1), device="cuda"), xy, xy + 10 + torch.rand((R, 2), generator=g, device="cuda") * 400], 1)
            logits = torch.randn((R, K), generator=g, device="cuda") * 3
            heads.append((rois, torch.softmax(logits, 1), torch.randn((R, 4 * K), generator=g, device="cuda") * 0.3, t % 2 == 1))

        def device_path():
            boxes = [ops.bbox_decode_raw(r, d, K, H, W, im_scale=SCALE, flip_width=W if hf else None) for r, _, d, hf in heads]
            return T.box_results_with_nms_and_limit(torch.cat([s for _, s, _, _ in heads]), torch.cat(boxes), num_classes=K)

        def host_path():
            scores, boxes = [], []
            for r, s, d, hf in heads:
                scores.append(s.cpu().numpy())
                boxes.append(O.decode(r.cpu().numpy(), d.cpu().numpy(), K, H, W, im_scale=SCALE, flip_width=W if hf else None))
            return T.box_results_with_nms_and_limit(np.vstack(scores), np.vstack(boxes), num_classes=K)

        device_path(); host_path(); torch.cuda.synchronize()                    # warm up both
        dev_ms, host_ms = [], []
        for _ in range(a.images):
            torch.cuda.synchronize(); t0 = time.perf_counter(); device_path(); dev_ms.append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize(); t0 = time.perf_counter(); host_path(); host_ms.append((time.perf_counter() - t0) * 1e3)
        # the decode alone, CUDA events
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for r, _, d, hf in heads:
            ops.bbox_decode_raw(r, d, K, H, W, im_scale=SCALE, flip_width=W if hf else None)
        e1.record(); torch.cuda.synchronize()
        d_cls, h_cls = device_path()[2], host_path()[2]
        same = all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(d_cls[1:], h_cls[1:]))
        res[name] = dict(rois=R, classes=K, transforms=n_t, device_ms_median=float(np.median(dev_ms)), host_ms_median=float(np.median(host_ms)),
                         device_decode_ms=e0.elapsed_time(e1), host_d2h_bytes=n_t * R * (5 + K + 4 * K) * 4,
                         detections=int(sum(len(c) for c in d_cls[1:])), same_detections=bool(same))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    res["gpu"] = q
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bbox_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
