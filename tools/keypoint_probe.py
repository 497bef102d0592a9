"""Wall time per image of the Keypoint R-CNN keypoint post-processing (keypoint_results, lib/core/test.py:850-866).

    python tools/keypoint_probe.py [--images 20] [--out DIR]

Load: 100 person-shaped detections (32-600 px wide) on an 800 x 1333 image, the keypoint head's 17 x 56 x 56 logits
already on the device.  Two timings per image, alternated:
  ours  core.test.keypoint_results on the CUDA tensor: one launch, the (100, 4, 17) result read once, the list of arrays;
  host  the reference's loop as written -- D2H copy of the logits, per detection cv2.resize(INTER_CUBIC) of the 17-channel
        map to the box, a numpy spatial softmax of every channel and an argmax per keypoint.
Both end with cls_keyps on the host.  Prints one JSON line, with the GPU's name and power limit.
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


def host_keypoints(maps_dev, rois, K=17):
    import cv2
    maps = maps_dev.cpu().numpy().transpose(0, 2, 3, 1)
    w = np.maximum(rois[:, 2] - rois[:, 0], 1)
    h = np.maximum(rois[:, 3] - rois[:, 1], 1)
    xy = np.zeros((len(rois), 4, K), np.float32)
    for i in range(len(rois)):
        mw, mh = int(np.ceil(w[i])), int(np.ceil(h[i]))
        m = np.ascontiguousarray(cv2.resize(maps[i], (mw, mh), interpolation=cv2.INTER_CUBIC).transpose(2, 0, 1))
        e = np.exp(m - m.max(axis=(1, 2), keepdims=True))
        probs = e / e.sum(axis=(1, 2), keepdims=True)
        for k in range(K):
            pos = m[k].argmax()
            xi, yi = pos % mw, pos // mw
            xy[i, 0, k] = (xi + 0.5) * (w[i] / mw) + rois[i, 0]
            xy[i, 1, k] = (yi + 0.5) * (h[i] / mh) + rois[i, 1]
            xy[i, 2, k] = m[k, yi, xi]
            xy[i, 3, k] = probs[k, yi, xi]
    return [[], [xy[i] for i in range(len(rois))]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from detectron.pytorch_b200.core.test import keypoint_results
    from tests import keypoint_cases as cases
    assert torch.cuda.is_available(), "keypoint_probe needs a GPU"
    D = 100
    rng = np.random.RandomState(0)
    rois = cases._person_boxes(rng, D)
    rois[:, 0::2] = np.clip(rois[:, 0::2], 0, cases.KP_IM_W - 1)
    rois[:, 1::2] = np.clip(rois[:, 1::2], 0, cases.KP_IM_H - 1)
    rois = rois.astype(np.float32)
    maps_dev = torch.from_numpy(cases._logits(rng, D)).cuda()
    cls_boxes = [np.zeros((0, 5), np.float32), np.concatenate([rois, np.ones((D, 1), np.float32)], 1)]
    kw = dict(num_classes=2, num_keypoints=17, inference_min_size=0, nms_oks=False)
    ours = keypoint_results(cls_boxes, maps_dev, rois, **kw)                 # warm-up (module load, allocator)
    host = host_keypoints(maps_dev, rois)
    a_xy, b_xy = np.stack(ours[1]), np.stack(host[1])
    same_xyl = bool(np.array_equal(a_xy[:, :3], b_xy[:, :3]))
    prob_rel = float(np.max(np.abs(a_xy[:, 3] - b_xy[:, 3]) / b_xy[:, 3]))
    t_ours, t_host = [], []
    for _ in range(a.images):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        keypoint_results(cls_boxes, maps_dev, rois, **kw)
        torch.cuda.synchronize(); t_ours.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        host_keypoints(maps_dev, rois)
        t_host.append(time.perf_counter() - t0)
    # kernel time alone, CUDA events around the launch
    from detectron.pytorch_b200 import ops
    rois_dev = torch.from_numpy(rois).cuda()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    t_kernel = []
    for _ in range(a.images):
        ev[0].record(); ops.heatmaps_to_keypoints_raw(maps_dev, rois_dev, 0); ev[1].record(); torch.cuda.synchronize()
        t_kernel.append(ev[0].elapsed_time(ev[1]))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    mw = np.ceil(np.maximum(rois[:, 2] - rois[:, 0], 1)); mh = np.ceil(np.maximum(rois[:, 3] - rois[:, 1], 1))
    res = dict(load="100 dets, 800x1333, 17x56x56 logits on the device", map_pixels=int((mw * mh).sum()), images=a.images,
               ours_ms_median=1e3 * float(np.median(t_ours)), ours_ms_min=1e3 * min(t_ours),
               kernel_ms_median=float(np.median(t_kernel)), host_ms_median=1e3 * float(np.median(t_host)),
               host_ms_min=1e3 * min(t_host), speedup_median=float(np.median(t_host) / np.median(t_ours)),
               xy_logit_identical_to_host=same_xyl, prob_max_rel_diff=prob_rel, host_cpus=os.cpu_count(), gpu=q)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "keypoint_probe.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
