"""Wall time per image of the Mask R-CNN mask post-processing (segm_results, lib/core/test.py:793-847).

    python tools/segm_probe.py [--images 50] [--out DIR]

Load: 100 detections on an 800 x 1333 image, M = 28, class-specific masks over 81 classes, the mask head's output already
on the device.  Two timings per image, alternated:
  ours  core.test.segm_results on the CUDA tensor: two launches, the sizes read, the string buffer's D2H copy, the dicts;
  host  the reference's loop as written -- D2H copy of the masks, box expansion, cv2.resize, threshold, paste into a zeroed
        full-image mask -- with a numpy column-major RLE in place of pycocotools.mask.encode (not installed here).
Both end with every result on the host.  Prints one JSON line, with the GPU's name and power limit.
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


def host_segm(cls_boxes, masks_dev, ref_boxes, im_h, im_w, M, thresh=0.5):
    import cv2
    from oracle.segms import rle_counts, rle_string
    masks = masks_dev.cpu().numpy().reshape(masks_dev.shape[0], -1, M, M)
    scale = (M + 2.0) / M
    b = ref_boxes
    w_half = (b[:, 2] - b[:, 0]) * .5; h_half = (b[:, 3] - b[:, 1]) * .5
    x_c = (b[:, 2] + b[:, 0]) * .5; y_c = (b[:, 3] + b[:, 1]) * .5
    w_half *= scale; h_half *= scale
    ib = np.stack([x_c - w_half, y_c - h_half, x_c + w_half, y_c + h_half], 1).astype(np.int32)
    padded = np.zeros((M + 2, M + 2), np.float32)
    out, d = [[] for _ in cls_boxes], 0
    for j in range(1, len(cls_boxes)):
        for _ in range(cls_boxes[j].shape[0]):
            padded[1:-1, 1:-1] = masks[d, j]
            r = ib[d]
            w = max(r[2] - r[0] + 1, 1); h = max(r[3] - r[1] + 1, 1)
            m = np.array(cv2.resize(padded, (int(w), int(h))) > thresh, dtype=np.uint8)
            im = np.zeros((im_h, im_w), np.uint8)
            x0, x1, y0, y1 = max(r[0], 0), min(r[2] + 1, im_w), max(r[1], 0), min(r[3] + 1, im_h)
            im[y0:y1, x0:x1] = m[(y0 - r[1]):(y1 - r[1]), (x0 - r[0]):(x1 - r[0])]
            out[j].append({"size": [im_h, im_w], "counts": rle_string(rle_counts(im)).decode("ascii")})
            d += 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from detectron.pytorch_b200.core.test import segm_results
    from scipy.ndimage import gaussian_filter
    assert torch.cuda.is_available(), "segm_probe needs a GPU"
    im_h, im_w, M, K, D = 800, 1333, 28, 81, 100
    rng = np.random.RandomState(0)
    x1 = rng.uniform(0, im_w - 60, D); y1 = rng.uniform(0, im_h - 60, D)
    bw = np.exp(rng.uniform(np.log(16), np.log(500), D)); bh = np.exp(rng.uniform(np.log(16), np.log(400), D))
    boxes = np.stack([x1, y1, np.minimum(x1 + bw, im_w - 1), np.minimum(y1 + bh, im_h - 1)], 1).astype(np.float32)
    cls = np.sort(rng.randint(1, K, D))
    cls_boxes = [np.zeros((0, 5), np.float32)] + [np.concatenate([boxes[cls == j], np.ones((int((cls == j).sum()), 1))], 1).astype(np.float32)
                                                  for j in range(1, K)]
    ref_boxes = np.concatenate([c[:, :4] for c in cls_boxes[1:]], 0)
    logits = gaussian_filter(rng.standard_normal((D, K, M, M)), sigma=(0, 0, 2, 2)) * 8.0
    masks_dev = torch.from_numpy((1 / (1 + np.exp(-logits))).astype(np.float32).reshape(D, K * M * M)).cuda()
    kw = dict(num_classes=K, resolution=M, cls_specific_mask=True, thresh_binarize=0.5)
    ours = segm_results(cls_boxes, masks_dev, ref_boxes, im_h, im_w, **kw)            # warm-up (module load, allocator)
    host_segm(cls_boxes, masks_dev, ref_boxes, im_h, im_w, M)
    import cv2
    cv2.ipp.setUseIPP(False)
    same = ours == host_segm(cls_boxes, masks_dev, ref_boxes, im_h, im_w, M)
    cv2.ipp.setUseIPP(True)
    t_ours, t_host = [], []
    for _ in range(a.images):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        segm_results(cls_boxes, masks_dev, ref_boxes, im_h, im_w, **kw)
        torch.cuda.synchronize(); t_ours.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        host_segm(cls_boxes, masks_dev, ref_boxes, im_h, im_w, M)
        t_host.append(time.perf_counter() - t0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(load="100 dets, 800x1333, M=28, 81 classes", images=a.images, ours_ms_median=1e3 * float(np.median(t_ours)),
               ours_ms_min=1e3 * min(t_ours), host_ms_median=1e3 * float(np.median(t_host)), host_ms_min=1e3 * min(t_host),
               speedup_median=float(np.median(t_host) / np.median(t_ours)), identical_to_host_ipp_off=bool(same),
               host_cpus=os.cpu_count(), gpu=q)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "segm_probe.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
