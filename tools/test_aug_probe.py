"""Time per image of combining the test-time augmentation transforms of the mask and keypoint heads.

    python tools/test_aug_probe.py [--images 10] [--out DIR]

Loads, with the head outputs synthetic and already on the device:
  mask   the X-152 mask TTA (TEST.MASK_AUG: identity, H_FLIP, 8 SCALES with SCALE_H_FLIP = 18 transforms), 100 detections x 81
         classes x 28 x 28, SOFT_AVG;
  kps    the keypoint TTA at the same 18 transforms, 100 x 17 x 56 x 56 (the keypoint baselines' HEATMAP_SIZE), HM_AVG.
Two timings per image, alternated:
  device  the running combine (ops.tta_combine_raw per transform, half of them mirrored, then ops.tta_finish_raw), CUDA events;
  host    the reference's path: each transform's D2H copy (.cpu().numpy()), the mirror view, np.mean over the list; wall clock
          from a synchronise to the result.
Also prints the bytes each moves.  One JSON line, with the GPU's name and power limit.
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

T = 18
LOADS = {"mask": (100, 81, 28, 28), "kps": (100, 17, 56, 56)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from detectron.pytorch_b200 import ops
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    res = {}
    for name, shape in LOADS.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        outs = [torch.rand(shape, generator=g, device="cuda") for _ in range(T)]
        hflips = [i % 2 == 1 for i in range(T)]
        acc = torch.empty(shape, device="cuda")

        def device_combine():
            for i, (o, hf) in enumerate(zip(outs, hflips)):
                ops.tta_combine_raw(o, acc, 0, op=ops.TTA_START if i == 0 else ops.TTA_FOLD, hflip=hf)
            ops.tta_finish_raw(acc, 0, count=T)

        def host_combine():
            ts = []
            for o, hf in zip(outs, hflips):
                m = o.cpu().numpy()
                ts.append(m[..., ::-1] if hf else m)
            return np.mean(ts, axis=0)

        device_combine(); host_combine(); torch.cuda.synchronize()              # warm up both
        dev_ms, host_ms = [], []
        for _ in range(a.images):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); device_combine(); e1.record(); torch.cuda.synchronize()
            dev_ms.append(e0.elapsed_time(e1))
            torch.cuda.synchronize(); t0 = time.perf_counter(); host_combine(); host_ms.append((time.perf_counter() - t0) * 1e3)
        # check once that both agree bit for bit
        assert np.array_equal(acc.cpu().numpy(), host_combine())
        nbytes = int(np.prod(shape)) * 4
        res[name] = dict(shape=list(shape), transforms=T, device_ms_median=float(np.median(dev_ms)), device_ms_min=float(np.min(dev_ms)),
                         host_ms_median=float(np.median(host_ms)), host_ms_min=float(np.min(host_ms)),
                         device_hbm_bytes=(3 * T - 1) * nbytes + 2 * nbytes,            # per transform: read src, read + write acc
                         host_d2h_bytes=T * nbytes,
                         device_gbps=((3 * T - 1) * nbytes + 2 * nbytes) / (np.median(dev_ms) * 1e-3) / 1e9)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    res["gpu"] = q
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "test_aug_probe.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
