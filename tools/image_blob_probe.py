"""Input image blob per call: the reference-style host path vs the device path.

    python tools/image_blob_probe.py [--iters 50] [--out DIR]

Two workloads: one 640 x 480 test image at TEST.SCALE 800 / MAX_SIZE 1333, and a two-image training step (640 x 480 and
480 x 640, the second flipped, TRAIN.SCALES 800 / MAX_SIZE 1333), FPN padding to 32 on both.
  host:   numpy mean subtraction, cv2.resize (IPP off, the arithmetic the device follows), im_list_to_blob and
          torch.from_numpy(blob).cuda(), timed to a device synchronise; the H2D copy is also timed on its own;
  device: the uint8 upload plus the one launch (ops.image_blob_raw), timed to a device synchronise; the kernel alone from
          torch.profiler's CUDA activity, in a pass of its own.
Medians.  The device blob is compared with the host path's blob.  Prints one JSON line with the card's name and power limit
read in the same run, and the algorithmic bytes (blob written + source read) over the kernel time.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from detectron.pytorch_b200 import _lib, ops  # noqa: E402
from detectron.pytorch_b200.utils import blob as B  # noqa: E402

MEANS = B.DEFAULT_PIXEL_MEANS


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def host_blob(ims, flipped, scales):
    out = []
    for im, f in zip(ims, flipped):
        x = (im[:, ::-1, :] if f else im).astype(np.float32, copy=False)
        x -= MEANS
        h, w = x.shape[:2]
        s = B.get_target_scale(min(h, w), max(h, w), scales, 1333)
        out.append(cv2.resize(x, None, None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR))
    hp, wp = B.get_max_shape([o.shape[:2] for o in out], fpn_on=True, coarsest_stride=32)
    blob = np.zeros((len(out), hp, wp, 3), np.float32)
    for i, o in enumerate(out):
        blob[i, :o.shape[0], :o.shape[1]] = o
    return blob.transpose(0, 3, 1, 2)


def median_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t))


def kernel_ms(fn, iters):
    """Median device time of image_blob_kernel over `iters` calls, from torch.profiler's CUDA activity (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    t = [e.device_time for e in prof.events() if "image_blob_kernel" in e.name]
    assert len(t) == iters, len(t)
    return float(np.median(t)) / 1e3


def workload(name, ims, flipped, iters):
    scales = [B.get_target_scale(min(im.shape[:2]), max(im.shape[:2]), 800, 1333) for im in ims]
    host_ms = median_ms(lambda: torch.from_numpy(np.ascontiguousarray(host_blob(ims, flipped, 800))).cuda(), iters)
    hb = np.ascontiguousarray(host_blob(ims, flipped, 800))
    copy_ms = median_ms(lambda: torch.from_numpy(hb).cuda(), iters)
    device_ms = median_ms(lambda: ops.image_blob_raw(ims, scales, flipped, MEANS, 32), iters)
    dims = [torch.from_numpy(im).cuda() for im in ims]
    out = torch.empty(hb.shape, dtype=torch.float32, device="cuda")
    n0 = _lib.launch_count()
    ops.image_blob_raw(dims, scales, flipped, MEANS, 32, out=out)
    launches = _lib.launch_count() - n0
    k_ms = kernel_ms(lambda: ops.image_blob_raw(dims, scales, flipped, MEANS, 32, out=out), iters)
    dev_blob, _ = ops.image_blob_raw(ims, scales, flipped, MEANS, 32)
    same = bool(np.array_equal(dev_blob.cpu().numpy(), hb))
    nbytes = hb.nbytes + sum(im.nbytes for im in ims)
    return dict(workload=name, images=len(ims), blob_shape=list(hb.shape), blob_mb=hb.nbytes / 1e6, uint8_mb=sum(im.nbytes for im in ims) / 1e6,
                host_path_ms_median=host_ms, host_h2d_copy_ms_median=copy_ms, device_path_ms_median=device_ms,
                kernel_ms_median=k_ms, launches_per_call=launches, algorithmic_mb=nbytes / 1e6,
                kernel_gb_per_s=nbytes / (k_ms * 1e-3) / 1e9, matches_host_ipp_off=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe measures the device path"
    cv2.ipp.setUseIPP(False)
    rng = np.random.RandomState(0)
    a640 = rng.randint(0, 256, (480, 640, 3)).astype(np.uint8)
    b480 = rng.randint(0, 256, (640, 480, 3)).astype(np.uint8)
    res = dict(card=card(), ipp=False, results=[workload("test_640x480", [a640], [False], a.iters),
                                                 workload("train_step_2img", [a640, b480], [False, True], a.iters)])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "image_blob_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
