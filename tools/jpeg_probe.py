"""Time the device JPEG decode (utils/image.imdecode) against cv2.imdecode plus the upload, on the GPU.

    python tools/jpeg_probe.py [--runs 50] [--out results.json]

Inputs are encoded here with cv2 (q90, 4:2:0): 1, 2 and 8 images of 640 x 480 and one of 1600 x 1200, with photo-like content
(smooth gradients, blocky texture and pixel noise).  Per configuration, medians over --runs runs after warm-up:
  cv2_ms        cv2.imdecode of every image plus torch's upload, to a synchronise (the reference's path)
  device_ms     utils/image.imdecode: parse, one pinned upload, three kernels, the status read-back
  parse_ms      utils/jpeg.parse of every image alone (host)
  gpu_ms        CUDA events around ops.jpeg_decode_raw on pre-parsed input (upload and kernels)
  kernels_us    per kernel, from torch.profiler (a separate run)
  host_bytes    bytes moved host -> device per image on each path
  sync          from the CPU restatement of the decomposition (oracle/jpeg.decode_sync, same S and threads): sync passes and the
                share of run boundaries already in sync after the first speculative decode
  nvjpeg_ms / nvjpeg_max_diff   torchvision.io.decode_jpeg(device="cuda"), for information: its time and its largest pixel
                difference from cv2
The card's name and power limit are printed in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def photo_like(h, w, seed):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([128 + 100 * np.sin(x / 53.0 + y / 71.0), 128 + 90 * np.cos(y / 37.0 - x / 90.0), 128 + 80 * np.sin((x + y) / 29.0)], -1)
    blocks = rng.randint(-30, 30, ((h + 15) // 16, (w + 15) // 16, 3)).repeat(16, 0).repeat(16, 1)[:h, :w]
    return np.clip(base + blocks + rng.normal(0, 6, (h, w, 3)), 0, 255).astype(np.uint8)


def median_ms(fn, runs, warmup=5):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t) * 1e3)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    from detectron.pytorch_b200 import ops
    from detectron.pytorch_b200.utils import image as I
    from detectron.pytorch_b200.utils import jpeg as J
    from oracle import jpeg as O

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    dev = torch.device("cuda", 0)
    configs = [("640x480 x1", 480, 640, 1), ("640x480 x2", 480, 640, 2), ("640x480 x8", 480, 640, 8), ("1600x1200 x1", 1200, 1600, 1)]
    results = {"card": card, "configs": []}
    for label, h, w, n in configs:
        files = []
        for k in range(n):
            ok, enc = cv2.imencode(".jpg", photo_like(h, w, k), [cv2.IMWRITE_JPEG_QUALITY, 90,
                                                              cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
            files.append(enc.tobytes())
        arrs = [np.frombuffer(f, np.uint8) for f in files]
        want = [cv2.imdecode(a, cv2.IMREAD_COLOR) for a in arrs]
        got = I.imdecode(files)
        exact = all(np.array_equal(g.cpu().numpy(), x) for g, x in zip(got, want))

        def cv2_path():
            return [torch.from_numpy(cv2.imdecode(a, cv2.IMREAD_COLOR)).to(dev) for a in arrs]

        def dev_path():
            return I.imdecode(files)

        parsed = [J.parse(f) for f in files]
        cv2_ms = median_ms(cv2_path, args.runs)
        dev_ms = median_ms(dev_path, args.runs)
        t = time.perf_counter()
        for _ in range(args.runs):
            [J.parse(f) for f in files]
        parse_ms = (time.perf_counter() - t) * 1e3 / args.runs
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(5):
            ops.jpeg_decode_raw(parsed)
        gpu = []
        for _ in range(args.runs):
            ev0.record()
            ops.jpeg_decode_raw(parsed)
            ev1.record()
            ev1.synchronize()
            gpu.append(ev0.elapsed_time(ev1))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                ops.jpeg_decode_raw(parsed)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if "jpeg" in e.key or "Memcpy" in e.key or "Memset" in e.key:
                kernels[e.key[:40]] = round(e.device_time_total / 10.0, 1)
        stats = {}
        O.decode_sync(parsed[0], parsed[0].intervals[0], ops.JPEG_SUBSEQ_BITS, 1024, stats)
        dev_bytes = [440 + 32 * len(p.intervals) + 1424 * 2 * p.ncomp + sum(len(iv[2]) for iv in p.intervals) for p in parsed]
        nv_ms, nv_diff = None, None
        try:
            import torchvision.io as tio
            datas = [torch.from_numpy(a.copy()) for a in arrs]
            nv_ms = median_ms(lambda: tio.decode_jpeg(datas, device="cuda"), args.runs)
            nv = tio.decode_jpeg(datas, device="cuda")
            nv_diff = int(max(np.abs(x.permute(1, 2, 0).cpu().numpy()[:, :, ::-1].astype(int) - y.astype(int)).max()
                              for x, y in zip(nv, want)))
        except Exception as exc:  # noqa: BLE001 -- information only
            nv_ms = "unavailable: %s" % exc
        r = dict(config=label, jpeg_bytes=[len(f) for f in files][:1], exact=exact, cv2_ms=round(cv2_ms, 3), device_ms=round(dev_ms, 3),
                 parse_ms=round(parse_ms, 3), gpu_ms=round(statistics.median(gpu), 3), kernels_us=kernels,
                 host_bytes=dict(cv2=h * w * 3, device=int(np.mean(dev_bytes))), sync=stats,
                 nvjpeg_ms=round(nv_ms, 3) if isinstance(nv_ms, float) else nv_ms, nvjpeg_max_diff=nv_diff)
        results["configs"].append(r)
        print(json.dumps(r))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
