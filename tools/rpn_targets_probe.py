"""Time of one training step's RPN labels and targets (add_rpn_blobs, lib/roi_data/rpn.py:40-261) on the device.

    python tools/rpn_targets_probe.py [--steps 20] [--out DIR]

Load: two 800 x 1333 images (TRAIN.MAX_SIZE 1333, FPN P2-P6, 3 aspect ratios: 451 143 anchors and 23.5 MB of blobs per
image) with G = 7 and G = 100 ground-truth boxes each.  Per G:
  step       roi_data.rpn.add_rpn_blobs with the device draw, host clock from the roidb to the CUDA blobs, synchronised;
  halves     CUDA events around ops.rpn_targets_raw: labelling half + the count read, then draw + emit half;
  launches   the library's launch counter over one call;
  oracle     oracle/rpn.py (numpy, float32 IoU in chunks) on the host for the same images, once: a stand-in for the
             reference's numpy + Cython _get_rpn_blobs, which this probe does not run.
Prints one JSON line, with the GPU's name and power limit.
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


def image(seed, G, h=800, w=1333):
    rng = np.random.RandomState(seed)
    cx, cy = rng.uniform(0, w, G), rng.uniform(0, h, G)
    bw, bh = np.exp(rng.uniform(np.log(8), np.log(w * 0.6), G)), np.exp(rng.uniform(np.log(8), np.log(h * 0.6), G))
    boxes = np.stack([np.clip(cx - bw / 2, 0, w - 1), np.clip(cy - bh / 2, 0, h - 1), np.clip(cx + bw / 2, 0, w - 1),
                      np.clip(cy + bh / 2, 0, h - 1)], 1).astype(np.float32)
    return dict(height=h, width=w, boxes=boxes, gt_classes=np.ones(G, np.int32), is_crowd=np.zeros(G, bool))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from detectron.pytorch_b200 import _lib, ops
    from detectron.pytorch_b200.roi_data import rpn as RPN
    from oracle import rpn as OR
    assert torch.cuda.is_available(), "rpn_targets_probe needs a GPU"
    p = dict(multilevel_rpn=True, max_size=1333)
    levels = RPN.anchor_levels(**p)
    anchors = sum(F * F * c.shape[0] for _, F, _, c in levels)
    res = dict(load="2 images 800x1333, FPN P2-P6, MAX_SIZE 1333", anchors_per_image=anchors,
               blob_bytes_per_image=anchors * (4 + 12 * 4), steps=a.steps)
    for G in (7, 100):
        roidb = [image(10 + G, G), image(20 + G, G)]
        scales = [1.0, 1.0]
        RPN.add_rpn_blobs({}, scales, roidb, **p)                             # warm-up (module load, allocator, randperm)
        torch.cuda.synchronize()
        c0 = _lib.launch_count()
        RPN.add_rpn_blobs({}, scales, roidb, **p)
        torch.cuda.synchronize()
        launches = _lib.launch_count() - c0
        t_step = []
        for _ in range(a.steps):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            RPN.add_rpn_blobs({}, scales, roidb, **p)
            torch.cuda.synchronize(); t_step.append(time.perf_counter() - t0)
        gt = torch.from_numpy(np.concatenate([e["boxes"] for e in roidb])).cuda()
        lv = [(F, s, c) for _, F, s, c in levels]
        t_lab, t_emit = [], []
        for _ in range(a.steps):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

            def draw(counts):
                ev[1].record()
                out = []
                for nf, nb, _ in counts.tolist():
                    n_dis = max(nf - 128, 0); num_bg = 256 - (nf - n_dis)
                    out.append((torch.randperm(nf, device="cuda")[:n_dis], torch.randint(nb, (num_bg if nb > num_bg else 0,), device="cuda")))
                return out
            torch.cuda.synchronize()
            ev[0].record()
            ops.rpn_targets_raw(gt, [G, G], np.array([[800.0, 1333.0]] * 2), lv, draw)
            ev[2].record(); torch.cuda.synchronize()
            t_lab.append(ev[0].elapsed_time(ev[1])); t_emit.append(ev[1].elapsed_time(ev[2]))
        t0 = time.perf_counter()
        OR.add_rpn_blobs(scales, roidb, levels, rng=np.random.RandomState(0))
        t_oracle = time.perf_counter() - t0
        res["G%d" % G] = dict(step_ms_median=1e3 * float(np.median(t_step)), step_ms_min=1e3 * min(t_step),
                              label_and_read_ms_median=float(np.median(t_lab)), draw_and_emit_ms_median=float(np.median(t_emit)),
                              launches_per_call=launches, oracle_host_ms=1e3 * t_oracle)
    res["host_cpus"] = os.cpu_count()
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                                text=True).stdout.strip()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "rpn_targets_probe.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
