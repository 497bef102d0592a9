"""A/B timing of the RoIAlign forward paths at BASELINE cfg2 (and an FPN-like P2 box-head shape) with CUDA events.

    python tools/fwd_ab.py [--iters 60] [--paths quad,stream,tiled] [--check]

Per path: time of the whole call (prepass + main), rotating over input sets larger than L2.
--check compares every path's output with the generic kernel's (bit-exact share).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--paths", default="quad,stream")
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--shapes", default="cfg2")
    args = ap.parse_args()
    import numpy as np
    import torch
    from detectron.pytorch_b200 import _lib, ops, synthetic as S
    shapes = {
        "cfg2": ((1, 256, 200, 272), 0.25, 7, 2, 512),
        "p2box": ((2, 256, 200, 336), 0.25, 7, 2, 1000),
        "p2mask": ((2, 256, 200, 336), 0.25, 14, 2, 256),
        "p4box": ((2, 256, 50, 84), 1.0 / 16, 7, 2, 1000),
    }
    res = {}
    for name in args.shapes.split(","):
        shape, s, P, sr, n = shapes[name]
        nset = 6
        feats = [torch.from_numpy(S.make_features(shape, seed=i)).cuda() for i in range(nset)]
        rois = [torch.from_numpy(S.make_rois(n, shape, s, seed=100 + i).astype(np.float32)).cuda() for i in range(nset)]
        ref = None
        if args.check:
            _lib.set_option("B200_ROI_ALIGN_PATH", "generic")
            ref = ops.roi_align_forward(feats[0], rois[0], P, P, s, sr).cpu().numpy()
        for path in args.paths.split(","):
            _lib.set_option("B200_ROI_ALIGN_PATH", path)
            row = {}
            for i in range(5):
                ops.roi_align_forward(feats[i % nset], rois[i % nset], P, P, s, sr)
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.iters):
                ops.roi_align_forward(feats[i % nset], rois[i % nset], P, P, s, sr)
            e1.record(); torch.cuda.synchronize()
            row["all_us"] = round(e0.elapsed_time(e1) * 1e3 / args.iters, 2)
            if ref is not None:
                out = ops.roi_align_forward(feats[0], rois[0], P, P, s, sr).cpu().numpy()
                row["exact_share"] = float(np.mean(out == ref))
                row["max_abs_diff"] = float(np.max(np.abs(out - ref)))
            res["%s/%s" % (name, path)] = row
            print(name, path, row, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
