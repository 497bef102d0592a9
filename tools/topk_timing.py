"""Time b200_topk_batched (the proposal layer's batched pre-NMS top-k) with CUDA events, on the two workloads of the reference's
training configurations:

    fpn   the five FPN levels of two 800 x 1333 images (A = 3, P2..P6), k = 2000 per map: 10 problems in one call
    c4    two C4 maps (A = 15, 50 x 84), k = 12000

each on unique scores and on float32 sigmoid scores whose k-th value is tied (tests/proposal_cases.py).  Several builds of
libb200_roi_ops.so can be compared in one run (--lib, repeatable; default: the in-tree library); their calls alternate
within every round, so they see the same clocks and neighbours.  Prints the card's name and power limit beside the numbers.

    python tools/topk_timing.py [--lib A.so --lib B.so] [--iters 200] [--rounds 5] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import proposal_cases as PC  # noqa: E402


def load(path):
    lib = ctypes.CDLL(path)
    lib.b200_topk_batched_workspace_bytes.restype = ctypes.c_size_t
    lib.b200_topk_batched_workspace_bytes.argtypes = [ctypes.c_int]
    lib.b200_topk_batched.restype = ctypes.c_int
    lib.b200_topk_batched.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_size_t, ctypes.c_void_p]
    return lib


def workloads():
    out = {}
    for kind in ("unique", "sigmoid"):
        maps, ks = [], []
        for i in range(2):
            for name, _ in PC.FPN_LEVELS:
                A, H, W = PC.SHAPES[name]
                maps.append(PC.scores(kind, (A, H, W), 2000, seed=10 * i + len(name)))
                ks.append(min(2000, A * H * W))
        out["fpn_%s" % kind] = (maps, ks)
        out["c4_%s" % kind] = ([PC.scores(kind, PC.SHAPES["c4"], 12000, seed=i) for i in range(2)], [12000, 12000])
    return out


class Call:
    def __init__(self, lib, maps, ks):
        self.lib = lib
        self.maps = [torch.from_numpy(m).cuda() for m in maps]
        P = len(maps)
        self.args = ((ctypes.c_void_p * P)(*[m.data_ptr() for m in self.maps]), (ctypes.c_int * P)(*[m.size(0) for m in self.maps]),
                     (ctypes.c_int * P)(*[m.size(1) * m.size(2) for m in self.maps]), (ctypes.c_int * P)(*ks))
        self.P = P
        self.order = torch.empty(sum(ks), dtype=torch.int64, device="cuda")
        self.scores = torch.empty(sum(ks), dtype=torch.float32, device="cuda")
        self.ws_bytes = int(lib.b200_topk_batched_workspace_bytes(P))
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device="cuda")

    def __call__(self):
        a = self.args
        rc = self.lib.b200_topk_batched(ctypes.cast(a[0], ctypes.c_void_p), ctypes.cast(a[1], ctypes.c_void_p), ctypes.cast(a[2], ctypes.c_void_p),
                                        ctypes.cast(a[3], ctypes.c_void_p), self.P, self.order.data_ptr(), self.scores.data_ptr(),
                                        self.ws.data_ptr(), self.ws_bytes, torch.cuda.current_stream().cuda_stream)
        if rc != 0:
            raise RuntimeError("b200_topk_batched returned %d" % rc)


def time_call(call, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        call()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / iters                  # microseconds per call


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", action="append", help="libb200_roi_ops.so to time (repeatable)")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", help="also write the result as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("topk_timing: needs a CUDA device")
    libs = args.lib or [os.path.join(ROOT, "detectron", "pytorch_b200", "libb200_roi_ops.so")]
    loaded = [load(p) for p in libs]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    result = {"gpu": gpu, "iters": args.iters, "rounds": args.rounds, "libs": libs, "us_per_call": {}}
    for wname, (maps, ks) in workloads().items():
        calls = [Call(lib, maps, ks) for lib in loaded]
        for c in calls:                                          # warm-up
            for _ in range(10):
                c()
        torch.cuda.synchronize()
        times = [[] for _ in calls]
        for _ in range(args.rounds):
            for i, c in enumerate(calls):
                times[i].append(time_call(c, args.iters))
        result["us_per_call"][wname] = [{"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))} for t in times]
        print("%-12s " % wname + "  ".join("%8.1f us (%.1f..%.1f)" % (np.median(t), np.min(t), np.max(t)) for t in times))
    print("GPU: %s" % gpu)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
