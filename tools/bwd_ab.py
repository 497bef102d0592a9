"""A/B timing of the RoIAlign backward at BASELINE cfg2 with CUDA events (rotating inputs larger than L2).
    python tools/bwd_ab.py [--iters 60]        # options come from the environment (B200_ROI_ALIGN_BWD_PATH)
"""
import argparse, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--iters", type=int, default=60); args = ap.parse_args()
    import numpy as np, torch
    from detectron.pytorch_b200 import ops, synthetic as S
    shape, s, P, sr, n = (1, 256, 200, 272), 0.25, 7, 2, 512
    nset = 6
    dys = [torch.randn((n, shape[1], P, P), device="cuda") for _ in range(nset)]
    rois = [torch.from_numpy(S.make_rois(n, shape, s, seed=100 + i).astype(np.float32)).cuda() for i in range(nset)]
    for i in range(5): ops.roi_align_backward(dys[i % nset], rois[i % nset], shape, P, P, s, sr)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.iters): ops.roi_align_backward(dys[i % nset], rois[i % nset], shape, P, P, s, sr)
    e1.record(); torch.cuda.synchronize()
    print("bwd cfg2: %.2f us" % (e0.elapsed_time(e1) * 1e3 / args.iters))
if __name__ == "__main__":
    main()
