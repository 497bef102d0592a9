"""Time one C4 labelling step (GenerateProposalLabelsOp: 2 images, RPN_POST_NMS_TOP_N 2000, 512 RoIs per image, MASK_ON) and
the FPN training branch (CollectAndDistributeFpnRpnProposalsOp) on the same inputs.  Wall time to a synchronise and CUDA
events; the card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/proposal_labels_probe.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import fast_rcnn_roidb_cases as C  # noqa: E402


def inputs():
    rng = np.random.RandomState(0)
    ims, rr = [], []
    for i, s in enumerate((1.6666666, 0.8)):
        gt, cl, cr = C.roster(60 + i, "mixed", 20, 81)
        props = C.proposals(60 + i, "mixed", gt, 2000)
        segms = [[[b[0], b[1], b[2], b[1], b[2], b[3], b[0], b[3]]] for b in gt]
        ims.append(dict(boxes=gt, gt_classes=cl, is_crowd=np.zeros_like(cr), segms=segms))
        rr.append(np.hstack([np.full((props.shape[0], 1), i, np.float32), props * np.float32(s)]))
    rr = np.concatenate(rr).astype(np.float32)
    return rr[rng.permutation(rr.shape[0])], ims, np.asarray([[800, 1333, 1.6666666], [640, 1066, 0.8]], np.float32)


def timed(fn, iters):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter(); e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return dict(wall_ms=(time.perf_counter() - t0) * 1e3 / iters, event_ms=e0.elapsed_time(e1) / iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("proposal_labels_probe: no CUDA device")
    from detectron.pytorch_b200.modeling.collect_and_distribute_fpn_rpn_proposals import CollectAndDistributeFpnRpnProposalsOp
    from detectron.pytorch_b200.modeling.generate_proposal_labels import GenerateProposalLabelsOp
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    rr, roidb, im_info = inputs()
    t = dict(C.TRAIN_CFG, BATCH_SIZE_PER_IM=512, MASK_ON=True, MRCNN_RESOLUTION=14, CLS_SPECIFIC_MASK=True)
    rr_d = torch.from_numpy(rr).cuda()
    c4 = GenerateProposalLabelsOp(train=t)
    out = dict(card=card, c4=timed(lambda: c4(rr_d, roidb, im_info), a.iters))
    scores = torch.rand(rr_d.shape[0], 1, device="cuda")
    cd = CollectAndDistributeFpnRpnProposalsOp(post_nms_topN=rr_d.shape[0])
    cd.train()
    inp = [rr_d] + [rr_d[:0]] * 4 + [scores] + [scores[:0]] * 4
    out["fpn"] = timed(lambda: cd(inp, roidb, im_info, train=t), a.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
