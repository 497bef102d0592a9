"""NMS on BASELINE cfg3 (6000 boxes): time per call (CUDA events) and the kept count; prints the card and its power limit."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from detectron.pytorch_b200 import ops, synthetic as S
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card:", card)
b = torch.from_numpy(S.make_nms_boxes(6000)).cuda()
for _ in range(3):
    keep, num = ops.nms_raw(b, 0.7)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20):
    ops.nms_raw(b, 0.7)
e1.record(); torch.cuda.synchronize()
print("nms 6000: %.1f us/call, kept %d" % (e0.elapsed_time(e1) / 20 * 1e3, int(num.item())))
