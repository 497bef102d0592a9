"""GPU test of the stream every op of ops.py launches on: the current torch stream of its device.

A handful of ops that never read the host are captured into one CUDA graph.  torch.cuda.graph captures on a side stream, so a
launch on the device's default stream makes the capture fail, and a launch on any other stream would leave the op out of the
graph.  The graph is then replayed on new inputs written into the captured tensors, and its outputs must equal an eager run on
those inputs.
"""
import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import ops, synthetic as S

pytestmark = pytest.mark.gpu

SHAPE, SCALE, P, SR = (1, 64, 50, 68), 1.0 / 16, 7, 2     # large enough for the workspace-backed RoIAlign paths
NMS_THRESH = 0.7
TOPK = (1000, 300)
D, K, M = 16, 17, 56                                        # keypoint heatmaps
R, C = 128, 81                                              # Fast R-CNN box head


def _inputs(seed):
    rs = np.random.RandomState(seed)
    rois = np.concatenate([S.make_rois(96, SHAPE, SCALE, seed=seed), S.make_edge_rois(SHAPE, SCALE)]).astype(np.float32)
    xy = rs.uniform(0, 400, (D, 2))
    kp_rois = np.concatenate([xy, xy + rs.uniform(16, 300, (D, 2))], axis=1)
    x = dict(feats=S.make_features(SHAPE, seed=seed), rois=rois,
             dy=rs.standard_normal((rois.shape[0], SHAPE[1], P, P)),
             boxes=S.make_nms_boxes(2000, seed=seed),
             maps=rs.standard_normal((2, 3, 50, 68)),
             heatmaps=rs.standard_normal((D, K, M, M)), kp_rois=kp_rois,
             cls_score=rs.standard_normal((R, C)), bbox_pred=rs.standard_normal((R, 4 * C)),
             labels=rs.randint(0, C, R).astype(np.int32), targets=rs.standard_normal((R, 4 * C)),
             inside=(rs.uniform(size=(R, 4 * C)) < 0.1), outside=(rs.uniform(size=(R, 4 * C)) < 0.1))
    return {k: torch.from_numpy(np.ascontiguousarray(v).astype(np.int32 if k == "labels" else np.float32)).cuda() for k, v in x.items()}


def _run(x):
    """Every op once on the tensors of `x`; returns their outputs."""
    feats = x["feats"].requires_grad_(True)
    out = ops._RoIAlign.apply(feats, x["rois"], P, P, SCALE, SR)
    (dx,) = torch.autograd.grad(out, feats, x["dy"])
    pool, argmax = ops.roi_pool_forward(x["feats"].detach(), x["rois"], P, P, SCALE)
    keep, num = ops.nms_raw(x["boxes"], NMS_THRESH)
    order, top = ops.topk_batched_raw([x["maps"][0], x["maps"][1]], TOPK)
    kps = ops.heatmaps_to_keypoints_raw(x["heatmaps"], x["kp_rois"])
    cls_score, bbox_pred = x["cls_score"].requires_grad_(True), x["bbox_pred"].requires_grad_(True)
    loss_cls, loss_bbox, accuracy = ops.fast_rcnn_losses(cls_score, bbox_pred, x["labels"], x["targets"], x["inside"], x["outside"])
    d_cls, d_bbox = torch.autograd.grad(loss_cls + loss_bbox, (cls_score, bbox_pred))
    return dict(out=out.detach(), dx=dx, pool=pool, argmax=argmax, keep=keep, num=num, order=order, top=top, kps=kps,
                losses=torch.stack([loss_cls.detach(), loss_bbox.detach(), accuracy]), d_cls=d_cls, d_bbox=d_bbox)


def test_ops_capture_into_a_cuda_graph_and_replay_like_eager():
    x = _inputs(1)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                             # warm-up off the default stream, as torch.cuda.graph asks
        _run(x)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _run(x)
    with torch.no_grad():
        for k, v in _inputs(2).items():
            x[k].copy_(v)
    graph.replay()
    eager = _run(x)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in captured.items()}
    want = {k: v.cpu().numpy() for k, v in eager.items()}
    n = int(want["num"][0])
    assert n > 0 and int(got["num"][0]) == n
    np.testing.assert_array_equal(got["keep"][:n], want["keep"][:n])
    np.testing.assert_allclose(got["dx"], want["dx"], rtol=1e-5, atol=1e-5)   # summed with fp32 atomics: order may differ
    for k in ("out", "pool", "argmax", "order", "top", "kps", "losses", "d_cls", "d_bbox"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
