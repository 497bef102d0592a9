"""Host-array front door of the device keypoint extraction, named like the reference's `utils.keypoints`
(lib/utils/keypoints.py): `heatmaps_to_keypoints(maps, rois)` (:103-157) and `nms_oks(kp_predictions, rois, thresh)`
(:225-266).  Both take numpy arrays like the reference's or CUDA tensors, and return numpy results.
`keypoints_to_heatmap_labels(keypoints, rois)` (:160-211), the training-time labels, returns CUDA tensors (the loss reads
them on the device).

The resize, argmax and coordinates reproduce the reference's numpy 2 / cv2 float32 INTER_CUBIC arithmetic bit for bit;
prob (the spatial softmax at the maximum) is summed in double on the device where numpy sums float32 pairwise, so it
agrees to ~1e-7 relative.  nms_oks takes equal scores the higher index first (the reference's order for ties comes from
numpy's unstable argsort), and its float64 exp may differ from numpy's by an ulp.
"""
import numpy as np
import torch

from .. import ops


def _device_of(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    return torch.device("cuda", torch.cuda.current_device())


def _f32(x, dev):
    t = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    return t.to(dev, dtype=torch.float32)


def heatmaps_to_keypoints(maps, rois, min_size=0):
    """(D, 4, K) float32 numpy array of (x, y, logit, prob) rows from the (D, K, M, M) logits and (D, >=4) boxes;
    min_size is KRCNN.INFERENCE_MIN_SIZE (<= 0: none)."""
    dev = _device_of(maps, rois)
    return ops.heatmaps_to_keypoints_raw(_f32(maps, dev), _f32(rois, dev), min_size).cpu().numpy()


def nms_oks(kp_predictions, rois, thresh):
    """Kept indices (list of int, greedy order) of the OKS NMS over (D, 4, 17) predictions and (D, >=4) boxes."""
    if kp_predictions.shape[0] == 0:
        return []
    dev = _device_of(kp_predictions, rois)
    keep, num_keep = ops.nms_oks_raw(_f32(kp_predictions, dev), _f32(rois, dev), thresh)
    return keep[:int(num_keep.item())].cpu().tolist()


def keypoints_to_heatmap_labels(keypoints, rois, heatmap_size=None, cfg=None):
    """The training-time labels of lib/utils/keypoints.py:160-211 on the device: keypoints (R, 3, K) int32 (x, y, v), rois (R, >=4)
    float32 [x1, y1, x2, y2] (numpy or CUDA; computed in float32 as the reference's float32 roidb boxes are).  heatmap_size is
    KRCNN.HEATMAP_SIZE (or taken from cfg).  Returns (heats, weights) as CUDA (R, K) tensors: heats int32 -- the reference's
    float32 labels after the caller's `.astype(np.int32)`, INT_MIN where they are NaN -- and weights float32 (0 / 1)."""
    if heatmap_size is None:
        if cfg is None:
            raise ValueError("keypoints_to_heatmap_labels needs heatmap_size (or cfg=)")
        heatmap_size = cfg.KRCNN.HEATMAP_SIZE
    dev = _device_of(keypoints, rois)
    return ops.keypoints_to_heatmap_labels_raw(keypoints, _f32(rois, dev), heatmap_size)


# The 17 COCO person keypoints in the dataset's order and their left / right pairs (lib/utils/keypoints.py:30-63).
KEYPOINTS = ["nose", "left_eye", "right_eye", "left_ear", "right_ear", "left_shoulder", "right_shoulder", "left_elbow",
             "right_elbow", "left_wrist", "right_wrist", "left_hip", "right_hip", "left_knee", "right_knee", "left_ankle", "right_ankle"]
KEYPOINT_FLIP_MAP = {"left_" + p: "right_" + p for p in ("eye", "ear", "shoulder", "elbow", "wrist", "hip", "knee", "ankle")}


def get_keypoints():
    """(keypoint names, left -> right flip map) like lib/utils/keypoints.py:30-63."""
    return list(KEYPOINTS), dict(KEYPOINT_FLIP_MAP)


def flip_permutation(num_keypoints=None):
    """(J,) int32: channel c of a horizontally flipped heatmap stack comes from channel perm[c] (each left / right pair of
    get_keypoints() swapped, the others in place), the channel half of flip_heatmaps.  J defaults to the 17 COCO keypoints."""
    keypoints, flip_map = get_keypoints()
    perm = np.arange(len(keypoints) if num_keypoints is None else int(num_keypoints), dtype=np.int32)
    for lkp, rkp in flip_map.items():
        lid, rid = keypoints.index(lkp), keypoints.index(rkp)
        perm[rid], perm[lid] = lid, rid
    return perm


def flip_heatmaps(heatmaps):
    """lib/utils/keypoints.py:90-100 on the device: heatmaps (R, J, M, M) (numpy or float32 CUDA) with the left / right
    keypoint channels swapped and mirrored along the last axis, in one launch (ops.tta_combine_raw copying through the
    permutation).  Returns a float32 CUDA tensor."""
    dev = _device_of(heatmaps)
    src = _f32(heatmaps, dev).contiguous()
    out = torch.empty_like(src)
    return ops.tta_combine_raw(src, out, ops.TTA_HEURISTICS["HM_MAX"], op=ops.TTA_START, hflip=True,
                               channel_perm=flip_permutation(src.size(1)))
