"""Seeded inputs of the Keypoint R-CNN keypoint tests (keypoint_results, lib/core/test.py:850-866) -- inputs only, expected
values come from the golden file tests/golden/keypoints.npz and from oracle/keypoints.py."""
import numpy as np

KP_IM_H, KP_IM_W = 800, 1333
KP_NUM_KEYPOINTS = 17
KP_HEATMAP_SIZE = 56
KP_NUM_CLASSES = 2                      # background + person
# (seed, detections, KRCNN.INFERENCE_MIN_SIZE, KRCNN.NMS_OKS).  min_size 1 stands for the default 0: every box side is
# clamped to >= 1 first, so both give the same heatmap sizes and the same float32 corrections.
KEYPOINT_CASES = ((0, 1, 1, False), (1, 7, 64, False), (2, 100, 1, False), (3, 100, 64, False), (4, 48, 1, True))
ZERO_CHANNEL, CONSTANT_CHANNEL = 3, 11  # of detection 0 in every case: all zeros / one constant nonzero logit


def _person_boxes(rng, n):
    w = np.exp(rng.uniform(np.log(32), np.log(600), n))
    h = np.minimum(w * rng.uniform(1.2, 3.0, n), KP_IM_H - 1.0)
    x1 = rng.uniform(0, KP_IM_W - 1 - w)
    y1 = rng.uniform(0, KP_IM_H - 1 - h)
    return np.stack([x1, y1, x1 + w, y1 + h], 1)


def _special_boxes(rng):
    X, Y = KP_IM_W - 1.0, KP_IM_H - 1.0
    x, y = rng.uniform(50, 600), rng.uniform(50, 400)
    return np.array([[x, y, x + 37.3, y + 91.7],                       # fractional sides
                     [100.0, 200.0, 156.0, 256.0],                     # exactly M x M: a copy when min_size < 56
                     [x, y, x + 0.4, y + 120.25],                      # width below 1 (clamped to 1)
                     [x + 10, y + 5, x + 60.5, y + 5.6],               # height below 1
                     [0.0, 0.0, X, Y],                                 # the whole image
                     [X - 30.8, Y - 70.1, X, Y]])                      # against the far corner


def _logits(rng, D, centers=None):
    """Gaussian blob per keypoint plus noise, (D, K, M, M) float32.  centers: optional (D, K, 2) blob centres."""
    M, K = KP_HEATMAP_SIZE, KP_NUM_KEYPOINTS
    g = np.arange(M, dtype=np.float64)
    if centers is None:
        centers = rng.uniform(4, M - 4, (D, K, 2))
    sig = rng.uniform(1.5, 4.0, (D, K, 1, 1))
    amp = rng.uniform(4.0, 12.0, (D, K, 1, 1))
    cx, cy = centers[..., 0][..., None, None], centers[..., 1][..., None, None]
    blob = amp * np.exp(-((g[None, None, None, :] - cx) ** 2 + (g[None, None, :, None] - cy) ** 2) / (2 * sig ** 2))
    maps = blob + 0.7 * rng.standard_normal((D, K, M, M)) + rng.uniform(-3, 1, (D, K, 1, 1))
    return maps.astype(np.float32)


def keypoint_case(seed, D, min_size, nms_oks):
    """Inputs of keypoint_results for one image: (cls_boxes list of KP_NUM_CLASSES arrays, background empty and (D, 5) at
    the person class; heatmaps (D, 17, 56, 56) float32; ref_boxes (D, 4) float32).  Detection 0 has an all-zero and a
    constant channel.  Without NMS the boxes are person-shaped plus, from D >= 7 on, the special boxes of _special_boxes;
    the NMS case has clusters of jittered boxes whose heatmap blobs sit at nearly the same relative places, so that some
    detections overlap in OKS and others do not."""
    rng = np.random.RandomState(1000 + seed)
    if nms_oks:
        n_clusters = 8
        per = D // n_clusters
        base = _person_boxes(rng, n_clusters)
        boxes, centers = [], []
        for c in range(n_clusters):
            kc = rng.uniform(6, KP_HEATMAP_SIZE - 6, (KP_NUM_KEYPOINTS, 2))
            for _ in range(per):
                bw, bh = base[c, 2] - base[c, 0], base[c, 3] - base[c, 1]
                j = rng.uniform(-0.08, 0.08, 4) * np.array([bw, bh, bw, bh])
                boxes.append(base[c] + j)
                centers.append(kc + rng.normal(0, rng.choice([0.3, 2.0, 6.0]), kc.shape))
        boxes = np.array(boxes)
        maps = _logits(rng, D, np.array(centers))
    else:
        boxes = _person_boxes(rng, D)
        if D >= 7:
            sp = _special_boxes(rng)
            boxes[1:1 + len(sp)] = sp
        maps = _logits(rng, D)
    boxes[:, 0::2] = np.clip(boxes[:, 0::2], 0, KP_IM_W - 1)
    boxes[:, 1::2] = np.clip(boxes[:, 1::2], 0, KP_IM_H - 1)
    boxes = boxes.astype(np.float32)
    maps[0, ZERO_CHANNEL] = 0
    maps[0, CONSTANT_CHANNEL] = np.float32(1.7)
    scores = rng.uniform(0.05, 1, (D, 1)).astype(np.float32)
    cls_boxes = [np.zeros((0, 5), np.float32), np.concatenate([boxes, scores], 1).astype(np.float32)]
    return cls_boxes, maps, boxes.copy()
