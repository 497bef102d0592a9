"""Seeded inputs of the Mask R-CNN mask-paste tests (segm_results, lib/core/test.py:793-847) -- inputs only, expected values
come from the golden file tests/golden/segms.npz and from oracle/segms.py."""
import numpy as np

# (seed, im_h, im_w, M, class-specific masks) of the mask-paste cases checked against the reference's segm_results
SEGM_CASES = ((0, 800, 1333, 28, True), (1, 427, 640, 28, False), (2, 427, 640, 14, True), (3, 800, 1333, 14, False))
SEGM_NUM_CLASSES = 8
SEGM_EMPTY_CLASSES = (3, 6)


def _segm_half_box(rng, M, im_h, im_w):
    """A box inside the image whose expanded int32 box is (M + 2) / 2 pixels on both sides (cv2's 2x INTER_AREA path)."""
    from oracle.segms import expand_boxes_int
    target = (M + 2) // 2
    while True:
        x1, y1 = rng.uniform(20, im_w - 60), rng.uniform(20, im_h - 60)
        side = (target - 1) * M / (M + 2.0) + rng.uniform(-0.4, 0.4)
        b = np.array([[x1, y1, x1 + side, y1 + side]], np.float32)
        e = expand_boxes_int(b, M)[0]
        if e[2] - e[0] + 1 == target and e[3] - e[1] + 1 == target:
            return b[0]


def segm_case(seed, im_h, im_w, M, cls_specific):
    """Inputs of segm_results for one image: (cls_boxes list of K arrays (n_j, 5), masks (D, Kc, M, M) float32, ref_boxes
    (D, 4) float32), detections stored class-major like the reference's im_detect_all.  About 60 boxes, clipped to the image
    like the detector's: random ones, boxes touching each border (their expanded boxes stick out), tiny boxes whose width or
    height collapses to one pixel, one expanding to exactly (M + 2) / 2 pixels, one spanning the image height.  Masks are
    sigmoids of smoothed seeded logits, plus one noisy mask (many runs) and one with exact-0.5 plateaus."""
    from scipy.ndimage import gaussian_filter
    rng = np.random.RandomState(100 + seed)
    K = SEGM_NUM_CLASSES
    boxes = []
    for _ in range(40):
        x1, y1 = rng.uniform(0, im_w - 2), rng.uniform(0, im_h - 2)
        boxes.append([x1, y1, x1 + rng.uniform(1, 350), y1 + rng.uniform(1, 300)])
    X, Y = im_w - 1.0, im_h - 1.0
    boxes += [[0, rng.uniform(50, 300), rng.uniform(30, 200), rng.uniform(320, Y)],          # left border
              [rng.uniform(100, 600), 0, rng.uniform(620, X), rng.uniform(20, 200)],         # top border
              [rng.uniform(300, X - 30), rng.uniform(10, 200), X, rng.uniform(210, Y)],      # right border
              [rng.uniform(10, 300), rng.uniform(200, Y - 30), rng.uniform(310, X), Y],      # bottom border
              [0, 0, X, Y], [0, 0, 40.5, 33.2], [X - 25.7, Y - 31.3, X, Y],                  # corners, whole image
              [rng.uniform(300, 500), 0, rng.uniform(510, 700), Y],                          # full height
              [0, 0, 120.0, Y], [X - 90.0, 0, X, Y]]                                         # full height at the sides
    for _ in range(6):                                                                       # tiny: one side collapses
        x1, y1 = rng.uniform(0, im_w - 40), rng.uniform(0, im_h - 40)
        if rng.rand() < 0.5:
            boxes.append([x1, y1, x1 + rng.uniform(0, 0.9), y1 + rng.uniform(0, 30)])
        else:
            boxes.append([x1, y1, x1 + rng.uniform(0, 30), y1 + rng.uniform(0, 0.9)])
    boxes.append([X - 0.4, 5.0, X, 6.0])
    boxes.append(list(_segm_half_box(rng, M, im_h, im_w)))
    boxes.append(list(_segm_half_box(rng, M, im_h, im_w)))
    b = np.array(boxes, dtype=np.float32)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, X); b[:, 1::2] = np.clip(b[:, 1::2], 0, Y)
    D = b.shape[0]
    live = [j for j in range(1, K) if j not in SEGM_EMPTY_CLASSES]
    cls_of = np.sort(np.asarray(live)[rng.randint(0, len(live), D)])
    order = rng.permutation(D)
    b = b[order]
    cls_boxes = [np.zeros((0, 5), np.float32)]
    for j in range(1, K):
        sel = b[cls_of == j]
        cls_boxes.append(np.concatenate([sel, rng.uniform(0.05, 1, (sel.shape[0], 1)).astype(np.float32)], 1).astype(np.float32))
    ref_boxes = np.concatenate([c[:, :4] for c in cls_boxes[1:]], 0).astype(np.float32)
    Kc = K if cls_specific else 1
    logits = np.stack([[gaussian_filter(rng.standard_normal((M, M)), sigma=rng.uniform(1.0, 3.0)) for _ in range(Kc)] for _ in range(D)])
    logits = logits / logits.std(axis=(2, 3), keepdims=True) * 3.0 + rng.uniform(-1.5, 1.5, (D, Kc, 1, 1))
    masks = (1.0 / (1.0 + np.exp(-logits))).astype(np.float32)
    ch = lambda d: int(cls_of[d]) if cls_specific else 0
    masks[1, ch(1)] = rng.rand(M, M).astype(np.float32)                                      # noisy: many runs
    plateau = np.full((M, M), 0.5, np.float32)
    plateau[:, M // 2:] = np.float32(0.25)
    plateau[M // 3:M // 2, :] = np.float32(0.75)
    masks[2, ch(2)] = plateau                                                                # strict > at exact 0.5
    return cls_boxes, masks, ref_boxes
