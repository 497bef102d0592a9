"""Seeded inputs of the image blob tests (get_image_blob, lib/utils/blob.py:37-60, and _get_image_blob,
lib/roi_data/minibatch.py:47-79) -- inputs only; expected values come from tests/golden/image_blob.npz and oracle/blob.py.

Images are small (sides up to 90 px) with scaled-down SCALE / MAX_SIZE so the golden file stays small; COCO-size parity is
checked against the oracle.  Between them the cases cover upscales, non-terminating scales, the MAX_SIZE cap, an exact 2x
shrink with even sides and with an odd last row or column, rint's half-to-even sizes, 1-px sides, blob widths that are not
a multiple of 4 (FPN off), flips and mixed sizes in one batch."""
import numpy as np

# test time: (name, seed, H, W, target_scale, target_max_size, fpn_on)
TEST_CASES = (
    ("up_nonterm", 0, 17, 23, 30, 50, True),            # 30 / 17: upscale, non-terminating scale
    ("up_nofpn", 1, 23, 17, 30, 50, False),             # blob width 30: scalar stores
    ("cap", 2, 40, 90, 30, 40, True),                   # MAX_SIZE cap, scale 4 / 9
    ("area_oddrow", 3, 47, 40, 20, 1000, True),         # 1 / s == 2, 47 rows -> 24 (last row has one source row)
    ("area_oddcol", 4, 40, 47, 20, 1000, False),        # the same on the columns
    ("area_even", 5, 60, 80, 30, 1000, True),           # 2x on even sides
    ("half_even", 6, 5, 14, 100, 7, False),             # cap to 0.5: 2.5 rows -> 2 (half to even)
    ("half_up", 7, 7, 14, 100, 7, True),                # 3.5 rows -> 4
    ("row1", 8, 1, 30, 2, 100, True),                   # a 1-px side, scale 2
    ("col1", 9, 30, 1, 3, 100, False),                  # a 1-px side, scale 3
    ("same", 10, 20, 31, 20, 1000, True),               # scale 1: cv2 copies
)

# training: (name, seed, [(H, W, flipped)], TRAIN.SCALES, TRAIN.MAX_SIZE, fpn_on, np.random seed of the scale draw)
TRAIN_CASES = (
    ("mixed_fpn", 20, [(23, 31, True), (40, 47, False), (9, 12, True)], (20, 30, 16), 50, True, 3),
    ("area_flip_nofpn", 21, [(47, 40, True), (1, 30, False)], (20,), 1000, False, 4),
    ("flip_pair", 22, [(33, 17, False), (33, 17, True)], (25, 18), 45, True, 5),
)


def image(seed, H, W):
    """A seeded uint8 (H, W, 3) BGR image: noise over a smooth ramp, with 0 and 255 present."""
    rng = np.random.RandomState(1000 + seed)
    ramp = (np.arange(H)[:, None, None] * 7 + np.arange(W)[None, :, None] * 3 + np.array([0, 85, 170])) % 256
    im = (ramp + rng.randint(-40, 41, (H, W, 3))).clip(0, 255).astype(np.uint8)
    im.reshape(-1)[:2] = (0, 255)
    return im


def train_images(seed, shapes):
    return [image(seed * 10 + k, H, W) for k, (H, W, _) in enumerate(shapes)]
