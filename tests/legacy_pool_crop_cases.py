"""Seeded cases for RoIPool, the legacy (lattice-corner) RoIAlign and RoICrop (inputs only -- expected values come from
the oracle / golden files).  Every case names the launch branch it is there to reach; tests/test_roi_pool_legacy_crop.py
restates the host-side choices of roi_pool.cu, roi_align_legacy.cu and roi_crop.cu and checks that it does:

  slabs      pool_c_per_cta / legacy_c_per_cta halve the channels per CTA while R x slabs < 8 x 132 CTAs and a slab
             still has >= 256 outputs; the RoIPool backward halves its slab (down to 8) while tiles x N x slabs < 4 x 132
  bins>1024  PH x PW > 1024: no shared-memory table of bin rectangles / lattice points, computed on the fly
  chunked    > 512 RoIs of one image meet one 8 x 32 tile of the RoIPool backward: its RoI list is consumed in chunks
  ties       post-ReLU, coarsely quantised features: most bins hold several cells equal to their maximum
  one-row    legacy RoIAlign on a map with H < 2 or W < 2 (never given to the reference kernel: it reads row / column -1)
  crop       RoICrop: the scalar kernel's channel split, R % N != 0 (RoIs whose image index R / (R / N) reaches N),
             the NHWC scatter backward with a partial last 256-channel chunk, and its shared tile over 200 KB (declines)

The RoIs of every case have valid batch indices; tests that need an out-of-range or negative one append them, so the
reference kernels (tests/golden/make_golden_legacy_pool_crop.py) never see one.
"""
import hashlib

import numpy as np

from detectron.pytorch_b200 import synthetic as S

NUM_SMS = 132           # kNumSMs of common.cuh (H100 SXM)


def _case(shape, scale, PH, PW, n_rois, branch, lo=32.0, hi=512.0, edge=True, feats="normal", golden=False):
    return dict(shape=shape, scale=scale, PH=PH, PW=PW, n_rois=n_rois, branch=branch, lo=lo, hi=hi, edge=edge, feats=feats,
                golden=golden)


# ---- RoIPool and legacy RoIAlign (the same inputs drive both)
POOL_LEGACY_CASES = {
    # BASELINE.json configs 1 and 2 at full size: 8 channels per CTA at cfg1, 64 at cfg2
    "cfg1": _case(S.CFG1["shape"], S.CFG1["scale"], 7, 7, S.CFG1["rois"], "slabs", edge=False, golden=True),
    "cfg2": _case(S.CFG2["shape"], S.CFG2["scale"], 7, 7, S.CFG2["rois"], "slabs", edge=False, golden=True),
    # rectangular bins; 1 x 16 is also the legacy P - 1 = 0 division (NaN) along h
    "rect_7x14": _case((2, 16, 30, 45), 1.0 / 8, 7, 14, 24, "rect", golden=True),
    "rect_14x7": _case((2, 16, 30, 45), 1.0 / 8, 14, 7, 24, "rect", golden=True),
    "rect_1x16": _case((2, 16, 30, 45), 1.0 / 8, 1, 16, 24, "rect", golden=True),
    # P = 1: one bin per RoI; the legacy lattice divides by P - 1 = 0
    "p1": _case((2, 16, 30, 45), 1.0 / 8, 1, 1, 24, "p1"),
    # more than 1024 bins per RoI
    "p33": _case((1, 8, 40, 48), 1.0 / 8, 33, 33, 16, "bins>1024", golden=True),
    "p40x28": _case((1, 8, 40, 48), 1.0 / 8, 40, 28, 16, "bins>1024", golden=True),
    # channel counts, three images with mixed batch indices
    "c1": _case((3, 1, 24, 40), 1.0 / 8, 7, 7, 48, "channels"),
    "c6": _case((3, 6, 24, 40), 1.0 / 8, 7, 7, 48, "channels"),
    "c33": _case((3, 33, 24, 40), 1.0 / 8, 7, 7, 48, "channels", golden=True),
    "c256": _case((3, 256, 24, 40), 1.0 / 8, 7, 7, 48, "slabs", golden=True),
    "c260": _case((3, 260, 24, 40), 1.0 / 8, 7, 7, 48, "slabs", golden=True),
    # most bins tie at their maximum (zeros and a few quantisation levels)
    "ties": _case((2, 16, 30, 45), 1.0 / 8, 7, 7, 64, "ties", feats="relu_quantised"),
    # RoIPool backward: > 512 RoIs of one image on one tile, several channel slabs, two images, partial tiles (37 % 8, 70 % 32)
    "chunked": _case((2, 256, 37, 70), 1.0 / 8, 7, 7, 1200, "chunked", lo=250.0, hi=560.0),
}

# ---- legacy RoIAlign on maps with one row or one column (and 2 x 2, the smallest map the reference handles)
LEGACY_MAP_CASES = {
    "map_1xW": _case((2, 8, 1, 40), 1.0 / 8, 7, 7, 24, "one-row", lo=4.0, hi=200.0),
    "map_Hx1": _case((2, 8, 30, 1), 1.0 / 8, 7, 7, 24, "one-row", lo=4.0, hi=200.0),
    "map_1x1": _case((2, 8, 1, 1), 1.0 / 8, 7, 7, 24, "one-row", lo=1.0, hi=16.0),
    "map_2x2": _case((2, 8, 2, 2), 1.0 / 8, 7, 7, 24, "one-row", lo=1.0, hi=24.0),
}


# ---- RoICrop.  grid "affine": utils.net.affine_grid_gen from the RoIs of a BASELINE config at 2P x 2P (the crop that
# model_builder's RoICrop transform max-pools 2 x 2 down to P x P); grid "random": synthetic.make_crop_grid plus samples on
# the border and outside the image
def _crop(shape, R, oh, ow, branch, grid="random", cfg=None, golden=False):
    return dict(shape=shape, R=R, oh=oh, ow=ow, branch=branch, grid=grid, cfg=cfg, golden=golden)


CROP_CASES = {
    "cfg1": _crop(S.CFG1["shape"], S.CFG1["rois"], 14, 14, "nhwc", grid="affine", cfg=S.CFG1, golden=True),
    "cfg2": _crop(S.CFG2["shape"], S.CFG2["rois"], 14, 14, "nhwc", grid="affine", cfg=S.CFG2, golden=True),
    # too few taps for the scatter path: the scalar kernel, 4 channels per CTA
    "scalar_slabs": _crop((2, 256, 50, 68), 8, 7, 7, "scalar", golden=True),
    # R % N != 0: per = 7 / 3 = 2, RoI 6 maps to image 3 = N -> zeros, no gradient
    "r_mod_n": _crop((3, 6, 20, 24), 7, 7, 7, "r%n"),
    # the scatter backward with C > 256: a full chunk + a partial one of 4 / 44 channels
    "c260": _crop((1, 260, 20, 24), 32, 7, 7, "nhwc", golden=True),
    "c300": _crop((1, 300, 20, 24), 32, 7, 7, "nhwc", golden=True),
    # the scatter path applies, but its shared tile (14 x 15 x 260 x 4 B = 218 400 B) exceeds 200 KB: the scalar kernel runs
    "tile_14x15": _crop((1, 256, 30, 40), 16, 14, 15, "declined", golden=True),
}

GOLDEN_SAMPLE = 2048


def features(c, seed=0):
    f = S.make_features(c["shape"], seed=seed)
    if c["feats"] == "relu_quantised":
        f = np.floor(np.maximum(f, 0.0))                      # {0, 1, 2, 3, 4}: ~84 % zeros
    return f.astype(np.float32)


def roi_case(c):
    """(features, rois, dy) of a RoIPool / legacy RoIAlign case; every batch index is valid."""
    f = features(c)
    rois = S.make_rois(c["n_rois"], c["shape"], c["scale"], seed=1, min_size=c["lo"], max_size=c["hi"])
    if c["edge"]:
        rois = np.concatenate([rois, S.make_edge_rois(c["shape"], c["scale"])])
    rois = rois.astype(np.float32)
    dy = np.random.RandomState(2).standard_normal((rois.shape[0], c["shape"][1], c["PH"], c["PW"])).astype(np.float32)
    return f, rois, dy


def crop_grid(c):
    """(R, oh, ow, 2) sampling grid in (y, x) order."""
    if c["grid"] == "affine":
        import torch
        from detectron.pytorch_b200.utils.net import affine_grid_gen
        cfg = c["cfg"]
        rois = S.make_rois(cfg["rois"], cfg["shape"], cfg["scale"])
        # built in float64 and rounded once, so that the grid does not depend on how the host's BLAS groups the
        # 3-term dot products of affine_grid (the golden outputs were recorded on another machine)
        g = affine_grid_gen(torch.from_numpy(rois.astype(np.float64)), cfg["shape"][2:], c["oh"]).numpy()
        return np.ascontiguousarray(np.stack([g[..., 1], g[..., 0]], axis=-1)).astype(np.float32)
    grid = S.make_crop_grid(c["R"], c["oh"], c["ow"], seed=3)
    grid[0, 0, 0] = (-1.0, -1.0)
    grid[0, 0, 1] = (1.0, 1.0)
    grid[1, 2, 2] = (-1.5, 0.2)
    grid[c["R"] - 1, 1, 1] = (0.3, 1.7)
    return grid.astype(np.float32)


def crop_case(c):
    """(image, grid, grad_output) of a RoICrop case."""
    img = S.make_features(c["shape"], seed=4)
    grid = crop_grid(c)
    go = np.random.RandomState(5).standard_normal((c["R"], c["shape"][1], c["oh"], c["ow"])).astype(np.float32)
    return img, grid, go


def golden_positions(size, seed, nonzero_of=None):
    """Sorted flat positions of a fixed, seeded sample (of the non-zero elements of `nonzero_of` when given)."""
    pool = np.flatnonzero(nonzero_of) if nonzero_of is not None else np.arange(size)
    pick = np.random.RandomState(seed).choice(pool.size, min(GOLDEN_SAMPLE, pool.size), replace=False)
    return np.sort(pool[pick]).astype(np.int32)


def digest(a):
    """sha256 of an array's bytes with every NaN written as the same quiet NaN: equal digests mean bit-identical arrays
    (up to NaN payloads), so a complete result can be compared without storing it."""
    a = np.ascontiguousarray(a)
    if a.dtype == np.float32:
        a = np.where(np.isnan(a), np.float32(np.nan), a).astype(np.float32)
    return hashlib.sha256(a.tobytes()).hexdigest()
