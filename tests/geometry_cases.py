"""Seeded RoIAlign cases at the geometry where index arithmetic and path choice go wrong (inputs only -- expected
values come from the oracle / golden files): rectangular bins, the pooled-size and sampling-ratio limits of every fast
path, maps at tile and strip boundaries, the 16-bit RoI field, partial channel groups and the shapes that make a path
decline.

Every case records which forced path must RUN on it and which must DECLINE (and fall back to the generic kernel):
  fwd: the fast forwards that accept the case, a subset of {"tiled", "stream", "quad"};
  bwd: the fast backwards that accept the case, a subset of {"nhwc", "rows"}.
The generic kernels accept everything.  The table restates the checks at the top of stream_geometry
(roi_align_stream.cu), strip_geometry (roi_align_strip.cu), roi_align_tiled_plan (roi_align_tiled.cuh), rows_plan
(roi_align_bwd_rows.cu) and roi_align_backward_nhwc (roi_align_bwd_nhwc.cu):
  stream, quad  sr in {1, 2}; PH * sr, PW * sr <= 32; PH, PW <= 31; R <= 65535; H, W >= 2; N x strips <= 96 strip
                columns (stream: 87-column strips + 10 halo at W = 2000; quad: 56 + 8); quad only: N x strips x H <= 6144 keys
  tiled         sr in {1..4}; PH * sr, PW * sr <= 32; R <= 65535
  nhwc          sr in {1..4}; PH * sr, PW * sr <= 32; PH * PW * (min(C, 256) rounded up to 4, + 4) * 4 B <= 200 KB
  rows          sr in {1, 2}; PW in {7, 14}; PH * sr <= 32; C % 64 == 0; R <= 65535
"""
import numpy as np

from detectron.pytorch_b200 import synthetic as S

FAST = ("tiled", "stream", "quad")


def _case(shape, scale, PH, PW, sr, n_rois, fwd, bwd, lo=32.0, hi=512.0, edge=True, pileup=False):
    return dict(shape=shape, scale=scale, PH=PH, PW=PW, sr=sr, n_rois=n_rois, fwd=frozenset(fwd), bwd=frozenset(bwd), lo=lo, hi=hi,
                edge=edge, pileup=pileup)


def _rows_ok(PW, sr, C):
    return PW in (7, 14) and sr in (1, 2) and C % 64 == 0


GEOMETRY_CASES = {}

# ---- rectangular bins (PH != PW): one map with C = 64, so that the rows backward runs wherever PW is 7 or 14
RECT_SHAPE, RECT_SCALE = (2, 64, 30, 45), 1.0 / 8
for _ph, _pw in ((7, 14), (14, 7), (1, 16), (16, 1), (3, 7), (16, 7), (7, 3)):
    for _sr in (1, 2):
        GEOMETRY_CASES["rect_%dx%d_sr%d" % (_ph, _pw, _sr)] = _case(
            RECT_SHAPE, RECT_SCALE, _ph, _pw, _sr, 24, FAST, ("nhwc", "rows") if _rows_ok(_pw, _sr, 64) else ("nhwc",))
# PW * sr = 33 > 32: every fast path declines
GEOMETRY_CASES["rect_5x11_sr3"] = _case(RECT_SHAPE, RECT_SCALE, 5, 11, 3, 24, (), ())
# adaptive sampling (grid_h != grid_w per RoI): only the generic kernels sample adaptively
GEOMETRY_CASES["rect_4x9_sr0"] = _case(RECT_SHAPE, RECT_SCALE, 4, 9, 0, 24, (), ())
RECT_CASES = tuple(sorted(n for n in GEOMETRY_CASES if n.startswith("rect_")))

# ---- pooled-size and sampling-ratio limits.  At 900 - 1024 samples per RoI the edge RoIs smaller than a cell (zero-area,
# sub-cell, hugging the last row) put thousands of fp32 addends on a few dX cells: pile-ups
_P = (1, 8, 40, 48)
GEOMETRY_CASES.update({
    "p16_sr2": _case(_P, 1.0 / 8, 16, 16, 2, 24, FAST, ("nhwc",), pileup=True),                 # PH * sr == 32 everywhere
    "p31_sr1": _case(_P, 1.0 / 8, 31, 31, 1, 24, FAST, ("nhwc",), pileup=True),                 # 5-bit field maximum, 961 bins
    "p31x3_sr1": _case(_P, 1.0 / 8, 31, 3, 1, 24, FAST, ("nhwc",)),
    "p3x31_sr1": _case(_P, 1.0 / 8, 3, 31, 1, 24, FAST, ("nhwc",)),
    "p8_sr4": _case(_P, 1.0 / 8, 8, 8, 4, 24, ("tiled",), ("nhwc",), pileup=True),
    "p10_sr3": _case(_P, 1.0 / 8, 10, 10, 3, 24, ("tiled",), ("nhwc",), pileup=True),
    # P 32 at sr 1: stream and quad decline (5-bit fields); the NHWC shared tile is 32 x 32 x (C + 4) floats:
    # 180 KB at C = 40 (runs), 208 KB at C = 48 (declines)
    "p32_sr1_c40": _case((1, 40, 40, 48), 1.0 / 8, 32, 32, 1, 24, ("tiled",), ("nhwc",), pileup=True),
    "p32_sr1_c48": _case((1, 48, 40, 48), 1.0 / 8, 32, 32, 1, 24, ("tiled",), (), pileup=True),
    "p17_sr2": _case(_P, 1.0 / 8, 17, 17, 2, 24, (), (), pileup=True),                          # PH * sr == 34
    "p3_sr5": _case(_P, 1.0 / 8, 3, 3, 5, 24, (), ()),                             # sr 5
})

# ---- map sizes at tile and strip boundaries (tiled core_w = 31, rows x-tiles of 32 cells) and the smallest maps
for _w in (31, 32, 33, 63, 64, 65):
    for _h in (1, 2, 3):
        GEOMETRY_CASES["map_h%d_w%d" % (_h, _w)] = _case(
            (2, 64, _h, _w), 1.0 / 8, 7, 7, 2, 16, FAST if _h >= 2 else ("tiled",), ("nhwc", "rows"))
GEOMETRY_CASES.update({
    # every tap of all 28 RoIs lands on the one cell: ~22 000 fp32 addends per dX element (a pile-up)
    "map_1x1": _case((1, 64, 1, 1), 1.0 / 8, 7, 7, 2, 16, ("tiled",), ("nhwc", "rows"), pileup=True),
    "map_h20_w2": _case((1, 64, 20, 2), 1.0 / 8, 7, 7, 2, 16, FAST, ("nhwc", "rows")),
    "map_2x2": _case((2, 64, 2, 2), 1.0 / 8, 7, 7, 1, 16, FAST, ("nhwc", "rows")),
})

# ---- RoI count (r is a 16-bit field of the fast paths' records) and channel counts
_R = (1, 64, 64, 256)
GEOMETRY_CASES.update({
    "r65535": _case(_R, 1.0 / 4, 1, 7, 1, 65535, FAST, ("nhwc", "rows"), lo=4.0, hi=64.0, edge=False),
    "r65536": _case(_R, 1.0 / 4, 1, 7, 1, 65536, (), ("nhwc",), lo=4.0, hi=64.0, edge=False),
})
for _c in (1, 6, 33, 64, 128, 256):                     # partial 32-channel groups; rows with 2 (C % 128 != 0) or 4 channels per lane
    GEOMETRY_CASES["c%d" % _c] = _case((2, _c, 24, 40), 1.0 / 8, 7, 7, 2, 32, FAST, ("nhwc", "rows") if _c % 64 == 0 else ("nhwc",))

# ---- geometry that makes a path decline
GEOMETRY_CASES.update({
    # W = 2000: the stream path cuts 23 strips per image (92 columns at N = 4: runs, 115 at N = 5: declines); the quad
    # strips cut 36 (144 and 180 columns: decline)
    "cols_n4_w2000": _case((4, 4, 2, 2000), 1.0 / 4, 7, 7, 2, 32, ("tiled", "stream"), ("nhwc",)),
    "cols_n5_w2000": _case((5, 4, 2, 2000), 1.0 / 4, 7, 7, 2, 32, ("tiled",), ("nhwc",)),
    # quad strips: 8 images x 2 strips x 800 rows = 12800 keys > 6144; the stream path holds W = 40 in one strip
    "keys_n8_h800": _case((8, 4, 800, 40), 1.0 / 4, 7, 7, 2, 32, ("tiled", "stream"), ("nhwc",)),
    # NHWC shared tile at C = 256: 14 x 14 x 260 x 4 = 203 840 B (runs), 15 x 14 -> 218 400 B > 200 KB (declines)
    "nhwc_14x14_c256": _case((1, 256, 20, 30), 1.0 / 8, 14, 14, 2, 16, FAST, ("nhwc", "rows")),
    "nhwc_15x14_c256": _case((1, 256, 20, 30), 1.0 / 8, 15, 14, 2, 16, FAST, ("rows",)),
})

# the cases whose reference-kernel outputs are recorded (tests/golden/roi_align_geometry_sm90a.npz)
GOLDEN_SAMPLE = 2048


def geometry_case(name):
    """(case, features, rois, dy) of one case; the RoIs are valid (batch index in range), edge RoIs included."""
    c = GEOMETRY_CASES[name]
    feats = S.make_features(c["shape"], seed=0)
    rois = S.make_rois(c["n_rois"], c["shape"], c["scale"], seed=1, min_size=c["lo"], max_size=c["hi"])
    if c["edge"]:
        rois = np.concatenate([rois, S.make_edge_rois(c["shape"], c["scale"])])
    rois = rois.astype(np.float32)
    dy = np.random.RandomState(2).standard_normal((rois.shape[0], c["shape"][1], c["PH"], c["PW"])).astype(np.float32)
    return c, feats, rois, dy


def golden_positions(size, seed, nonzero_of=None):
    """Sorted flat positions of a fixed, seeded sample (of the non-zero elements of `nonzero_of` when given)."""
    pool = np.flatnonzero(nonzero_of) if nonzero_of is not None else np.arange(size)
    pick = np.random.RandomState(seed).choice(pool.size, min(GOLDEN_SAMPLE, pool.size), replace=False)
    return np.sort(pool[pick]).astype(np.int32)
