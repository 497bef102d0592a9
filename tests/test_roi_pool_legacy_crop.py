"""RoIPool, the legacy (lattice-corner) RoIAlign and RoICrop at full size and at their geometry limits
(tests/legacy_pool_crop_cases.py).

CPU part (no marker):
  * a numpy restatement of legacy_point (roi_align_legacy.cu) shows that the reference's tap formula,
    min(floor(h), H - 2), reads row / column -1 on one-row and one-column maps, and that the clamped taps stay inside
    [0, H - 1] x [0, W - 1] for every sample of every case (and equal the reference's wherever H, W >= 2);
  * the host-side launch choices of roi_pool.cu, roi_align_legacy.cu and roi_crop.cu, restated, show that every case
    reaches the branch it names (channel slabs, > 1024 bins, the chunked RoI list, ties, the RoICrop paths);
  * a numpy restatement of the RoIPool backward (argmax scatter in ascending (RoI, ph, pw) order with the reference's
    rounded-rectangle and feasible-bin test) equals oracle_roi_pool_backward bit for bit.  Its per-cell loop over all RoIs
    is ~7e9 RoI checks at BASELINE cfg2, so the GPU part uses the restatement on the large cases.

GPU part (`-m gpu`), with the tolerances of test_gpu_parity.py: RoIPool forward, argmax and backward bit-exact; legacy
RoIAlign forward bit-exact (NaN exactly where the oracle has NaN: P = 1 divides by P - 1 = 0); legacy and RoICrop image
gradients within |a - b| <= 1e-5 + 1e-5 |b| of the fp64 oracle; RoICrop forward bit-exact.  RoIs with an out-of-range or
negative batch index give exact zeros and no gradient.  The golden file legacy_pool_crop_sm90a.npz holds the reference
kernels' results on an H100 (tests/golden/make_golden_legacy_pool_crop.py): digests of the complete bit-exact results and
seeded samples.  Maps with one row or one column run only on the fixed kernel, inside NaN-sentinel guard bands.
"""
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200.model.roi_align.functions.roi_align import RoIAlignFunction as LegacyRoIAlignFunction
from detectron.pytorch_b200.model.roi_crop.functions.roi_crop import RoICropFunction
from detectron.pytorch_b200.model.roi_pooling.functions.roi_pool import RoIPoolFunction
from detectron.pytorch_b200 import synthetic as S
from oracle import cpu as O
from tests import cases as RC
from tests import legacy_pool_crop_cases as LC

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
GOLDEN_FILE = os.path.join(GOLDEN, "legacy_pool_crop_sm90a.npz")
GRAD_TOL = dict(rtol=1e-5, atol=1e-5)
SENTINEL = 0x7FC0DEAD                 # a quiet NaN with a payload no kernel produces
GUARD = 1024                          # sentinel elements before and after every buffer of the guard-band test
PL_NAMES = sorted(LC.POOL_LEGACY_CASES)
MAP_NAMES = sorted(LC.LEGACY_MAP_CASES)
CROP_NAMES = sorted(LC.CROP_CASES)
ORACLE_POOL_BWD_MAX = 2e8             # N C H W R above which the RoIPool backward reference is the numpy scatter


# ------------------------------------------------------------------------------------------ restated host-side choices
def ceil_div(a, b):
    return -(-a // b)


def c_per_cta(R, C, bins):
    """pool_c_per_cta (roi_pool.cu) == legacy_c_per_cta (roi_align_legacy.cu): channels per CTA of the forward."""
    cpc = C
    while cpc > 1 and R * ceil_div(C, cpc) < 8 * LC.NUM_SMS and (cpc // 2) * bins >= 256:
        cpc //= 2
    return cpc


def pool_bwd_c_per_cta(N, C, H, W):
    """roi_pool_backward: channels per CTA over 8 x 32 tiles."""
    tiles = ceil_div(H, 8) * ceil_div(W, 32)
    cpc = C
    while cpc > 8 and tiles * N * ceil_div(C, cpc) < 4 * LC.NUM_SMS:
        cpc //= 2
    return cpc


def crop_c_per_cta(C, npix):
    """crop_grid (roi_crop.cu): channels per CTA of the scalar kernel."""
    xb = ceil_div(npix, 256)
    cpc = C
    while cpc > 4 and xb * ceil_div(C, cpc) < 8 * LC.NUM_SMS:
        cpc //= 2
    return cpc


def crop_backward_path(N, C, H, W, R, oh, ow):
    """crop_nhwc_applies + the checks of roi_crop_backward_nhwc: 'nhwc', 'declined' (the path applies but its shared tile
    exceeds 200 KB) or 'scalar'."""
    if C & 3 or C < 16 or N <= 0 or R <= 0 or R % N:
        return "scalar"
    if 4 * R * oh * ow * C < 2 * N * C * H * W:
        return "scalar"
    chunk = min(C, 256)
    if chunk & 3:
        return "scalar"
    return "declined" if oh * ow * (chunk + 4) * 4 > 200 * 1024 else "nhwc"


def _roundf(x):
    """C roundf of a float32 array (halves away from zero)."""
    x = x.astype(np.float64)
    return (np.sign(x) * np.floor(np.abs(x) + 0.5)).astype(np.int64)


def pool_rois(rois, scale):
    """pool_roi (roi_pool.cu): batch index, rounded rectangle, fp32 bin sizes."""
    s = np.float32(scale)
    r = rois.astype(np.float32)
    b = r[:, 0].astype(np.int64)
    sw, sh, ew, eh = (_roundf(r[:, k] * s) for k in (1, 2, 3, 4))
    rw = np.maximum(ew - sw + 1, 1)
    rh = np.maximum(eh - sh + 1, 1)
    return b, sw, sh, ew, eh, rh.astype(np.float32), rw.astype(np.float32)


def pool_tile_hits(rois, scale, N, H, W):
    """Largest number of RoIs that the RoIPool backward lists for one 8 x 32 tile (its per-image hit test)."""
    b, sw, sh, ew, eh, _, _ = pool_rois(rois, scale)
    best = 0
    for n in range(N):
        for h0 in range(0, H, 8):
            for w0 in range(0, W, 32):
                hit = (b == n) & ~((ew < w0) | (sw >= w0 + 32) | (eh < h0) | (sh >= h0 + 8))
                best = max(best, int(hit.sum()))
    return best


def pool_backward_scatter(dy, argmax, rois, shape, PH, PW, scale):
    """The RoIPool backward restated as a scatter: every pooled element adds its gradient to its argmax cell, in ascending
    (RoI, ph, pw) order -- the order of the reference's per-cell loop -- if the cell lies in the RoI's rounded rectangle and
    the bin lies in the cell's feasible bin range (reference ROIPoolBackward)."""
    N, C, H, W = shape
    R = rois.shape[0]
    b, sw, sh, ew, eh, rh, rw = pool_rois(rois, scale)
    bh = rh / np.float32(PH)
    bw = rw / np.float32(PW)
    flat = np.ascontiguousarray(argmax, dtype=np.int64).reshape(-1)
    o = np.flatnonzero((flat >= 0) & (flat < N * C * H * W))
    idx = flat[o]
    r, rem = np.divmod(o, C * PH * PW)
    c, rem = np.divmod(rem, PH * PW)
    ph, pw = np.divmod(rem, PW)
    n, cell = np.divmod(idx, C * H * W)
    cc, hw = np.divmod(cell, H * W)
    h, w = np.divmod(hw, W)
    ok = (n == b[r]) & (cc == c) & (w >= sw[r]) & (w <= ew[r]) & (h >= sh[r]) & (h <= eh[r])

    def feasible(p, x, x0, bin_, P):
        lo = np.floor((x - x0).astype(np.float32) / bin_).astype(np.int64)
        hi = np.ceil((x - x0 + 1).astype(np.float32) / bin_).astype(np.int64)
        return (p >= np.clip(lo, 0, P)) & (p < np.clip(hi, 0, P))

    ok &= feasible(ph, h, sh[r], bh[r], PH) & feasible(pw, w, sw[r], bw[r], PW)
    grad = np.zeros(N * C * H * W, np.float32)
    np.add.at(grad, idx[ok], np.ascontiguousarray(dy, dtype=np.float32).reshape(-1)[o[ok]])
    return grad.reshape(shape)


def pool_backward_reference(dy, argmax, rois, shape, PH, PW, scale):
    N, C, H, W = shape
    if N * C * H * W * rois.shape[0] <= ORACLE_POOL_BWD_MAX:
        return O.roi_pool_backward(dy, argmax, rois, shape, PH, PW, scale)
    return pool_backward_scatter(dy, argmax, rois, shape, PH, PW, scale)


def legacy_taps(rois, scale, PH, PW, H, W, clamped):
    """legacy_point (roi_align_legacy.cu) restated: for every lattice sample (R, PH, PW) whether it is read (the kernel
    skips a sample only when h < 0, h >= H, w < 0 or w >= W, so a NaN coordinate is read) and its tap rows / columns,
    with the reference's min(floor(h), H - 2) (clamped=False) or the clamped taps."""
    s = np.float32(scale)
    r = rois.astype(np.float32)
    sw, sh = r[:, 1] * s, r[:, 2] * s

    def extent(x2, x1s):                      # fmaxf(FADD(FFMA(x2, scale, -start), 1), 0)
        return np.maximum(((x2.astype(np.float64) * np.float64(s) - x1s).astype(np.float32) + np.float32(1)), np.float32(0))

    rw, rh = extent(r[:, 3], sw), extent(r[:, 4], sh)
    with np.errstate(divide="ignore", invalid="ignore"):
        bh = (rh.astype(np.float64) / (PH - 1.0)).astype(np.float32)
        bw = (rw.astype(np.float64) / (PW - 1.0)).astype(np.float32)
        h = (np.arange(PH)[None, :, None] * bh[:, None, None].astype(np.float64) + sh[:, None, None]).astype(np.float32)
        w = (np.arange(PW)[None, None, :] * bw[:, None, None].astype(np.float64) + sw[:, None, None]).astype(np.float32)
    h, w = np.broadcast_arrays(h, w)
    read = ~((h < 0) | (h >= H) | (w < 0) | (w >= W))

    def taps(x, size):
        lo = np.fmin(np.floor(x), np.float32(size - 2))          # fminf: a NaN coordinate gives size - 2
        if clamped:
            lo = np.fmax(lo, np.float32(0))
        lo = lo.astype(np.int64)
        return lo, (np.minimum(lo + 1, size - 1) if clamped else lo + 1)

    hs, hs2 = taps(h, H)
    ws, ws2 = taps(w, W)
    return read, hs, hs2, ws, ws2


def all_legacy_cases():
    return [(n, c) for n, c in sorted(LC.POOL_LEGACY_CASES.items())] + [(n, c) for n, c in sorted(LC.LEGACY_MAP_CASES.items())]


# ---------------------------------------------------------------------------------------------- CPU
def test_reference_legacy_taps_read_row_and_column_minus_one_on_one_row_and_one_column_maps():
    """The reference's tap formula on H = 1 / W = 1 maps gives index -1 for every sample it reads; the clamped one never
    leaves the map."""
    for name in ("map_1xW", "map_Hx1", "map_1x1"):
        c = LC.LEGACY_MAP_CASES[name]
        _, r, _ = LC.roi_case(c)
        _, _, H, W = c["shape"]
        read, hs, hs2, ws, ws2 = legacy_taps(r, c["scale"], c["PH"], c["PW"], H, W, clamped=False)
        assert read.sum() > 100
        if H == 1:
            assert np.all(hs[read] == -1) and np.all(hs2[read] == 0)
        if W == 1:
            assert np.all(ws[read] == -1) and np.all(ws2[read] == 0)
        read, hs, hs2, ws, ws2 = legacy_taps(r, c["scale"], c["PH"], c["PW"], H, W, clamped=True)
        if H == 1:
            assert np.all(hs[read] == 0) and np.all(hs2[read] == 0)
        if W == 1:
            assert np.all(ws[read] == 0) and np.all(ws2[read] == 0)


@pytest.mark.parametrize("name,c", all_legacy_cases(), ids=[n for n, _ in all_legacy_cases()])
def test_clamped_legacy_taps_stay_in_the_map_and_equal_the_reference_on_larger_maps(name, c):
    _, r, _ = LC.roi_case(c)
    _, _, H, W = c["shape"]
    read, hs, hs2, ws, ws2 = legacy_taps(r, c["scale"], c["PH"], c["PW"], H, W, clamped=True)
    assert read.any()
    for lo, hi, size in ((hs, hs2, H), (ws, ws2, W)):
        assert lo[read].min() >= 0 and hi[read].max() <= size - 1 and np.all(hi[read] - lo[read] <= 1)
    if H >= 2 and W >= 2:
        ref = legacy_taps(r, c["scale"], c["PH"], c["PW"], H, W, clamped=False)
        for a, b in zip((hs, hs2, ws, ws2), ref[1:]):
            assert np.array_equal(a[read], b[read])


def test_every_pool_and_legacy_case_reaches_its_branch():
    for name, c in LC.POOL_LEGACY_CASES.items():
        N, C, H, W = c["shape"]
        _, r, _ = LC.roi_case(c)
        R, bins = r.shape[0], c["PH"] * c["PW"]
        fwd_slabs = ceil_div(C, c_per_cta(R, C, bins))
        if c["branch"] == "slabs":
            assert fwd_slabs > 1 and ceil_div(C, pool_bwd_c_per_cta(N, C, H, W)) > 1, name
        if c["branch"] == "bins>1024":
            assert bins > 1024, name
        if c["branch"] == "channels":
            assert N == 3 and set(r[:, 0].astype(int)) == {0, 1, 2}, name
        if c["branch"] == "chunked":
            assert N == 2 and H % 8 and W % 32 and ceil_div(C, pool_bwd_c_per_cta(N, C, H, W)) > 1
            assert pool_tile_hits(r, c["scale"], N, H, W) > 512
    assert c_per_cta(32, 256, 49) == 8 and c_per_cta(512, 256, 49) == 64        # BASELINE cfg1 / cfg2


def test_ties_case_ties_in_most_bins():
    """The ties case: most non-empty bins hold their maximum in more than one cell, so the argmax is decided by the
    first-maximum rule alone."""
    c = LC.POOL_LEGACY_CASES["ties"]
    f, r, _ = LC.roi_case(c)
    N, C, H, W = c["shape"]
    PH, PW = c["PH"], c["PW"]
    b, sw, sh, _, _, rh, rw = pool_rois(r, c["scale"])
    bh, bw = rh / np.float32(PH), rw / np.float32(PW)
    tied = total = 0
    for i in range(r.shape[0]):
        for ph in range(PH):
            hs = int(np.clip(np.floor(np.float32(ph) * bh[i]) + sh[i], 0, H)); he = int(np.clip(np.ceil(np.float32(ph + 1) * bh[i]) + sh[i], 0, H))
            for pw in range(PW):
                ws = int(np.clip(np.floor(np.float32(pw) * bw[i]) + sw[i], 0, W)); we = int(np.clip(np.ceil(np.float32(pw + 1) * bw[i]) + sw[i], 0, W))
                if he <= hs or we <= ws:
                    continue
                v = f[b[i], :, hs:he, ws:we].reshape(C, -1)
                tied += int(((v == v.max(axis=1, keepdims=True)).sum(axis=1) > 1).sum())
                total += C
    assert total > 0 and tied > 0.5 * total


def test_every_crop_case_reaches_its_branch():
    for name, c in LC.CROP_CASES.items():
        N, C, H, W = c["shape"]
        R, oh, ow = c["R"], c["oh"], c["ow"]
        path = crop_backward_path(N, C, H, W, R, oh, ow)
        if c["branch"] in ("nhwc", "declined"):
            assert path == c["branch"], name
        else:
            assert path == "scalar", name
        if name in ("c260", "c300"):
            assert C > 256 and C % 256
        if c["branch"] == "scalar":
            assert ceil_div(C, crop_c_per_cta(C, R * oh * ow)) > 1
        if c["branch"] == "r%n":
            assert R % N and (R - 1) // (R // N) == N           # the last RoI's image index is N: no image
    assert crop_backward_path(1, 256, 30, 40, 16, 14, 14) == "nhwc"       # 14 x 14 x 260 x 4 B = 203 840 B fits


def test_crop_affine_grids_sample_inside_the_map():
    """The affine grids of the BASELINE configs are those of whole RoIs: (y, x) in [-1, 1] up to the RoI clipping."""
    for name in ("cfg1", "cfg2"):
        c = LC.CROP_CASES[name]
        g = LC.crop_grid(c)
        assert g.shape == (c["R"], c["oh"], c["ow"], 2) and g.dtype == np.float32
        assert np.isfinite(g).all() and np.mean(np.abs(g) <= 1.0) > 0.5


def _pool_scatter_check(f, r, shape, PH, PW, s, dy):
    _, arg = O.roi_pool_forward(f, r, PH, PW, s)
    ref = O.roi_pool_backward(dy, arg, r, shape, PH, PW, s)
    got = pool_backward_scatter(dy, arg, r, shape, PH, PW, s)
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))
    return ref


@pytest.mark.parametrize("name", sorted(RC.ROI_CASES) + ["cfg1", "pileup", "ties"])
def test_pool_backward_scatter_restatement_equals_the_oracle(name):
    if name in RC.ROI_CASES:
        c, f, r, dy = RC.roi_case(name)
        _pool_scatter_check(f, r, c["shape"], c["P"], c["P"], c["scale"], dy)
    elif name == "pileup":              # 1400 RoIs piled on a 20 x 24 map: up to hundreds of addends per cell, in order
        shape = (2, 3, 20, 24)
        f = S.make_features(shape)
        r = S.make_rois(1400, shape, 0.25, seed=2, min_size=40, max_size=96)
        dy = np.random.RandomState(1).standard_normal((1400, 3, 3, 3)).astype(np.float32)
        ref = _pool_scatter_check(f, r, shape, 3, 3, 0.25, dy)
        assert np.count_nonzero(ref) > 0
    else:
        c = LC.POOL_LEGACY_CASES[name]
        f, r, dy = LC.roi_case(c)
        _pool_scatter_check(f, r, c["shape"], c["PH"], c["PW"], c["scale"], dy)


def test_golden_covers_the_recorded_cases():
    g = np.load(GOLDEN_FILE)
    for name, c in LC.POOL_LEGACY_CASES.items():
        if c["golden"]:
            for k in ("legacy_out_sha256", "legacy_dx_idx", "legacy_dx", "pool_out_sha256", "pool_argmax_sha256",
                      "pool_argmax_idx", "pool_argmax", "pool_dx_sha256", "pool_dx_idx", "pool_dx"):
                assert g["pl/%s/%s" % (name, k)].size > 0
    for name, c in LC.CROP_CASES.items():
        if c["golden"]:
            for k in ("out_sha256", "out_idx", "out", "grad_img_idx", "grad_img", "grad_grid_nonzero"):
                assert g["crop/%s/%s" % (name, k)].size > 0


# ---------------------------------------------------------------------------------------------- GPU
def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


_golden = {}


def golden(prefix):
    if not _golden:
        _golden.update(np.load(GOLDEN_FILE))
    return {k[len(prefix):]: v for k, v in _golden.items() if k.startswith(prefix)}


def with_bad_rois(N, r, dy):
    """The case's RoIs + one with batch index N + 2 and one with -1 (and two rows of dY for them); returns rois, dy and the
    index of the valid rows."""
    extra = r[:2].copy()
    extra[0, 0] = N + 2
    extra[1, 0] = -1
    rois = np.concatenate([r, extra]).astype(np.float32)
    dy = np.concatenate([dy, np.random.RandomState(9).standard_normal((2,) + dy.shape[1:]).astype(np.float32)])
    return rois, dy, np.arange(r.shape[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", PL_NAMES)
def test_pool_and_legacy_vs_oracle_and_reference(name):
    from detectron.pytorch_b200 import ops
    c = LC.POOL_LEGACY_CASES[name]
    N, C, H, W = shape = c["shape"]
    PH, PW, s = c["PH"], c["PW"], c["scale"]
    f, r, dy = LC.roi_case(c)
    rois, dy, good = with_bad_rois(N, r, dy)
    R0 = r.shape[0]

    # ---- RoIPool: output, argmax and dX bit-exact; the bad-batch rows give 0 / -1 and nothing to dX
    fn = RoIPoolFunction(PH, PW, s)
    F = dev(f).requires_grad_(True)
    pout = fn(F, dev(rois))
    pout.backward(dev(dy))
    pout, parg, pdx = pout.detach().cpu().numpy(), fn.argmax.cpu().numpy(), F.grad.cpu().numpy()
    o_out, o_arg = O.roi_pool_forward(f, r, PH, PW, s)
    assert np.array_equal(pout[:R0], o_out) and not np.any(pout[R0:])
    assert np.array_equal(parg[:R0], o_arg) and np.all(parg[R0:] == -1)
    ref_pdx = pool_backward_reference(dy[good], o_arg, r, shape, PH, PW, s)
    assert np.array_equal(pdx, ref_pdx)
    # run to run: the backward has no atomics, every cell sums in the reference's order
    again = ops.roi_pool_backward(dev(dy), fn.argmax, dev(rois), shape, PH, PW, s).cpu().numpy()
    assert np.array_equal(again.view(np.int32), pdx.view(np.int32))

    # ---- legacy RoIAlign: forward bit-exact (NaN where the oracle has NaN), dX within 1e-5 of the fp64 oracle
    LF = dev(f).requires_grad_(True)
    lout = LegacyRoIAlignFunction(PH, PW, s)(LF, dev(rois))
    lout.backward(dev(dy))
    lout, ldx = lout.detach().cpu().numpy(), LF.grad.cpu().numpy()
    ref = O.roi_align_legacy_forward(f, r, PH, PW, s)
    assert np.array_equal(lout[:R0], ref, equal_nan=True) and not np.any(lout[R0:])
    assert np.any(np.isnan(ref)) == (PH == 1 or PW == 1)        # P - 1 = 0: the reference's lattice divides by zero
    np.testing.assert_allclose(ldx, O.roi_align_legacy_backward(dy[good], r, shape, PH, PW, s, acc64=True), **GRAD_TOL)

    # ---- the reference kernels on an H100 (tests/golden/make_golden_legacy_pool_crop.py)
    if c["golden"]:
        g = golden("pl/%s/" % name)
        assert LC.digest(lout[:R0]) == str(g["legacy_out_sha256"])
        np.testing.assert_allclose(ldx.reshape(-1)[g["legacy_dx_idx"]], g["legacy_dx"], **GRAD_TOL)
        assert LC.digest(pout[:R0]) == str(g["pool_out_sha256"])
        assert np.array_equal(parg[:R0].reshape(-1)[g["pool_argmax_idx"]], g["pool_argmax"])
        assert LC.digest(parg[:R0]) == str(g["pool_argmax_sha256"])
        assert np.array_equal(pdx.reshape(-1)[g["pool_dx_idx"]], g["pool_dx"])
        assert LC.digest(pdx) == str(g["pool_dx_sha256"])


def sentinel_buffer(n):
    """n float32 elements between two guard bands of GUARD elements, every one holding the NaN bit pattern SENTINEL;
    returns the int32 buffer and the float32 view of its middle."""
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(torch.float32)


def assert_guards_intact(buf, n):
    assert bool((buf[:GUARD] == SENTINEL).all()), "a kernel wrote before the start of its buffer"
    assert bool((buf[GUARD + n:] == SENTINEL).all()), "a kernel wrote past the end of its buffer"


@pytest.mark.gpu
@pytest.mark.parametrize("name", MAP_NAMES)
def test_legacy_one_row_and_one_column_maps_stay_inside_their_tensors(name):
    """Legacy RoIAlign on 1 x W, H x 1, 1 x 1 and 2 x 2 maps through the C entry points, with the features and dX in the
    middle of NaN-sentinel buffers: a read outside the features would bring a NaN into the output, a write outside dX
    would change a guard element.  Values equal the (clamped) oracle; bad batch indices give zeros and no gradient."""
    from detectron.pytorch_b200 import _lib
    c = LC.LEGACY_MAP_CASES[name]
    N, C, H, W = shape = c["shape"]
    PH, PW, s = c["PH"], c["PW"], c["scale"]
    f, r, dy = LC.roi_case(c)
    rois, dy, good = with_bad_rois(N, r, dy)
    R, R0 = rois.shape[0], r.shape[0]
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    n_in, n_out = N * C * H * W, R * C * PH * PW
    in_buf, feats = sentinel_buffer(n_in)
    feats.copy_(dev(f).reshape(-1))
    out_buf, out = sentinel_buffer(n_out)
    Rt = dev(rois)
    _lib.check(lib.b200_roi_align_legacy_forward(feats.data_ptr(), s, N, R, H, W, C, PH, PW, Rt.data_ptr(), out.data_ptr(),
                                                 stream), "legacy forward")
    DY = dev(dy)
    dx_buf, dx = sentinel_buffer(n_in)
    _lib.check(lib.b200_roi_align_legacy_backward(DY.data_ptr(), s, N, R, H, W, C, PH, PW, Rt.data_ptr(), dx.data_ptr(),
                                                  stream), "legacy backward")
    torch.cuda.synchronize()
    assert_guards_intact(in_buf, n_in)
    assert_guards_intact(out_buf, n_out)
    assert_guards_intact(dx_buf, n_in)
    got = out.cpu().numpy().reshape(R, C, PH, PW)
    ref = O.roi_align_legacy_forward(f, r, PH, PW, s)
    assert not np.any(np.isnan(got)), "an output read a guard element (or was never written)"
    assert np.array_equal(got[:R0], ref) and not np.any(got[R0:])
    assert np.count_nonzero(ref) > 0.2 * ref.size
    if H == 1 and W == 1:                    # every tap is the one cell and the weights sum to 1
        b = r[:, 0].astype(int)
        cell = np.broadcast_to(f[b, :, 0, 0][:, :, None, None], ref.shape)
        hit = ref != 0
        np.testing.assert_allclose(ref[hit], cell[hit], rtol=1e-6, atol=0)
    gdx = dx.cpu().numpy().reshape(shape)
    ref_dx = O.roi_align_legacy_backward(dy[good], r, shape, PH, PW, s, acc64=True)
    np.testing.assert_allclose(gdx, ref_dx, **GRAD_TOL)
    assert np.count_nonzero(ref_dx) > 0
    # the gradient is conserved: every sample puts weights summing to 1 on cells of its own plane
    read = legacy_taps(r, s, PH, PW, H, W, clamped=True)[0]
    total = np.einsum("rchw,rhw->", dy[good].astype(np.float64), read.astype(np.float64))
    assert abs(float(gdx.astype(np.float64).sum()) - total) <= 1e-4 * max(1.0, abs(total))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CROP_NAMES)
def test_roi_crop_vs_oracle_and_reference(name, lib_option):
    """RoICrop forward bit-exact and image gradient within 1e-5 of the fp64 oracle; the launch counter shows which backward
    ran (NHWC scatter + transpose: 2, scalar kernel: 1); RoIs whose image index reaches N give zeros and no gradient."""
    from detectron.pytorch_b200 import _lib, ops
    c = LC.CROP_CASES[name]
    N, C, H, W = shape = c["shape"]
    img, grid, go = LC.crop_case(c)
    R = c["R"]
    valid = (R // N) * N                                   # RoI b reads image b / (R / N): the last R % N have none
    out = RoICropFunction()(dev(img), dev(grid)).cpu().numpy()
    ref = O.roi_crop_forward(img, grid[:valid])
    assert np.array_equal(out[:valid], ref) and not np.any(out[valid:])
    before = _lib.launch_count()
    gi, gg = ops.roi_crop_backward(dev(go), dev(grid), shape)
    launches = _lib.launch_count() - before
    assert launches == (2 if c["branch"] == "nhwc" else 1), "%s backward: %d launches" % (name, launches)
    gi = gi.cpu().numpy()
    ref_gi = O.roi_crop_backward(go[:valid], grid[:valid], shape, acc64=True)
    np.testing.assert_allclose(gi, ref_gi, **GRAD_TOL)
    assert np.count_nonzero(ref_gi) > 0 and torch.count_nonzero(gg) == 0
    if c["branch"] == "nhwc":                              # A/B: the scalar-atomic kernel forced
        lib_option("B200_ROI_ALIGN_BWD_PATH", "generic")
        before = _lib.launch_count()
        gi2, _ = ops.roi_crop_backward(dev(go), dev(grid), shape)
        assert _lib.launch_count() - before == 1
        np.testing.assert_allclose(gi2.cpu().numpy(), ref_gi, **GRAD_TOL)
    if c["golden"]:
        g = golden("crop/%s/" % name)
        assert LC.digest(out) == str(g["out_sha256"])
        assert np.array_equal(out.reshape(-1)[g["out_idx"]], g["out"])
        np.testing.assert_allclose(gi.reshape(-1)[g["grad_img_idx"]], g["grad_img"], **GRAD_TOL)
        assert int(g["grad_grid_nonzero"]) == 0
