"""RoIAlign at the geometry where index arithmetic and path choice go wrong (tests/geometry_cases.py).

CPU part (no marker): the oracle (oracle/roi_ops_oracle.c), which the GPU part trusts, against torchvision at every case:
the unfused oracle bit for bit, the fused oracle within 1e-4, the fp64 backward within 2e-4 of torchvision's autograd.

GPU part (`-m gpu`):
  * every case under each forced forward path (generic, tiled, stream, quad) and each forced backward path (generic, nhwc,
    rows: 4 channels per lane at P = 7 and C % 128 == 0, else 2).  The launch counter proves which path ran: a case a path
    must accept runs it (forward: stream 3 launches, quad 2, tiled 2; backward: rows 2, nhwc 2), a case it must decline falls back to the
    generic kernel (1 launch).  Values against the oracle with the tolerances of test_gpu_parity.py (generic forward
    bit-exact; tiled / stream / quad forward 1e-6; backward 1e-5 against fp64), and on the rectangular-bin cases against
    the reference kernel's sm_90a build (tests/golden/roi_align_geometry_sm90a.npz);
  * the C entry points with NaN-sentinel output buffers and a guard band behind them: every element must be written,
    nothing past the end, and an indexed call must leave the rows it does not map alone.  RoIs with an out-of-range batch
    index and RoIs outside the map come back as exact zeros;
  * RoIAlignFPNFunction (restore index through the indexed entry points) on the row-stationary backward, the tiled forward,
    pyramids whose TMA-staged and cp.async levels interleave, 5 / 6 / 7 levels, a 1 x 1 level, empty levels and a level
    whose RoIs all have a bad batch index.
"""
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import synthetic as S
from oracle import cpu as O
from tests import geometry_cases as GC

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
GRAD_TOL = dict(rtol=1e-5, atol=1e-5)
NAMES = sorted(GC.GEOMETRY_CASES)
FWD_LAUNCHES = {"generic": 1, "tiled": 2, "stream": 3, "quad": 2}     # prepass + main (+ fill for stream); memsets are not counted
BWD_LAUNCHES = {"generic": 1, "nhwc": 2, "rows": 2}
SENTINEL = 0x7FC0DEAD                 # a quiet NaN with a payload no kernel produces
GUARD = 1024                          # elements behind every output buffer that must stay untouched

_cache = {}


def oracle_case(name):
    """(case, features, rois, dy, oracle forward, oracle backward in fp64), computed once per case."""
    if name not in _cache:
        c, f, r, dy = GC.geometry_case(name)
        PH, PW, s, sr = c["PH"], c["PW"], c["scale"], c["sr"]
        _cache[name] = (c, f, r, dy, O.roi_align_forward(f, r, PH, PW, s, sr),
                        O.roi_align_backward(dy, r, c["shape"], PH, PW, s, sr, acc64=True))
    return _cache[name]


# ---------------------------------------------------------------------------------------------- CPU: pin the oracle
@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_torchvision_at_geometry_case(name):
    import torchvision
    c, f, r, dy, ref, ref_dx = oracle_case(name)
    PH, PW, s, sr = c["PH"], c["PW"], c["scale"], c["sr"]
    O.set_fused(False)
    try:
        unfused = O.roi_align_forward(f, r, PH, PW, s, sr)
    finally:
        O.set_fused(True)
    ft = torch.from_numpy(f).requires_grad_(True)
    tv = torchvision.ops.roi_align(ft, torch.from_numpy(r), (PH, PW), s, sr, aligned=False)
    assert np.array_equal(unfused, tv.detach().numpy())                  # the index and weight logic, bit for bit
    np.testing.assert_allclose(ref, tv.detach().numpy(), rtol=0, atol=1e-4)      # FMA contraction moves samples by <= 1 ulp
    tv.backward(torch.from_numpy(dy))
    # torchvision accumulates in fp32: where every tap piles onto a few cells (the 1 x 1 map: |dX| ~ 50) its own rounding error
    # grows with |dX|, hence the relative term
    np.testing.assert_allclose(ref_dx, ft.grad.numpy(), rtol=1e-5, atol=2e-4)


# ---------------------------------------------------------------------------------------------- GPU
def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def assert_fwd_matches(out, ref, path):
    """As test_gpu_parity.assert_fwd_matches: generic bit-exact; tiled / stream / quad within 1e-6 (bins cut into partial sums)."""
    if path == "generic":
        assert np.array_equal(out, ref)
        return
    np.testing.assert_allclose(out, ref, rtol=1e-6, atol=1e-6)
    assert np.mean(out == ref) > (0.5 if path == "tiled" else 0.9)


_golden = {}


def golden():
    if not _golden:
        _golden.update(np.load(os.path.join(GOLDEN, "roi_align_geometry_sm90a.npz")))
    return _golden


def test_geometry_golden_covers_the_rectangular_cases():
    g = golden()
    for name in GC.RECT_CASES:
        for k in ("out_idx", "out", "dx_idx", "dx"):
            assert g[name + "/" + k].size > 0


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["generic", "tiled", "stream", "quad"])
@pytest.mark.parametrize("name", NAMES)
def test_forward_forced_path(name, path, lib_option):
    """Forced forward path: runs where the case table says it accepts the geometry, falls back to the generic kernel (one
    launch) where it declines; the values match the oracle (and the reference kernel on the rectangular cases)."""
    from detectron.pytorch_b200 import _lib, ops
    c, f, r, _, ref, _ = oracle_case(name)
    PH, PW, s, sr = c["PH"], c["PW"], c["scale"], c["sr"]
    lib_option("B200_ROI_ALIGN_PATH", path)
    F, Rt = dev(f), dev(r)
    before = _lib.launch_count()
    out = ops.roi_align_forward(F, Rt, PH, PW, s, sr)
    launches = _lib.launch_count() - before
    ran = path if path in c["fwd"] else "generic"
    assert launches == FWD_LAUNCHES[ran], "%s forward on %s: %d launches, expected %s" % (path, name, launches, ran)
    got = out.cpu().numpy()
    assert_fwd_matches(got, ref, ran)
    if ran in ("generic", "stream", "quad"):              # at most two partial sums per element: order independent
        assert torch.equal(ops.roi_align_forward(F, Rt, PH, PW, s, sr), out)
    if name in GC.RECT_CASES:
        g = golden()
        np.testing.assert_allclose(got.reshape(-1)[g[name + "/out_idx"]], g[name + "/out"], rtol=1e-6, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["generic", "nhwc", "rows"])
@pytest.mark.parametrize("name", NAMES)
def test_backward_forced_path(name, path, lib_option):
    from detectron.pytorch_b200 import _lib, ops
    c, f, r, dy, _, ref_dx = oracle_case(name)
    PH, PW, s, sr = c["PH"], c["PW"], c["scale"], c["sr"]
    lib_option("B200_ROI_ALIGN_BWD_PATH", path)
    DY, Rt = dev(dy), dev(r)
    before = _lib.launch_count()
    dx = ops.roi_align_backward(DY, Rt, c["shape"], PH, PW, s, sr)
    launches = _lib.launch_count() - before
    ran = path if path in c["bwd"] else "generic"
    assert launches == BWD_LAUNCHES[ran], "%s backward on %s: %d launches, expected %s" % (path, name, launches, ran)
    got = dx.cpu().numpy()
    # a pile-up is only good to ~n eps sum|terms| in fp32 (ours and the reference's atomics alike): the tolerance of
    # test_gpu_parity.py::test_roi_align_backward_rows_path_row_overflow
    np.testing.assert_allclose(got, ref_dx, **(dict(rtol=1e-4, atol=1e-4) if c["pileup"] else GRAD_TOL))
    if name in GC.RECT_CASES:
        g = golden()
        np.testing.assert_allclose(got.reshape(-1)[g[name + "/dx_idx"]], g[name + "/dx"], **GRAD_TOL)


# ------------------------------------------------------------------ C entry points: sentinel-filled outputs, guard band
SENTINEL_FWD_CASES = ("rect_7x14_sr2", "rect_16x1_sr1", "p31_sr1", "p8_sr4", "map_h2_w33", "c33", "keys_n8_h800", "cols_n4_w2000")
SENTINEL_BWD_CASES = ("rect_16x7_sr2", "rect_3x7_sr1", "rect_1x16_sr2", "map_h1_w65", "c128")


def sentinel_buffer(n):
    """n float32 elements + GUARD, every one holding the NaN bit pattern SENTINEL (int32 view returned)."""
    return torch.full((n + GUARD,), SENTINEL, dtype=torch.int32, device="cuda")


def assert_guard_intact(buf, n):
    assert bool((buf[n:] == SENTINEL).all()), "a kernel wrote past the end of its output"


def with_bad_rois(c, r):
    """The case's RoIs + one with batch index N + 2 and one with -1; returns rois, index of those two, index of the RoIs that
    lie entirely outside the map (make_edge_rois rows 3 and 4), and the RoIs with the bad indices replaced by 0."""
    N = c["shape"][0]
    extra = r[:2].copy()
    extra[0, 0] = N + 2
    extra[1, 0] = -1
    rois = np.concatenate([r, extra]).astype(np.float32)
    bad = np.array([len(r), len(r) + 1])
    outside = np.array([c["n_rois"] + 3, c["n_rois"] + 4])
    fixed = rois.copy()
    fixed[bad, 0] = 0
    return rois, bad, outside, fixed


def _ws(nbytes):
    t = torch.empty((max(int(nbytes), 1),), dtype=torch.uint8, device="cuda")
    return t, (t.data_ptr() if nbytes else None), int(nbytes)


@pytest.mark.gpu
@pytest.mark.parametrize("indexed", [False, True], ids=["ws", "indexed"])
@pytest.mark.parametrize("path", ["generic", "tiled", "stream", "quad"])
@pytest.mark.parametrize("name", SENTINEL_FWD_CASES)
def test_forward_writes_every_element_once_and_nothing_else(name, path, indexed, lib_option):
    from detectron.pytorch_b200 import _lib
    c, f, r, _, _, _ = oracle_case(name)
    N, C, H, W = c["shape"]
    PH, PW, s, sr = c["PH"], c["PW"], c["scale"], c["sr"]
    rois, bad, outside, fixed = with_bad_rois(c, r)
    ref = O.roi_align_forward(f, fixed, PH, PW, s, sr)
    ref[bad] = 0
    R = rois.shape[0]
    lib_option("B200_ROI_ALIGN_PATH", path)
    lib = _lib.load()
    keep_ws, ws_ptr, ws_bytes = _ws(lib.b200_roi_align_workspace_bytes(N, R, H, W, PH, PW, sr))
    F, Rt = dev(f), dev(rois)
    per_row = C * PH * PW
    R_out = 2 * R + 5 if indexed else R
    buf = sentinel_buffer(R_out * per_row)
    stream = torch.cuda.current_stream().cuda_stream
    before = _lib.launch_count()
    if indexed:
        rows = np.random.RandomState(7).choice(R_out, R, replace=False).astype(np.int32)
        Rows = dev(rows)
        st = lib.b200_roi_align_forward_indexed(F.data_ptr(), s, N, R, H, W, C, PH, PW, sr, Rt.data_ptr(), Rows.data_ptr(),
                                                buf.data_ptr(), ws_ptr, ws_bytes, stream)
    else:
        rows = np.arange(R, dtype=np.int32)
        st = lib.b200_roi_align_forward_ws(F.data_ptr(), s, N, R, H, W, C, PH, PW, sr, Rt.data_ptr(), buf.data_ptr(), ws_ptr,
                                           ws_bytes, stream)
    _lib.check(st, "forward")
    launches = _lib.launch_count() - before
    ran = path if path in c["fwd"] else "generic"
    assert launches == FWD_LAUNCHES[ran]
    torch.cuda.synchronize()
    assert_guard_intact(buf, R_out * per_row)
    bits = buf[:R_out * per_row].view(R_out, C, PH, PW).cpu().numpy()
    got = bits[rows].view(np.float32)
    assert not np.any(bits[rows] == SENTINEL), "an output element of a mapped row was never written"
    assert_fwd_matches(got, ref, ran)
    assert not np.any(got[bad]) and not np.any(got[outside]), "rows of bad-batch / outside RoIs must be exact zeros"
    unmapped = np.setdiff1d(np.arange(R_out), rows)
    assert np.all(bits[unmapped] == SENTINEL), "an indexed call wrote a row it does not map"


@pytest.mark.gpu
@pytest.mark.parametrize("indexed", [False, True], ids=["ws", "indexed"])
@pytest.mark.parametrize("name,axis", [("keys_n8_h800", 0), ("cols_n4_w2000", 1)])
def test_tiled_prepass_roi_spanning_more_than_32_tile_rows_or_columns(name, axis, indexed, lib_option):
    """Regression: the tiled forward's prepass kept the bin count of each tile row / column of a RoI in 32-entry shared
    arrays indexed by the offset from the RoI's first tile.  The whole-image RoI of an 800-row map spans 45 tile rows (18-row
    cores), the whole-width RoI of a 2000-column map 65 tile columns (31-column cores): the writes ran past the arrays,
    into the other axis' counts and the split-bin list, and 56 outputs of the 800-row case came back wrong (up to 0.7)."""
    from detectron.pytorch_b200 import _lib
    c, _, r, _, _, _ = oracle_case(name)
    lo = r[c["n_rois"], 2 - axis] * c["scale"]             # make_edge_rois row 0: the whole image
    hi = r[c["n_rois"], 4 - axis] * c["scale"]
    assert (hi - lo) > 33 * (18 if axis == 0 else 31)
    test_forward_writes_every_element_once_and_nothing_else(name, "tiled", indexed, lib_option)


@pytest.mark.gpu
@pytest.mark.parametrize("indexed", [False, True], ids=["ws", "indexed"])
@pytest.mark.parametrize("path", ["generic", "nhwc", "rows"])
@pytest.mark.parametrize("name", SENTINEL_BWD_CASES)
def test_backward_writes_every_element_once_and_nothing_else(name, path, indexed, lib_option):
    """dX in a sentinel-filled buffer: every element written (generic: memset + atomics; nhwc: transpose; rows: one store per
    element, no memset), nothing behind it.  The indexed call reads dY through top_rows: the rows it does not map hold NaN."""
    from detectron.pytorch_b200 import _lib
    c, f, r, dy, _, _ = oracle_case(name)
    N, C, H, W = c["shape"]
    PH, PW, s, sr = c["PH"], c["PW"], c["scale"], c["sr"]
    rois, bad, _, fixed = with_bad_rois(c, r)
    R = rois.shape[0]
    dy = np.concatenate([dy, np.random.RandomState(5).standard_normal((2,) + dy.shape[1:]).astype(np.float32)])
    dyr = dy.copy()
    dyr[bad] = 0                                           # RoIs with a bad batch index contribute nothing
    ref_dx = O.roi_align_backward(dyr, fixed, c["shape"], PH, PW, s, sr, acc64=True)
    lib_option("B200_ROI_ALIGN_BWD_PATH", path)
    lib = _lib.load()
    keep_ws, ws_ptr, ws_bytes = _ws(lib.b200_roi_align_backward_workspace_bytes(N, R, C, H, W, PH, PW, sr))
    Rt = dev(rois)
    n = N * C * H * W
    buf = sentinel_buffer(n)
    stream = torch.cuda.current_stream().cuda_stream
    before = _lib.launch_count()
    if indexed:
        R_out = 2 * R + 5
        rows = np.random.RandomState(8).choice(R_out, R, replace=False).astype(np.int32)
        big = np.full((R_out,) + dy.shape[1:], np.nan, np.float32)
        big[rows] = dy
        DY, Rows = dev(big), dev(rows)
        st = lib.b200_roi_align_backward_indexed(DY.data_ptr(), Rows.data_ptr(), s, N, R, H, W, C, PH, PW, sr, Rt.data_ptr(),
                                                 buf.data_ptr(), ws_ptr, ws_bytes, stream)
    else:
        DY = dev(dy)
        st = lib.b200_roi_align_backward_ws(DY.data_ptr(), s, N, R, H, W, C, PH, PW, sr, Rt.data_ptr(), buf.data_ptr(), ws_ptr,
                                            ws_bytes, stream)
    _lib.check(st, "backward")
    launches = _lib.launch_count() - before
    ran = path if path in c["bwd"] else "generic"
    assert launches == BWD_LAUNCHES[ran]
    torch.cuda.synchronize()
    assert_guard_intact(buf, n)
    bits = buf[:n].cpu().numpy()
    assert not np.any(bits == SENTINEL), "a dX element was never written"
    np.testing.assert_allclose(bits.view(np.float32).reshape(c["shape"]), ref_dx, **GRAD_TOL)


# ------------------------------------------------------------------ FPN: the restore index through the indexed entry points
def fpn_inputs(shapes, scales, counts, P, seed, lo=16.0, hi=256.0, bad_level=None):
    feats = [S.make_features(sh, seed=seed + i) for i, sh in enumerate(shapes)]
    rois = [S.make_rois(n, sh, sc, seed=seed + 10 + i, min_size=lo * 2 ** i, max_size=hi * 2 ** i).astype(np.float32) if n
            else np.zeros((0, 5), np.float32) for i, (n, sh, sc) in enumerate(zip(counts, shapes, scales))]
    if bad_level is not None:
        rois[bad_level][0::2, 0] = shapes[0][0] + 2
        rois[bad_level][1::2, 0] = -1
    rng = np.random.RandomState(seed)
    total = sum(counts)
    restore = rng.permutation(total).astype(np.int32)
    dy = rng.standard_normal((total, shapes[0][1], P, P)).astype(np.float32)
    return feats, rois, restore, dy


def fpn_oracle(feats, rois, scales, restore, dy, P, sr):
    """The reference flow on the CPU: per-level RoIAlign, concatenation, gather by the restore index; and each level's dX
    from the gradient rows its RoIs were moved to (bad batch index: zeros, no contribution)."""
    inv = np.argsort(restore)                              # concatenated position k lands on output row inv[k]
    parts, dxs, off = [], [], 0
    for f, r, sc in zip(feats, rois, scales):
        n = len(r)
        C = f.shape[1]
        if n == 0:
            parts.append(np.zeros((0, C, P, P), np.float32))
            dxs.append(np.zeros_like(f))
            continue
        bad = (r[:, 0] < 0) | (r[:, 0] >= f.shape[0])
        rr = r.copy()
        rr[bad, 0] = 0
        o = O.roi_align_forward(f, rr, P, P, sc, sr)
        o[bad] = 0
        parts.append(o)
        dyl = dy[inv[off:off + n]].copy()
        dyl[bad] = 0
        dxs.append(O.roi_align_backward(dyl, rr, f.shape, P, P, sc, sr, acc64=True))
        off += n
    return np.concatenate(parts)[restore], dxs


def fpn_run(feats, rois, scales, restore, dy, P, sr, backward=True):
    """RoIAlignFPNFunction forward (+ backward); returns out, level grads, forward launches, backward launches."""
    from detectron.pytorch_b200 import _lib
    from detectron.pytorch_b200.modeling.roi_xfrom.roi_align.functions.roi_align_fpn import RoIAlignFPNFunction
    F = [f if isinstance(f, torch.Tensor) else dev(f) for f in feats]
    if backward:
        F = [f.requires_grad_(True) for f in F]
    before = _lib.launch_count()
    out = RoIAlignFPNFunction(P, P, scales, sr)(F, [dev(r) for r in rois], restore)
    torch.cuda.synchronize()
    fwd = _lib.launch_count() - before
    grads, bwd = None, 0
    if backward:
        before = _lib.launch_count()
        out.backward(dev(dy))
        torch.cuda.synchronize()
        bwd = _lib.launch_count() - before
        grads = [f.grad.cpu().numpy() for f in F]
    return out.detach().cpu().numpy(), grads, fwd, bwd


def fpn_check(out, grads, ref, ref_dxs, exact=0.9):
    np.testing.assert_allclose(out, ref, rtol=1e-6, atol=1e-6)
    assert np.mean(out == ref) > exact
    if grads is not None:
        for g, rd in zip(grads, ref_dxs):
            np.testing.assert_allclose(g, rd, **GRAD_TOL)


def fpn_ws_bytes(shapes, counts, P, sr):
    import ctypes
    from detectron.pytorch_b200 import _lib
    live = [sh for sh, n in zip(shapes, counts) if n]
    hs = (ctypes.c_int * len(live))(*[sh[2] for sh in live])
    ws = (ctypes.c_int * len(live))(*[sh[3] for sh in live])
    return int(_lib.load().b200_roi_align_fpn_workspace_bytes(len(live), ctypes.cast(hs, ctypes.c_void_p), ctypes.cast(ws, ctypes.c_void_p),
                                                              shapes[0][0], sum(counts), P, P, sr))


FPN_SHAPES = [(2, 64, 40, 56), (2, 64, 20, 28), (2, 64, 10, 14), (2, 64, 5, 7)]
FPN_SCALES = [1.0 / 4, 1.0 / 8, 1.0 / 16, 1.0 / 32]


@pytest.mark.gpu
@pytest.mark.parametrize("P", [7, 14])
def test_fpn_restore_index_through_rows_backward(P, lib_option):
    """The row-stationary backward reads dY through row_map (the mask head at FPN P2 takes it in production)."""
    lib_option("B200_ROI_ALIGN_BWD_PATH", "rows")
    counts = [60, 30, 0, 9]
    feats, rois, restore, dy = fpn_inputs(FPN_SHAPES, FPN_SCALES, counts, P, seed=31)
    ref, ref_dxs = fpn_oracle(feats, rois, FPN_SCALES, restore, dy, P, 2)
    out, grads, _, bwd = fpn_run(feats, rois, FPN_SCALES, restore, dy, P, 2)
    assert bwd == 2 * 3                                    # tables + main per non-empty level
    fpn_check(out, grads, ref, ref_dxs)
    assert not np.any(grads[2])                            # the empty level


@pytest.mark.gpu
@pytest.mark.parametrize("P", [7, 14])
def test_fpn_restore_index_through_tiled_forward_and_nhwc_backward(P, lib_option):
    """The tiled forward with top_rows (per-level loop: the pyramid call runs the quad strips only) and the NHWC backward."""
    lib_option("B200_ROI_ALIGN_PATH", "tiled")
    lib_option("B200_ROI_ALIGN_BWD_PATH", "nhwc")
    counts = [60, 30, 0, 9]
    feats, rois, restore, dy = fpn_inputs(FPN_SHAPES, FPN_SCALES, counts, P, seed=32)
    assert fpn_ws_bytes(FPN_SHAPES, counts, P, 2) == 0
    ref, ref_dxs = fpn_oracle(feats, rois, FPN_SCALES, restore, dy, P, 2)
    out, grads, fwd, bwd = fpn_run(feats, rois, FPN_SCALES, restore, dy, P, 2)
    assert fwd == 2 * 3 and bwd == 2 * 3
    fpn_check(out, grads, ref, ref_dxs, exact=0.5)


@pytest.mark.gpu
def test_fpn_tma_and_cp_async_levels_interleave():
    """Widths 64, 42, 32, 10: TMA-staged (W % 4 == 0) and cp.async levels alternate -> four launch sequences of prep + main."""
    shapes = [(2, 32, 48, 64), (2, 32, 32, 42), (2, 32, 24, 32), (2, 32, 8, 10)]
    counts = [40, 30, 20, 10]
    feats, rois, restore, dy = fpn_inputs(shapes, FPN_SCALES, counts, 7, seed=33)
    assert fpn_ws_bytes(shapes, counts, 7, 2) > 0
    ref, ref_dxs = fpn_oracle(feats, rois, FPN_SCALES, restore, dy, 7, 2)
    out, grads, fwd, _ = fpn_run(feats, rois, FPN_SCALES, restore, dy, 7, 2)
    assert fwd == 2 * 4
    fpn_check(out, grads, ref, ref_dxs)


@pytest.mark.gpu
def test_fpn_level_with_misaligned_base_takes_cp_async():
    """A 64-wide level whose base is 4 bytes off 16-byte alignment (a contiguous view into a larger buffer) cannot be staged by
    TMA: the pyramid splits into three launch sequences (TMA | cp.async | TMA)."""
    shapes = [(2, 32, 40, 64), (2, 32, 32, 64), (2, 32, 16, 32)]
    scales = FPN_SCALES[:3]
    counts = [30, 25, 15]
    feats, rois, restore, dy = fpn_inputs(shapes, scales, counts, 7, seed=34)
    big = torch.empty((feats[1].size + 1,), dtype=torch.float32, device="cuda")
    view = big[1:].view(shapes[1])
    view.copy_(dev(feats[1]))
    assert view.is_contiguous() and view.data_ptr() % 16 == 4
    ref, _ = fpn_oracle(feats, rois, scales, restore, dy, 7, 2)
    out, _, fwd, _ = fpn_run([feats[0], view, feats[2]], rois, scales, restore, dy, 7, 2, backward=False)
    assert fwd == 2 * 3
    fpn_check(out, None, ref, None)


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [5, 6, 7])
def test_fpn_five_six_levels_fused_seven_per_level(levels):
    """Up to six levels run as one launch sequence; a seventh sizes no pyramid workspace and takes the per-level loop."""
    shapes = [(2, 32, 64, 96), (2, 32, 32, 48), (2, 32, 16, 24), (2, 32, 8, 12), (2, 32, 4, 8), (2, 32, 2, 4), (2, 32, 2, 4)][:levels]
    scales = [1.0 / 2 ** (i + 2) for i in range(levels)]
    counts = [24, 20, 16, 12, 8, 6, 4][:levels]
    feats, rois, restore, dy = fpn_inputs(shapes, scales, counts, 7, seed=35, lo=8.0, hi=128.0)
    ws = fpn_ws_bytes(shapes, counts, 7, 2)
    ref, ref_dxs = fpn_oracle(feats, rois, scales, restore, dy, 7, 2)
    out, grads, fwd, _ = fpn_run(feats, rois, scales, restore, dy, 7, 2)
    if levels <= 6:
        assert ws > 0 and fwd == 2
    else:
        assert ws == 0
    fpn_check(out, grads, ref, ref_dxs)


@pytest.mark.gpu
def test_fpn_one_by_one_top_level_takes_per_level_loop():
    """Stream and quad strips need maps of at least 2 x 2: a 1 x 1 level sends the whole pyramid to the per-level loop."""
    shapes = [(2, 32, 32, 48), (2, 32, 16, 24), (2, 32, 1, 1)]
    scales = FPN_SCALES[:3]
    counts = [20, 12, 6]
    feats, rois, restore, dy = fpn_inputs(shapes, scales, counts, 7, seed=36)
    assert fpn_ws_bytes(shapes, counts, 7, 2) == 0
    ref, ref_dxs = fpn_oracle(feats, rois, scales, restore, dy, 7, 2)
    out, grads, _, _ = fpn_run(feats, rois, scales, restore, dy, 7, 2)
    fpn_check(out, grads, ref, ref_dxs)


@pytest.mark.gpu
def test_fpn_empty_levels_between_non_empty_ones():
    shapes = [(2, 32, 40, 56), (2, 32, 20, 28), (2, 32, 10, 14), (2, 32, 5, 7), (2, 32, 3, 4)]
    scales = [1.0 / 2 ** (i + 2) for i in range(5)]
    counts = [25, 0, 15, 0, 6]
    feats, rois, restore, dy = fpn_inputs(shapes, scales, counts, 7, seed=37)
    ref, ref_dxs = fpn_oracle(feats, rois, scales, restore, dy, 7, 2)
    out, grads, fwd, _ = fpn_run(feats, rois, scales, restore, dy, 7, 2)
    fpn_check(out, grads, ref, ref_dxs)
    assert not np.any(grads[1]) and not np.any(grads[3])


@pytest.mark.gpu
@pytest.mark.parametrize("bwd", ["auto", "generic", "nhwc", "rows"])
def test_fpn_level_whose_rois_all_have_a_bad_batch_index(bwd, lib_option):
    """Every RoI of level 1 has batch index N + 2 or -1: its rows come back as zeros and its dX is exactly zero."""
    if bwd != "auto":
        lib_option("B200_ROI_ALIGN_BWD_PATH", bwd)
    counts = [40, 12, 8, 5]
    feats, rois, restore, dy = fpn_inputs(FPN_SHAPES, FPN_SCALES, counts, 7, seed=38, bad_level=1)
    ref, ref_dxs = fpn_oracle(feats, rois, FPN_SCALES, restore, dy, 7, 2)
    out, grads, _, _ = fpn_run(feats, rois, FPN_SCALES, restore, dy, 7, 2)
    fpn_check(out, grads, ref, ref_dxs)
    assert not np.any(out[np.argsort(restore)[40:52]])
    assert not np.any(grads[1])
