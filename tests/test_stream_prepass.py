"""GPU tests of the streaming-strip forward's prepass (roi_align_stream.cu: clear, one prepass kernel with a grid barrier,
main kernel launched as its programmatic dependent) at the edges of its launch geometry, each bit-exact against the generic
kernel: more RoIs than one resident prepass grid holds (the grid loops over them), a single RoI, a workspace one byte
short of the queried size (the call declines to the generic kernel), and the FPN pyramid levels of an 800 x 1333 image
through single-level calls on the streaming path.

The RoIs are kept small enough (at most 64 feature cells a side) that every bin's samples are resident together: no bin
is cut into partial sums, so the streaming path computes every element as the generic kernel does, bit for bit.
"""
import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import _lib, synthetic as S

pytestmark = pytest.mark.gpu

STREAM_LAUNCHES = 3                                           # clear + prepass + main
GENERIC_LAUNCHES = 1


def _forward(f, r, P, scale, sr, ws_bytes=None):
    """One b200_roi_align_forward_ws call on a garbage-filled workspace of ws_bytes (default: the queried size).
    Returns (output, launches)."""
    lib = _lib.load()
    N, C, H, W = f.shape
    R = r.shape[0]
    if ws_bytes is None:
        ws_bytes = int(lib.b200_roi_align_workspace_bytes(N, R, H, W, P, P, sr))
    ws = torch.randint(0, 256, (max(ws_bytes, 1),), dtype=torch.uint8, device="cuda")
    F = torch.from_numpy(np.ascontiguousarray(f)).cuda()
    Rt = torch.from_numpy(np.ascontiguousarray(r)).cuda()
    out = torch.empty((R, C, P, P), dtype=torch.float32, device="cuda")
    before = _lib.launch_count()
    _lib.check(lib.b200_roi_align_forward_ws(F.data_ptr(), scale, N, R, H, W, C, P, P, sr, Rt.data_ptr(), out.data_ptr(),
                                             ws.data_ptr() if ws_bytes else None, ws_bytes, torch.cuda.current_stream().cuda_stream),
               "forward")
    launches = _lib.launch_count() - before
    return out.cpu().numpy(), launches


def _generic(f, r, P, scale, sr, lib_option):
    lib_option("B200_ROI_ALIGN_PATH", "generic")
    out, launches = _forward(f, r, P, scale, sr)
    assert launches == GENERIC_LAUNCHES
    lib_option("B200_ROI_ALIGN_PATH", "stream")
    return out


def _small_rois(n, shape, scale, seed):
    return S.make_rois(n, shape, scale, seed=seed, min_size=4.0 / scale, max_size=64.0 / scale)


def test_stream_more_rois_than_one_resident_prepass_grid(lib_option):
    """4000 RoIs: a prepass CTA has 128 threads, so at most 2048 / 128 = 16 of them fit on one SM, 2112 on 132 SMs -- the
    prepass grid is capped there and every CTA takes several RoIs, before and after the grid barrier."""
    shape, scale, P, sr = (2, 64, 60, 100), 1.0 / 8, 7, 2
    f = S.make_features(shape, seed=11)
    r = _small_rois(4000, shape, scale, seed=12)
    assert r.shape[0] > 16 * 132
    ref = _generic(f, r, P, scale, sr, lib_option)
    out, launches = _forward(f, r, P, scale, sr)
    assert launches == STREAM_LAUNCHES
    assert np.array_equal(out, ref)


@pytest.mark.parametrize("sr", [1, 2])
def test_stream_single_roi(sr, lib_option):
    """R = 1: a one-CTA prepass grid computes every piece boundary of the 132 main-kernel CTAs, most of them empty."""
    shape, scale, P = (1, 96, 50, 84), 1.0 / 16, 7
    f = S.make_features(shape, seed=13)
    r = np.array([[0, 100.0, 120.0, 700.0, 500.0]], dtype=np.float32)
    ref = _generic(f, r, P, scale, sr, lib_option)
    out, launches = _forward(f, r, P, scale, sr)
    assert launches == STREAM_LAUNCHES
    assert np.array_equal(out, ref)


def test_stream_workspace_one_byte_short_declines(lib_option):
    """A workspace one byte smaller than b200_roi_align_workspace_bytes returns: the streaming path declines and the call
    falls back to the generic kernel (one launch), with its result."""
    lib_option("B200_ROI_ALIGN_PATH", "stream")
    shape, scale, P, sr = (1, 64, 50, 84), 1.0 / 16, 7, 2
    f = S.make_features(shape, seed=14)
    r = _small_rois(200, shape, scale, seed=15)
    need = int(_lib.load().b200_roi_align_workspace_bytes(1, r.shape[0], 50, 84, P, P, sr))
    assert need > 0
    _, launches = _forward(f, r, P, scale, sr, ws_bytes=need)
    assert launches == STREAM_LAUNCHES
    ref = _generic(f, r, P, scale, sr, lib_option)
    out, launches = _forward(f, r, P, scale, sr, ws_bytes=need - 1)
    assert launches == GENERIC_LAUNCHES
    assert np.array_equal(out, ref)


FPN_LEVELS = {                                                # an 800 x 1333 image pair: P2 .. P5 (DESIGN.md 4.1)
    "p2": ((2, 256, 200, 336), 1.0 / 4, 1000),
    "p3": ((2, 256, 100, 168), 1.0 / 8, 1000),
    "p4": ((2, 256, 50, 84), 1.0 / 16, 1000),
    "p5": ((2, 256, 25, 42), 1.0 / 32, 500),
}


@pytest.mark.parametrize("P", [7, 14], ids=["box", "mask"])
@pytest.mark.parametrize("level", sorted(FPN_LEVELS))
def test_stream_fpn_levels(level, P, lib_option):
    shape, scale, n = FPN_LEVELS[level]
    if P == 14:
        n = 256
    f = S.make_features(shape, seed=16)
    r = _small_rois(n, shape, scale, seed=17)
    ref = _generic(f, r, P, scale, 2, lib_option)
    out, launches = _forward(f, r, P, scale, 2)
    assert launches == STREAM_LAUNCHES
    assert np.array_equal(out, ref)
