"""GPU tests of the streaming-strip forward's output staging (roi_align_stream.cu): the main kernel stores every bin's result
into its output row laid out (bin, channel) and, after a grid barrier, transposes each row in place to (channel, bin) through
shared memory.  A call whose row block does not fit the kernel's shared memory declines.

Each case runs the indexed entry point into a NaN-sentinel buffer of 2R + 5 rows (the rows it does not map must stay untouched)
and checks the launch count of the path that ran against the generic kernel.
"""
import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import _lib, synthetic as S

pytestmark = pytest.mark.gpu

STREAM_LAUNCHES = 3                                           # clear + prepass + main (the transpose is the main kernel's tail)
GENERIC_LAUNCHES = 1
SENTINEL = 0x7FC0DEAD                                         # a quiet NaN with a payload no kernel produces


def _indexed(f, r, P, scale, sr, rows, n_out):
    """b200_roi_align_forward_indexed into a sentinel buffer of n_out rows.  Returns (rows as int32 bits, launches)."""
    lib = _lib.load()
    N, C, H, W = f.shape
    R = r.shape[0]
    ws_bytes = int(lib.b200_roi_align_workspace_bytes(N, R, H, W, P, P, sr))
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device="cuda")
    F = torch.from_numpy(np.ascontiguousarray(f)).cuda()
    Rt = torch.from_numpy(np.ascontiguousarray(r)).cuda()
    Rows = torch.from_numpy(rows).cuda()
    buf = torch.full((n_out * C * P * P,), SENTINEL, dtype=torch.int32, device="cuda")
    before = _lib.launch_count()
    _lib.check(lib.b200_roi_align_forward_indexed(F.data_ptr(), scale, N, R, H, W, C, P, P, sr, Rt.data_ptr(), Rows.data_ptr(),
                                                  buf.data_ptr(), ws.data_ptr() if ws_bytes else None, ws_bytes,
                                                  torch.cuda.current_stream().cuda_stream), "forward")
    launches = _lib.launch_count() - before
    return buf.view(n_out, C, P, P).cpu().numpy(), launches


def _run(f, r, P, scale, sr, lib_option, launches_expected):
    """(stream-path output, generic output) of the mapped rows; checks the launch counts and the unmapped rows."""
    R = r.shape[0]
    n_out = 2 * R + 5
    rows = np.random.RandomState(7).choice(n_out, R, replace=False).astype(np.int32)
    unmapped = np.setdiff1d(np.arange(n_out), rows)
    lib_option("B200_ROI_ALIGN_PATH", "generic")
    ref, launches = _indexed(f, r, P, scale, sr, rows, n_out)
    assert launches == GENERIC_LAUNCHES
    lib_option("B200_ROI_ALIGN_PATH", "stream")
    bits, launches = _indexed(f, r, P, scale, sr, rows, n_out)
    assert launches == launches_expected
    assert np.all(bits[unmapped] == SENTINEL), "an indexed call wrote a row it does not map"
    assert not np.any(bits[rows] == SENTINEL), "an output element of a mapped row was never written"
    return bits[rows].view(np.float32), ref[rows].view(np.float32)


def _small_rois(n, shape, scale, seed):
    # at most 64 cells a side: every bin's samples are resident together, so no bin is cut into partial sums
    return S.make_rois(n, shape, scale, seed=seed, min_size=4.0 / scale, max_size=64.0 / scale)


def test_largest_row_block_runs_on_stream_path(lib_option):
    """14 x 14 bins at C = 288: a row block of 196 bins x 289 words (odd stride) = 226 576 B, the largest multiple of 32
    channels whose block fits the main kernel's shared memory; one row at a time in the tail."""
    shape, scale, P, sr = (1, 288, 100, 168), 1.0 / 8, 14, 2
    f = S.make_features(shape, seed=21)
    r = _small_rois(200, shape, scale, seed=22)
    out, ref = _run(f, r, P, scale, sr, lib_option, STREAM_LAUNCHES)
    assert np.array_equal(out, ref)


def test_row_block_one_channel_group_over_declines(lib_option):
    """C = 320 at 14 x 14: 196 x 321 x 4 = 251 664 B does not fit; the stream path declines to the generic kernel."""
    shape, scale, P, sr = (1, 320, 100, 168), 1.0 / 8, 14, 2
    f = S.make_features(shape, seed=23)
    r = _small_rois(64, shape, scale, seed=24)
    out, ref = _run(f, r, P, scale, sr, lib_option, GENERIC_LAUNCHES)
    assert np.array_equal(out, ref)


@pytest.mark.parametrize("C", [40, 35], ids=["c40_16byte", "c35_scalar"])
def test_several_rows_per_cta_with_split_bins(C, lib_option):
    """More output rows than 8 per main-kernel CTA, a partial last channel group (C % 32 != 0; C = 35 takes the tail's
    4-byte path), RoIs up to 200 cells wide, so that bins whose two x samples straddle a strip's end are cut into partial sums
    (red.global.add onto elements the prepass zeroed in the staging layout), and one RoI with a batch index out of range (its
    row is all zeros).  Split bins add their partial sums in another order than the generic kernel: within 1e-6 of it."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    shape, scale, P, sr = (2, C, 64, 200), 1.0 / 4, 7, 2
    R = 8 * sms + 300
    f = S.make_features(shape, seed=25)
    r = S.make_rois(R, shape, scale, seed=26, min_size=32.0, max_size=800.0)
    r[5, 0] = shape[0] + 2
    out, ref = _run(f, r, P, scale, sr, lib_option, STREAM_LAUNCHES)
    assert not np.any(out[5]) and not np.any(ref[5])
    np.testing.assert_allclose(out, ref, rtol=1e-6, atol=1e-6)
    assert np.mean(out == ref) > 0.9
