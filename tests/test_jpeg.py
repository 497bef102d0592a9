"""JPEG decode on the device (utils/image.imdecode / imread, ops.jpeg_decode_raw, csrc/jpeg.cu) against cv2.imread.

CPU: the numpy oracle (oracle/jpeg.py) equals cv2's pixels stored in tests/golden/jpeg.npz (make_golden_jpeg.py) on every
device-decodable case; the restatement of the device's self-synchronising decomposition gives the sequential decoder's
coefficients for every subsequence length from 1 bit to more than the interval; the parser's classification, restart splitting,
unstuffing and orientation; malformed headers raise ValueError; the C ABI rejects bad arguments.
GPU: the device equals the goldens and the oracle, in one mixed batch and one image at a time; fallback cases report their
status and imdecode returns cv2's pixels for them; the decoded CUDA images chain into the input blob; the current stream is
honoured."""
import hashlib
import os

import numpy as np
import pytest
import torch

from detectron.pytorch_b200 import _lib, ops
from detectron.pytorch_b200.utils import image as I
from detectron.pytorch_b200.utils import jpeg as J
from oracle import jpeg as O
from tests import jpeg_cases as cases

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "jpeg.npz"))
NAMES = cases.NAMES
DEVICE = [n for n in NAMES if cases.CASES[n]["status"] == 0]
FALLBACK = [n for n in NAMES if cases.CASES[n]["status"] != 0]
EINVAL, EWORKSPACE = -1, -2


def _data(name):
    return GOLD[name + "/jpeg"].tobytes()


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest().encode()


def _assert_golden(name, im):
    im = im.cpu().numpy() if torch.is_tensor(im) else im
    assert tuple(im.shape) == tuple(GOLD[name + "/shape"]), name
    if name + "/pixels" in GOLD:
        np.testing.assert_array_equal(im, GOLD[name + "/pixels"], err_msg=name)
    assert _sha(im) == GOLD[name + "/sha256"].tobytes(), name


# ---- CPU ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", DEVICE)
def test_oracle_equals_cv2(name):
    _assert_golden(name, O.decode(_data(name)))


def _interval_cases():
    return ["size_9x17_420", "quality_100_444", "noise_q100_420", "restart_3_420", "orientation_6", "optimized_gray",
            "checker_q100_420"]


@pytest.mark.parametrize("name", _interval_cases())
@pytest.mark.parametrize("S", [1, 2, 5, 16, 27, 31, 64, 512, 1 << 22])
def test_sync_restatement_equals_sequential(name, S):
    """Subsequences of S bits, from 1 bit (below one codeword plus its magnitude bits: sync cannot happen inside one) to more
    than the whole interval, and 1, 3 or 256 threads: the same coefficients as the sequential decode."""
    p = J.parse(_data(name))
    for iv in p.intervals:
        want = O.decode_sequential(p, iv)
        assert want is not None
        for T in (1, 3, 256):
            stats = {}
            got = O.decode_sync(p, iv, S, T, stats)
            assert got is not None and np.array_equal(got, want), (name, S, T)
            assert stats["passes"] <= max(stats["boundaries"], 0) + 1


@pytest.mark.parametrize("name", ["fallback_truncated", "fallback_corrupt"])
def test_bad_entropy_data_is_reported(name):
    p = J.parse(_data(name))
    assert p.fallback is None
    assert O.coefficients(p) is None
    for S in (1, 7, 64, 512):
        assert O.coefficients(p, sync=(S, 8)) is None


def test_parser_classification():
    want = {"fallback_progressive": "progressive", "fallback_411": "sampling 4x1,1x1,1x1"}
    for name in NAMES:
        p = J.parse(_data(name))
        if name in want:
            assert p.fallback == want[name], name
        else:
            assert p.fallback is None, (name, p.fallback)
            assert p.out_shape == tuple(GOLD[name + "/shape"][:2]), name
    assert J.parse(_data("orientation_6")).orientation == 6
    assert J.parse(_data("orientation_6")).out_shape == (37, 23)
    assert J.parse(_data("size_9x17_420")).orientation == 1


def test_parser_restart_split_and_unstuffing():
    for name in ("restart_1_420", "restart_3_440", "restart_row_gray", "size_16x16_444"):
        p = J.parse(_data(name))
        total = p.mcus_x * p.mcus_y
        r = p.restart or total
        assert [iv[:2] for iv in p.intervals] == [(f, min(r, total - f)) for f in range(0, total, r)], name
        # the scan between SOS and EOI, unstuffed and without its RSTn markers, is the intervals' concatenation
        data = _data(name)
        sos = data.index(b"\xff\xda")
        start = sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
        scan = data[start:data.rindex(b"\xff\xd9")]
        for m in range(0xD0, 0xD8):
            scan = scan.replace(bytes([0xFF, m]), b"")
        assert scan.replace(b"\xff\x00", b"\xff") == b"".join(iv[2] for iv in p.intervals), name
    stuffed = [iv[2] for n in NAMES if cases.CASES[n]["status"] == 0 for iv in J.parse(_data(n)).intervals]
    assert any(b"\xff" in b for b in stuffed)          # the fixtures do contain stuffed bytes


def _replace_segment(data, marker, fn):
    i = data.index(bytes([0xFF, marker]))
    n = int.from_bytes(data[i + 2:i + 4], "big")
    return data[:i] + fn(data[i:i + 2 + n]) + data[i + 2 + n:]


def test_malformed_headers_raise():
    good = _data("size_16x16_420")
    bad = {
        "no SOI": good[2:],
        "length past the end": good[:20],
        "zero height": _replace_segment(good, 0xC0, lambda s: s[:5] + b"\x00\x00" + s[7:]),
        "zero width": _replace_segment(good, 0xC0, lambda s: s[:7] + b"\x00\x00" + s[9:]),
        "DQT id out of range": _replace_segment(good, 0xDB, lambda s: s[:4] + bytes([0x07]) + s[5:]),
        "DHT id out of range": _replace_segment(good, 0xC4, lambda s: s[:4] + bytes([0x05]) + s[5:]),
        "DHT class out of range": _replace_segment(good, 0xC4, lambda s: s[:4] + bytes([0x20]) + s[5:]),
        "bad segment length": _replace_segment(good, 0xDB, lambda s: s[:2] + b"\x00\x01" + s[4:]),
        "missing table": _replace_segment(good, 0xDA, lambda s: s[:6] + bytes([0x33]) + s[7:]),
        "scan component not in frame": _replace_segment(good, 0xDA, lambda s: s[:5] + bytes([9]) + s[6:]),
        "bogus Huffman table": _replace_segment(good, 0xC4, lambda s: s[:5] + bytes([3]) + s[6:]),
    }
    for what, data in bad.items():
        with pytest.raises(ValueError):
            J.parse(data)
            pytest.fail(what)


def test_fallback_reasons():
    data = _data("size_16x16_420")
    adobe = data[:2] + bytes([0xFF, 0xEE, 0, 14]) + b"Adobe" + bytes([0, 100, 0, 0, 0, 0, 0]) + data[2:]
    jfif_free = adobe.replace(b"JFIF\x00", b"JFIX\x00")
    assert J.parse(jfif_free).fallback == "Adobe transform 0"
    xmp = data[:2] + bytes([0xFF, 0xE1, 0, 6]) + b"http" + data[2:]
    assert J.parse(xmp).fallback == "first APP1 segment is not EXIF"


def test_abi_rejects_bad_arguments():
    lib = _lib.load()
    assert lib.b200_jpeg_decode_workspace_bytes(0, 1) == 0
    assert lib.b200_jpeg_decode_workspace_bytes(10, 3) >= 10 * 192 + 3 * 32
    # well-formed but for the one argument changed below; every case returns before any launch
    args = [8, 8, 1, 8, 1, 8, 512, 4, 1, 4, 16, 8, 1 << 20, 8, 8, None]
    for i in (0, 1, 3, 5, 11, 13, 14):                                    # each null pointer
        a = list(args)
        a[i] = None
        assert lib.b200_jpeg_decode(*a) == EINVAL, i
    for i, v in ((2, 0), (2, 65536), (4, 0), (6, 0), (7, 0), (8, 0), (9, 0), (9, 5), (10, 0)):
        a = list(args)
        a[i] = v
        assert lib.b200_jpeg_decode(*a) == EINVAL, (i, v)
    a = list(args)
    a[12] = 100
    assert lib.b200_jpeg_decode(*a) == EWORKSPACE


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
def _status(names, status):
    return {n: int(s) for n, s in zip(names, status.cpu().numpy())}


@pytest.mark.gpu
def test_device_equals_goldens_in_one_batch():
    parsed = [J.parse(_data(n)) for n in DEVICE]
    images, status = ops.jpeg_decode_raw(parsed)
    assert set(_status(DEVICE, status).values()) == {ops.JPEG_DECODED}
    for n, im in zip(DEVICE, images):
        _assert_golden(n, im)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DEVICE)
def test_device_equals_goldens_one_at_a_time(name):
    _assert_golden(name, I.imdecode([_data(name)])[0])


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 13, 64, 4096, 1 << 24])
def test_device_subsequence_length_does_not_change_the_result(S):
    names = ["large_480x640_420_q90", "noise_q100_420_optimized", "restart_1_440", "orientation_7", "checker_q100_444"]
    images, status = ops.jpeg_decode_raw([J.parse(_data(n)) for n in names], subseq_bits=S)
    assert set(_status(names, status).values()) == {ops.JPEG_DECODED}
    for n, im in zip(names, images):
        _assert_golden(n, im)


@pytest.mark.gpu
def test_device_equals_oracle_on_every_stored_jpeg():
    parsed = [J.parse(_data(n)) for n in NAMES]
    images, status = ops.jpeg_decode_raw(parsed)
    st = _status(NAMES, status)
    for n, p, im in zip(NAMES, parsed, images):
        assert st[n] == cases.CASES[n]["status"], n
        if p.fallback:
            assert im is None
            continue
        want = O.decode(p)
        if want is None:
            assert st[n] == ops.JPEG_ENTROPY_ERROR
        else:
            np.testing.assert_array_equal(im.cpu().numpy(), want, err_msg=n)


@pytest.mark.gpu
def test_fallback_cases_return_cv2_pixels():
    for n in FALLBACK:
        _assert_golden(n, I.imdecode([_data(n)])[0])
    # one fallback of each kind in the middle of a batch
    names = ["size_15x15_420", "fallback_progressive", "large_481x639_420_q75", "fallback_corrupt", "orientation_5",
             "fallback_truncated", "fallback_411", "size_1x1_gray"]
    images = I.imdecode([_data(n) for n in names])
    for n, im in zip(names, images):
        assert im.is_cuda and im.dtype == torch.uint8
        _assert_golden(n, im)


@pytest.mark.gpu
def test_parsed_payload_and_imread(tmp_path):
    import pickle
    names = ["restart_row_large_optimized", "fallback_progressive", "orientation_3"]
    payloads = [pickle.loads(pickle.dumps(J.parse(_data(n)))) for n in names]     # what a loader worker hands over
    for n, im in zip(names, I.imdecode(payloads)):
        _assert_golden(n, im)
    path = tmp_path / "a.jpg"
    path.write_bytes(_data("large_640x480_422_q95"))
    _assert_golden("large_640x480_422_q95", I.imread(str(path)))


@pytest.mark.gpu
def test_non_default_stream():
    names = ["large_768x1024_444_q50", "restart_3_420", "noise_q100_444"]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        images, status = ops.jpeg_decode_raw([J.parse(_data(n)) for n in names])
        torch.cuda._sleep(1000000)
        host = [im.cpu() for im in images]
        st = status.cpu()
    assert int(st.max()) == 0
    for n, im in zip(names, host):
        _assert_golden(n, im)


@pytest.mark.gpu
@pytest.mark.parametrize("flipped", [False, True])
def test_decoded_images_chain_into_the_input_blob(flipped):
    from detectron.pytorch_b200.roi_data import minibatch as MB
    from detectron.pytorch_b200.utils import blob as B
    test_names = ["large_481x639_420_q75", "orientation_6"]
    for n in test_names:
        ref = GOLD[n + "/pixels"] if n + "/pixels" in GOLD else None
        im = I.imdecode([_data(n)])[0]
        if ref is None:
            ref = im.cpu().numpy()
            assert _sha(ref) == GOLD[n + "/sha256"].tobytes()
        got = B.get_image_blob(im, 600, 1000, _hflip=flipped)
        want = B.get_image_blob(ref, 600, 1000, _hflip=flipped)
        assert torch.equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2]), n
    # a two-image training step
    names = ["large_480x640_420_q90", "large_640x480_422_q95"]
    roidb = [{"flipped": flipped}, {"flipped": not flipped}]
    ims = I.imdecode([_data(n) for n in names])
    host = [im.cpu().numpy() for im in ims]
    for n, h in zip(names, host):
        assert _sha(h) == GOLD[n + "/sha256"].tobytes()
    kw = dict(scales=(600,), max_size=1000, fpn_on=True, coarsest_stride=32)
    got, s1 = MB.get_image_blob(roidb, ims, [0, 0], **kw)
    want, s2 = MB.get_image_blob(roidb, host, [0, 0], **kw)
    assert s1 == s2 and torch.equal(got, want)
