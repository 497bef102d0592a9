"""JPEG files for tests/test_jpeg.py, written with cv2's and PIL's encoders (tests/golden/make_golden_jpeg.py stores their bytes
and cv2's decode of them in tests/golden/jpeg.npz, so the tests need no encoder).

Each case: name -> dict(h, w, content, sampling, quality, optimize, restart, orientation, extra, mutate, status)
  content      natural (gradients plus texture and pixel noise), smooth (gradients plus coarse texture: the large cases, whose
               sizes matter and whose bytes should stay few), flat (DC only), checker (0 / 255 at 1 pixel), noise (uniform)
  sampling     444, 422, 420, 440, 411 (cv2 writer) or gray; orientation (1-8) switches to PIL's writer with an EXIF APP1
  restart      MCUs per restart interval (cv2's IMWRITE_JPEG_RST_INTERVAL), "row" = one MCU row, 0 = none
  extra        True: APP2, APP13 and COM segments inserted after SOI
  mutate       "progressive", "truncate", "corrupt"
  status       what the device reports: 0 decoded, 1 format fallback, 2 entropy data that does not decode
Cases of at most SMALL pixels store cv2's pixels; larger ones their SHA-256.
"""
import io

import numpy as np

SMALL = 40 * 40
_SAMPLING = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def _case(h, w, content="natural", sampling="420", quality=90, optimize=False, restart=0, orientation=None, extra=False, mutate=None,
          status=0):
    return dict(h=h, w=w, content=content, sampling=sampling, quality=quality, optimize=optimize, restart=restart,
                orientation=orientation, extra=extra, mutate=mutate, status=status)


CASES = {}
for _h, _w in [(1, 1), (1, 37), (37, 1), (8, 8), (9, 17), (15, 15), (16, 16), (3, 4)]:
    for _s in ("444", "422", "420", "440", "gray"):
        CASES["size_%dx%d_%s" % (_h, _w, _s)] = _case(_h, _w, sampling=_s)
for _h, _w, _s, _q in [(481, 639, "420", 75), (480, 640, "420", 90), (640, 480, "422", 95), (768, 1024, "444", 50), (480, 640, "gray", 90),
                       (481, 639, "440", 90)]:
    CASES["large_%dx%d_%s_q%d" % (_h, _w, _s, _q)] = _case(_h, _w, content="smooth", sampling=_s, quality=_q)
for _q in (50, 75, 90, 95, 100):
    for _s in ("420", "444"):
        CASES["quality_%d_%s" % (_q, _s)] = _case(48, 72, sampling=_s, quality=_q)
for _s in ("420", "422", "gray"):
    CASES["optimized_%s" % _s] = _case(57, 83, sampling=_s, optimize=True)
for _r in (1, 3, "row"):
    for _s in ("420", "440", "gray"):
        CASES["restart_%s_%s" % (_r, _s)] = _case(41, 67, sampling=_s, restart=_r)
CASES["restart_row_large_optimized"] = _case(480, 640, content="smooth", sampling="420", restart="row", optimize=True)
for _o in range(1, 9):
    CASES["orientation_%d" % _o] = _case(23, 37, sampling="420", orientation=_o)
CASES["orientation_6_gray"] = _case(19, 30, sampling="gray", orientation=6)
CASES["orientation_8_444"] = _case(19, 30, sampling="444", orientation=8)
CASES["extra_segments"] = _case(30, 40, sampling="420", extra=True)
CASES["flat_dc_only"] = _case(40, 56, content="flat", sampling="420", quality=75)
for _s in ("444", "420", "gray"):
    CASES["checker_q100_%s" % _s] = _case(32, 40, content="checker", sampling=_s, quality=100)
    CASES["noise_q100_%s" % _s] = _case(48, 40, content="noise", sampling=_s, quality=100)
CASES["noise_q100_420_optimized"] = _case(64, 64, content="noise", sampling="420", quality=100, optimize=True)
CASES["fallback_progressive"] = _case(45, 61, mutate="progressive", status=1)
CASES["fallback_411"] = _case(45, 61, sampling="411", status=1)
CASES["fallback_truncated"] = _case(45, 61, mutate="truncate", status=2)
CASES["fallback_corrupt"] = _case(45, 61, mutate="corrupt", status=2)

NAMES = sorted(CASES)


def pixels(c, seed):
    """The BGR uint8 source image of a case (gray: (h, w))."""
    rng = np.random.RandomState(seed)
    h, w = c["h"], c["w"]
    if c["content"] == "flat":
        im = np.empty((h, w, 3), np.uint8)
        im[...] = (37, 140, 201)
    elif c["content"] == "checker":
        y, x = np.mgrid[0:h, 0:w]
        im = np.repeat((((x + y) & 1) * 255).astype(np.uint8)[:, :, None], 3, axis=2)
        im[:, :, 1] = 255 - im[:, :, 1]
    elif c["content"] == "noise":
        im = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    elif c["content"] == "smooth":
        y, x = np.mgrid[0:h, 0:w].astype(np.float64)
        base = np.stack([128 + 100 * np.sin(x / 61.0 + y / 83.0), 128 + 90 * np.cos(y / 47.0), 128 + 80 * np.sin((x - y) / 37.0)], -1)
        coarse = rng.randint(-24, 25, ((h + 31) // 32, (w + 31) // 32, 3)).repeat(32, 0).repeat(32, 1)[:h, :w]
        im = np.clip(base + coarse, 0, 255).astype(np.uint8)
    else:
        y, x = np.mgrid[0:h, 0:w].astype(np.float64)
        base = np.stack([128 + 100 * np.sin(x / 23.0 + y / 41.0), 128 + 90 * np.cos(y / 17.0), (x * 3 + y * 2) % 256], -1)
        small = rng.randint(-40, 40, ((h + 7) // 8, (w + 7) // 8, 3)).repeat(8, 0).repeat(8, 1)[:h, :w]
        im = np.clip(base + small + rng.randint(-6, 7, (h, w, 3)), 0, 255).astype(np.uint8)
    if c["sampling"] == "gray":
        import cv2
        im = cv2.cvtColor(im, cv2.COLOR_BGR2GRAY)
    return im


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def encode(c, seed):
    """The JPEG bytes of a case."""
    import cv2
    im = pixels(c, seed)
    if c["orientation"] is not None or c["mutate"] == "progressive":
        from PIL import Image
        rgb = im if im.ndim == 2 else im[:, :, ::-1]
        kw = dict(quality=c["quality"])
        if c["orientation"] is not None:
            exif = Image.Exif()
            exif[0x0112] = c["orientation"]
            kw["exif"] = exif.tobytes()
        if c["mutate"] == "progressive":
            kw["progressive"] = True
        if im.ndim == 3:
            kw["subsampling"] = {"444": 0, "422": 1, "420": 2}[c["sampling"]]
        buf = io.BytesIO()
        Image.fromarray(rgb).save(buf, "JPEG", **kw)
        data = buf.getvalue()
    else:
        params = [cv2.IMWRITE_JPEG_QUALITY, c["quality"], cv2.IMWRITE_JPEG_OPTIMIZE, int(c["optimize"])]
        if c["sampling"] != "gray":
            params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, _SAMPLING[c["sampling"]]]
        r = c["restart"]
        if r == "row":
            hmax = 2 if c["sampling"] in ("420", "422", "411") else 1
            hmax = 4 if c["sampling"] == "411" else hmax
            r = -(-c["w"] // (8 * hmax))
        if r:
            params += [cv2.IMWRITE_JPEG_RST_INTERVAL, r]
        ok, enc = cv2.imencode(".jpg", im, params)
        assert ok
        data = enc.tobytes()
    if c["extra"]:
        data = (data[:2] + _segment(0xE2, b"ICC_PROFILE\x00" + bytes(range(40))) + _segment(0xFE, b"a comment")
                + _segment(0xED, b"Photoshop 3.0\x00" + b"\x00" * 20) + data[2:])
    if c["mutate"] in ("truncate", "corrupt"):
        sos = data.index(b"\xff\xda")
        start = sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
        end = data.rindex(b"\xff\xd9")
        if c["mutate"] == "truncate":
            data = data[:start + (end - start) // 2] + b"\xff\xd9"
        else:
            b = bytearray(data)
            for k in range(8):                       # overwrite a run in the middle of the scan with 0xFE 0xFE ...
                b[start + (end - start) // 3 + k] = 0xFE
            data = bytes(b)
    return data
