"""JPEG file parsing for the device decoder (ops.jpeg_decode_raw, utils/image.imdecode).

`parse(data)` walks the markers of one file (SOI, APPn, COM, DQT, SOF, DHT, DRI, SOS, RSTn, EOI), reads the EXIF orientation
that cv2.imread applies, and classifies the file:

  * device-decodable: Huffman-coded sequential 8-bit (SOF0 / SOF1) in one interleaved scan, either 3 YCbCr components with luma
    sampling H, V in {1, 2} and chroma 1x1 (4:4:4, 4:2:2, 4:2:0, 4:4:0) or 1 component (grayscale);
  * fallback (`Parsed.fallback` names the reason): everything else cv2 can read -- progressive, arithmetic, 12-bit, other
    sampling factors, several scans, CMYK / YCCK, Adobe RGB -- is decoded by cv2.imdecode on the host.

Malformed headers raise ValueError: a segment length that runs past the data, a table id out of range, a zero dimension, a
bogus Huffman table, a scan that references a missing table.  Entropy data is not decoded here; the scan is split into its
restart intervals and unstuffed (0xFF00 -> 0xFF) with compiled regular expressions and bytes.replace, which run at C speed, so this module runs in
a loader worker on the CPU without CUDA.  The result pickles: a worker can hand the parsed, still compressed payload to the
main process instead of the pixels.
"""
import re
import struct

import numpy as np

# natural-order index of the k-th zig-zag coefficient (ITU-T T.81, figure A.6)
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63], dtype=np.int32)

LOOKUP_BITS = 9          # codes up to this length decode with one table lookup
# one Huffman decode table as the device reads it (b200_jpeg_huff_table in include/b200_roi_ops.h)
HUFF_TABLE = np.dtype([("lookup", "<u2", (1 << LOOKUP_BITS,)), ("maxcode", "<i4", (18,)), ("valoff", "<i4", (18,)),
                       ("values", "u1", (256,))])


class Huffman:
    """A decode table derived from a DHT segment (T.81 annex C and F.2.2.3).

    lookup[p]:  for a code of length l <= LOOKUP_BITS that is the prefix of the 9-bit window p, (l << 8) | symbol; 0 otherwise.
    maxcode[l]: the largest code of length l, -1 when there is none; maxcode[17] is a sentinel above every 17-bit value.
    valoff[l]:  values index of a length-l code = code + valoff[l].
    """

    def __init__(self, bits, values, is_dc):
        bits = [int(b) for b in bits]
        values = bytes(values)
        if sum(bits) != len(values) or len(values) > 256:
            raise ValueError("bogus Huffman table: %d symbols for %d codes" % (len(values), sum(bits)))
        if is_dc and any(v > 15 for v in values):
            raise ValueError("bogus Huffman table: DC symbol above 15")
        self.values = values
        self.maxcode = [-1] * 18
        self.valoff = [0] * 18
        self.maxcode[17] = 1 << 20
        # codes in increasing order fill consecutive ranges of the 9-bit lookup from 0: one np.repeat builds it
        entries, reps = [], []
        code, p = 0, 0
        maxlen = max([l for l in range(1, 17) if bits[l - 1]], default=0)
        for l in range(1, maxlen + 1):
            n = bits[l - 1]
            if n:
                self.valoff[l] = p - code
                if l <= LOOKUP_BITS:
                    entries.extend((l << 8) | v for v in values[p:p + n])
                    reps.extend([1 << (LOOKUP_BITS - l)] * n)
                code += n
                p += n
                self.maxcode[l] = code - 1
            # libjpeg's check: the codes of each length fit in it, and the all-ones code stays unassigned
            if code >= (1 << l):
                raise ValueError("bogus Huffman table: codes of length %d overflow" % l)
            code <<= 1
        self.lookup = np.zeros((1 << LOOKUP_BITS,), np.uint16)
        filled = np.repeat(np.array(entries, np.uint16), reps)
        self.lookup[:len(filled)] = filled
        self._packed = None

    def decode(self, window16):
        """(length, symbol) of the code at the front of a 16-bit window, or (0, 0) for a bad code."""
        e = int(self.lookup[window16 >> (16 - LOOKUP_BITS)])
        if e:
            return e >> 8, e & 0xFF
        for l in range(LOOKUP_BITS + 1, 17):
            c = window16 >> (16 - l)
            if c <= self.maxcode[l]:
                return l, self.values[c + self.valoff[l]]
        return 0, 0

    def packed(self):
        if self._packed is not None:
            return self._packed
        t = np.zeros((), HUFF_TABLE)
        t["lookup"] = self.lookup
        t["maxcode"] = self.maxcode
        t["valoff"] = self.valoff
        t["values"][:len(self.values)] = np.frombuffer(self.values, np.uint8)
        self._packed = t
        return t


class Parsed:
    """What parse() finds in one file.

    data           the file's bytes (the fallback decodes them with cv2.imdecode)
    fallback       None when the device decodes the file, else the reason it does not
    height, width  the coded size; orientation the EXIF orientation (1-8, 1 without one)
    out_shape      (H, W) of the decoded image after the orientation (5-8 transpose it)
    ncomp          1 or 3; h, v: the luma sampling factors (1 for grayscale); mcus_x, mcus_y: the MCU grid
    quant          (ncomp, 64) int32 quantisation tables in natural order
    dc, ac         per component its Huffman table
    restart        the restart interval in MCUs (0: none)
    intervals      [(first_mcu, num_mcus, unstuffed entropy bytes)] in scan order
    """
    fallback = None
    orientation = 1

    @property
    def blocks_per_mcu(self):
        return self.h * self.v + (2 if self.ncomp == 3 else 0)

    @property
    def num_blocks(self):
        return self.mcus_x * self.mcus_y * self.blocks_per_mcu

    @property
    def out_shape(self):
        return (self.width, self.height) if self.orientation >= 5 else (self.height, self.width)

    def __repr__(self):
        return "Parsed(%dx%d, %s, orientation %d)" % (self.width, self.height, self.fallback or "device", self.orientation)


_SOF_OTHER = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "differential sequential", 0xC6: "differential progressive",
              0xC7: "differential lossless", 0xC9: "arithmetic coding", 0xCA: "progressive arithmetic coding",
              0xCB: "lossless arithmetic coding", 0xCD: "differential arithmetic coding",
              0xCE: "differential progressive arithmetic coding", 0xCF: "differential lossless arithmetic coding"}


def _exif_orientation(seg):
    """The orientation tag of IFD0 of an APP1 payload, as cv2 reads it from the first APP1 segment: (value, None), or (1, None)
    when there is none, or (None, reason) for anything this reader does not follow to the letter."""
    if not seg.startswith(b"Exif\x00\x00"):
        return None, "first APP1 segment is not EXIF"
    t = seg[6:]
    if len(t) < 8 or t[:2] not in (b"II", b"MM"):
        return None, "unreadable EXIF header"
    e = "<" if t[:2] == b"II" else ">"
    if struct.unpack(e + "H", t[2:4])[0] != 42:
        return None, "unreadable EXIF header"
    ifd = struct.unpack(e + "I", t[4:8])[0]
    if ifd + 2 > len(t):
        return None, "unreadable EXIF IFD"
    n = struct.unpack(e + "H", t[ifd:ifd + 2])[0]
    if ifd + 2 + 12 * n > len(t):
        return None, "unreadable EXIF IFD"
    for i in range(n):
        tag, typ, count = struct.unpack(e + "HHI", t[ifd + 2 + 12 * i:ifd + 10 + 12 * i])
        if tag == 0x0112:
            if typ != 3 or count != 1:
                return None, "unusual EXIF orientation entry"
            o = struct.unpack(e + "H", t[ifd + 10 + 12 * i:ifd + 12 + 12 * i])[0]
            if not 1 <= o <= 8:
                return None, "EXIF orientation %d" % o
            return o, None
    return 1, None


# the scan ends at the first 0xFF followed by neither 0x00 (stuffing) nor RST0-7
_SCAN_END = re.compile(rb"\xff[^\x00\xd0-\xd7]")
_RST = re.compile(rb"\xff[\xd0-\xd7]")


def _scan_end(data, start):
    """Offset of the marker that ends the entropy-coded segment starting at `start`, or None when the data ends first."""
    m = _SCAN_END.search(data, start)
    return None if m is None else m.start()


def _split_scan(data, start, end, restart, total_mcus):
    """The entropy-coded segment data[start:end] split at its RSTn markers and unstuffed: (intervals, fallback reason or None)."""
    pieces = [(m.start(), data[m.start() + 1]) for m in _RST.finditer(data, start, end)]
    if restart == 0:
        if pieces:
            return None, "RST marker without a restart interval"
        return [(0, total_mcus, data[start:end].replace(b"\xff\x00", b"\xff"))], None
    bounds, prev = [], start
    for j, m in pieces:
        bounds.append((prev, j, m))
        prev = j + 2
    bounds.append((prev, end, None))
    count = -(-total_mcus // restart)
    if len(bounds) != count:
        return None, "%d restart intervals, %d expected" % (len(bounds), count)
    out = []
    for idx, (a, b, m) in enumerate(bounds):
        if m is not None and m != 0xD0 + (idx & 7):
            return None, "restart markers out of sequence"
        first = idx * restart
        out.append((first, min(restart, total_mcus - first), data[a:b].replace(b"\xff\x00", b"\xff")))
    return out, None


def parse(data):
    """Parse one JPEG file (bytes-like).  Returns a Parsed; raises ValueError on a malformed header."""
    data = bytes(data)
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise ValueError("not a JPEG file (no SOI marker)")
    p = Parsed()
    p.data = data
    qt, dht = {}, {}
    frame = None
    restart = 0
    saw_jfif = saw_adobe = False
    adobe_transform = None
    app1_seen = False
    fallback = None
    scans = 0
    pos = 2

    def fail(reason):
        nonlocal fallback
        if fallback is None:
            fallback = reason

    while True:
        # a marker: 0xFF, optional 0xFF fill bytes, the code
        if pos >= n or data[pos] != 0xFF:
            raise ValueError("expected a marker at byte %d" % pos)
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise ValueError("file ends inside a marker")
        m = data[pos]
        pos += 1
        if m == 0xD9:                                                 # EOI
            break
        if m == 0xD8 or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise ValueError("unexpected marker 0x%02X" % m)
        if pos + 2 > n:
            raise ValueError("segment length past the end of the data")
        length = (data[pos] << 8) | data[pos + 1]
        if length < 2 or pos + length > n:
            raise ValueError("bad length %d of segment 0x%02X" % (length, m))
        seg = data[pos + 2:pos + length]
        pos += length
        if m == 0xDB:                                                 # DQT
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                if tq > 3 or pq > 1:
                    raise ValueError("DQT table id %d precision %d" % (tq, pq))
                size = 64 * (pq + 1)
                if i + 1 + size > len(seg):
                    raise ValueError("DQT segment too short")
                vals = np.frombuffer(seg[i + 1:i + 1 + size], ">u2" if pq else "u1").astype(np.int32)
                t = np.zeros(64, np.int32)
                t[ZIGZAG] = vals
                qt[tq] = t
                i += 1 + size
        elif m == 0xC4:                                               # DHT
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise ValueError("DHT segment too short")
                tc, th = seg[i] >> 4, seg[i] & 15
                if tc > 1 or th > 3:
                    raise ValueError("DHT table class %d id %d" % (tc, th))
                bits = list(seg[i + 1:i + 17])
                cnt = sum(bits)
                if cnt > 256 or i + 17 + cnt > len(seg):
                    raise ValueError("DHT segment too short")
                dht[(tc, th)] = Huffman(bits, seg[i + 17:i + 17 + cnt], tc == 0)
                i += 17 + cnt
        elif m == 0xDD:                                               # DRI
            if len(seg) != 2:
                raise ValueError("DRI segment of %d bytes" % len(seg))
            restart = (seg[0] << 8) | seg[1]
        elif 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):       # SOFn
            if frame is not None:
                raise ValueError("two frame headers")
            if len(seg) < 6:
                raise ValueError("SOF segment too short")
            prec, H, W, nc = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if H == 0 or W == 0 or nc == 0:
                raise ValueError("zero dimension in the frame header (%d x %d, %d components)" % (W, H, nc))
            if len(seg) != 6 + 3 * nc:
                raise ValueError("SOF segment of %d bytes for %d components" % (len(seg), nc))
            comps = []
            for c in range(nc):
                cid, hv, tq = seg[6 + 3 * c], seg[7 + 3 * c], seg[8 + 3 * c]
                h, v = hv >> 4, hv & 15
                if not (1 <= h <= 4 and 1 <= v <= 4) or tq > 3:
                    raise ValueError("component %d: sampling %dx%d, table %d" % (c, h, v, tq))
                comps.append((cid, h, v, tq))
            frame = (m, prec, H, W, comps)
            if m in _SOF_OTHER:
                fail(_SOF_OTHER[m])
            elif prec != 8:
                fail("%d-bit samples" % prec)
        elif m == 0xDA:                                               # SOS
            if frame is None:
                raise ValueError("scan before the frame header")
            ns = seg[0] if seg else 0
            if ns < 1 or ns > 4 or len(seg) != 4 + 2 * ns:
                raise ValueError("bad SOS segment")
            comps = frame[4]
            ids = [c[0] for c in comps]
            sel = []
            for j in range(ns):
                cid, t = seg[1 + 2 * j], seg[2 + 2 * j]
                if cid not in ids:
                    raise ValueError("scan references component %d, not in the frame" % cid)
                td, ta = t >> 4, t & 15
                if td > 3 or ta > 3:
                    raise ValueError("scan table ids %d / %d" % (td, ta))
                sel.append((ids.index(cid), td, ta))
            ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            scans += 1
            if frame[0] in (0xC0, 0xC1):
                for ci, td, ta in sel:
                    if (0, td) not in dht or (1, ta) not in dht:
                        raise ValueError("scan references a missing Huffman table")
                for c in comps:
                    if c[3] not in qt:
                        raise ValueError("frame references missing quantisation table %d" % c[3])
            if scans > 1:
                fail("more than one scan")
            elif ns != len(comps):
                fail("non-interleaved scans")
            elif [s[0] for s in sel] != list(range(ns)):
                fail("scan component order differs from the frame's")
            elif (ss, se, ahal) != (0, 63, 0) and frame[0] in (0xC0, 0xC1):
                fail("scan parameters Ss=%d Se=%d Ah/Al=0x%02X" % (ss, se, ahal))
            end = _scan_end(data, pos)
            if fallback is not None:
                # skip this scan's entropy data to the next marker
                if end is None:
                    break
                pos = end
                continue
            p.sel = sel
            p.dc = [dht[(0, td)] for _, td, _ in sorted(sel)]
            p.ac = [dht[(1, ta)] for _, _, ta in sorted(sel)]
            p.quant = np.stack([qt[c[3]] for c in comps])
            p.scan = (pos, n if end is None else end, restart)
            if end is None:
                fail("truncated scan")
                break
            pos = end
        elif m == 0xE1 and not app1_seen:                             # the first APP1: EXIF
            app1_seen = True
            o, why = _exif_orientation(seg)
            if why:
                fail(why)
            else:
                p.orientation = o
        elif m == 0xE0:
            if seg.startswith(b"JFIF\x00"):
                saw_jfif = True
        elif m == 0xEE:
            if len(seg) >= 12 and seg.startswith(b"Adobe"):
                saw_adobe = True
                adobe_transform = seg[11]
        # other APPn, COM and reserved markers: skipped
    if frame is None:
        raise ValueError("no frame header")
    if scans == 0:
        raise ValueError("no scan")
    sof, prec, H, W, comps = frame
    p.height, p.width, p.ncomp = H, W, len(comps)
    if fallback is None:
        if len(comps) == 3:
            if not saw_jfif and saw_adobe and adobe_transform != 1:
                fail("Adobe transform %d" % adobe_transform)
            elif not saw_jfif and not saw_adobe and [c[0] for c in comps] == [82, 71, 66]:
                fail("RGB components")
            else:
                (_, h, v, _), c1, c2 = comps
                if c1[1:3] != (1, 1) or c2[1:3] != (1, 1) or h > 2 or v > 2:
                    fail("sampling %s" % ",".join("%dx%d" % (c[1], c[2]) for c in comps))
        elif len(comps) != 1:
            fail("%d components" % len(comps))
        if fallback is None and int(p.quant.max()) > 255:
            fail("quantisation values above 255")
    if fallback is not None:
        p.fallback = fallback
        return p
    if len(comps) == 1:
        p.h = p.v = 1
        p.mcus_x, p.mcus_y = -(-W // 8), -(-H // 8)
    else:
        p.h, p.v = comps[0][1], comps[0][2]
        p.mcus_x, p.mcus_y = -(-W // (8 * p.h)), -(-H // (8 * p.v))
    start, end, restart = p.scan
    intervals, why = _split_scan(data, start, end, restart, p.mcus_x * p.mcus_y)
    if why:
        p.fallback = why
        return p
    p.restart = restart
    p.intervals = intervals
    del p.scan, p.sel
    return p
