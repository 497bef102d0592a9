"""numpy restatement of the device JPEG decoder (csrc/jpeg.cu), the checker for ops.jpeg_decode_raw.

Derived from ITU-T T.81 and the integer "islow" algorithm that cv2's libjpeg-turbo applies by default:
  * sequential Huffman decode (T.81 F.2.2), coefficients de-zigzagged, DC differences summed per component and restart
    interval, stored as 16-bit values (libjpeg's JCOEF);
  * dequantisation and the islow IDCT: CONST_BITS 13, PASS1_BITS 2, 32-bit integer arithmetic, descale by rounding shifts,
    libjpeg's range-limit table (10-bit wrap, then clamp to 0..255);
  * fancy upsampling of 1x1 chroma: h2v1 and h1v2 triangle filters with biases 1 / 2, h2v2 with biases 8 / 7; a neighbour past
    the image edge is the edge sample itself (the real chroma size, not the MCU padding);
  * libjpeg's integer YCbCr -> BGR (16-bit fixed point tables, ONE_HALF rounding), clamped;
  * the EXIF orientation as cv2 applies it (flip / transpose).

`decode_run` is the one decoding step both decompositions share: from a codeword-boundary state (bit offset, block in the MCU,
coefficient index) up to the first boundary at or past a given bit.  `decode_sequential` runs it over a whole restart interval;
`decode_sync` restates the device's self-synchronising decomposition of the same interval (subsequences of S bits, speculative
decode, sync passes, block-count scan, a second decode that writes).
"""
import numpy as np

from detectron.pytorch_b200.utils import jpeg as J


def _window32(buf, pos):
    """The 32 bits of `buf` (zero-padded) starting at bit `pos`."""
    b = pos >> 3
    x = int.from_bytes(buf[b:b + 5].ljust(5, b"\x00"), "big")
    return (x >> (8 - (pos & 7))) & 0xFFFFFFFF


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def decode_run(buf, L, state, end, dc, ac, comp_of_blk, out=None, first=0, limit=0):
    """Decode the interval's bits `buf` (L bits long) from the boundary state (pos, blk, k) to the first codeword boundary at
    or past `end`.  Returns ((pos, blk, k), blocks completed, error).  With `out`, block `first + n` (n-th completed here,
    below `limit`) receives the DC difference at [0] and the AC values at their natural positions.

    A run of fewer than 8 one-bits before L at a block start is the encoder's byte padding and ends the interval.  Data that a
    valid stream never contains sets `error` and the decode goes on, so that a decode started from a guessed state can still
    fall into step with the true one: a bad code skips one bit, a code or magnitude past L ends the interval, a coefficient
    index past 63 ends the block."""
    pos, blk, k = state
    bpm = len(comp_of_blk)
    n, err = 0, False
    while pos < end:
        rem = L - pos
        w = _window32(buf, pos)
        if k == 0 and rem < 8 and (w >> (32 - rem)) == (1 << rem) - 1:
            pos = L
            break
        c = comp_of_blk[blk]
        tab = dc[c] if k == 0 else ac[c]
        ln, sym = tab.decode(w >> 16)
        if ln == 0:
            err = True
            pos += 1
            continue
        if k == 0:
            s = sym
            if ln + s > rem:
                err, pos = True, L
                break
            if out is not None and first + n < limit:
                out[first + n, 0] = _extend((w >> (32 - ln - s)) & ((1 << s) - 1), s) if s else 0
            pos += ln + s
            k = 1
            continue
        r, s = sym >> 4, sym & 15
        if s:
            if ln + s > rem:
                err, pos = True, L
                break
            pos += ln + s
            k += r
            if k > 63:
                err, done = True, True
            else:
                if out is not None and first + n < limit:
                    out[first + n, J.ZIGZAG[k]] = _extend((w >> (32 - ln - s)) & ((1 << s) - 1), s)
                k += 1
                done = k == 64
        elif r == 15:
            if ln > rem:
                err, pos = True, L
                break
            pos += ln
            k += 16
            done = k > 63
            err = err or done
        else:
            if ln > rem:
                err, pos = True, L
                break
            pos += ln
            done = True                                               # EOB
        if done:
            n += 1
            blk = blk + 1 if blk + 1 < bpm else 0
            k = 0
    return (pos, blk, k), n, err


def comp_of_blk(p):
    return [0] * (p.h * p.v) + ([1, 2] if p.ncomp == 3 else [])


def _dc_sum(coefs, cob):
    """DC differences -> values per component within one interval (int32 accumulation, stored as int16)."""
    bpm = len(cob)
    dc = coefs[:, 0].astype(np.int64).reshape(-1, bpm)
    for c in set(cob):
        cols = [b for b in range(bpm) if cob[b] == c]
        run = np.cumsum(dc[:, cols].reshape(-1)).reshape(-1, len(cols))
        dc[:, cols] = run
    coefs[:, 0] = dc.reshape(-1).astype(np.int32).astype(np.int16)


def decode_sequential(p, iv):
    """Coefficients (blocks of the interval, 64) int16 of interval `iv` = (first_mcu, num_mcus, bytes); None when the entropy
    data does not decode to exactly the interval's blocks."""
    _, nm, buf = iv
    cob = comp_of_blk(p)
    want = nm * len(cob)
    out = np.zeros((want, 64), np.int16)
    L = 8 * len(buf)
    st, n, err = decode_run(buf, L, (0, 0, 0), L, p.dc, p.ac, cob, out, 0, want)
    if err or st != (L, 0, 0) or n != want:
        return None
    _dc_sum(out, cob)
    return out


def decode_sync(p, iv, S, T, stats=None):
    """The device's decomposition of one interval: the L bits are cut into subsequences of S bits, thread t of T owns the
    contiguous run of subsequences [t R, (t + 1) R), R = ceil(n / T).

    1. Every thread decodes its run in order.  Its first subsequence starts from a guess -- its first bit, block 0 of an MCU,
       the DC coefficient -- the others from the exit state of the one before.  in[j] / out[j] record each subsequence's
       entry and exit state (the exit is the first boundary at or past its last bit) and its block count.
    2. Sync passes: thread t compares out[last subsequence of t - 1] with its own in[first]; on a difference it decodes again
       from that state and stops as soon as a subsequence's new entry state equals the recorded one (the decode has met the
       previous one: everything after is unchanged).  Passes repeat until none changes anything.  Each pass makes at least one
       more run exact, so a decode that never syncs ends as the sequential decode: slower, never wrong.
    3. An exclusive scan of the runs' block counts gives each run its first block; the interval is valid when the last exit is
       (L, block 0, DC), no subsequence's exact decode met an error and the count is the interval's block count.
    4. Each thread decodes its run once more from its exact entry state and writes its blocks; then the DC differences are
       summed per component.
    Returns the coefficients as decode_sequential does.  `stats` (a dict) receives the number of sync passes that changed a
    run ("passes"), and of the T - 1 run boundaries ("boundaries") how many the first sync pass found in sync: the run's guessed
    decode had met the true one inside the run ("synced_first")."""
    _, nm, buf = iv
    cob = comp_of_blk(p)
    want = nm * len(cob)
    L = 8 * len(buf)
    nsub = max(1, -(-L // S))
    R = -(-nsub // T)
    runs = [(t * R, min((t + 1) * R, nsub)) for t in range(T) if t * R < nsub]
    ends = [min((j + 1) * S, L) for j in range(nsub)]
    st_in, st_out, cnt, err = [None] * nsub, [None] * nsub, [0] * nsub, [False] * nsub

    def run_from(j0, j1, state, stop_on_match):
        """Decode subsequences j0 .. j1 - 1 from `state`; True when it stopped at a recorded entry state (in sync)."""
        for j in range(j0, j1):
            if stop_on_match and j > j0 and st_in[j] == state:
                return True
            st_in[j] = state
            state, cnt[j], err[j] = decode_run(buf, L, state, ends[j], p.dc, p.ac, cob)
            st_out[j] = state
        return False

    for j0, j1 in runs:
        run_from(j0, j1, (0, 0, 0) if j0 == 0 else (j0 * S, 0, 0), False)
    passes, synced = 0, None
    while True:
        cand = [st_out[j0 - 1] if j0 else st_in[0] for j0, _ in runs]
        stale = [t for t, (j0, _) in enumerate(runs) if cand[t] != st_in[j0]]
        if not stale:
            break
        passes += 1
        met = [run_from(runs[t][0], runs[t][1], cand[t], True) for t in stale]
        if synced is None:
            synced = sum(met) + (len(runs) - 1 - len(stale))
    if stats is not None:
        stats.update(passes=passes, synced_first=synced or 0, boundaries=len(runs) - 1)
    if st_out[-1] != (L, 0, 0) or sum(cnt) != want or any(err):
        return None
    out = np.zeros((want, 64), np.int16)
    base = 0
    for j0, j1 in runs:
        state = st_in[j0]
        for j in range(j0, j1):
            state, c, _ = decode_run(buf, L, state, ends[j], p.dc, p.ac, cob, out, base, want)
            base += c
    _dc_sum(out, cob)
    return out


def coefficients(p, sync=None):
    """All blocks of the image in MCU order, (num_blocks, 64) int16; None on undecodable entropy data.  sync = (S, T) decodes
    each interval with decode_sync instead of decode_sequential."""
    parts = []
    for iv in p.intervals:
        c = decode_sequential(p, iv) if sync is None else decode_sync(p, iv, *sync)
        if c is None:
            return None
        parts.append(c)
    return np.concatenate(parts)


# ---- islow IDCT ----------------------------------------------------------------------------------------------------------
_F = dict(F0298=2446, F0390=3196, F0541=4433, F0765=6270, F0899=7373, F1175=9633, F1501=12299, F1847=15137, F1961=16069,
          F2053=16819, F2562=20995, F3072=25172)


def _idct_1d(d0, d1, d2, d3, d4, d5, d6, d7, shift):
    """One islow pass over int32 arrays; returns the 8 outputs descaled by `shift` with rounding."""
    i32 = np.int32
    z2, z3 = d2, d6
    z1 = (z2 + z3) * i32(_F["F0541"])
    tmp2 = z1 + z3 * i32(-_F["F1847"])
    tmp3 = z1 + z2 * i32(_F["F0765"])
    tmp0 = (d0 + d4) << i32(13)
    tmp1 = (d0 - d4) << i32(13)
    tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
    tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = d7, d5, d3, d1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * i32(_F["F1175"])
    t0 = t0 * i32(_F["F0298"])
    t1 = t1 * i32(_F["F2053"])
    t2 = t2 * i32(_F["F3072"])
    t3 = t3 * i32(_F["F1501"])
    z1 = z1 * i32(-_F["F0899"])
    z2 = z2 * i32(-_F["F2562"])
    z3 = z3 * i32(-_F["F1961"]) + z5
    z4 = z4 * i32(-_F["F0390"]) + z5
    t0 = t0 + z1 + z3
    t1 = t1 + z2 + z4
    t2 = t2 + z2 + z3
    t3 = t3 + z1 + z4
    r = i32(1 << (shift - 1))
    s = i32(shift)
    return [(tmp10 + t3 + r) >> s, (tmp11 + t2 + r) >> s, (tmp12 + t1 + r) >> s, (tmp13 + t0 + r) >> s,
            (tmp13 - t0 + r) >> s, (tmp12 - t1 + r) >> s, (tmp11 - t2 + r) >> s, (tmp10 - t3 + r) >> s]


def range_limit(x):
    """libjpeg's post-IDCT range limit: the value + 128 taken modulo 1024 as a signed 10-bit number, clamped to 0..255."""
    v = ((x.astype(np.int32) + 128 + 512) & 1023) - 512
    return np.clip(v, 0, 255).astype(np.uint8)


def idct_islow(coefs, quant):
    """(n, 64) int16 coefficients (natural order), (n, 64) or (64,) quantisation -> (n, 8, 8) uint8 samples."""
    with np.errstate(over="ignore"):
        d = (coefs.astype(np.int32) * np.asarray(quant, np.int32)).reshape(-1, 8, 8)
        # pass 1: columns (over the row index), descale by CONST_BITS - PASS1_BITS
        ws = np.stack(_idct_1d(*[d[:, r, :] for r in range(8)], 11), axis=1)
        # pass 2: rows, descale by CONST_BITS + PASS1_BITS + 3
        out = np.stack(_idct_1d(*[ws[:, :, c] for c in range(8)], 18), axis=2)
    return range_limit(out)


def planes(p, coefs):
    """The component sample planes (padded to whole MCUs) from coefficients in MCU order."""
    cob = comp_of_blk(p)
    bpm = len(cob)
    samples = idct_islow(coefs, p.quant[np.tile(cob, coefs.shape[0] // bpm)])
    s = samples.reshape(p.mcus_y, p.mcus_x, bpm, 8, 8)
    h, v = p.h, p.v
    y = s[:, :, :h * v].reshape(p.mcus_y, p.mcus_x, v, h, 8, 8).transpose(0, 2, 4, 1, 3, 5)
    out = [y.reshape(p.mcus_y * v * 8, p.mcus_x * h * 8)]
    for c in (1, 2) if p.ncomp == 3 else ():
        out.append(s[:, :, h * v + c - 1].transpose(0, 2, 1, 3).reshape(p.mcus_y * 8, p.mcus_x * 8))
    return out


def upsample(p, c):
    """Fancy upsampling of one 1x1 chroma plane to the luma grid, (height, width) int32."""
    H, W, h, v = p.height, p.width, p.h, p.v
    cw, ch = -(-W // h), -(-H // v)
    c = c[:ch, :cw].astype(np.int32)
    if h == 2 and cw <= 2:
        # libjpeg-turbo filters h2v1 / h2v2 only when the chroma row is wider than 2 samples; else it replicates each sample
        return np.repeat(np.repeat(c, v, axis=0), 2, axis=1)[:H, :W]
    if v == 2:
        up = np.concatenate([c[:1], c[:-1]])
        dn = np.concatenate([c[1:], c[-1:]])
        if h == 2:
            rows = np.empty((2 * ch, cw), np.int32)
            rows[0::2] = 3 * c + up                                   # column sums
            rows[1::2] = 3 * c + dn
        else:
            rows = np.empty((2 * ch, cw), np.int32)
            rows[0::2] = (3 * c + up + 1) >> 2
            rows[1::2] = (3 * c + dn + 2) >> 2
            return rows[:H, :W]
    else:
        rows = c
    if h == 2:
        left = np.concatenate([rows[:, :1], rows[:, :-1]], axis=1)
        right = np.concatenate([rows[:, 1:], rows[:, -1:]], axis=1)
        out = np.empty((rows.shape[0], 2 * cw), np.int32)
        if v == 2:
            out[:, 0::2] = (3 * rows + left + 8) >> 4
            out[:, 1::2] = (3 * rows + right + 7) >> 4
        else:
            out[:, 0::2] = (3 * rows + left + 1) >> 2
            out[:, 1::2] = (3 * rows + right + 2) >> 2
        return out[:H, :W]
    return rows[:H, :W]


def ycc_to_bgr(y, cb, cr):
    """libjpeg's ycc_rgb_convert, channels written B, G, R."""
    y, cb, cr = (a.astype(np.int64) for a in (y, cb, cr))
    xb, xr = cb - 128, cr - 128
    r = y + ((91881 * xr + 32768) >> 16)
    g = y + ((-22554 * xb + 32768 - 46802 * xr) >> 16)
    b = y + ((116130 * xb + 32768) >> 16)
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def orient(im, o):
    """cv2's EXIF orientation transform of an (H, W, 3) image."""
    if o >= 5:
        im = im.transpose(1, 0, 2)
    flip = {1: None, 2: 1, 3: -1, 4: 0, 5: None, 6: 1, 7: -1, 8: 0}[o]
    if flip == 1:
        im = im[:, ::-1]
    elif flip == 0:
        im = im[::-1]
    elif flip == -1:
        im = im[::-1, ::-1]
    return np.ascontiguousarray(im)


def pixels(p, coefs):
    """(out_h, out_w, 3) uint8 BGR from the coefficients."""
    pl = planes(p, coefs)
    y = pl[0][:p.height, :p.width]
    if p.ncomp == 1:
        im = np.repeat(y[:, :, None], 3, axis=2)
    else:
        im = ycc_to_bgr(y, upsample(p, pl[1]), upsample(p, pl[2]))
    return orient(im, p.orientation)


def decode(data, sync=None):
    """The oracle's decode of a device-decodable file: (out_h, out_w, 3) uint8 BGR, or None when its entropy data does not
    decode.  Raises ValueError for a file the device does not take (`Parsed.fallback`)."""
    p = data if isinstance(data, J.Parsed) else J.parse(data)
    if p.fallback:
        raise ValueError("not device-decodable: %s" % p.fallback)
    c = coefficients(p, sync)
    return None if c is None else pixels(p, c)
