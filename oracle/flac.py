"""Restatement of ``librosa.load(path, sr=..., mono=True)`` for FLAC files: librosa 0.9 reads them with
``soundfile.SoundFile(path).read(dtype='float32')`` -> libsndfile -> libFLAC, then ``to_mono`` and ``resample``
(res_type='kaiser_best', oracle/resample.py).  FLAC is lossless and integer-only, so the decoded samples are a pure function
of the bitstream; libsndfile scales them to float32 as x * 2^-(bps-1).

- ``decode``: a sequential FLAC decoder (frame by frame, as libFLAC walks a stream), strict: a CRC-8 or CRC-16 mismatch, a
  truncated frame, a reserved code, a gap or overlap in frame or sample numbers, or a length that differs from STREAMINFO
  raises ValueError naming the stream, 'FLAC' and the byte offset (libFLAC would resync and libsndfile pad instead).  An
  ID3v2 tag in front of 'fLaC' and metadata blocks other than STREAMINFO are skipped; the MD5 is not checked (libsndfile
  does not check it); bytes after the last frame are ignored once STREAMINFO's sample count is reached.
- ``encode``: a FLAC encoder that exists to make test vectors and can force every feature: CONSTANT / VERBATIM / FIXED 0-4 /
  LPC 1-32 subframes with any precision (1-15) and shift (0-15), Rice methods 0 and 1, escaped partitions, partition orders
  0-15, wasted bits, all four channel assignments, 1-8 channels, bps 4-24, fixed and variable blocking, block sizes 1-65535
  through every block-size code, every sample-rate code, metadata blocks of every type and an ID3v2 prefix.  Left to itself
  it picks the cheapest of those per subframe (like ``flac -5``: LPC order <= 8, partition order <= 5).
- ``load``: decode -> scale -> to_mono -> oracle.resample.resample.

Both are written from the FLAC format description (RFC 9639), with the frame loops compiled by numba.  NOT verified here:
no libFLAC, libsndfile or output of the reference encoder was available where this was written, so the decoder has only
been checked against this encoder and against frames assembled bit by bit in tests/test_flac_cpu.py.  Also unverified:
how libsndfile treats bit depths other than 8, 16 and 24 (this restatement scales every depth up to 24 the same way).

TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
from __future__ import annotations

import numba
import numpy as np

from . import resample as ors

BLOCK_TYPES = {'STREAMINFO': 0, 'PADDING': 1, 'APPLICATION': 2, 'SEEKTABLE': 3, 'VORBIS_COMMENT': 4, 'CUESHEET': 5,
               'PICTURE': 6}
SR_TABLE = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000, 11: 96000}
BPS_TABLE = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24}
CHANNEL_MODES = {'independent': -1, 'left_side': 8, 'side_right': 9, 'mid_side': 10}

# status codes (the device's SOME_FLAC_* values, plus the stream-level ones)
OK, TRUNCATED, BAD_CRC16, BAD_PADDING, RESERVED_SUBFRAME, BAD_WASTED, BAD_ORDER, BAD_LPC, BAD_RESIDUAL, BAD_PARTITION = range(10)
NO_HEADER = 10
REASONS = {TRUNCATED: 'truncated frame', BAD_CRC16: 'CRC-16 mismatch', BAD_PADDING: 'non-zero padding bits',
           RESERVED_SUBFRAME: 'reserved subframe type', BAD_WASTED: 'invalid wasted-bits count',
           BAD_ORDER: 'predictor order larger than the block', BAD_LPC: 'invalid LPC precision or shift',
           BAD_RESIDUAL: 'reserved residual coding method', BAD_PARTITION: 'invalid partition order',
           NO_HEADER: 'no valid frame header (sync, reserved code, CRC-8 or STREAMINFO mismatch)'}


def _crc_table(poly, width):
    top, mask = 1 << (width - 1), (1 << width) - 1
    t = np.zeros(256, np.int64)
    for i in range(256):
        c = i << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else (c << 1)
        t[i] = c & mask
    return t


CRC8_T, CRC16_T = _crc_table(0x07, 8), _crc_table(0x8005, 16)


@numba.njit(nogil=True)
def _crc8(data, a, b, t):
    c = 0
    for i in range(a, b):
        c = t[c ^ data[i]]
    return c


@numba.njit(nogil=True)
def _crc16(data, a, b, t):
    c = 0
    for i in range(a, b):
        c = ((c << 8) ^ t[((c >> 8) ^ data[i]) & 0xFF]) & 0xFFFF
    return c


def crc8(b: bytes) -> int:
    return int(_crc8(np.frombuffer(b, np.uint8), 0, len(b), CRC8_T))


def crc16(b: bytes) -> int:
    return int(_crc16(np.frombuffer(b, np.uint8), 0, len(b), CRC16_T))


# ---------------------------------------------------------------------------------------------- metadata
def id3_size(data: bytes) -> int:
    """Bytes of an ID3v2 tag at the start of data (0 if none): 10 + syncsafe size (+ 10 with the footer flag 0x10)."""
    if len(data) >= 10 and data[:3] == b'ID3':
        size = (data[6] & 0x7F) << 21 | (data[7] & 0x7F) << 14 | (data[8] & 0x7F) << 7 | (data[9] & 0x7F)
        return 10 + size + (10 if data[5] & 0x10 else 0)
    return 0


def parse_metadata(data: bytes, name='<stream>') -> dict:
    off = id3_size(data)
    if data[off:off + 4] != b'fLaC':
        raise ValueError(f'{name}: not a FLAC stream (no fLaC marker at byte offset {off})')
    p, info, first = off + 4, None, True
    while True:
        if p + 4 > len(data):
            raise ValueError(f'{name}: FLAC metadata block header truncated at byte offset {p}')
        last, kind, length = data[p] >> 7, data[p] & 0x7F, int.from_bytes(data[p + 1:p + 4], 'big')
        if first and (kind != 0 or length != 34):
            raise ValueError(f'{name}: FLAC stream does not start with a 34-byte STREAMINFO block at byte offset {p}')
        if kind == 127:
            raise ValueError(f'{name}: invalid FLAC metadata block type 127 at byte offset {p}')
        if p + 4 + length > len(data):
            raise ValueError(f'{name}: FLAC metadata block truncated at byte offset {p}')
        if kind == 0:
            if not first:
                raise ValueError(f'{name}: second FLAC STREAMINFO block at byte offset {p}')
            b = int.from_bytes(data[p + 4:p + 4 + 18], 'big')           # the 144 bits before the MD5
            info = dict(min_blocksize=b >> 128, max_blocksize=(b >> 112) & 0xFFFF, rate=(b >> 44) & 0xFFFFF,
                        channels=((b >> 41) & 7) + 1, bps=((b >> 36) & 31) + 1, total=b & ((1 << 36) - 1))
        first = False
        p += 4 + length
        if last:
            break
    if info['bps'] > 24:
        raise ValueError(f'{name}: FLAC streams with {info["bps"]} bits per sample are not supported (at most 24; '
                         f'STREAMINFO at byte offset {off + 8})')
    if info['rate'] == 0 or info['max_blocksize'] == 0:
        raise ValueError(f'{name}: invalid FLAC STREAMINFO at byte offset {off + 8}')
    info['audio_offset'] = p
    return info


# ---------------------------------------------------------------------------------------------- decoder
@numba.njit(nogil=True)
def _bits(data, pos, lim, n):
    """(value of the n <= 32 bits at bit position pos, MSB first; past lim bytes reads zeros), new pos, overrun flag"""
    v = 0
    over = False
    while n > 0:
        byte, off = pos >> 3, pos & 7
        c = min(8 - off, n)
        b = 0
        if byte < lim:
            b = data[byte]
        else:
            over = True
        v = (v << c) | ((b >> (8 - off - c)) & ((1 << c) - 1))
        pos += c
        n -= c
    return v, pos, over


@numba.njit(nogil=True)
def _signed(v, n):
    if n == 0:
        return 0
    if v >= (1 << (n - 1)):
        v -= 1 << n
    return v


@numba.njit(nogil=True)
def _header(data, p, lim, channels, bps, max_bs, t8):
    """-> (ok, header_len, blocksize, chan_code, number, variable)"""
    if p + 6 > lim or data[p] != 0xFF or (data[p + 1] & 0xFE) != 0xF8:
        return False, 0, 0, 0, 0, 0
    variable = data[p + 1] & 1
    bs_code, sr_code = data[p + 2] >> 4, data[p + 2] & 15
    ch_code, bps_code = data[p + 3] >> 4, (data[p + 3] >> 1) & 7
    if bs_code == 0 or sr_code == 15 or ch_code > 10 or bps_code == 3 or bps_code == 7 or (data[p + 3] & 1):
        return False, 0, 0, 0, 0, 0
    q = p + 4
    x = data[q]
    q += 1
    if x < 0x80:
        num, extra = x, 0
    elif 0xC0 <= x < 0xE0:
        num, extra = x & 0x1F, 1
    elif 0xE0 <= x < 0xF0:
        num, extra = x & 0x0F, 2
    elif 0xF0 <= x < 0xF8:
        num, extra = x & 0x07, 3
    elif 0xF8 <= x < 0xFC:
        num, extra = x & 0x03, 4
    elif 0xFC <= x < 0xFE:
        num, extra = x & 0x01, 5
    elif x == 0xFE and variable:
        num, extra = 0, 6
    else:
        return False, 0, 0, 0, 0, 0
    if q + extra > lim:
        return False, 0, 0, 0, 0, 0
    for _ in range(extra):
        c = data[q]
        q += 1
        if (c & 0xC0) != 0x80:
            return False, 0, 0, 0, 0, 0
        num = (num << 6) | (c & 0x3F)
    nb = 1 if bs_code == 6 else (2 if bs_code == 7 else 0)
    ns = 1 if sr_code == 12 else (2 if sr_code == 13 or sr_code == 14 else 0)
    if q + nb + ns + 1 > lim:
        return False, 0, 0, 0, 0, 0
    if bs_code == 1:
        bs = 192
    elif bs_code <= 5:
        bs = 576 << (bs_code - 2)
    elif bs_code >= 8:
        bs = 256 << (bs_code - 8)
    elif bs_code == 6:
        bs = data[q] + 1
    else:
        bs = (data[q] << 8 | data[q + 1]) + 1
    q += nb + ns
    if _crc8(data, p, q, t8) != data[q]:
        return False, 0, 0, 0, 0, 0
    ch = ch_code + 1 if ch_code < 8 else 2
    fb = bps if bps_code == 0 else (8 if bps_code == 1 else (12 if bps_code == 2 else bps_code * 4))
    if ch != channels or fb != bps or bs > max_bs:
        return False, 0, 0, 0, 0, 0
    return True, q + 1 - p, bs, ch_code, num, variable


@numba.njit(nogil=True)
def _unary(data, pos, lim):
    q = 0
    while True:
        if (pos >> 3) >= lim:
            return q, pos, True
        if (pos & 7) == 0 and data[pos >> 3] == 0:
            q += 8
            pos += 8
            continue
        if (data[pos >> 3] >> (7 - (pos & 7))) & 1:
            return q, pos + 1, False
        q += 1
        pos += 1


@numba.njit(nogil=True)
def _residual(data, pos, lim, bs, order, out):
    """-> (status, pos); out[order:bs] = residuals"""
    method, pos, o1 = _bits(data, pos, lim, 2)
    if method > 1:
        return BAD_RESIDUAL, pos
    pbits, esc = (5, 31) if method else (4, 15)
    porder, pos, o2 = _bits(data, pos, lim, 4)
    psize = bs >> porder
    if (psize << porder) != bs or psize < order:
        return BAD_PARTITION, pos
    i = order
    for part in range(1 << porder):
        k, pos, ov = _bits(data, pos, lim, pbits)
        stop = (part + 1) * psize
        if k == esc:
            w, pos, ov = _bits(data, pos, lim, 5)
            while i < stop:
                v, pos, ov2 = _bits(data, pos, lim, w)
                out[i] = _signed(v, w)
                i += 1
                if ov2:
                    return TRUNCATED, pos
        else:
            while i < stop:
                q, pos, ov2 = _unary(data, pos, lim)
                low, pos, ov3 = _bits(data, pos, lim, k)
                if ov2 or ov3:
                    return TRUNCATED, pos
                u = ((q << k) | low) & 0xFFFFFFFF
                out[i] = (u >> 1) ^ -(u & 1)
                i += 1
        if ov:
            return TRUNCATED, pos
    return OK, pos


@numba.njit(nogil=True)
def _subframe(data, pos, lim, bs, sbps, out):
    """-> (status, pos); out[:bs] = samples (int64, wrapped to int32 like the device)"""
    pad, pos, ov = _bits(data, pos, lim, 1)
    if pad:
        return BAD_PADDING, pos
    kind, pos, ov = _bits(data, pos, lim, 6)
    flag, pos, ov = _bits(data, pos, lim, 1)
    wasted = 0
    if flag:
        q, pos, ov = _unary(data, pos, lim)
        wasted = q + 1
        if wasted >= sbps:
            return BAD_WASTED, pos
    b = sbps - wasted
    if ov:
        return TRUNCATED, pos
    if kind == 0:
        v, pos, ov = _bits(data, pos, lim, b)
        out[:bs] = _signed(v, b)
    elif kind == 1:
        for i in range(bs):
            v, pos, ov = _bits(data, pos, lim, b)
            out[i] = _signed(v, b)
    elif (kind & 0x38) == 0x08 or kind & 0x20:
        lpc = bool(kind & 0x20)
        order = (kind & 31) + 1 if lpc else kind & 7
        if not lpc and order > 4:
            return RESERVED_SUBFRAME, pos
        if order > bs:
            return BAD_ORDER, pos
        for i in range(order):
            v, pos, ov = _bits(data, pos, lim, b)
            out[i] = _signed(v, b)
        coef = np.zeros(32, np.int64)
        shift = 0
        if lpc:
            prec, pos, ov = _bits(data, pos, lim, 4)
            prec += 1
            if prec == 16:
                return BAD_LPC, pos
            s, pos, ov = _bits(data, pos, lim, 5)
            shift = _signed(s, 5)
            if shift < 0:
                return BAD_LPC, pos
            for j in range(order):
                c, pos, ov = _bits(data, pos, lim, prec)
                coef[j] = _signed(c, prec)
        else:
            fixed = ((0, 0, 0, 0), (1, 0, 0, 0), (2, -1, 0, 0), (3, -3, 1, 0), (4, -6, 4, -1))
            for j in range(order):
                coef[j] = fixed[order][j]
        st, pos = _residual(data, pos, lim, bs, order, out)
        if st != OK:
            return st, pos
        for i in range(order, bs):
            acc = 0
            for j in range(order):
                acc += coef[j] * out[i - 1 - j]
            v = out[i] + (acc >> shift)
            out[i] = ((v + 2 ** 31) & 0xFFFFFFFF) - 2 ** 31
    else:
        return RESERVED_SUBFRAME, pos
    if ov or (pos >> 3) > lim:
        return TRUNCATED, pos
    if wasted:
        for i in range(bs):
            out[i] = (((out[i] << wasted) + 2 ** 31) & 0xFFFFFFFF) - 2 ** 31
    return OK, pos


@numba.njit(nogil=True)
def _frame(data, p, lim, channels, bps, max_bs, out, t8, t16):
    """Decodes the frame at byte p into out[:channels, :blocksize].
    -> (status, end or problem byte, blocksize, number, variable)"""
    ok, hlen, bs, ch_code, num, variable = _header(data, p, lim, channels, bps, max_bs, t8)
    if not ok:
        return NO_HEADER, p, 0, 0, 0
    pos = (p + hlen) * 8
    for c in range(channels):
        side = (ch_code == 8 and c == 1) or (ch_code == 9 and c == 0) or (ch_code == 10 and c == 1)
        st, pos = _subframe(data, pos, lim, bs, bps + (1 if side else 0), out[c])
        if st != OK:
            return st, min(pos >> 3, lim), bs, num, variable
    padn = (8 - (pos & 7)) & 7
    pad, pos, ov = _bits(data, pos, lim, padn)
    if pad:
        return BAD_PADDING, min(pos >> 3, lim), bs, num, variable
    want, pos, ov2 = _bits(data, pos, lim, 16)
    if ov or ov2:
        return TRUNCATED, lim, bs, num, variable
    end = pos >> 3
    if _crc16(data, p, end - 2, t16) != want:
        return BAD_CRC16, end, bs, num, variable
    if ch_code >= 8:
        for i in range(bs):
            a, s = out[0, i], out[1, i]
            if ch_code == 8:
                out[1, i] = a - s
            elif ch_code == 9:
                out[0, i] = a + s
            else:
                m = (a << 1) | (s & 1)
                out[0, i] = (m + s) >> 1
                out[1, i] = (m - s) >> 1
    return OK, end, bs, num, variable


def decode(data: bytes, name='<stream>'):
    """(int32 samples [n, channels], metadata dict) of a FLAC stream, decoded frame by frame."""
    info = parse_metadata(data, name)
    buf = np.frombuffer(data, np.uint8)
    lim, ch, bps, total, max_bs = len(data), info['channels'], info['bps'], info['total'], info['max_blocksize']
    scratch = np.zeros((ch, max(max_bs, 1)), np.int64)
    pieces, got, k, pos, strategy = [], 0, 0, info['audio_offset'], None
    while not (total and got == total) and not (not total and pos == lim):
        if pos >= lim:
            raise ValueError(f'{name}: FLAC stream ends at byte offset {pos} after {got} of {total} samples')
        st, end, bs, num, variable = _frame(buf, pos, lim, ch, bps, max_bs, scratch, CRC8_T, CRC16_T)
        if st != OK:
            raise ValueError(f'{name}: FLAC frame at byte offset {pos}: {REASONS[st]} (at byte offset {end})')
        if strategy is None:
            strategy = variable
        want = got if variable else k
        if variable != strategy or num != want:
            raise ValueError(f'{name}: FLAC frame at byte offset {pos}: {"sample" if variable else "frame"} number {num}, '
                             f'expected {want} (gap, overlap or changed blocking strategy)')
        got += bs
        if total and got > total:
            raise ValueError(f'{name}: FLAC frame at byte offset {pos} decodes past STREAMINFO\'s {total} samples')
        pieces.append(scratch[:, :bs].T.astype(np.int32))
        k += 1
        pos = end
    x = np.concatenate(pieces) if pieces else np.zeros((0, ch), np.int32)
    return np.ascontiguousarray(x), info                                # [n, ch] C order, as soundfile returns it


def scale(x: np.ndarray, bps: int) -> np.ndarray:
    """libsndfile's integer -> float32: x * 2^-(bps-1)"""
    return x.astype(np.float32) * np.float32(2.0 ** -(bps - 1))


def decode_file(path):
    """(float32 [n] (mono) or [n, channels], rate) as soundfile hands them to librosa.load."""
    with open(path, 'rb') as f:
        data = f.read()
    x, info = decode(data, str(path))
    y = scale(x, info['bps'])
    return (y[:, 0].copy() if info['channels'] == 1 else y), info['rate']


def load(path, sr=22050, mono=True):
    """librosa.load(path, sr=sr, mono=mono, res_type='kaiser_best') for FLAC files; returns (y, sr)."""
    x, native = decode_file(path)
    y = x.T
    if mono and y.ndim > 1:
        y = np.mean(y, axis=0)                                            # librosa.to_mono
    if sr is not None and sr != native:
        if y.ndim > 1:
            y = np.stack([ors.resample(np.ascontiguousarray(c), native, sr) for c in y])
        else:
            y = ors.resample(np.ascontiguousarray(y), native, sr)
        return y, sr
    return y, native


# ---------------------------------------------------------------------------------------------- encoder
@numba.njit(nogil=True)
def _put(buf, pos, value, n):
    value &= (1 << n) - 1 if n < 63 else -1
    while n > 0:
        room = 8 - (pos & 7)
        c = min(room, n)
        buf[pos >> 3] |= ((value >> (n - c)) & ((1 << c) - 1)) << (room - c)
        pos += c
        n -= c
    return pos


@numba.njit(nogil=True)
def _zigzag(r):
    return (r << 1) ^ (r >> 63)


@numba.njit(nogil=True)
def _part_cost(res, a, b, k):
    c = (b - a) * (k + 1)
    for i in range(a, b):
        c += _zigzag(res[i]) >> k
    return c


@numba.njit(nogil=True)
def _escape_width(res, a, b):
    w = 0
    for i in range(a, b):
        r = res[i]
        m = r if r >= 0 else -r - 1
        n = 1
        while m >> (n - 1):
            n += 1
        if m or r < 0:
            w = max(w, n)
    return w


@numba.njit(nogil=True)
def _plan_partitions(res, bs, order, porder, method, params):
    """Cheapest Rice parameter (or escape, params = -(width + 1)) per partition for a fixed method and order;
    returns the bits of the residual section."""
    kmax, pbits = (30, 5) if method else (14, 4)
    psize = bs >> porder
    bits = 6
    for part in range(1 << porder):
        a, b = max(part * psize, order), (part + 1) * psize
        s = 0
        for i in range(a, b):
            s += _zigzag(res[i])
        mean = s // max(b - a, 1)
        k0 = 0
        while k0 < kmax and (mean >> (k0 + 1)):
            k0 += 1
        best, bk = -1, 0
        for k in range(max(0, k0 - 1), min(kmax, k0 + 1) + 1):
            c = _part_cost(res, a, b, k)
            if best < 0 or c < best:
                best, bk = c, k
        w = _escape_width(res, a, b)
        esc = 5 + (b - a) * w
        if esc < best:
            best, bk = esc, -(w + 1)
        params[part] = bk
        bits += pbits + best
    return bits


@numba.njit(nogil=True)
def _params_bits(res, bs, order, porder, method, params):
    psize = bs >> porder
    bits = 6
    for part in range(1 << porder):
        a, b = max(part * psize, order), (part + 1) * psize
        k = params[part]
        bits += (5 if method else 4) + (5 + (b - a) * (-k - 1) if k < 0 else _part_cost(res, a, b, k))
    return bits


@numba.njit(nogil=True)
def _best_k(res, a, b, kmax):
    best, bk = -1, 0
    for k in range(kmax + 1):
        c = _part_cost(res, a, b, k)
        if best < 0 or c < best:
            best, bk = c, k
    return bk


@numba.njit(nogil=True)
def _write_residual(buf, pos, res, bs, order, method, porder, params):
    pos = _put(buf, pos, method, 2)
    pos = _put(buf, pos, porder, 4)
    pbits, esc = (5, 31) if method else (4, 15)
    psize = bs >> porder
    for part in range(1 << porder):
        a, b = max(part * psize, order), (part + 1) * psize
        k = params[part]
        if k < 0:
            w = -k - 1
            pos = _put(buf, pos, esc, pbits)
            pos = _put(buf, pos, w, 5)
            for i in range(a, b):
                pos = _put(buf, pos, res[i], w)
        else:
            pos = _put(buf, pos, k, pbits)
            for i in range(a, b):
                u = _zigzag(res[i])
                pos += u >> k                                          # the zeros are already in buf
                pos = _put(buf, pos, 1, 1)
                pos = _put(buf, pos, u & ((1 << k) - 1), k)
    return pos


@numba.njit(nogil=True)
def _predict_residual(x, order, coef, shift, res):
    """res[i] = x[i] - ((sum_j coef[j] x[i-1-j]) >> shift) for i >= order (64-bit sums)"""
    for i in range(order):
        res[i] = 0
    for i in range(order, x.shape[0]):
        acc = 0
        for j in range(order):
            acc += coef[j] * x[i - 1 - j]
        res[i] = x[i] - (acc >> shift)


@numba.njit(nogil=True)
def _lpc(x, order):
    """Float LPC coefficients (autocorrelation + Levinson-Durbin, Welch window), predicting x[i] from x[i-1-j]."""
    n = x.shape[0]
    w = np.empty(n)
    for i in range(n):
        t = (2.0 * i - (n - 1)) / (n + 1)
        w[i] = x[i] * (1.0 - t * t)
    r = np.zeros(order + 1)
    for lag in range(order + 1):
        s = 0.0
        for i in range(lag, n):
            s += w[i] * w[i - lag]
        r[lag] = s
    a = np.zeros(order)
    if r[0] <= 0:
        return a
    r[0] *= 1.0 + 1e-9
    err = r[0]
    tmp = np.zeros(order)
    for m in range(order):
        acc = r[m + 1]
        for j in range(m):
            acc -= a[j] * r[m - j]
        k = acc / err
        for j in range(m):
            tmp[j] = a[j] - k * a[m - 1 - j]
        for j in range(m):
            a[j] = tmp[j]
        a[m] = k
        err *= 1.0 - k * k
        if err <= 0:
            break
    return a


def _quantize(a, precision, shift=None):
    cmax = float(np.max(np.abs(a))) if len(a) else 0.0
    if shift is None:
        log2c = int(np.frexp(cmax)[1]) if cmax > 0 else 0
        shift = min(15, max(0, precision - 1 - log2c))
    lo, hi = -(1 << (precision - 1)), (1 << (precision - 1)) - 1
    q, e = np.zeros(len(a), np.int64), 0.0
    for j, c in enumerate(a):                                          # with error feedback, like libFLAC
        e += c * (1 << shift)
        q[j] = min(hi, max(lo, int(np.round(e))))
        e -= q[j]
    return q, shift


FIXED_COEFS = [[], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1]]


def _valid_porders(bs, order, max_porder):
    return [p for p in range(0, max_porder + 1) if (bs >> p) << p == bs and (bs >> p) >= order and (p == 0 or bs >> p > 0)]


def _subframe_plan(x, sbps, spec, max_lpc_order, max_porder):
    """Chooses (or forces, spec) one subframe's coding; returns (bits, writer args)."""
    spec = dict(spec or {})
    bs = len(x)
    wasted = spec.get('wasted')
    if wasted is None:
        acc = int(np.bitwise_or.reduce(x.astype(np.int64))) if bs else 0
        wasted = 0
        if acc:
            while not (acc >> wasted) & 1 and wasted < sbps - 1:
                wasted += 1
    if wasted and np.any(x.astype(np.int64) & ((1 << wasted) - 1)):
        raise ValueError(f'encode: samples are not multiples of 2^{wasted}')
    xs = (x.astype(np.int64) >> wasted)
    b = sbps - wasted
    lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
    if xs.min(initial=0) < lo or xs.max(initial=0) > hi:
        raise ValueError(f'encode: samples do not fit {sbps} bits')
    head = 8 + (wasted if wasted else 0)
    kind = spec.get('type')
    cands = []

    def residual_plan(order, coef, shift, extra_bits, tag):
        res = np.zeros(bs, np.int64)
        _predict_residual(xs, order, np.asarray(coef, np.int64), shift, res)
        if np.abs(res).max(initial=0) >= 1 << 30:
            return None                                                # not representable (escape width <= 31 bits)
        methods = [spec['method']] if 'method' in spec else [0, 1]
        porders = _valid_porders(bs, order, spec.get('porder', max_porder))
        if 'porder' in spec:                                           # the forced order, or the largest this block allows
            porders = porders[-1:]
        best = None
        for m in methods:
            for p in porders:
                params = np.zeros(1 << p, np.int64)
                bits = _plan_partitions(res, bs, order, p, m, params)
                esc = spec.get('escape')
                if esc is not None:                                    # force (True: all; list: those) partitions escaped
                    psize = bs >> p
                    for part in (range(1 << p) if esc is True else [e for e in esc if e < 1 << p]):
                        a, e = max(part * psize, order), (part + 1) * psize
                        params[part] = -(_escape_width(res, a, e) + 1)
                    if esc is False:
                        for part in range(1 << p):
                            if params[part] < 0:
                                params[part] = _best_k(res, max(part * psize, order), (part + 1) * psize, 30 if m else 14)
                    bits = _params_bits(res, bs, order, p, m, params)
                if m == 0 and np.any(params > 14):
                    continue
                if best is None or bits < best[0]:
                    best = (bits, m, p, params)
        if best is None:
            return None
        bits, m, p, params = best
        return (head + order * b + extra_bits + bits, tag, order, coef, shift, res, m, p, params, xs)

    if kind in (None, 'constant') and bs and np.all(xs == xs[0]):
        cands.append((head + b, 'constant', 0, None, 0, xs, 0, 0, None, xs))
    elif kind == 'constant':
        raise ValueError('encode: CONSTANT subframe of non-constant samples')
    if kind in (None, 'verbatim'):
        cands.append((head + bs * b, 'verbatim', 0, None, 0, xs, 0, 0, None, xs))
    if kind in (None, 'fixed'):
        orders = [spec['order']] if 'order' in spec else range(min(4, bs) + 1)
        for o in orders:
            c = residual_plan(o, FIXED_COEFS[o], 0, 0, 'fixed')
            if c is not None:
                cands.append(c)
    if kind in (None, 'lpc') and bs > 1:
        orders = [spec['order']] if 'order' in spec else [min(max_lpc_order, bs - 1)] if max_lpc_order else []
        for o in orders:
            prec = spec.get('precision', 15 if b > 16 else 12 if bs > 1152 else 10)
            coef, shift = _quantize(_lpc(xs.astype(np.float64), o), prec, spec.get('shift'))
            c = residual_plan(o, coef, shift, 4 + 5 + o * prec, ('lpc', prec))
            if c is not None:
                cands.append(c)
    if not cands:
        raise ValueError(f'encode: the forced subframe {spec} cannot code these samples')
    return min(cands, key=lambda c: c[0]), wasted, b


def _write_subframe(buf, pos, plan, wasted, b):
    bits, tag, order, coef, shift, res, m, p, params, xs = plan
    kind = tag[0] if isinstance(tag, tuple) else tag
    code = {'constant': 0, 'verbatim': 1}.get(kind, 8 + order if kind == 'fixed' else 32 + order - 1)
    pos = _put(buf, pos, code << 1 | (1 if wasted else 0), 8)
    if wasted:
        pos = _put(buf, pos, 1, wasted)                                 # wasted - 1 zeros, then a 1
    if kind == 'constant':
        return _put(buf, pos, int(xs[0]), b)
    n = len(xs) if kind == 'verbatim' else order
    for i in range(n):                                                 # every sample, or the warm-up samples
        pos = _put(buf, pos, int(xs[i]), b)
    if kind == 'lpc':
        prec = tag[1]
        pos = _put(buf, pos, prec - 1, 4)
        pos = _put(buf, pos, shift, 5)
        for c in coef:
            pos = _put(buf, pos, int(c), prec)
    if kind in ('fixed', 'lpc'):
        pos = _write_residual(buf, pos, res, len(res), order, m, p, params)
    return pos


def _utf8(v: int, variable: bool) -> bytes:
    if v < 0x80:
        return bytes([v])
    for n in range(2, 8):
        if v < 1 << (5 * n + 1) or n == 7:
            break
    if n == 7 and not variable or v >= 1 << 36:
        raise ValueError(f'encode: frame/sample number {v} cannot be coded')
    out = [0x80 | ((v >> (6 * i)) & 0x3F) for i in range(n - 1)][::-1]
    first = (0xFF << (8 - n)) & 0xFF | (v >> (6 * (n - 1)))
    return bytes([first & 0xFF] + out)


def _bs_code(bs, force):
    if force in (6, 7):
        return force
    if bs == 192:
        return 1
    for c in range(2, 6):
        if bs == 576 << (c - 2):
            return c
    for c in range(8, 16):
        if bs == 256 << (c - 8):
            return c
    return 6 if bs <= 256 else 7


def _sr_code(rate, force):
    if force is None:
        for c, r in SR_TABLE.items():
            if r == rate:
                return c
        force = 12 if rate % 1000 == 0 and rate // 1000 < 256 else 13 if rate < 65536 else 14 if rate % 10 == 0 and rate // 10 < 65536 else 0
    if force in SR_TABLE and SR_TABLE[force] != rate or force == 12 and (rate % 1000 or rate >= 256000) or \
            force == 13 and rate >= 65536 or force == 14 and (rate % 10 or rate >= 655360):
        raise ValueError(f'encode: sample-rate code {force} cannot give {rate} Hz')
    return force


def _frame_bytes(x, rate, bps, number, variable, ch_code, spec, max_lpc_order, max_porder, bs_force, sr_force, bps_code0):
    bs, ch = x.shape
    bsc, src = _bs_code(bs, bs_force), _sr_code(rate, sr_force)
    bpc = 0 if bps_code0 or bps not in BPS_TABLE.values() else {v: k for k, v in BPS_TABLE.items()}[bps]
    cc = ch - 1 if ch_code < 0 else ch_code
    head = bytearray([0xFF, 0xF8 | int(variable), bsc << 4 | src, cc << 4 | bpc << 1])
    head += _utf8(number, variable)
    if bsc == 6:
        head += bytes([bs - 1])
    elif bsc == 7:
        head += (bs - 1).to_bytes(2, 'big')
    if src == 12:
        head += bytes([rate // 1000])
    elif src == 13:
        head += rate.to_bytes(2, 'big')
    elif src == 14:
        head += (rate // 10).to_bytes(2, 'big')
    head += bytes([crc8(bytes(head))])
    xs = x.astype(np.int64)
    chans = [xs[:, c] for c in range(ch)]
    sb = [bps] * ch
    if cc == 8:
        chans, sb = [xs[:, 0], xs[:, 0] - xs[:, 1]], [bps, bps + 1]
    elif cc == 9:
        chans, sb = [xs[:, 0] - xs[:, 1], xs[:, 1]], [bps + 1, bps]
    elif cc == 10:
        chans, sb = [(xs[:, 0] + xs[:, 1]) >> 1, xs[:, 0] - xs[:, 1]], [bps, bps + 1]
    plans = [_subframe_plan(c, s, spec(c_i) if callable(spec) else spec, max_lpc_order, max_porder)
             for c_i, (c, s) in enumerate(zip(chans, sb))]
    nbits = len(head) * 8 + sum(p[0][0] for p in plans) + 8 + 16
    buf = np.zeros(nbits // 8 + 16, np.uint8)
    buf[:len(head)] = np.frombuffer(bytes(head), np.uint8)
    pos = len(head) * 8
    for plan, wasted, b in plans:
        pos = _write_subframe(buf, pos, plan, wasted, b)
    end = (pos + 7) >> 3
    body = buf[:end].tobytes()
    return body + crc16(body).to_bytes(2, 'big')


def id3_tag(body: bytes = b'TIT2\x00\x00\x00\x05\x00\x00test', footer: bool = False) -> bytes:
    """An ID3v2.4 tag (10-byte header, syncsafe size, optional 10-byte footer) around ``body``."""
    n = len(body)
    size = bytes([(n >> 21) & 0x7F, (n >> 14) & 0x7F, (n >> 7) & 0x7F, n & 0x7F])
    flags = 0x10 if footer else 0
    tag = b'ID3\x04\x00' + bytes([flags]) + size + body
    return tag + (b'3DI\x04\x00' + bytes([flags]) + size if footer else b'')


def encode(x, rate: int, bps: int, *, blocksize=4096, variable=False, channel_mode='independent', subframe=None,
           max_lpc_order=8, max_porder=5, metadata=(), id3=None, total_samples=None, min_blocksize=None,
           max_blocksize=None, bs_code=None, sr_code=None, bps_code0=False, frame_numbers=None) -> bytes:
    """FLAC bytes for integer samples ``x`` [n] or [n, channels] (each within ``bps`` signed bits).

    blocksize: an int (fixed blocking, the last frame shorter) or a list of block sizes (summing to n).
    variable: variable blocking (coded sample numbers) instead of fixed (coded frame numbers).
    channel_mode: 'independent', 'left_side', 'side_right' or 'mid_side' (the last three for 2 channels).
    subframe: None (cheapest), a dict forcing the coding of every subframe, or f(frame, channel) -> dict.  Keys: type
      ('constant' | 'verbatim' | 'fixed' | 'lpc'), order, precision, shift, method (0/1), porder, escape (True / list
      of partitions / False), wasted (bits).
    metadata: [(type name or number, payload bytes)] blocks after STREAMINFO.  id3: bytes put in front of 'fLaC'.
    total_samples / min_blocksize / max_blocksize: STREAMINFO overrides (total 0 = unknown).
    bs_code: 6 or 7 forces an explicit block size; sr_code forces a sample-rate code (0, 1-11, 12, 13, 14);
    bps_code0: the frame headers take bps from STREAMINFO.  frame_numbers: overrides the coded numbers."""
    x = np.asarray(x)
    if x.ndim == 1:
        x = x[:, None]
    n, ch = x.shape
    if not (1 <= ch <= 8 and 4 <= bps <= 24):
        raise ValueError('encode: 1-8 channels of 4-24 bits')
    sizes = list(blocksize) if not np.isscalar(blocksize) else [min(blocksize, n - a) for a in range(0, n, blocksize)]
    assert sum(sizes) == n and all(1 <= s <= 65535 for s in sizes)
    ch_code = CHANNEL_MODES[channel_mode]
    assert ch_code < 0 or ch == 2, 'stereo decorrelation needs 2 channels'
    frames, a = [], 0
    for k, s in enumerate(sizes):
        num = frame_numbers[k] if frame_numbers is not None else (a if variable else k)
        spec = (lambda c, k=k: subframe(k, c)) if callable(subframe) else subframe
        frames.append(_frame_bytes(x[a:a + s], rate, bps, num, variable, ch_code, spec, max_lpc_order, max_porder,
                                   bs_code, sr_code, bps_code0))
        a += s
    mn = min_blocksize if min_blocksize is not None else (min(sizes) if variable or len(sizes) == 1 else max(sizes))
    mx = max_blocksize if max_blocksize is not None else max(sizes, default=16)
    total = n if total_samples is None else total_samples
    fmin, fmax = min(map(len, frames), default=0), max(map(len, frames), default=0)
    si = (mn << 128 | mx << 112 | fmin << 88 | fmax << 64 | rate << 44 | (ch - 1) << 41 | (bps - 1) << 36 | total)
    blocks = [(0, si.to_bytes(18, 'big') + bytes(16))] + [(BLOCK_TYPES.get(t, t), bytes(p)) for t, p in metadata]
    out = bytearray(id3 or b'') + b'fLaC'
    for i, (t, p) in enumerate(blocks):
        out += bytes([(0x80 if i == len(blocks) - 1 else 0) | t]) + len(p).to_bytes(3, 'big') + p
    return bytes(out) + b''.join(frames)


# ---------------------------------------------------------------------------------------------- test vectors
def test_signal(n: int, channels: int, bps: int, seed: int, level: float = 0.4) -> np.ndarray:
    """int64 [n, channels]: a few sines plus noise at ``level`` of full scale, different per channel."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    full = (1 << (bps - 1)) - 1
    out = np.empty((n, channels), np.int64)
    for c in range(channels):
        f = rng.uniform(0.002, 0.05, 3)
        y = sum(np.sin(2 * np.pi * fi * t + rng.uniform(0, 6)) for fi in f) / 3 + rng.normal(0, 0.02, n)
        out[:, c] = np.clip(np.round(level * full * y), -full - 1, full)
    return out


def feature_cases():
    """[(name, samples [n, ch], encode kwargs)] covering every feature encode() can force."""
    cases = []
    add = lambda name, x, **kw: cases.append((name, x, kw))                 # noqa: E731
    s16 = test_signal(5000, 2, 16, 1)
    m16 = s16[:, :1]
    add('constant', np.full((3000, 1), -1234, np.int64), rate=44100, bps=16, subframe={'type': 'constant'})
    add('verbatim', m16, rate=44100, bps=16, subframe={'type': 'verbatim'})
    for o in range(5):
        add(f'fixed{o}', m16, rate=44100, bps=16, subframe={'type': 'fixed', 'order': o})
    for o in range(1, 33):
        add(f'lpc{o}', test_signal(1500, 1, 16, o), rate=44100, bps=16, blocksize=750,
            subframe={'type': 'lpc', 'order': o, 'precision': 15 - (o % 15), 'shift': o % 16})
    add('lpc_shift0', m16, rate=44100, bps=16, subframe={'type': 'lpc', 'order': 2, 'precision': 15, 'shift': 0})
    add('lpc_prec1', m16, rate=44100, bps=16, subframe={'type': 'lpc', 'order': 4, 'precision': 1, 'shift': 3})
    for m in (0, 1):
        add(f'rice{m}', m16, rate=44100, bps=16, subframe={'type': 'fixed', 'order': 2, 'method': m})
        add(f'escape_all{m}', m16, rate=44100, bps=16, subframe={'type': 'fixed', 'order': 1, 'method': m, 'porder': 3,
                                                                 'escape': True})
    add('escape_some', m16, rate=44100, bps=16, blocksize=4096,
        subframe={'type': 'lpc', 'order': 6, 'porder': 4, 'escape': [0, 5, 15]})
    add('escape_zero', np.concatenate([np.zeros((2048, 1), np.int64), m16[:2048]]), rate=44100, bps=16, blocksize=4096,
        subframe={'type': 'fixed', 'order': 0, 'porder': 1, 'escape': [0]})
    for p in range(9):
        add(f'porder{p}', m16, rate=44100, bps=16, blocksize=4096, subframe={'type': 'fixed', 'order': 2, 'porder': p})
    for k in (1, 3, 7):
        add(f'wasted{k}', (m16 >> k) << k, rate=44100, bps=16)
    add('wasted_forced', (s16 >> 2) << 2, rate=44100, bps=16, subframe={'wasted': 2, 'type': 'lpc', 'order': 3})
    for mode in CHANNEL_MODES:
        add(f'stereo_{mode}', s16, rate=48000, bps=16, channel_mode=mode)
        add(f'stereo24_{mode}', test_signal(5000, 2, 24, 3, level=0.9), rate=48000, bps=24, channel_mode=mode)
    for ch in range(1, 9):
        add(f'channels{ch}', test_signal(3000, ch, 16, 10 + ch), rate=32000, bps=16)
    for bps in range(4, 25):
        add(f'bps{bps}', test_signal(2500, 2, bps, 40 + bps), rate=44100, bps=bps, channel_mode='mid_side',
            bps_code0=bps == 16)
    add('variable', s16, rate=44100, bps=16, variable=True, blocksize=[1, 700, 192, 2000, 2107])
    add('fixed_short_last', s16[:4097], rate=44100, bps=16, blocksize=1024)
    for bs in (1, 17, 192, 256, 576, 1152, 2304, 4608, 512, 1024, 2048, 8192, 16384, 32768):
        add(f'bs{bs}', test_signal(min(max(bs * 2, 40), 40000), 1, 12, bs), rate=8000, bps=12, blocksize=bs)
    add('bs_explicit8', m16[:2000], rate=44100, bps=16, blocksize=200)
    add('bs_explicit8_forced', m16[:1000], rate=44100, bps=16, blocksize=192, bs_code=6)
    add('bs_explicit16', m16[:3000], rate=44100, bps=16, blocksize=1000)
    add('bs_explicit16_forced', m16[:1000], rate=44100, bps=16, blocksize=256, bs_code=7)
    add('bs65535', test_signal(70000, 1, 8, 5), rate=44100, bps=8, blocksize=65535)
    for code, rate in SR_TABLE.items():
        add(f'sr_code{code}', m16[:1000], rate=rate, bps=16, blocksize=500)
    add('sr_code0', m16[:1000], rate=44100, bps=16, sr_code=0)
    add('sr_code12', m16[:1000], rate=11000, bps=16)
    add('sr_code13', m16[:1000], rate=11025, bps=16)
    add('sr_code14', m16[:1000], rate=100000, bps=16, sr_code=14)
    add('metadata', s16, rate=44100, bps=16, metadata=[
        ('PADDING', bytes(100)), ('APPLICATION', b'abcd' + bytes(8)), ('SEEKTABLE', bytes(18 * 2)),
        ('VORBIS_COMMENT', b'\x05\x00\x00\x00hello\x00\x00\x00\x00'), ('CUESHEET', bytes(396)),
        ('PICTURE', bytes(32) + b'\xff\xf8\xc9\x08\x00\x00' * 4), (99, b'unknown')])
    add('id3', s16, rate=44100, bps=16, id3=id3_tag())
    add('id3_footer', s16, rate=44100, bps=16, id3=id3_tag(footer=True))
    add('total_unknown', s16, rate=44100, bps=16, total_samples=0)
    return cases
