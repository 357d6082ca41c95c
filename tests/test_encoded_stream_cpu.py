"""CPU tests of the resumable halves of encoded streams (csrc/audio_host.cu; the library loads without a GPU): the container
walk fed in pieces (some_audio_walk_*) against some_audio_info on the whole file, and the FLAC chain continued window by
window (some_flac_chain_resume) against the whole-list walk."""
import ctypes as C
import struct

import numpy as np
import pytest

import test_encoded_cpu as tc
from oracle import flac as of
from some_b200 import _lib

lib = _lib.load()
META = [name for name, _ in _lib.AudioMeta._fields_ if name != 'reserved']


def whole(data: bytes):
    """some_audio_info: (meta dict, None) or (None, message)."""
    try:
        m = tc.info(data)
    except ValueError as e:
        return None, str(e)
    return {k: getattr(m, k) for k in META}, None


def walked(data: bytes, cuts, stream=True):
    """The walk fed data split at `cuts`, then the end: (meta dict, None, audio ranges, largest held) or (None, message, ...)."""
    w = C.c_void_p()
    assert lib.some_audio_walk_create(int(stream), C.byref(w)) == 0
    known, m = C.c_int(), _lib.AudioMeta()
    a, b, held = C.c_longlong(), C.c_longlong(), C.c_longlong()
    ranges, most = [], 0
    try:
        bounds = [0] + sorted(set(c for c in cuts if 0 < c < len(data))) + [len(data)]
        for k in range(len(bounds) - 1):
            piece = data[bounds[k]:bounds[k + 1]]
            end = int(k == len(bounds) - 2)
            if lib.some_audio_walk_feed(w, piece, len(piece), end, C.byref(known), C.byref(m), C.byref(a), C.byref(b),
                                        C.byref(held)):
                return None, lib.some_last_error().decode(), ranges, most
            most = max(most, held.value)
            if b.value > a.value:
                assert a.value >= bounds[k] - 64 and b.value <= bounds[k + 1]   # the feed's own bytes (and a lookahead)
                ranges.append((a.value, b.value))
        assert known.value == 1
        return {k: getattr(m, k) for k in META}, None, ranges, most
    finally:
        lib.some_audio_walk_destroy(w)


def frame_bytes(meta):
    if meta['container'] == _lib.AUDIO_FLAC:
        return 1
    return meta['channels'] * {_lib.PCM_U8: 1, _lib.PCM_S16: 2, _lib.PCM_S24: 3, _lib.PCM_S32: 4, _lib.PCM_F32: 4,
                               _lib.PCM_F64: 8}[meta['kind']]


def splits(data: bytes, seed: int, meta_end: int):
    """Every split point up to the audio and a little past it, single bytes (short files) and random splits."""
    rng = np.random.default_rng(seed)
    out = [[c] for c in range(1, min(len(data), meta_end + 24, 2000))]
    if len(data) <= 4000:
        out.append(list(range(1, len(data))))
    for _ in range(4):
        out.append(np.cumsum(rng.integers(1, max(2, len(data) // rng.integers(2, 40)), len(data))).tolist())
    return out


def check_walks(data: bytes, seed=0):
    want, err = whole(data)
    meta_end = want['data_offset'] if want else len(data)
    for cuts in splits(data, seed, meta_end):
        got, gerr, ranges, most = walked(data, cuts)
        assert most <= 48, f'the walker held {most} bytes'
        assert (got, gerr) == (want, err), cuts[:8]
        if got is None:
            continue
        # the audio ranges follow each other from the first audio byte, cover the decoded bytes and, past them, at most
        # an incomplete sample frame
        if ranges:
            assert ranges[0][0] == want['data_offset']
            assert all(r[1] == s[0] for r, s in zip(ranges, ranges[1:]))
        reported = ranges[-1][1] - ranges[0][0] if ranges else 0
        assert want['data_bytes'] <= reported < want['data_bytes'] + frame_bytes(want)


# ---------------------------------------------------------------------------------------------- the walk: WAV
@pytest.mark.parametrize('kind,ch,ext', [(k, ch, ext) for k in tc.KINDS for ch in (1, 2, 3, 8) for ext in (False, True)])
def test_wav_walk_equals_audio_info(kind, ch, ext):
    data = tc.wav_bytes(kind, ch, 257 + ch, rate=22050 + ch, seed=ch, extensible=ext,
                        extra=[(b'LIST', b'INFOabc'), (b'fact', b'\x01\x02\x03\x04')], after=[(b'junk', b'12345')])
    check_walks(data, seed=ch)


def test_wav_walk_truncated_and_odd_chunks():
    full = tc.wav_bytes('s16', 2, 1000, seed=3)
    s24 = tc.wav_bytes('s24', 1, 100, seed=5)
    for data in (full[:-100], full[:-101], full[:-102], tc.wav_bytes('s16', 1, 1000, seed=4)[:-33], s24[:-30], s24[:-31],
                 tc.wav_bytes('s16', 1, 0), tc.wav_bytes('s16', 2, 0), tc.wav_bytes('u8', 1, 7, after=[(b'LIST', b'odd')]),
                 tc.wav_bytes('f32', 3, 5, extra=[(b'abc ', b'x' * 3), (b'JUNK', b'y')]),
                 tc.wav_bytes('s24', 2, 50, data=bytes(301)), tc.wav_bytes('s16', 3, 50, data=bytes(301))):
        check_walks(data)


@pytest.mark.parametrize('case', range(9))
def test_wav_walk_refusals(case):
    data, _, _ = [
        (tc._riff(tc._fmt(tag=6), tc.chunk(b'data', bytes(8))), 0, 0),
        (tc._riff(tc._fmt(tag=0xFFFE, size=18), tc.chunk(b'data', bytes(8))), 0, 0),
        (tc._riff(tc._fmt(tag=3, bits=16, block=2), tc.chunk(b'data', bytes(8))), 0, 0),
        (tc._riff(tc._fmt(bits=72, block=9), tc.chunk(b'data', bytes(18))), 0, 0),
        (tc._riff(tc._fmt(rate_bytes=1), tc.chunk(b'data', bytes(8))), 0, 0),
        (tc._riff(tc.chunk(b'fmt ', bytes(8)), tc.chunk(b'data', bytes(8))), 0, 0),
        (tc._riff(tc.chunk(b'data', bytes(8)), tc._fmt()), 0, 0),
        (tc._riff(tc.chunk(b'LIST', bytes(4))) + b'da', 0, 0),
        (tc._riff(tc.chunk(b'LIST', bytes(4)))[:-2], 0, 0)][case]
    data = data[:4] + struct.pack('<I', max(len(data) - 8, 100)) + data[8:]
    assert whole(data)[1]
    check_walks(data)


def test_wav_walk_without_fmt_or_data_and_riff_size():
    good = tc.wav_bytes('s16', 1, 10)
    short = good[:4] + struct.pack('<I', 12 + 8 + 16 - 8) + good[8:]
    for data in (tc._riff(tc._fmt()), tc._riff(tc.chunk(b'LIST', bytes(4))), short, b'', b'RIF', b'RIFF\0\0\0\0WAV'):
        check_walks(data)


def test_wav_walk_placeholder_sizes_read_to_the_end():
    """A recorder writing to a pipe leaves the RIFF and data sizes at a placeholder: the whole frames present are read."""
    for size in (0xFFFFFFFF, 0x7FFFFFFF, 0x7FFFF000):
        data = bytearray(tc.wav_bytes('s16', 2, 3001, seed=9))
        data[4:8] = struct.pack('<I', size)
        data[40:44] = struct.pack('<I', size)
        for cut in (0, 4, 8, 2):
            d = bytes(data[:len(data) - cut])
            meta, err = whole(d)
            assert (meta['frames'], err) == (3001 - cut // 4, None) if cut % 4 == 0 else 'whole frames' in err
            check_walks(d, seed=cut)


def test_wav_second_data_chunk_is_refused_by_a_stream():
    data = tc.wav_bytes('s16', 1, 100, seed=1, after=[(b'LIST', b'ab'), (b'data', bytes(40))])
    want, _ = whole(data)
    assert want['frames'] == 20                                  # some_audio_info reads the last data chunk, as scipy
    second = data.rindex(b'data')
    for cuts in ([], [second + 1], [second + 4], [second + 8], list(range(1, len(data)))):
        got, err, ranges, _ = walked(data, cuts)
        assert got is None and f'a second data chunk at byte offset {second}' in err
        if len(cuts) > 1:                                        # pushed before the refusal: the first chunk's audio
            assert sum(b - a for a, b in ranges) == 200 and ranges[0][0] == 44
        assert walked(data, cuts, stream=False)[0] == want


def test_wav_fmt_after_data_is_refused_by_a_stream():
    """scipy reads a fmt chunk after the data chunk and decodes with it; a stream has decoded with the first one."""
    fmt48 = tc._fmt(rate=48000, block=2, bits=16)
    data = tc.wav_bytes('s16', 1, 100, seed=2, after=[(b'LIST', b'ab')]) + fmt48
    data = data[:4] + struct.pack('<I', len(data) - 8) + data[8:]
    want, _ = whole(data)
    assert want['rate'] == 48000                                 # some_audio_info: the last fmt chunk, as scipy
    second = data.rindex(b'fmt ')
    for cuts in ([], [second + 2], [second + 8], list(range(1, len(data)))):
        got, err, _, _ = walked(data, cuts)
        assert got is None and f'a fmt chunk after the data chunk at byte offset {second}' in err
        assert walked(data, cuts, stream=False)[0] == want


# ---------------------------------------------------------------------------------------------- the walk: FLAC
@pytest.mark.parametrize('name,x,kw', of.feature_cases(), ids=[c[0] for c in of.feature_cases()])
def test_flac_walk_equals_audio_info(name, x, kw):
    check_walks(of.encode(x, **kw), seed=len(name))


def test_flac_walk_refusals_and_large_skipped_blocks():
    for _, data, message in tc.FLAC_REFUSALS:
        if 'not a FLAC stream' not in message:                  # the walk's own FLAC refusals
            check_walks(data)
    x = of.test_signal(3000, 2, 16, 7)
    big = of.encode(x, rate=44100, bps=16, id3=of.id3_tag(bytes(300000)),
                    metadata=[('PICTURE', b'\xff\xf8\xc9\x08' * 250000), ('PADDING', bytes(5000))])
    for cuts in ([], list(range(1, len(big), 997)), list(range(1, 200))):
        got, err, ranges, most = walked(big, cuts)
        assert err is None and got == whole(big)[0] and most <= 48
    for cut in (100, 300020, 300100, 900000, len(big) - 1):
        want = whole(big[:cut])
        for cuts in ([], list(range(1, cut, 4099)), [5, 299999, 300021, 300050]):
            assert walked(big[:cut], cuts)[:2] == want


@pytest.mark.parametrize('data', [b'OggS' + bytes(40), b'ID3\x04\x00\x00\x00\x00\x00\x02ab' + bytes(40),
                                  b'\xff\xfb\x90\x00' + bytes(40), b'FORM\x00\x00\x00\x20AIFF' + bytes(40),
                                  of.id3_tag() + b'OggS' + bytes(30)])
def test_other_containers_refused_as_by_audio_info(data):
    assert whole(data)[1]
    check_walks(data)


# ---------------------------------------------------------------------------------------------- the chain
def resumed(fr, rec, cuts):
    """some_flac_chain_resume over windows of the file ending at `cuts`, then the final one: (chained positions, length) or
    the refusal's message.  A window holds the candidates a scan of its bytes finds: those whose header fits in it, and a
    frame running past its end is SOME_FLAC_TRUNCATED there."""
    base, start, stop, total = rec
    w = _lib.FlacWalk(start - base, 0, 0, -1, 0)
    chained = []
    for c in [c for c in cuts if start < c < stop] + [stop]:
        final = int(c == stop)
        lo = base + w.pos
        rows = []
        for r in fr:
            if r['pos'] >= lo and r['pos'] + r['header_len'] <= c:
                r = r.copy()
                if r['end'] > c:
                    r['status'], r['end'] = 1, c
                rows.append(r)
        win = np.array(rows, dtype=fr.dtype)
        chain = np.zeros(max(len(win), 1), np.int32)
        k = C.c_int()
        if lib.some_flac_chain_resume(win.ctypes.data if len(win) else None, len(win), base, c, total, final, C.byref(w),
                                      chain.ctypes.data, len(win), C.byref(k)):
            return lib.some_last_error().decode()
        chained += [int(win[j]['pos']) for j in chain[:k.value]]
        assert not (final and not w.done)
    return chained, w.got


@pytest.mark.parametrize('name,rows,recs', tc.chain_cases(), ids=[c[0] for c in tc.chain_cases()])
def test_resumed_chain_equals_whole_walk(name, rows, recs):
    fr = tc.frames(rows)
    for rec in recs:
        try:
            chains, lengths = tc.python_chain(fr, [rec])
            want = ([int(fr[i]['pos']) for i in chains[0]], lengths[0])
        except ValueError as e:
            want = str(e)
        edges = sorted({v + d for r in rows for v in (r[0], r[1]) for d in (-1, 0, 1, 2, 3)})
        for cuts in [[c] for c in edges] + [edges, list(range(rec[1], rec[2]))]:
            assert resumed(fr, rec, cuts) == want, cuts


def test_resumed_chain_waits_on_short_windows():
    fr = tc.frames([(100, 150, 0, 10, 0, 0), (150, 190, 1, 10, 0, 0)])
    rec = (90, 100, 190, 20)
    w = _lib.FlacWalk(10, 0, 0, -1, 0)
    chain, k = np.zeros(2, np.int32), C.c_int()
    # a truncated frame and a window of fewer than 16 bytes without a header: no error before the end
    t = fr[:1].copy()
    t['status'], t['end'] = 1, 120
    assert lib.some_flac_chain_resume(t.ctypes.data, 1, 90, 120, 20, 0, C.byref(w), chain.ctypes.data, 2, C.byref(k)) == 0
    assert (k.value, w.pos) == (0, 10)
    assert lib.some_flac_chain_resume(None, 0, 90, 115, 20, 0, C.byref(w), chain.ctypes.data, 2, C.byref(k)) == 0
    assert lib.some_flac_chain_resume(None, 0, 90, 116, 20, 0, C.byref(w), chain.ctypes.data, 2, C.byref(k)) == -1
    assert 'no valid FLAC frame header' in lib.some_last_error().decode() and 'byte offset 10' in lib.some_last_error().decode()
