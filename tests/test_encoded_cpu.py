"""CPU tests of the host half of the encoded-file path (csrc/audio_host.cu; the library loads without a GPU):
some_audio_info against audio.decode_wav and oracle/flac.py, audio.parse_flac's refusals word for word, some_flac_chain
against the Python walk FlacBatch used to do (kept here as the comparison), and some_midi_write against
midi.build_midi_file(...).to_bytes()."""
import ctypes as C
import struct
import warnings

import numpy as np
import pytest

from oracle import aiff as oa
from oracle import flac as of
from some_b200 import _lib, audio, midi

lib = _lib.load()


def info(data: bytes):
    m = _lib.AudioMeta()
    buf = C.create_string_buffer(data, len(data))
    rc = lib.some_audio_info(buf, len(data), C.byref(m))
    if rc:
        raise ValueError(lib.some_last_error().decode())
    return m


# ---------------------------------------------------------------------------------------------- WAV files
KINDS = {  # kind: (format tag, bits, container bytes, numpy dtype of the raw samples)
    'u8': (1, 8, 1, np.uint8), 's16': (1, 16, 2, np.int16), 's24': (1, 24, 3, None), 's32': (1, 32, 4, np.int32),
    'f32': (3, 32, 4, np.float32), 'f64': (3, 64, 8, np.float64)}
CODE = {'u8': _lib.PCM_U8, 's16': _lib.PCM_S16, 's24': _lib.PCM_S24, 's32': _lib.PCM_S32, 'f32': _lib.PCM_F32,
        'f64': _lib.PCM_F64}
FLOAT_GUID = b'\x03\x00\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x008\x9bq'
PCM_GUID = b'\x01\x00\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x008\x9bq'


def raw_samples(kind: str, n: int, ch: int, seed: int) -> bytes:
    rng = np.random.default_rng(seed)
    if kind == 's24':
        return rng.integers(0, 256, n * ch * 3, dtype=np.uint8).tobytes()
    dt = KINDS[kind][3]
    if dt in (np.float32, np.float64):
        return (rng.standard_normal(n * ch) * 0.3).astype(dt).tobytes()
    info_ = np.iinfo(dt)
    return rng.integers(info_.min, info_.max, n * ch, dtype=dt, endpoint=True).tobytes()


def chunk(cid: bytes, body: bytes) -> bytes:
    return cid + struct.pack('<I', len(body)) + body + (b'\0' if len(body) % 2 else b'')


def wav_bytes(kind: str, ch: int, n: int, rate=44100, seed=0, extensible=False, extra=(), after=(), data=None,
              riff_size=None) -> bytes:
    tag, bits, cb, _ = KINDS[kind]
    block = cb * ch
    if extensible:
        fmt = struct.pack('<HHIIHHHHI', 0xFFFE, ch, rate, rate * block, block, bits, 22, bits, 0) + \
            (FLOAT_GUID if tag == 3 else PCM_GUID)
    else:
        fmt = struct.pack('<HHIIHH', tag, ch, rate, rate * block, block, bits)
    body = b'WAVE' + b''.join(chunk(c, b) for c, b in extra) + chunk(b'fmt ', fmt)
    body += chunk(b'data', raw_samples(kind, n, ch, seed) if data is None else data)
    body += b''.join(chunk(c, b) for c, b in after)
    return b'RIFF' + struct.pack('<I', len(body) if riff_size is None else riff_size) + body


def decode_wav_bytes(tmp_path, data: bytes):
    p = tmp_path / 'x.wav'
    p.write_bytes(data)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return audio.decode_wav(p)


def host_decode(data: bytes, m) -> np.ndarray:
    """The samples some_audio_info points at, scaled as decode_wav scales them (numpy, for the offset check)."""
    raw = np.frombuffer(data, np.uint8, count=m.data_bytes, offset=m.data_offset)
    if m.kind == _lib.PCM_S24:
        b = raw.reshape(-1, 3).astype(np.int32)
        x = ((b[:, 0] << 8) | (b[:, 1] << 16) | (b[:, 2] << 24)).astype(np.float32) / np.float32(2 ** 31)
    else:
        dt = {_lib.PCM_U8: np.uint8, _lib.PCM_S16: '<i2', _lib.PCM_S32: '<i4', _lib.PCM_F32: '<f4', _lib.PCM_F64: '<f8'}[m.kind]
        v = raw.view(dt)
        if m.kind == _lib.PCM_U8:
            x = (v.astype(np.float32) - 128.0) / 128.0
        elif m.kind in (_lib.PCM_S16, _lib.PCM_S32):
            x = v.astype(np.float32) / float(1 << (8 * v.dtype.itemsize - 1))
        else:
            x = v.astype(np.float32)
    return x.reshape(-1, m.channels) if m.channels > 1 else x


WAV_CASES = [(k, ch, ext) for k in KINDS for ch in range(1, 9) for ext in (False, True)]


@pytest.mark.parametrize('kind,ch,ext', WAV_CASES)
def test_wav_info_equals_decode_wav(tmp_path, kind, ch, ext):
    n = 257 + ch
    data = wav_bytes(kind, ch, n, rate=22050 + ch, seed=ch, extensible=ext,
                     extra=[(b'LIST', b'INFOabc'), (b'fact', b'\x01\x02\x03\x04')], after=[(b'junk', b'12345')])
    x, rate = decode_wav_bytes(tmp_path, data)
    m = info(data)
    assert (m.container, m.rate, m.channels, m.kind, m.frames) == (_lib.AUDIO_WAV, rate, ch, CODE[kind], x.shape[0])
    assert m.bits == KINDS[kind][1] and m.data_bytes == n * ch * KINDS[kind][2]
    np.testing.assert_array_equal(host_decode(data, m), x)


def test_wav_truncated_data_chunk_keeps_the_whole_frames(tmp_path):
    """scipy.io.wavfile.read returns the whole frames present when the data chunk runs past the end of the file (with a
    warning); a partial frame of several channels is refused (scipy cannot reshape it), as is a partial 24-bit sample."""
    full = wav_bytes('s16', 2, 1000, seed=3)
    cut = full[:-101]                                # 24 whole stereo frames and one extra sample missing
    x, _ = decode_wav_bytes(tmp_path, full[:-100])
    m = info(full[:-100])
    assert m.frames == x.shape[0] == 975
    np.testing.assert_array_equal(host_decode(full[:-100], m), x)
    with pytest.raises(ValueError):
        decode_wav_bytes(tmp_path, cut[:-1])
    with pytest.raises(ValueError, match='whole frames'):
        info(cut[:-1])
    mono = wav_bytes('s16', 1, 1000, seed=4)[:-33]
    x, _ = decode_wav_bytes(tmp_path, mono)
    assert info(mono).frames == x.shape[0] == 983
    s24 = wav_bytes('s24', 1, 100, seed=5)
    x, _ = decode_wav_bytes(tmp_path, s24[:-30])
    assert info(s24[:-30]).frames == x.shape[0] == 90
    with pytest.raises(ValueError):
        decode_wav_bytes(tmp_path, s24[:-31])
    with pytest.raises(ValueError, match='24-bit'):
        info(s24[:-31])


def test_wav_empty_and_odd_chunks(tmp_path):
    for data in (wav_bytes('s16', 1, 0), wav_bytes('s16', 2, 0), wav_bytes('u8', 1, 7, after=[(b'LIST', b'odd')]),
                 wav_bytes('f32', 3, 5, extra=[(b'abc ', b'x' * 3), (b'JUNK', b'y')])):
        x, rate = decode_wav_bytes(tmp_path, data)
        m = info(data)
        assert (m.rate, m.frames) == (rate, x.shape[0])
        np.testing.assert_array_equal(host_decode(data, m), x)


@pytest.mark.parametrize('data,reason', [
    (b'OggS' + bytes(40), 'Ogg'),
    (b'ID3\x04\x00\x00\x00\x00\x00\x02ab' + bytes(40), 'MP3 (ID3 tag)'),
    (b'\xff\xfb\x90\x00' + bytes(40), 'MPEG audio (MP3)'),
    (b'FORM\x00\x00\x00\x20AIFF' + bytes(40), 'AIFF/IFF'),
    (b'RIFX' + bytes(40), 'big-endian RIFX'),
    (b'RF64' + bytes(40), 'RF64'),
    (b'caff' + bytes(40), 'Core Audio (CAF)'),
    (b'.snd' + bytes(40), 'Sun/NeXT AU'),
    (b'RIFF\x00\x00\x00\x00AVI ' + bytes(40), 'unrecognised header'),
])
def test_other_containers_are_refused_by_name(tmp_path, data, reason):
    with pytest.raises(ValueError, match=reason.replace('(', r'\(').replace(')', r'\)')):
        decode_wav_bytes(tmp_path, data)
    with pytest.raises(ValueError, match=reason.replace('(', r'\(').replace(')', r'\)')):
        info(data)


def _fmt(tag=1, ch=1, rate=8000, block=2, bits=16, rate_bytes=None, size=16):
    body = struct.pack('<HHIIHH', tag, ch, rate, rate * block if rate_bytes is None else rate_bytes, block, bits)
    return chunk(b'fmt ', body + bytes(size - 16))


def _riff(*chunks_):
    body = b'WAVE' + b''.join(chunks_)
    return b'RIFF' + struct.pack('<I', len(body)) + body


@pytest.mark.parametrize('data,reason,offset', [
    (_riff(_fmt(tag=6), chunk(b'data', bytes(8))), 'Unknown wave file format', 12),
    (_riff(_fmt(tag=0xFFFE, size=18), chunk(b'data', bytes(8))), 'not compliant', 12),
    (_riff(_fmt(tag=3, bits=16, block=2), chunk(b'data', bytes(8))), 'Unsupported bit depth', 36),
    (_riff(_fmt(bits=72, block=9), chunk(b'data', bytes(18))), 'Unsupported bit depth', 36),
    (_riff(_fmt(rate_bytes=1), chunk(b'data', bytes(8))), 'nAvgBytesPerSec', 12),
    (_riff(chunk(b'fmt ', bytes(8)), chunk(b'data', bytes(8))), 'not compliant', 12),
    (_riff(chunk(b'data', bytes(8)), _fmt()), 'No fmt chunk before data', 12),
    (_riff(chunk(b'LIST', bytes(4))) + b'da', 'Incomplete chunk ID', 24),
    (_riff(chunk(b'LIST', bytes(4)))[:-2], 'Unexpected end of file', 24),
])
def test_wav_refusals_name_the_reason_and_offset(tmp_path, data, reason, offset):
    data = data[:4] + struct.pack('<I', max(len(data) - 8, 100)) + data[8:]
    with pytest.raises(ValueError, match=reason):           # scipy's own text, which decode_wav passes on
        decode_wav_bytes(tmp_path, data)
    with pytest.raises(ValueError, match=reason) as e:
        info(data)
    assert f'byte offset {offset}' in str(e.value)


def test_wav_without_fmt_or_data_is_refused(tmp_path):
    for data, reason in ((_riff(_fmt()), 'no data chunk'), (_riff(chunk(b'LIST', bytes(4))), 'no fmt chunk')):
        with pytest.raises(Exception):                       # scipy: UnboundLocalError
            decode_wav_bytes(tmp_path, data)
        with pytest.raises(ValueError, match=reason):
            info(data)


def test_wav_riff_size_bounds_the_walk(tmp_path):
    """scipy reads chunks only up to the RIFF size: a data chunk after it is never seen."""
    good = wav_bytes('s16', 1, 10)
    fmt_end = 12 + 8 + 16
    short = good[:4] + struct.pack('<I', fmt_end - 8) + good[8:]
    with pytest.raises(Exception):
        decode_wav_bytes(tmp_path, short)
    with pytest.raises(ValueError, match='no data chunk'):
        info(short)


# ---------------------------------------------------------------------------------------------- FLAC metadata
@pytest.mark.parametrize('name,x,kw', of.feature_cases(), ids=[c[0] for c in of.feature_cases()])
def test_flac_info_equals_oracle(name, x, kw):
    data = of.encode(x, **kw)
    want = of.parse_metadata(data)
    m = info(data)
    assert (m.container, m.rate, m.channels, m.bits, m.frames) == \
        (_lib.AUDIO_FLAC, want['rate'], want['channels'], want['bps'], want['total'])
    assert (m.min_blocksize, m.max_blocksize, m.data_offset, m.data_bytes) == \
        (want['min_blocksize'], want['max_blocksize'], want['audio_offset'], len(data) - want['audio_offset'])


def _flac_refusals():
    x = of.test_signal(1000, 1, 16, 1)
    good = of.encode(x, rate=44100, bps=16)
    si = good.index(b'fLaC') + 4
    b32 = bytearray(good)
    b32[si + 4 + 12] = (b32[si + 4 + 12] & 0xFE) | 1         # bps - 1 = 31 -> 32 bits (high bit of the 5-bit field)
    b32[si + 4 + 13] = (b32[si + 4 + 13] & 0x0F) | 0xF0
    rate0 = bytearray(good)
    rate0[si + 4 + 10:si + 4 + 12] = b'\0\0'
    rate0[si + 4 + 12] &= 0x0F
    not_flac = 'f: not a FLAC stream (no fLaC marker at byte offset 0)'
    return [
        ('bps_32', bytes(b32), "f: FLAC stream of 32 bits per sample (at byte offset 8); only up to 24 bits are decoded "
                               "(libsndfile's float scaling is exact up to 24 bits)"),
        ('rate_0', bytes(rate0), 'f: invalid FLAC STREAMINFO (sample rate 0, max block size 1000) at byte offset 8'),
        ('second_streaminfo', good[:si] + bytes([0x00, 0, 0, 34]) + good[si + 4:si + 38] + bytes([0x80, 0, 0, 34]) +
         good[si + 4:], 'f: second STREAMINFO FLAC metadata block at byte offset 42'),
        ('block_127', good[:si] + bytes([0x00, 0, 0, 34]) + good[si + 4:si + 38] + bytes([0xFF, 0, 0, 0]) + good[si + 38:],
         'f: invalid FLAC metadata block at byte offset 42'),
        ('first_not_streaminfo', good[:si] + bytes([0x81, 0, 0, 34]) + good[si + 4:],
         'f: FLAC stream does not start with a 34-byte STREAMINFO block (type 1, 34 bytes at byte offset 4)'),
        ('block_truncated', good[:si + 20], 'f: FLAC metadata block truncated at byte offset 4'),
        ('header_truncated', good[:si + 2], 'f: FLAC metadata block header truncated at byte offset 4'),
        ('id3_block_truncated', of.id3_tag() + good[:si + 20], 'f: FLAC metadata block truncated at byte offset 28'),
        # bytes the walk takes for, or refuses as, another container
        ('no_marker', b'fLaX' + good[4:], not_flac),
        ('id3_no_marker', of.id3_tag() + b'fLaX' + good[4:], 'f: not a FLAC stream (no fLaC marker at byte offset 24)'),
        ('wav', wav_bytes('s16', 1, 10), not_flac),
        ('bad_wav', _riff(_fmt(tag=6), chunk(b'data', bytes(8))), not_flac),
        ('aiff', oa.aiff_bytes(bytes(20), 1, 16, 8000.0), not_flac),
        ('bad_aiff', b'FORM\x00\x00\x00\x20' + b'8SVX' + bytes(40), not_flac),
    ]


FLAC_REFUSALS = _flac_refusals()


@pytest.mark.parametrize('name,data,message', FLAC_REFUSALS, ids=[c[0] for c in FLAC_REFUSALS])
def test_flac_refusal_messages(name, data, message):
    """audio.parse_flac's refusals, word for word: the walk's FLAC reason and byte offset, or 'not a FLAC stream' and
    where the marker was looked for."""
    with pytest.raises(ValueError) as e:
        audio.parse_flac(data, 'f')
    assert str(e.value) == message


# ---------------------------------------------------------------------------------------------- the frame chain
_REASONS = {1: 'truncated frame', 2: 'CRC-16 mismatch', 3: 'non-zero padding bits', 4: 'reserved subframe type',
            5: 'invalid wasted-bits count', 6: 'predictor order larger than the block',
            7: 'invalid LPC precision or shift', 8: 'reserved residual coding method', 9: 'invalid partition order'}


def python_chain(fr, recs):
    """The walk FlacBatch._chain did in Python before it called some_flac_chain (the comparison)."""
    pos, end, status = fr['pos'].tolist(), fr['end'].tolist(), fr['status'].tolist()
    number, variable, bs = fr['number'].tolist(), fr['variable'].tolist(), fr['blocksize'].tolist()
    n = len(pos)
    chains, lengths = [], []
    i = 0
    for base, start, stop, total in recs:
        p = start
        chain, got, strategy = [], 0, None
        while not (total and got == total) and not (not total and p == stop):
            if p >= stop:
                raise ValueError(f'FLAC stream ends at byte offset {p - base} after {got} of {total} samples')
            while i < n and pos[i] < p:
                i += 1
            if i >= n or pos[i] != p:
                raise ValueError(f'no valid FLAC frame header (sync, reserved code, CRC-8 or STREAMINFO '
                                 f'mismatch) at byte offset {p - base}')
            if status[i]:
                raise ValueError(f'FLAC frame at byte offset {p - base}: '
                                 f'{_REASONS.get(status[i], status[i])} (at byte offset {end[i] - base})')
            strategy = variable[i] if strategy is None else strategy
            want = got if variable[i] else len(chain)
            if variable[i] != strategy or number[i] != want:
                raise ValueError(f'FLAC frame at byte offset {p - base}: {"sample" if variable[i] else "frame"} '
                                 f'number {number[i]}, expected {want} (gap, overlap or changed blocking strategy)')
            got += bs[i]
            if total and got > total:
                raise ValueError(f'FLAC frame at byte offset {p - base} decodes past the {total} samples '
                                 f'STREAMINFO states')
            chain.append(i)
            p = end[i]
        chains.append(chain)
        lengths.append(got)
    return chains, lengths


def c_chain(fr, recs):
    n, k = len(fr), len(recs)
    fr = np.ascontiguousarray(fr)
    rr = (_lib.FlacRange * max(k, 1))(*[_lib.FlacRange(*r) for r in recs])
    chain = np.zeros(max(n, 1), np.int32)
    first = np.zeros(k + 1, np.int64)
    lengths = np.zeros(max(k, 1), np.int64)
    failed = C.c_int(-1)
    if lib.some_flac_chain(fr.ctypes.data if n else None, n, rr, k, chain.ctypes.data, n, first.ctypes.data,
                           lengths.ctypes.data, C.byref(failed)):
        raise ValueError(lib.some_last_error().decode(), failed.value)
    return [chain[first[r]:first[r + 1]].tolist() for r in range(k)], lengths[:k].tolist()


def frames(rows):
    fr = np.zeros(len(rows), audio._FRAME_DTYPE)
    for i, (pos, end, number, bs, variable, status) in enumerate(rows):
        fr[i] = (pos, number, end, 0, bs, 4, 0, variable, status)
    return fr


def chain_cases():
    ok = [(100, 150, 0, 10, 0, 0), (150, 190, 1, 10, 0, 0), (190, 230, 2, 5, 0, 0)]
    var = [(100, 150, 0, 10, 1, 0), (150, 190, 10, 10, 1, 0), (190, 230, 20, 5, 1, 0)]
    false_sync = [(100, 150, 0, 10, 0, 0), (120, 121, 7, 10, 0, 3), (150, 190, 1, 10, 0, 0), (190, 230, 2, 5, 0, 0)]
    two = ok + [(1100, 1150, 0, 10, 1, 0), (1150, 1200, 10, 20, 1, 0)]
    cases = [
        ('fixed', ok, [(90, 100, 230, 25)]),
        ('variable', var, [(90, 100, 230, 25)]),
        ('unknown_length', ok, [(90, 100, 230, 0)]),
        ('false_sync_skipped', false_sync, [(0, 100, 230, 25)]),
        ('two_recordings', two, [(90, 100, 230, 25), (1000, 1100, 1200, 0)]),
        ('empty_unknown', [], [(0, 50, 50, 0)]),
        ('no_header', ok, [(90, 100, 230, 30)]),
        ('no_header_at_start', ok, [(90, 101, 230, 25)]),
        ('bad_status', [ok[0], (150, 170, 1, 10, 0, 2), ok[2]], [(90, 100, 230, 25)]),
        ('unknown_status', [ok[0], (150, 170, 1, 10, 0, 42), ok[2]], [(90, 100, 230, 25)]),
        ('frame_gap', [ok[0], (150, 190, 2, 10, 0, 0), ok[2]], [(90, 100, 230, 25)]),
        ('sample_overlap', [var[0], (150, 190, 5, 10, 1, 0), var[2]], [(90, 100, 230, 25)]),
        ('strategy_change', [ok[0], (150, 190, 10, 10, 1, 0), ok[2]], [(90, 100, 230, 25)]),
        ('past_streaminfo', ok, [(90, 100, 230, 22)]),
        ('ends_early', ok, [(90, 100, 230, 40)]),
        ('ends_early_unknown', ok[:2], [(90, 100, 230, 0)]),
        ('second_fails', two[:4] + [(1150, 1200, 5, 20, 1, 0)], [(90, 100, 230, 25), (1000, 1100, 1200, 0)]),
    ]
    return cases


@pytest.mark.parametrize('name,rows,recs', chain_cases(), ids=[c[0] for c in chain_cases()])
def test_flac_chain_equals_python_walk(name, rows, recs):
    fr = frames(rows)
    try:
        want = python_chain(fr, recs)
    except ValueError as e:
        with pytest.raises(ValueError) as got:
            c_chain(fr, recs)
        assert got.value.args[0] == str(e)
        return
    assert c_chain(fr, recs) == want


# ---------------------------------------------------------------------------------------------- MIDI
def c_midi(offsets, segs, timestep, tempo):
    counts = np.array([len(s[0]) for s in segs] or [0], np.int32)
    cat = lambda i, dt: np.concatenate([np.asarray(s[i], dt) for s in segs] + [np.zeros(1, dt)])   # noqa: E731
    midi_, dur, rest = cat(0, np.float32), cat(1, np.int32), cat(2, np.uint8)
    off = np.array(list(offsets) or [0.0], np.float64)
    size = C.c_size_t()
    args = (len(segs), off.ctypes.data, counts.ctypes.data, midi_.ctypes.data, dur.ctypes.data, rest.ctypes.data,
            timestep, tempo)
    if lib.some_midi_write(*args, None, 0, C.byref(size)):
        raise ValueError(lib.some_last_error().decode())
    buf = (C.c_uint8 * max(size.value, 1))()
    small = C.c_size_t()
    assert lib.some_midi_write(*args, buf, size.value - 1, C.byref(small)) == 0 and small.value == size.value
    assert lib.some_midi_write(*args, buf, size.value, C.byref(size)) == 0
    return bytes(buf[:size.value])


def py_midi(offsets, segs, timestep, tempo):
    segments = [{'note_midi': np.asarray(m, np.float32), 'note_dur': np.asarray(d, np.int32) * timestep,
                 'note_rest': np.asarray(r, bool)} for m, d, r in segs]
    return midi.build_midi_file(list(offsets), segments, tempo).to_bytes()


def random_case(seed):
    rng = np.random.default_rng(seed)
    timestep = [512 / 44100, 512 / 48000, 0.01, 1 / 96][seed % 4]
    tempo = [120, 90.5, 37, 1000][(seed // 4) % 4]
    tps = tempo * 8
    k = int(rng.integers(0, 6))
    offsets, segs, t = [], [], 0.0
    for _ in range(k):
        if rng.random() < 0.3:     # a chunk offset on a half-tick tie
            t = (np.floor(t * tps) + 0.5 + rng.integers(0, 50)) / tps
        else:
            t += rng.uniform(0, 5)
        offsets.append(t)
        n = int(rng.integers(0, 40))
        dur = rng.integers(0, 60, n).astype(np.int32)
        dur[rng.random(n) < 0.1] = 0
        if rng.random() < 0.3 and n:
            dur[-1] = 5000           # runs past the next chunk
        m = (rng.uniform(30, 90, n)).astype(np.float32)
        half = rng.random(n) < 0.15
        m[half] = np.floor(m[half]) + 0.5          # rounding ties of the pitch
        rest = (rng.random(n) < 0.2).astype(np.uint8)
        segs.append((m, dur, rest))
        t += rng.uniform(0, 3)
    return offsets, segs, timestep, tempo


@pytest.mark.parametrize('seed', range(320))
def test_midi_bytes_equal_build_midi_file(seed):
    offsets, segs, timestep, tempo = random_case(seed)
    assert c_midi(offsets, segs, timestep, tempo) == py_midi(offsets, segs, timestep, tempo)


def test_midi_half_tick_duration_ties():
    """Cumulative durations that land exactly on half ticks (np.round: half to even)."""
    timestep = 1 / 1920            # 0.5 tick at 120 bpm (960 ticks per second)
    for tempo in (120, 90.5, 37, 1000):
        segs = [(np.full(9, 60.0, np.float32), np.arange(1, 10, dtype=np.int32), np.zeros(9, np.uint8))] * 3
        offsets = [0.0, 0.5 / (tempo * 8) + 0.02, 2.5 / (tempo * 8) + 0.04]
        assert c_midi(offsets, segs, timestep, tempo) == py_midi(offsets, segs, timestep, tempo)


def test_midi_empty_result():
    for tempo in (120, 90.5, 37, 1000):
        assert c_midi([], [], 0.01, tempo) == py_midi([], [], 0.01, tempo)
        assert c_midi([1.0], [([], [], [])], 0.01, tempo) == py_midi([1.0], [([], [], [])], 0.01, tempo)


def test_midi_refusals():
    with pytest.raises(ValueError, match='0..127'):
        py_midi([0.0], [([128.0], [10], [0])], 0.01, 120)
    with pytest.raises(ValueError, match='0..127'):
        c_midi([0.0], [([128.0], [10], [0])], 0.01, 120)
    with pytest.raises(ValueError, match='0..127'):
        c_midi([0.0], [([-0.6], [10], [0])], 0.01, 120)
    neg = ([0.0], [([60.0, 61.0, 62.0], [10, -5, 10], [0, 0, 0])], 0.01, 120)     # a negative duration moves back
    with pytest.raises(ValueError, match='non-negative'):
        py_midi(*neg)
    with pytest.raises(ValueError, match='non-negative'):
        c_midi(*neg)
    with pytest.raises(ValueError, match='24'):     # Python truncates this tempo to 24 bits; C refuses it
        c_midi([0.0], [([60.0], [10], [0])], 0.01, 3.5)
    assert c_midi([0.0], [([60.0], [10], [0])], 0.01, 3.6) == py_midi([0.0], [([60.0], [10], [0])], 0.01, 3.6)


def test_integer_pcm_wider_than_4_bytes_is_refused(tmp_path):
    """audio.load reads 40-64 bit integer PCM (scipy: int64, x / 2^63); some_audio_info refuses it and names the container.
    This is the one kind of file the two disagree on."""
    for bits, cb in ((64, 8), (40, 5)):
        raw = np.arange(-6, 6, dtype='<i8').tobytes() if cb == 8 else bytes(range(60))
        data = _riff(_fmt(bits=bits, block=cb, rate_bytes=8000 * cb), chunk(b'data', raw))
        x, _ = decode_wav_bytes(tmp_path, data)
        assert x.dtype == np.float32 and x.shape == (12,)
        with pytest.raises(ValueError, match=f'{bits}-bit PCM in {cb}-byte containers is not read'):
            info(data)
