"""CPU tests of AIFF / AIFF-C reading on the host (csrc/audio_host.cu; the library loads without a GPU): some_audio_info
against oracle/aiff.py's walk on every coding, channel count, sample size and chunk layout; the oracle against Python's
aifc and audioop; every refusal's reason and byte offset; and the resumable walk (some_audio_walk_*) fed in pieces against
the whole-file walk."""
import ctypes as C
import math
import struct
import warnings

import numpy as np
import pytest

import test_encoded_stream_cpu as ts
from oracle import aiff as oa
from some_b200 import _lib

lib = _lib.load()
META = ts.META

# (compression type or None for plain AIFF, sampleSize) of every row of the coding table
ROWS = ([(None, b) for b in (8, 12, 16, 20, 24, 32)] +
        [(c, b) for c in (b'NONE', b'twos', b'sowt') for b in (1, 8, 12, 16, 20, 24, 32)] + [(b'raw ', 8), (b'fl32', 32), (b'FL32', 32), (b'fl64', 64), (b'FL64', 64), (b'ulaw', 16), (b'ULAW', 8),
         (b'alaw', 16), (b'ALAW', 8)])


def meta_of(data: bytes):
    """some_audio_info: (meta dict, None) or (None, message)."""
    return ts.whole(data)


def oracle_meta(data: bytes):
    try:
        m = oa.walk(data)
    except oa.AiffError as e:
        return None, e
    return {k: m[k] for k in META}, None


def case(comp, bits, ch, n=101, rate=44100.0, seed=0, **kw):
    kind = oa._kind_of(comp, bits)
    return oa.aiff_bytes(oa.raw_samples(kind, n, ch, seed), ch, bits, rate, comp=comp, **kw)


def layout_cases():
    """(name, bytes): chunk layouts, sizes and rates around one coding."""
    skip = [(b'MARK', b'\0\x01abc'), (b'(c) ', b'x'), (b'ANNO', b'odd'), (b'ID3 ', b'ID3\3\0' + bytes(6)), (b'APPL', b'appl')]
    good = case(b'twos', 16, 2, n=300, seed=5)
    out = [
        ('skipped_odd_chunks', case(None, 16, 2, before=skip[:3], between=skip[3:], after=[(b'COMT', b'late')])),
        ('aifc_named', case(b'sowt', 24, 3, name=b'little-endian 24-bit PCM', before=skip, seed=2)),
        ('ssnd_offset', case(b'NONE', 16, 2, offset=7, block_size=4096, seed=3)),
        ('ssnd_offset_even', case(None, 24, 1, offset=64, seed=4)),
        ('truncated_ssnd', good[:-37]),
        ('truncated_to_header', good[:len(good) - 1200 + 3]),
        ('ssnd_size_placeholder', case(None, 16, 2, ssnd_size=0xFFFFFFF0, n=77)),
        ('form_size_past_end', case(None, 16, 1, form_size=0xFFFFFFFF)),
        ('form_size_placeholders_cut', case(b'fl32', 32, 2, ssnd_size=0x7FFFFFFF, form_size=0xFFFFFFFF, n=90)[:-5]),
        ('non_integer_rate', case(None, 16, 1, rate=22254.545454545454)),
        ('rate_below_2_31', case(None, 8, 1, rate=2.0 ** 31 - 0.25, n=3)),
        ('rate_one', case(None, 8, 1, rate=1.0, n=3)),
        ('empty_ssnd', case(b'alaw', 16, 2, n=0)),
        ('partial_frame', case(None, 16, 3, n=20)[:-1]),
        ('frames_field_ignored', case(None, 16, 2, frames=12345)),
        ('second_comm_after_ssnd', case(None, 16, 1, after=[(b'COMM', oa.comm_body(2, 32, 8000.0))])),
        ('second_comm_before_ssnd', case(None, 16, 1, between=[(b'COMM', oa.comm_body(2, 8, 8000.0))])),
        ('offset_past_file_end', case(None, 16, 1, offset=500, n=0)[:60]),
    ]
    return out


def all_cases():
    out = [(f'{(c or b"AIFF").decode().strip()}_{b}bit', case(c, b, 2, seed=b)) for c, b in ROWS]
    out += [(f'channels{ch}', case(b'NONE', 16, ch, seed=ch)) for ch in list(range(1, 9)) + [12]]
    out += [(f'ulaw_channels{ch}', case(b'ulaw', 16, ch, seed=ch)) for ch in (1, 5, 12)]
    return out + layout_cases()


CASES = all_cases()


@pytest.mark.parametrize('name,data', CASES, ids=[c[0] for c in CASES])
def test_audio_info_equals_oracle(name, data):
    want, err = oracle_meta(data)
    assert err is None, err
    got, gerr = meta_of(data)
    assert gerr is None, gerr
    assert got == want
    x = oa.samples(data, oa.walk(data))
    assert x.shape == (want['frames'], want['channels']) and x.dtype == np.float32


def test_coding_table_and_layouts():
    """The kinds and byte ranges the table and the layouts give (fixed, so that the oracle is held to the issue's table)."""
    kinds = {(c, b): meta_of(case(c, b, 2))[0]['kind'] for c, b in ROWS}
    assert kinds[(None, 12)] == _lib.PCM_S16BE and kinds[(None, 20)] == _lib.PCM_S24BE and kinds[(None, 8)] == _lib.PCM_S8
    assert kinds[(b'sowt', 8)] == _lib.PCM_S8 and kinds[(b'sowt', 12)] == _lib.PCM_S16 and kinds[(b'sowt', 32)] == _lib.PCM_S32
    assert kinds[(b'raw ', 8)] == _lib.PCM_U8 and kinds[(b'FL64', 64)] == _lib.PCM_F64BE
    assert kinds[(b'ULAW', 8)] == _lib.PCM_ULAW and kinds[(b'alaw', 16)] == _lib.PCM_ALAW
    lay = dict(layout_cases())
    m = meta_of(lay['ssnd_offset'])[0]
    assert m['data_offset'] == lay['ssnd_offset'].index(b'SSND') + 16 + 7 and m['frames'] == 101
    assert meta_of(lay['truncated_ssnd'])[0]['frames'] == 300 - 10           # 37 bytes: 9 whole frames and a partial one
    assert meta_of(lay['non_integer_rate'])[0]['rate'] == 22254
    assert meta_of(lay['rate_below_2_31'])[0]['rate'] == 2 ** 31 - 1
    assert meta_of(lay['ssnd_size_placeholder'])[0]['frames'] == 77
    assert meta_of(lay['partial_frame'])[0]['frames'] == 19
    assert meta_of(lay['frames_field_ignored'])[0]['frames'] == 101
    assert meta_of(lay['second_comm_after_ssnd'])[0]['channels'] == 1
    assert meta_of(lay['second_comm_before_ssnd'])[0]['channels'] == 2        # the last COMM before SSND
    assert meta_of(lay['offset_past_file_end'])[0]['frames'] == 0


# ---------------------------------------------------------------------------------------------- the standard library
def _stdlib(name):
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', DeprecationWarning)
        return pytest.importorskip(name)


@pytest.mark.parametrize('comp,width', [(b'NONE', 1), (b'NONE', 2), (b'NONE', 3), (b'NONE', 4), (b'sowt', 2), (b'ulaw', 2),
                                        (b'alaw', 2), (None, 2), (None, 3)])
@pytest.mark.parametrize('ch', [1, 2, 3])
def test_oracle_agrees_with_aifc(tmp_path, comp, width, ch):
    aifc = _stdlib('aifc')
    rng = np.random.default_rng(width * 10 + ch)
    n = 256          # an even byte count: aifc counts the pad byte of odd sample data in the SSND size, so its frames differ
    path = tmp_path / 'x.aif'
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', DeprecationWarning)
        w = aifc.open(str(path), 'wb')
        if comp is None:
            w.aiff()
        else:
            w.setcomptype(comp, b'x')
        w.setnchannels(ch)
        w.setsampwidth(width)
        w.setframerate(22050 + ch)
        if comp in (b'ulaw', b'alaw'):
            lin = rng.integers(-32768, 32768, n * ch).astype(np.int16)
            w.writeframes(lin.tobytes())                          # native 16-bit linear, encoded by aifc
        else:
            w.writeframes(rng.integers(0, 256, n * ch * width, dtype=np.uint8).tobytes())   # big-endian samples
        w.close()
        r = aifc.open(str(path), 'rb')
        got = (r.getnchannels(), r.getframerate(), r.getnframes())
        frames = r.readframes(r.getnframes())
        r.close()
    data = path.read_bytes()
    m = oa.walk(data)
    assert (m['channels'], m['rate'], m['frames']) == got
    assert meta_of(data)[0] == {k: m[k] for k in META}
    x = oa.samples(data, m)
    if comp in (b'ulaw', b'alaw'):                                 # aifc decodes G.711 with audioop, to native int16
        np.testing.assert_array_equal(x.reshape(-1) * 32768, np.frombuffer(frames, np.int16).astype(np.float32))
    else:                                                          # aifc hands over big-endian samples
        b = np.frombuffer(frames, np.uint8).reshape(-1, width).astype(np.int64)
        v = np.zeros(len(b), np.int64)
        for k in range(width):
            v = v << 8 | b[:, k]
        v = np.where(v >= 1 << (8 * width - 1), v - (1 << 8 * width), v)
        want = v.astype(np.float32) / np.float32(2 ** (8 * width - 1)) if width != 4 else \
            v.astype(np.int32).astype(np.float32) / np.float32(2 ** 31)
        np.testing.assert_array_equal(x.reshape(-1), want)


def test_g711_equals_audioop():
    audioop = _stdlib('audioop')
    codes = bytes(range(256))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', DeprecationWarning)
        ulaw = np.frombuffer(audioop.ulaw2lin(codes, 2), np.int16)
        alaw = np.frombuffer(audioop.alaw2lin(codes, 2), np.int16)
    np.testing.assert_array_equal(oa.ULAW_TABLE, ulaw)
    np.testing.assert_array_equal(oa.ALAW_TABLE, alaw)
    assert oa.ULAW_TABLE[0] == -32124 and oa.ALAW_TABLE[0] == -5504 and oa.ULAW_TABLE[0xFF] == 0


def test_extended_rate_round_trip():
    for v in (1.0, 8000.0, 22050.0, 44100.0, 22254.545454545454, 96000.0, 2.0 ** 31 - 1, 12345.999):
        assert oa.extended_int(oa.extended(v)) == math.floor(v)
    for v in (0.0, 0.999, -44100.0, 2.0 ** 31, float('inf'), float('nan')):
        assert oa.extended_int(oa.extended(v)) is None
    # an unnormalised mantissa (no explicit integer bit) with a large exponent: 3 * 2^2 = 12
    raw = struct.pack('>HQ', 16383 + 65, 3)
    assert oa.extended_int(raw) == 12
    data = case(None, 16, 1)
    c = data.index(b'COMM') + 16
    assert meta_of(data[:c] + raw + data[c + 10:])[0]['rate'] == 12


# ---------------------------------------------------------------------------------------------- refusals
def refusal_cases():
    good = case(None, 16, 2, n=10)
    comm = good.index(b'COMM')
    ssnd = good.index(b'SSND')

    def comm_at(body, comp=False):
        """COMM at byte 12 (no FVER chunk), then an SSND chunk of 40 sample bytes."""
        rest = oa.chunk(b'COMM', body) + oa.chunk(b'SSND', bytes(48))
        return b'FORM' + struct.pack('>I', 4 + len(rest)) + (b'AIFC' if comp else b'AIFF') + rest

    out = [
        ('form_type', b'FORM' + good[4:8] + b'WAVE' + good[12:], 'is neither AIFF nor AIFC', 8),
        ('form_truncated', b'FORM\0\0\0\x20AI', 'FORM header truncated', 0),
        ('no_comm', b'FORM\x00\x00\x00\x20AIFF' + bytes(40), 'no COMM chunk before', 36),
        ('no_comm_marks', b'FORM\x00\x00\x00\x10AIFF' + oa.chunk(b'MARK', b'\0\0'), 'no COMM chunk before', 22),
        ('no_ssnd', good[:ssnd], 'no SSND chunk before', ssnd),
        ('no_ssnd_form_size', good[:4] + struct.pack('>I', ssnd - 8) + good[8:], 'no SSND chunk before', ssnd),
        ('comm_cut', good[:comm + 20], 'COMM chunk truncated', comm),
        ('comm_short', good[:comm + 4] + struct.pack('>I', 16) + good[comm + 8:], 'COMM chunk of', comm),
        ('aifc_comm_short', comm_at(oa.comm_body(1, 16, 8000.0), comp=True), 'COMM chunk of', 12),
        ('ssnd_before_comm', b'FORM' + good[4:12] + good[ssnd:] + good[12:ssnd], 'SSND chunk before the COMM chunk', 12),
        ('ssnd_header_cut', good[:ssnd + 12], 'SSND chunk header truncated', ssnd),
        ('ssnd_offset', good[:ssnd + 8] + struct.pack('>I', 41) + good[ssnd + 12:], 'past its chunk', ssnd),
        ('ssnd_size_7', good[:ssnd + 4] + struct.pack('>I', 7) + good[ssnd + 8:], 'past its chunk', ssnd),
        ('zero_channels', comm_at(oa.comm_body(0, 16, 8000.0)), 'channels (COMM chunk', 12),
        ('negative_channels', comm_at(oa.comm_body(-2, 16, 8000.0)), 'channels (COMM chunk', 12),
        ('sample_size_0', comm_at(oa.comm_body(1, 0, 8000.0)), 'sampleSize', 12),
        ('sample_size_33', comm_at(oa.comm_body(1, 33, 8000.0)), 'sampleSize', 12),
        ('raw_16', comm_at(oa.comm_body(1, 16, 8000.0, b'raw '), comp=True), 'sampleSize', 12),
        ('fl32_64', comm_at(oa.comm_body(1, 64, 8000.0, b'fl32'), comp=True), 'sampleSize', 12),
        ('fl64_32', comm_at(oa.comm_body(1, 32, 8000.0, b'FL64'), comp=True), 'sampleSize', 12),
        ('rate_0', comm_at(oa.comm_body(1, 16, 0.0)), 'sample rate', 12),
        ('rate_half', comm_at(oa.comm_body(1, 16, 0.5)), 'sample rate', 12),
        ('rate_2_31', comm_at(oa.comm_body(1, 16, 2.0 ** 31)), 'sample rate', 12),
        ('rate_negative', comm_at(oa.comm_body(1, 16, -44100.0)), 'sample rate', 12),
        ('rate_inf', comm_at(oa.comm_body(1, 16, float('inf'))), 'sample rate', 12),
        ('rate_nan', comm_at(oa.comm_body(1, 16, float('nan'))), 'sample rate', 12),
    ]
    for comp in (b'ima4', b'GSM ', b'in24', b'\0\x01zz'):
        out.append((f'comp_{comp!r}', comm_at(oa.comm_body(1, 16, 8000.0, comp, b'name'), comp=True),
                    'AIFF-C compression type', 12))
    return out


REFUSALS = refusal_cases()


@pytest.mark.parametrize('name,data,reason,offset', REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_name_the_reason_and_offset(name, data, reason, offset):
    with pytest.raises(oa.AiffError) as e:
        oa.walk(data)
    assert (e.value.reason, e.value.offset) == (reason, offset)
    got, err = meta_of(data)
    assert got is None and err.startswith('AIFF/IFF: ') and reason in err and f'byte offset {offset}' in err, err


def test_compression_type_is_named():
    for comp, shown in ((b'ima4', "'ima4'"), (b'GSM ', "'GSM '"), (b'in24', "'in24'"), (b'\0\x01zz', r"'\x00\x01zz'")):
        data = oa.aiff_bytes(bytes(8), 1, 16, 8000.0, comp=comp, frames=4)
        assert shown in meta_of(data)[1]


def test_other_containers_keep_their_refusal():
    for data, text in ((b'OggS' + bytes(40), 'not a RIFF/WAVE file (Ogg)'), (b'RIFX' + bytes(40), '(big-endian RIFX)'),
                       (b'RF64' + bytes(40), '(RF64)'), (b'caff' + bytes(40), '(Core Audio (CAF))'),
                       (b'.snd' + bytes(40), '(Sun/NeXT AU)'), (b'\xff\xfb\x90\x00' + bytes(40), '(MPEG audio (MP3))')):
        assert text in meta_of(data)[1]


# ---------------------------------------------------------------------------------------------- the resumable walk
def boundaries(data: bytes):
    """Every chunk's first byte, its size field and its body, and the first sample byte (when the walk gets there)."""
    out, p = {4, 8, 12}, 12
    while p + 8 <= len(data):
        out |= {p, p + 4, p + 8}
        size = struct.unpack('>I', data[p + 4:p + 8])[0]
        if data[p:p + 4] == b'SSND':
            out |= {p + 12, p + 16}
            break
        p += 8 + size + (size & 1)
    return sorted(c for b in out for c in (b - 1, b, b + 1))


def check_walk(data: bytes):
    want, err = meta_of(data)
    head = want['data_offset'] + 24 if want else len(data)
    splits = [[], list(range(997, len(data), 997)), list(range(1, min(head, len(data)))), boundaries(data)]
    for cuts in splits + [[c] for c in boundaries(data)]:
        got, gerr, ranges, most = ts.walked(data, cuts)
        assert most <= 48, f'the walker held {most} bytes'
        assert (got, gerr) == (want, err), cuts[:8]
        if got is None:
            continue
        if ranges:
            assert ranges[0][0] == want['data_offset']
            assert all(r[1] == s[0] for r, s in zip(ranges, ranges[1:]))
        reported = ranges[-1][1] - ranges[0][0] if ranges else 0
        frame = want['channels'] * _lib.PCM_BYTES[want['kind']]
        assert want['data_bytes'] <= reported < want['data_bytes'] + frame


@pytest.mark.parametrize('name,data', CASES, ids=[c[0] for c in CASES])
def test_walk_in_pieces_equals_audio_info(name, data):
    check_walk(data)


@pytest.mark.parametrize('name,data,reason,offset', REFUSALS, ids=[c[0] for c in REFUSALS])
def test_walk_refusals_in_pieces(name, data, reason, offset):
    check_walk(data)


def test_known_once_the_ssnd_header_is_read():
    data = case(b'NONE', 16, 2, offset=9, before=[(b'MARK', b'abc')])
    ssnd = data.index(b'SSND')
    w = C.c_void_p()
    assert lib.some_audio_walk_create(1, C.byref(w)) == 0
    known, m = C.c_int(), _lib.AudioMeta()
    a, b, held = C.c_longlong(), C.c_longlong(), C.c_longlong()
    try:
        for i in range(ssnd + 17):
            assert lib.some_audio_walk_feed(w, data[i:i + 1], 1, 0, C.byref(known), C.byref(m), C.byref(a), C.byref(b),
                                            C.byref(held)) == 0
            assert known.value == (i >= ssnd + 15), i
        assert (m.container, m.channels, m.data_offset, m.frames) == (_lib.AUDIO_AIFF, 2, ssnd + 16 + 9, 101)
    finally:
        lib.some_audio_walk_destroy(w)
