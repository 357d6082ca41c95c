"""CPU tests of the FLAC restatement (oracle/flac.py) and of the host half of some_b200.audio's FLAC path: the CRC check
values, frames assembled bit by bit here from the format description (independently of the oracle's encoder), the
encoder -> decoder round trip over every feature the encoder can force, every refusal, and the ID3v2 skip."""
import re

import numpy as np
import pytest
import torch

from oracle import flac as of
from some_b200 import audio

REFUSAL = re.compile(r'FLAC.*byte offset \d+')


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, value, n):
        self.bits += [(value >> (n - 1 - i)) & 1 for i in range(n)]

    def unary(self, q):
        self.bits += [0] * q + [1]

    def pad(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def bytes(self):
        assert len(self.bits) % 8 == 0
        return bytes(int(''.join(map(str, self.bits[i:i + 8])), 2) for i in range(0, len(self.bits), 8))


def streaminfo(min_bs, max_bs, rate, channels, bps, total, last=True):
    w = BitWriter()
    w.put(0x80 if last else 0, 8)
    w.put(34, 24)
    for v, n in ((min_bs, 16), (max_bs, 16), (0, 24), (0, 24), (rate, 20), (channels - 1, 3), (bps - 1, 5), (total, 36)):
        w.put(v, n)
    w.put(0, 128)
    return b'fLaC' + w.bytes()


def frame(number, bs_code, sr_code, ch_code, bps_code, body, extra=b'', variable=True, crc8_fix=0, crc16_fix=0):
    """A frame: header (+ explicit block-size / rate bytes ``extra``), CRC-8, the subframes written by ``body(w)``,
    zero padding, CRC-16.  The *_fix arguments corrupt a CRC."""
    w = BitWriter()
    w.put(0xFFF8 | int(variable), 16)
    w.put(bs_code, 4)
    w.put(sr_code, 4)
    w.put(ch_code, 4)
    w.put(bps_code, 3)
    w.put(0, 1)
    assert number < 0x80
    w.put(number, 8)
    head = w.bytes() + extra
    head += bytes([of.crc8(head) ^ crc8_fix])
    w = BitWriter()
    body(w)
    w.pad()
    data = head + w.bytes()
    return data + ((of.crc16(data) ^ crc16_fix).to_bytes(2, 'big'))


def sub_header(w, kind, wasted=0):
    w.put(0, 1)
    w.put(kind, 6)
    w.put(1 if wasted else 0, 1)
    if wasted:
        w.unary(wasted - 1)


def b_constant(w):                                    # CONSTANT -5
    sub_header(w, 0b000000)
    w.put(-5, 16)


def b_verbatim(w):
    sub_header(w, 0b000001)
    for v in (1, -2, 3, 32767):
        w.put(v, 16)


def b_fixed2(w):
    """FIXED order 2, warm-up 10, 12; method 0, partition order 1: partition 0 = Rice k=1 (residuals 1, -1),
    partition 1 escaped at 4 bits (3, -4, 0, 7)."""
    sub_header(w, 0b001010)
    w.put(10, 16)
    w.put(12, 16)
    w.put(0, 2)
    w.put(1, 4)
    w.put(1, 4)
    w.unary(1)                                        # 1 -> u = 2: q = 1, low bit 0
    w.put(0, 1)
    w.unary(0)                                        # -1 -> u = 1: q = 0, low bit 1
    w.put(1, 1)
    w.put(15, 4)
    w.put(4, 5)
    for v in (3, -4, 0, 7):
        w.put(v, 4)


def b_lpc3(w):
    """LPC order 3, warm-up 100, 110, 118, precision 4, shift 2, coefficients 6, -3, 1; Rice k=2: 1, -2, 0."""
    sub_header(w, 0b100010)
    for v in (100, 110, 118):
        w.put(v, 16)
    w.put(4 - 1, 4)
    w.put(2, 5)
    for c in (6, -3, 1):
        w.put(c, 4)
    w.put(0, 2)
    w.put(0, 4)
    w.put(2, 4)
    for u in (2, 3, 0):                               # zigzag of 1, -2, 0
        w.unary(u >> 2)
        w.put(u & 3, 2)


def b_wasted(w):                                      # VERBATIM with 2 wasted bits: 3, -1, 5, 0 at 14 bits
    sub_header(w, 0b000001, wasted=2)
    for v in (3, -1, 5, 0):
        w.put(v, 14)


def b_midside(w):                                     # mid 16 bits, side 17 bits, both VERBATIM
    sub_header(w, 0b000001)
    for v in (5, -3, 0, 100):
        w.put(v, 16)
    sub_header(w, 0b000001)
    for v in (1, 2, -1, 7):
        w.put(v, 17)


MONO_WANT = [-5] * 4 + [1, -2, 3, 32767] + [10, 12, 15, 17, 22, 23, 24, 32] + [100, 110, 118, 120, 117, 115] + [12, -4, 20, 0]


def hand_mono(corrupt=None):
    """Variable blocking, 16-bit mono: CONSTANT (8-bit explicit block size, 16-bit sample-rate code), VERBATIM, FIXED-2,
    LPC-3, wasted bits."""
    frames = [(4, b_constant), (4, b_verbatim), (8, b_fixed2), (6, b_lpc3), (4, b_wasted)]
    out, n = streaminfo(4, 8, 44100, 1, 16, 26), 0
    for k, (bs, body) in enumerate(frames):
        kw = dict(crc8_fix=1) if corrupt == ('crc8', k) else dict(crc16_fix=1) if corrupt == ('crc16', k) else {}
        if k == 0:
            out += frame(n, 6, 13, 0, 4, body, extra=bytes([bs - 1]) + (44100).to_bytes(2, 'big'), **kw)
        else:
            out += frame(n, 6, 9, 0, 4, body, extra=bytes([bs - 1]), **kw)
        n += bs
    return out


def test_crc_check_values():
    assert of.crc8(b'123456789') == 0xF4
    assert of.crc16(b'123456789') == 0xFEE8


def test_hand_assembled_frames_decode_to_the_written_samples():
    x, info = of.decode(hand_mono())
    assert (info['rate'], info['channels'], info['bps']) == (44100, 1, 16)
    assert x[:, 0].tolist() == MONO_WANT
    stereo = streaminfo(4, 4, 48000, 2, 16, 4) + frame(0, 6, 10, 10, 4, b_midside, extra=bytes([3]), variable=False)
    x, _ = of.decode(stereo)
    assert x.tolist() == [[6, 5], [-2, -4], [0, 1], [104, 97]]


@pytest.mark.parametrize('case', of.feature_cases(), ids=lambda c: c[0])
def test_encoder_decoder_round_trip(case):
    name, x, kw = case
    data = of.encode(x, **kw)
    y, info = of.decode(data, name)
    np.testing.assert_array_equal(y, x)
    assert (info['rate'], info['channels'], info['bps']) == (kw['rate'], x.shape[1], kw['bps'])
    rec = audio.parse_flac(data, name)                      # the native container walk agrees with the oracle's metadata
    assert (rec.rate, rec.channels, rec.bps, rec.length, rec.min_blocksize, rec.max_blocksize, rec.audio_offset) == \
        (info['rate'], info['channels'], info['bps'], info['total'], info['min_blocksize'], info['max_blocksize'],
         info['audio_offset'])
    assert rec.length == (0 if kw.get('total_samples') == 0 else len(x))


def test_encoder_forces_what_it_is_asked():
    x = of.test_signal(4096, 1, 16, 3)
    data = of.encode(x, 44100, 16, subframe={'type': 'lpc', 'order': 7, 'precision': 9, 'shift': 5, 'method': 1,
                                             'porder': 2}, id3=of.id3_tag())
    head = data[of.id3_size(data) + 42:]
    assert head[:2] == b'\xff\xf8' and head[2] >> 4 == 12 and head[2] & 15 == 9   # 4096 -> code 12, 44.1 kHz -> 9
    sub = int.from_bytes(head[6:8], 'big')                                          # after the 6-byte header
    assert sub >> 8 == (0b100000 | 6) << 1                                          # LPC, order 7, no wasted bits
    v = of.encode(x, 44100, 16, blocksize=[96, 4000], variable=True)
    assert v[42 + 1] == 0xF9


def _metadata_refusals():
    good = of.encode(of.test_signal(100, 1, 16, 0), 44100, 16)
    si = bytearray(good)
    si[4 + 4 + 12] |= 0x01                                      # bps - 1 = 31: 32 bits per sample (5 bits over bytes 20-21)
    si[4 + 4 + 13] |= 0xF0
    return [
        ('streaminfo_length_0', b'fLaC' + b'\x00' * 60),
        ('no_marker', b'fLaX' + good[4:]),
        ('first_not_streaminfo', b'fLaC' + b'\x01' + good[5:]),
        ('metadata_truncated', good[:30]),
        ('block_127', good[:4] + bytes([good[4] & 0x7F]) + good[5:42] + b'\xff\x00\x00\x00' + good[42:]),
        ('bps_32', bytes(si)),
    ]


@pytest.mark.parametrize('name,data', _metadata_refusals(), ids=lambda v: v if isinstance(v, str) else '')
def test_metadata_refusals(name, data, tmp_path):
    with pytest.raises(ValueError, match=REFUSAL):
        of.parse_metadata(data, name)
    with pytest.raises(ValueError, match=REFUSAL):
        audio.parse_flac(data, name)
    p = tmp_path / 'x.flac'
    p.write_bytes(data)
    if data[:4] == b'fLaC':                                     # load() takes it for FLAC and refuses before any device work
        with pytest.raises(ValueError, match=REFUSAL):
            audio.load(p, sr=None)


def _bad_subframe(kind):
    def body(w):
        sub_header(w, kind)
        w.put(0, 64)
    return body


def _frame_refusals():
    x = of.test_signal(10000, 2, 16, 7)
    good = of.encode(x, 44100, 16, blocksize=4096)
    first = 42                                                  # fLaC + STREAMINFO
    hdr = lambda body: streaminfo(4, 4, 44100, 1, 16, 4) + frame(0, 6, 9, 0, 4, body, extra=b'\x03')   # noqa: E731

    def lpc_bad(prec_code, shift):
        def body(w):
            sub_header(w, 0b100000)
            w.put(7, 16)
            w.put(prec_code, 4)
            w.put(shift, 5)
            w.put(0, 64)
        return body

    def residual_method(m):
        def body(w):
            sub_header(w, 0b001000)
            w.put(m, 2)
            w.put(0, 64)
        return body
    flipped = bytearray(good)
    flipped[first + 3000] ^= 0x10                               # inside frame 0's subframes
    return [
        ('crc8', hand_mono(corrupt=('crc8', 2))),
        ('crc16', hand_mono(corrupt=('crc16', 3))),
        ('flipped_bit', bytes(flipped)),
        ('truncated_last_frame', good[:-5]),
        ('truncated_stream', good[:first + 10]),
        ('reserved_subframe', hdr(_bad_subframe(0b000010))),
        ('fixed_order_5', hdr(_bad_subframe(0b001101))),
        ('lpc_precision_1111', hdr(lpc_bad(15, 2))),
        ('lpc_negative_shift', hdr(lpc_bad(3, 0b11110))),
        ('residual_method_2', hdr(residual_method(2))),
        ('frame_gap', of.encode(x, 44100, 16, blocksize=4096, frame_numbers=[0, 1, 3])),
        ('frame_overlap', of.encode(x, 44100, 16, blocksize=4096, frame_numbers=[0, 0, 1])),
        ('sample_gap', of.encode(x, 44100, 16, blocksize=[5000, 5000], variable=True, frame_numbers=[0, 5001])),
        ('blocking_changed', of.encode(x[:5000], 44100, 16, blocksize=[4096, 904], variable=True)[:42] +
         of.encode(x[:4096], 44100, 16, blocksize=4096)[42:] + of.encode(x[4096:5000], 44100, 16, blocksize=[904],
                                                                          variable=True, frame_numbers=[4096])[42:]),
        ('more_than_streaminfo', of.encode(x, 44100, 16, blocksize=4096, total_samples=9000)),
        ('fewer_than_streaminfo', of.encode(x, 44100, 16, blocksize=4096, total_samples=10001)),
        ('reserved_blocksize_code', good[:first] + good[first:first + 2] + bytes([good[first + 2] & 0x0F]) + good[first + 3:]),
        ('reserved_channel_code', good[:first] + good[first:first + 3] + bytes([0xB0 | (good[first + 3] & 0x0F)]) +
         good[first + 4:]),
        ('trailing_garbage_unknown_total', of.encode(x, 44100, 16, total_samples=0) + b'\x00' * 7),
    ]


FRAME_REFUSALS = _frame_refusals()


@pytest.mark.parametrize('name,data', FRAME_REFUSALS, ids=[n for n, _ in FRAME_REFUSALS])
def test_frame_refusals(name, data):
    with pytest.raises(ValueError, match=REFUSAL):
        of.decode(data, name)


def test_trailing_bytes_after_the_stated_length_are_ignored():
    x = of.test_signal(5000, 1, 16, 2)
    y, _ = of.decode(of.encode(x, 44100, 16) + b'\xff\xf8 anything')
    np.testing.assert_array_equal(y, x)


@pytest.mark.parametrize('footer', [False, True])
def test_id3v2_tagged_flac_is_read_as_flac(footer, tmp_path, monkeypatch):
    x = of.test_signal(3000, 2, 16, 4)
    tag = of.id3_tag(b'TIT2\x00\x00\x00\x06\x00\x00\xff\xf8\xc9\x08', footer=footer)   # a sync pattern inside the tag
    data = of.encode(x, 44100, 16, id3=tag)
    assert of.id3_size(data) == len(tag) and data[len(tag):len(tag) + 4] == b'fLaC'
    y, info = of.decode(data)
    np.testing.assert_array_equal(y, x)
    assert audio.parse_flac(data).audio_offset == info['audio_offset']
    p = tmp_path / 'tagged.flac'
    p.write_bytes(data)
    taken = []                                                  # load() takes it for FLAC: the record goes to the device path

    def flac_device(rec, mono):
        taken.append(rec)
        return torch.zeros(rec.length), None
    monkeypatch.setattr(audio, '_flac_device', flac_device)
    assert audio.load(p, sr=None)[1] == 44100
    assert [(r.audio_offset, r.length, r.channels) for r in taken] == [(info['audio_offset'], len(x), 2)]
    assert taken[0].data == data and taken[0].name == str(p)
    with pytest.raises(ValueError, match='not a RIFF/WAVE file'):  # decode_wav keeps refusing FLAC files
        audio.decode_wav(p)
    p.write_bytes(data[len(tag):])
    with pytest.raises(ValueError, match='FLAC'):
        audio.decode_wav(p)


def test_read_encoded_parses_without_decoding(tmp_path):
    x = of.test_signal(7000, 3, 20, 5)
    p = tmp_path / 'a.flac'
    p.write_bytes(of.encode(x, 22050, 20))
    rec = audio.read_encoded(p, 44100)
    assert (rec.rate, rec.channels, rec.bps, rec.length, rec.name) == (22050, 3, 20, 7000, str(p))
    assert rec.data == p.read_bytes()


def test_oracle_load_scales_and_downmixes(tmp_path):
    x = of.test_signal(3000, 3, 24, 6, level=0.99)
    p = tmp_path / 'b.flac'
    p.write_bytes(of.encode(x, 44100, 24))
    y, sr = of.load(p, sr=None)
    f = x.astype(np.float32) * np.float32(2.0 ** -23)
    assert sr == 44100
    np.testing.assert_array_equal(y, audio.to_mono(f.T))
    y2, _ = of.load(p, sr=None, mono=False)
    np.testing.assert_array_equal(y2, f.T)
