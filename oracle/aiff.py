"""Restatement of ``librosa.load(path, sr=..., mono=True)`` for AIFF and AIFF-C files: librosa 0.9 reads them with
``soundfile.SoundFile(path).read(dtype='float32')`` -> libsndfile (aiff.c), then ``to_mono`` and ``resample``
(res_type='kaiser_best', oracle/resample.py).  Every coding read here is integer or IEEE PCM or G.711, so each sample has
one right float32 value.

- ``walk``: the container walk some_audio_info does (csrc/audio_host.cu), in plain Python: ``FORM`` + ``AIFF`` / ``AIFC``,
  big-endian chunks padded to an even length within the FORM size; COMM (numChannels, numSampleFrames, sampleSize, an
  80-bit extended sampleRate and, in AIFF-C, the compression type; its pascal-string name is skipped with the chunk) must
  come before SSND (offset, blockSize); the walk ends at SSND.  Returns the metadata and the byte range of the samples, or
  raises ``AiffError`` with the reason's key words and the byte offset.
- ``samples``: the bytes of that range as libsndfile scales them: integer samples left-justified in ceil(sampleSize / 8)
  bytes divided by 2^(8 bytes - 1) (int32 rounded to float32 first), ``raw `` 8-bit (x - 128) / 128, ``fl32`` as is,
  ``fl64`` rounded to float32, ``ulaw`` / ``alaw`` the 16-bit G.711 value / 32768.
- ``aiff_bytes`` / ``raw_samples``: a writer for test vectors that can place every chunk, offset and size.
- ``load``: walk -> samples -> to_mono -> oracle.resample.resample.

Restated from libsndfile's aiff.c, ulaw.c and alaw.c (as published) WITHOUT being compared with the library, which was not
available where this was written: the truncation of the extended rate to its integer part; the frame count taken from the
SSND bytes (whole frames within its stated size and the file) rather than COMM's numSampleFrames; the scaling of 1-8 bit
signed samples by 1/128; the G.711 tables (computed here with the standard bit arithmetic of Sun's g711.c).

Cross-checked against independent implementations in Python 3.12's standard library (tests/test_aiff_cpu.py): ``aifc`` for
the chunk walk, channels, rate and frames of the files it writes (NONE, sowt, ulaw, alaw), and ``audioop.ulaw2lin`` /
``alaw2lin`` for all 256 G.711 codes.

TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction

import numpy as np

from . import resample as ors

# the device's SOME_PCM_* codes
U8, S16, S24, S32, F32, F64, S8, S16BE, S24BE, S32BE, F32BE, F64BE, ULAW, ALAW = range(1, 15)
SAMPLE_BYTES = {U8: 1, S16: 2, S24: 3, S32: 4, F32: 4, F64: 8, S8: 1, S16BE: 2, S24BE: 3, S32BE: 4, F32BE: 4, F64BE: 8,
                ULAW: 1, ALAW: 1}


class AiffError(ValueError):
    """A refusal: ``reason`` (key words of some_audio_info's message) at byte ``offset``."""

    def __init__(self, reason: str, offset: int):
        super().__init__(f'AIFF/IFF: {reason} (at byte offset {offset})')
        self.reason, self.offset = reason, offset


# ---------------------------------------------------------------------------------------------- G.711
def ulaw_value(code: int) -> int:
    u = ~code & 0xFF
    t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
    return 0x84 - t if u & 0x80 else t - 0x84


def alaw_value(code: int) -> int:
    a = code ^ 0x55
    t = (a & 0x0F) << 4
    seg = (a & 0x70) >> 4
    t = t + 8 if seg == 0 else (t + 0x108) << (seg - 1)
    return t if a & 0x80 else -t


ULAW_TABLE = np.array([ulaw_value(c) for c in range(256)], np.int16)
ALAW_TABLE = np.array([alaw_value(c) for c in range(256)], np.int16)


# ---------------------------------------------------------------------------------------------- the 80-bit rate
def extended(value: float) -> bytes:
    """An IEEE 754 80-bit extended value (the one a float64 holds exactly; inf and nan too)."""
    sign = 0x8000 if math.copysign(1.0, value) < 0 else 0
    if math.isnan(value):
        return struct.pack('>HQ', 0x7FFF, 0xC000000000000000)
    if math.isinf(value):
        return struct.pack('>HQ', sign | 0x7FFF, 1 << 63)
    if value == 0:
        return struct.pack('>HQ', sign, 0)
    m, e = math.frexp(abs(value))                      # 0.5 <= m < 1
    return struct.pack('>HQ', sign | (e - 1 + 16383), int(m * (1 << 64)))


def extended_int(b: bytes):
    """The integer part of the extended value (libsndfile's conversion), or None when it is not finite, below 1 or at
    least 2^31."""
    se, mant = struct.unpack('>HQ', b)
    sign, e = se >> 15, (se & 0x7FFF) - 16383
    if (se & 0x7FFF) == 0x7FFF or sign:
        return None
    ip = math.floor(Fraction(mant) * Fraction(2) ** (e - 63))
    return ip if 1 <= ip < 1 << 31 else None


# ---------------------------------------------------------------------------------------------- the walk
def coding(comp: bytes, bits: int):
    """(kind, None) for a compression type and sampleSize, or (None, reason)."""
    if comp in (b'NONE', b'twos', b'sowt'):
        le = comp == b'sowt'
        for lo, hi, be_kind, le_kind in ((1, 8, S8, S8), (9, 16, S16BE, S16), (17, 24, S24BE, S24), (25, 32, S32BE, S32)):
            if lo <= bits <= hi:
                return (le_kind if le else be_kind), None
        return None, 'sampleSize'
    if comp == b'raw ':
        return (U8, None) if bits == 8 else (None, 'sampleSize')
    if comp in (b'fl32', b'FL32'):
        return (F32BE, None) if bits == 32 else (None, 'sampleSize')
    if comp in (b'fl64', b'FL64'):
        return (F64BE, None) if bits == 64 else (None, 'sampleSize')
    if comp in (b'ulaw', b'ULAW'):
        return ULAW, None
    if comp in (b'alaw', b'ALAW'):
        return ALAW, None
    return None, 'AIFF-C compression type'


def walk(data: bytes) -> dict:
    """The metadata some_audio_info reports for an AIFF / AIFF-C file (container 3), or AiffError."""
    if len(data) < 12:
        raise AiffError('FORM header truncated', 0)
    assert data[:4] == b'FORM'
    if data[8:12] not in (b'AIFF', b'AIFC'):
        raise AiffError('is neither AIFF nor AIFC', 8)
    aifc = data[8:12] == b'AIFC'
    form_end = struct.unpack('>I', data[4:8])[0] + 8
    p, comm = 12, None
    while True:
        if p + 8 > form_end or p + 8 > len(data):
            raise AiffError(f'no {"SSND" if comm else "COMM"} chunk before', p)
        cid, size = data[p:p + 4], struct.unpack('>I', data[p + 4:p + 8])[0]
        if cid == b'COMM':
            need = 22 if aifc else 18
            if size < need:
                raise AiffError('COMM chunk of', p)
            if p + 8 + need > len(data):
                raise AiffError('COMM chunk truncated', p)
            ch, _, bits = struct.unpack('>hIh', data[p + 8:p + 16])
            if ch < 1:
                raise AiffError('channels (COMM chunk', p)
            comp = data[p + 26:p + 30] if aifc else b'NONE'
            kind, why = coding(comp, bits)
            if kind is None:
                raise AiffError(why, p)
            rate = extended_int(data[p + 16:p + 26])
            if rate is None:
                raise AiffError('sample rate', p)
            comm = dict(rate=rate, channels=ch, bits=bits, kind=kind)
        elif cid == b'SSND':
            if comm is None:
                raise AiffError('SSND chunk before the COMM chunk', p)
            if p + 16 > len(data):
                raise AiffError('SSND chunk header truncated', p)
            offset = struct.unpack('>I', data[p + 8:p + 12])[0]
            if size < 8 or offset > size - 8:
                raise AiffError('past its chunk', p)
            frame = comm['channels'] * SAMPLE_BYTES[comm['kind']]
            begin = p + 16 + offset
            avail = min(size - 8 - offset, max(len(data) - begin, 0))
            frames = avail // frame
            return dict(container=3, min_blocksize=0, max_blocksize=0, frames=frames, data_offset=begin,
                        data_bytes=frames * frame, **comm)
        p += 8 + size + (size & 1)


def samples(data: bytes, meta: dict) -> np.ndarray:
    """float32 [frames, channels] as libsndfile hands them to librosa."""
    if meta['data_bytes'] == 0:
        return np.zeros((0, meta['channels']), np.float32)
    raw = np.frombuffer(data, np.uint8, count=meta['data_bytes'], offset=meta['data_offset'])
    k = meta['kind']
    if k in (S24, S24BE):
        b = raw.reshape(-1, 3).astype(np.uint32)
        if k == S24BE:
            b = b[:, ::-1]
        v = ((b[:, 0] << 8) | (b[:, 1] << 16) | (b[:, 2] << 24)).view(np.int32)
        x = v.astype(np.float32) / np.float32(2 ** 31)
    elif k in (ULAW, ALAW):
        x = (ULAW_TABLE if k == ULAW else ALAW_TABLE)[raw].astype(np.float32) / np.float32(32768)
    elif k == U8:
        x = (raw.astype(np.float32) - np.float32(128)) / np.float32(128)
    else:
        dt = {S8: 'i1', S16: '<i2', S16BE: '>i2', S32: '<i4', S32BE: '>i4', F32: '<f4', F32BE: '>f4', F64: '<f8',
              F64BE: '>f8'}[k]
        v = raw.view(dt)
        x = v.astype(np.float32)
        if v.dtype.kind == 'i':
            x = x / np.float32(2 ** (8 * v.dtype.itemsize - 1))
    return x.reshape(-1, meta['channels'])


def to_mono(x: np.ndarray) -> np.ndarray:
    """librosa.to_mono of librosa's (channels, n) view: np.mean in float32 (one channel: the samples themselves)."""
    return x[:, 0].copy() if x.shape[1] == 1 else np.mean(x.T, axis=0)


def load(data: bytes, sr=None, mono=True):
    """librosa.load of an AIFF file's bytes: (y, rate), y [n] (mono or one channel) or [channels, n]."""
    m = walk(data)
    x = samples(data, m)
    y = to_mono(x) if mono or x.shape[1] == 1 else np.ascontiguousarray(x.T)
    if sr is None or sr == m['rate']:
        return y, m['rate']
    return ors.resample(y, m['rate'], sr), sr


# ---------------------------------------------------------------------------------------------- test vectors
def raw_samples(kind: int, n: int, ch: int, seed: int) -> bytes:
    """n frames of ch channels of random samples in a kind's byte layout (floats: normal values of scale 0.3)."""
    rng = np.random.default_rng(seed)
    if kind in (F32, F32BE, F64, F64BE):
        dt = {F32: '<f4', F32BE: '>f4', F64: '<f8', F64BE: '>f8'}[kind]
        return (rng.standard_normal(n * ch) * 0.3).astype(dt).tobytes()
    return rng.integers(0, 256, n * ch * SAMPLE_BYTES[kind], dtype=np.uint8).tobytes()


def chunk(cid: bytes, body: bytes, size=None) -> bytes:
    """An IFF chunk: id, big-endian size (the body's unless given), body, pad byte to an even length."""
    return cid + struct.pack('>I', len(body) if size is None else size) + body + (b'\0' if len(body) % 2 else b'')


def comm_body(channels: int, bits: int, rate: float, comp=None, name=b'', frames=0) -> bytes:
    body = struct.pack('>hIh', channels, frames, bits) + extended(rate)
    if comp is not None:
        pstr = bytes([len(name)]) + name
        body += comp + pstr + (b'\0' if len(pstr) % 2 else b'')
    return body


def aiff_bytes(raw: bytes, channels: int, bits: int, rate: float, comp=None, name=b'', before=(), between=(), after=(),
               offset=0, block_size=0, frames=None, ssnd_size=None, form_size=None, form_type=None) -> bytes:
    """An AIFF (comp None) or AIFF-C file: FORM, the chunks `before`, COMM, the chunks `between`, SSND (`offset` bytes of
    zeros in front of the samples), the chunks `after`.  frames: COMM's numSampleFrames (default: from raw)."""
    if frames is None:
        frames = len(raw) // max(channels, 1) // SAMPLE_BYTES.get(_kind_of(comp, bits), 1)
    aifc = comp is not None
    body = (form_type or (b'AIFC' if aifc else b'AIFF'))
    if aifc:
        body += chunk(b'FVER', struct.pack('>I', 0xA2805140))
    body += b''.join(chunk(c, b) for c, b in before)
    body += chunk(b'COMM', comm_body(channels, bits, rate, comp, name, frames))
    body += b''.join(chunk(c, b) for c, b in between)
    ssnd = struct.pack('>II', offset, block_size) + bytes(offset) + raw
    body += chunk(b'SSND', ssnd, ssnd_size)
    body += b''.join(chunk(c, b) for c, b in after)
    return b'FORM' + struct.pack('>I', len(body) if form_size is None else form_size) + body


def _kind_of(comp, bits):
    kind, _ = coding(comp if comp is not None else b'NONE', bits)
    return kind
