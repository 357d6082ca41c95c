"""Audio loading as the reference's callers do it: ``librosa.load(path, sr=config['audio_sample_rate'], mono=True)``
(infer.py:34, batch_infer.py:51, webui.py:47), with librosa<0.10 (requirements.txt:10), whose default ``res_type`` is
``'kaiser_best'`` = ``resampy.resample(x, sr_orig, sr_new, filter='kaiser_best')``.

- ``decode_wav`` / ``to_mono``: libsndfile's integer -> float32 scaling for RIFF/WAVE files and librosa.to_mono.
- ``resample``: librosa.resample(res_type='kaiser_best') on the GPU (csrc/resample.cu, some_resample_kaiser), BIT-identical to
  resampy's float32 loop; numpy in -> numpy out, CUDA tensor in -> CUDA tensor out on the current stream.
- ``audio_info``: the native container walk (some_audio_info, csrc/audio_host.cu) on a file's bytes, the one reader of
  FLAC and AIFF headers: container, rate, channels, sample kind, frames and where the audio starts.
- ``read_encoded`` / ``parse_flac`` / ``EncodedAudio`` / ``FlacBatch`` / ``decode_flac``: FLAC files (libsndfile reads them
  through libFLAC) decoded on the GPU (csrc/flac.cu): the file's bytes and its STREAMINFO (from ``audio_info``) are read on
  the host, the frames are found, checked and decoded on the device, many recordings in one set of launches, straight to
  mono if wanted.
- ``decode_aiff``: AIFF and AIFF-C files as libsndfile reads them, decoded on the GPU: the container is walked on the host
  (``audio_info``), the SSND bytes go up and one some_pcm_decode (csrc/pcm.cu) scales them (integer PCM of 1-32 bits in
  either byte order, 8-bit unsigned, big-endian float32 / float64, G.711 u-law and A-law).
- ``load``: librosa.load for RIFF/WAVE files (PCM 8/16/24/32-bit, float32/64, WAVE_FORMAT_EXTENSIBLE; read by
  ``decode_wav``), and, through ``audio_info``, for FLAC files (``fLaC``, optionally behind an ID3v2 tag; up to 24 bits
  per sample) and AIFF / AIFF-C files (``FORM``), chosen by the file's content.  Other containers (Ogg, MP3, ...) raise:
  librosa decodes those through libsndfile / audioread, which this module does not restate.
- ``load_native``: the decoded recording at its own rate, for batch.batch_infer_dataset's device-resident resampling.

The arithmetic is restated in oracle/resample.py, oracle/flac.py and oracle/aiff.py (test infrastructure), which document
what was restated and what could not be compared with the libraries themselves.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import functools
import re
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

NUM_ZEROS, NUM_TABLE = 64, 512                       # kaiser_best: 64 zero crossings, precision 9
ROLLOFF, BETA = 0.9475937167399596, 14.769656459379492

_FORMATS = {b'fLaC': 'FLAC', b'OggS': 'Ogg', b'ID3': 'MP3 (ID3 tag)', b'FORM': 'AIFF/IFF', b'RIFX': 'big-endian RIFX',
            b'RF64': 'RF64', b'caff': 'Core Audio (CAF)', b'.snd': 'Sun/NeXT AU'}


# ---------------------------------------------------------------------------------------------- decode (host)
def decode_wav(path) -> Tuple[np.ndarray, int]:
    """(samples, native rate) of a RIFF/WAVE file as libsndfile hands them to librosa.load: float32 [n] or [n, channels];
    8-bit unsigned -> (x - 128) / 128, 16/24/32-bit signed -> x / 2^(bits - 1), float / double -> cast to float32.
    scipy reads 24-bit samples left-justified in int32, so x / 2^31 is libsndfile's x / 2^23 exactly."""
    from scipy.io import wavfile
    with open(path, 'rb') as f:
        head = f.read(12)
    if len(head) < 12 or head[:4] != b'RIFF' or head[8:12] != b'WAVE':
        kind = next((name for magic, name in _FORMATS.items() if head.startswith(magic)), None)
        if kind is None and len(head) >= 2 and head[0] == 0xFF and (head[1] & 0xE0) == 0xE0:
            kind = 'MPEG audio (MP3)'
        raise ValueError(f'{path}: not a RIFF/WAVE file ({kind or "unrecognised header " + repr(head[:12])}); '
                         f'some_b200.audio reads WAV files only')
    rate, data = wavfile.read(path)
    if data.dtype.kind == 'i':
        x = data.astype(np.float32) / float(1 << (8 * data.dtype.itemsize - 1))
    elif data.dtype.kind == 'u':
        x = (data.astype(np.float32) - 128.0) / 128.0
    else:
        x = data.astype(np.float32)
    return x, int(rate)


def to_mono(y: np.ndarray) -> np.ndarray:
    """librosa.to_mono for librosa's (channels, n) layout: the float32 mean over channels."""
    return np.mean(y, axis=0) if y.ndim > 1 else y


# ---------------------------------------------------------------------------------------------- resampling (device)
def as_rate(sr) -> int:
    """A sample rate as the int the kernel takes (44100.0 is accepted, 44100.5 is not)."""
    if int(sr) != sr or int(sr) <= 0:
        raise ValueError(f'sample rates must be positive integers, got {sr!r}')
    return int(sr)


def resampled_length(n: int, orig_sr: int, target_sr: int) -> int:
    """Length of librosa.resample's output (fix_length to ceil(n * ratio)); raises ValueError like resampy when its own
    output, floor(n * target / orig) samples, would be empty."""
    if orig_sr == target_sr:
        return n
    if n * target_sr // orig_sr < 1:
        raise ValueError(f'Input signal length={n} is too small to resample from {orig_sr}->{target_sr}')
    return int(np.ceil(n * (float(target_sr) / orig_sr)))


@functools.lru_cache(maxsize=None)
def kaiser_best_table() -> np.ndarray:
    """resampy's kaiser_best interpolation table (float64 [32769]) from its published parameters."""
    import scipy.signal
    n = NUM_TABLE * NUM_ZEROS
    sinc = ROLLOFF * np.sinc(ROLLOFF * np.linspace(0, NUM_ZEROS, num=n + 1, endpoint=True))
    taper = scipy.signal.windows.kaiser(2 * n + 1, BETA)[n:]
    win = taper * sinc
    win.setflags(write=False)
    return win


_device_tables: dict = {}


def _device_table(orig_sr: int, target_sr: int, device):
    """The table for one rate pair (scaled by the ratio when downsampling, as resampy does), built once in float64 numpy and
    kept on the device."""
    import torch
    ratio = float(target_sr) / orig_sr
    key = (torch.device(device), ratio if ratio < 1 else 1.0)
    t = _device_tables.get(key)
    if t is None:
        win = kaiser_best_table()
        if ratio < 1:
            win = ratio * win
        t = torch.from_numpy(np.array(win, dtype=np.float64)).to(device)
        torch.cuda.current_stream(device).synchronize()     # once per rate pair: usable from any stream afterwards
        _device_tables[key] = t
    return t


def resample_into(src, src_starts: Sequence[int], src_lens: Sequence[int], dst, dst_starts: Sequence[int],
                  orig_sr: int, target_sr: int) -> None:
    """One some_resample_kaiser launch on the current stream of ``dst``'s device: recording b = src[src_starts[b] :
    + src_lens[b]] (float32 CUDA tensor, at orig_sr) -> dst[dst_starts[b] : + resampled_length(...)] (float32, target_sr)."""
    import torch
    from . import _lib
    orig_sr, target_sr = as_rate(orig_sr), as_rate(target_sr)
    assert src.dtype == torch.float32 and dst.dtype == torch.float32 and src.is_cuda and dst.device == src.device
    lens = [int(n) for n in src_lens]
    outs = [resampled_length(n, orig_sr, target_sr) for n in lens]
    for a, n, d, m in zip(src_starts, lens, dst_starts, outs):
        assert 0 <= a and a + n <= src.numel() and 0 <= d and d + m <= dst.numel(), 'recording outside its buffer'
    if not lens:
        return
    dev = dst.device
    meta = torch.tensor(np.array([list(src_starts), lens, list(dst_starts)], dtype=np.int64), device=dev)
    table = _device_table(orig_sr, target_sr, dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    lib = _lib.load()
    _lib.check(lib.some_resample_kaiser(src.data_ptr(), meta[0].data_ptr(), meta[1].data_ptr(), dst.data_ptr(),
                                        meta[2].data_ptr(), len(lens), max(outs), orig_sr, target_sr, table.data_ptr(),
                                        int(table.numel()), stream), 'some_resample_kaiser')


def resample(y, orig_sr: int, target_sr: int):
    """librosa.resample(y, orig_sr=orig_sr, target_sr=target_sr, res_type='kaiser_best') on the GPU, bit for bit.

    ``y``: float32 samples [n] or [channels, n], a numpy array (returns numpy; runs on the current CUDA device) or a CUDA
    tensor (returns a new CUDA tensor, enqueued on the current stream, no synchronisation).  Equal rates return ``y``
    itself, like librosa.  librosa would compute float64 input in float64; this kernel takes float32 (librosa.load's
    dtype) only."""
    import torch
    orig_sr, target_sr = as_rate(orig_sr), as_rate(target_sr)
    is_np = isinstance(y, np.ndarray)
    if y.dtype != (np.float32 if is_np else torch.float32):
        raise TypeError(f'resample takes float32 samples (librosa.load\'s dtype), got {y.dtype}')
    if y.ndim not in (1, 2):
        raise ValueError(f'resample takes [n] or [channels, n] samples, got shape {tuple(y.shape)}')
    if is_np and not np.isfinite(y).all():                  # librosa.util.valid_audio
        raise ValueError('Audio buffer is not finite everywhere')
    if orig_sr == target_sr:
        return y
    rows, n = (1, y.shape[0]) if y.ndim == 1 else tuple(y.shape)
    m = resampled_length(n, orig_sr, target_sr)
    if is_np:
        src = torch.from_numpy(np.ascontiguousarray(y)).to(torch.device('cuda', torch.cuda.current_device()))
    else:
        if not y.is_cuda:
            raise ValueError('resample takes a numpy array or a CUDA tensor')
        src = y.contiguous()
    with torch.cuda.device(src.device):
        dst = torch.empty((rows, m) if y.ndim == 2 else (m,), dtype=torch.float32, device=src.device)
        resample_into(src, [r * n for r in range(rows)], [n] * rows, dst, [r * m for r in range(rows)], orig_sr, target_sr)
    return dst.cpu().numpy() if is_np else dst


# ---------------------------------------------------------------------------------------------- container metadata (host)
def audio_info(data: bytes, name: str = '<bytes>'):
    """some_audio_info on a file's bytes (host): its _lib.AudioMeta, or ValueError naming the file, the container and the
    byte offset."""
    from . import _lib
    lib = _lib.load()
    m = _lib.AudioMeta()
    if lib.some_audio_info(data, len(data), C.byref(m)):
        raise ValueError(f'{name}: {lib.some_last_error().decode("utf8", "replace")}')
    return m


@dataclasses.dataclass(frozen=True, eq=False)
class EncodedAudio:
    """A FLAC recording as read from disk, not yet decoded: the file's bytes and its STREAMINFO.  ``length`` is the
    STREAMINFO sample count (0 = not stated: known once the frames are decoded)."""
    name: str
    data: bytes
    rate: int
    channels: int
    bps: int
    length: int
    audio_offset: int           # byte offset of the first frame (after any ID3v2 tag, 'fLaC' and the metadata blocks)
    min_blocksize: int
    max_blocksize: int


# How the container walk's refusals of bytes it does not take for FLAC begin; its FLAC refusals name FLAC instead.
_OTHER_CONTAINERS = ('not a RIFF/WAVE file', 'RIFF/WAVE: ', 'AIFF/IFF: ')


def _flac_record(data: bytes, name: str, m) -> EncodedAudio:
    """The record of FLAC bytes from the _lib.AudioMeta some_audio_info gave for them."""
    return EncodedAudio(name=name, data=bytes(data), rate=m.rate, channels=m.channels, bps=m.bits, length=m.frames,
                        audio_offset=m.data_offset, min_blocksize=m.min_blocksize, max_blocksize=m.max_blocksize)


def parse_flac(data: bytes, name: str = '<bytes>') -> EncodedAudio:
    """The metadata of a FLAC stream, read by the native container walk (``audio_info``).  Malformed metadata raises
    ValueError naming the file, FLAC and the byte offset (the first block must be a 34-byte STREAMINFO, type 127 is
    invalid, more than 24 bits per sample are refused); bytes of any other container raise 'not a FLAC stream' with the
    byte offset where the fLaC marker was looked for (after any ID3v2 tag)."""
    from . import _lib
    off = 0
    try:
        m = audio_info(data, name)
    except ValueError as e:
        reason = str(e)[len(name) + 2:]
        if not reason.startswith(_OTHER_CONTAINERS):
            raise
        at = re.search(r'no fLaC marker at byte offset (\d+)', reason)     # the walk names it after an ID3v2 tag
        m, off = None, int(at.group(1)) if at else 0
    if m is None or m.container != _lib.AUDIO_FLAC:
        raise ValueError(f'{name}: not a FLAC stream (no fLaC marker at byte offset {off})')
    return _flac_record(data, name, m)


def read_encoded(path, sr=None) -> EncodedAudio:
    """Reads a FLAC file and parses its metadata on the host; no decoding happens here.  The second argument is the rate
    the caller wants (batch.batch_infer_dataset passes it) and is ignored: the dataset driver decodes the records on the
    device and resamples them straight into the batch's wave buffer."""
    with open(path, 'rb') as f:
        return parse_flac(f.read(), str(path))


# ---------------------------------------------------------------------------------------------- FLAC (device)
_STREAM_DTYPE = np.dtype([('audio_start', '<i8'), ('end', '<i8'), ('channels', '<i4'), ('bps', '<i4'),
                          ('max_blocksize', '<i4'), ('reserved', '<i4')])                       # some_flac_stream
_FRAME_DTYPE = np.dtype([('pos', '<i8'), ('number', '<i8'), ('end', '<i8'), ('stream', '<i4'), ('blocksize', '<i4'),
                         ('header_len', '<i2'), ('chan_code', 'u1'), ('variable', 'u1'), ('status', '<i4')])  # some_flac_frame


class FlacBatch:
    """FLAC recordings uploaded into one device buffer, their frames found, checked and chained (some_flac_scan, then one
    device-to-host copy of the candidate list and the chain on the host).  Raises ValueError naming the file, FLAC and the
    byte offset for a corrupt stream.  ``lengths`` are then known, and ``emit`` enqueues the decode of any of the
    recordings into slices of a float32 CUDA tensor on the current stream, without synchronising."""

    def __init__(self, records: Sequence[EncodedAudio], device):
        import torch
        from . import _lib
        self.records = list(records)
        self.device = torch.device(device)
        sizes = [len(r.data) for r in self.records]
        bases = np.zeros(len(sizes) + 1, dtype=np.int64)
        np.cumsum(sizes, out=bases[1:])
        streams = np.zeros(len(self.records), _STREAM_DTYPE)
        for i, r in enumerate(self.records):
            streams[i] = (bases[i] + r.audio_offset, bases[i + 1], r.channels, r.bps, r.max_blocksize, 0)
        lib = _lib.load()
        stream = torch.cuda.current_stream(self.device)
        host = np.empty(max(int(bases[-1]), 1), np.uint8)
        for r, a in zip(self.records, bases):
            host[a:a + len(r.data)] = np.frombuffer(r.data, np.uint8)
        self.data = torch.from_numpy(host).to(self.device)
        self.streams = torch.from_numpy(streams.view(np.uint8).copy()).to(self.device)
        ws = torch.empty(int(lib.some_flac_scan_workspace_bytes(int(bases[-1]))), dtype=torch.uint8, device=self.device)
        count = torch.zeros(1, dtype=torch.int32, device=self.device)
        # real frames: at most length / min block size + 1 each; false sync patterns are rare (a CRC-8 and the STREAMINFO
        # must both match), and a larger list is made if they do not fit
        capacity = 64 + sum((r.length // max(r.min_blocksize, 1) + 2) if r.length else (len(r.data) // 16 + 2)
                            for r in self.records)
        while True:
            frames = torch.empty(capacity * _FRAME_DTYPE.itemsize, dtype=torch.uint8, device=self.device)
            _lib.check(lib.some_flac_scan(self.data.data_ptr(), int(bases[-1]), self.streams.data_ptr(), len(self.records),
                                          frames.data_ptr(), capacity, count.data_ptr(), ws.data_ptr(),
                                          C.c_void_p(stream.cuda_stream)), 'some_flac_scan')
            n = int(count.item())                                             # syncs
            if n <= capacity:
                break
            capacity = n
        self.frames, self.n_candidates = frames, n
        fr = frames[:n * _FRAME_DTYPE.itemsize].cpu().numpy().view(_FRAME_DTYPE)
        self._chain(fr, bases)

    def _chain(self, fr, bases):
        """Walks every recording from its first audio byte (some_flac_chain, the walk the session uses too): each next frame
        starts where the current one ends and carries the next frame number (fixed blocking) or sample number (variable
        blocking)."""
        from . import _lib
        n, k = len(fr), len(self.records)
        frames = np.ascontiguousarray(fr)
        recs = (_lib.FlacRange * max(k, 1))()
        for r, rec in enumerate(self.records):
            recs[r] = _lib.FlacRange(int(bases[r]), int(bases[r]) + rec.audio_offset, int(bases[r + 1]), rec.length)
        chain = np.zeros(max(n, 1), np.int32)
        first = np.zeros(k + 1, np.int64)
        lengths = np.zeros(max(k, 1), np.int64)
        failed = C.c_int(-1)
        lib = _lib.load()
        if lib.some_flac_chain(frames.ctypes.data if n else None, n, recs, k, chain.ctypes.data, n, first.ctypes.data,
                               lengths.ctypes.data, C.byref(failed)):
            msg = lib.some_last_error().decode('utf8', 'replace')
            if failed.value < 0:
                raise _lib.SomeB200Error(f'some_flac_chain failed: {msg}')
            raise ValueError(f'{self.records[failed.value].name}: {msg}')
        self.chains: List[np.ndarray] = [chain[first[r]:first[r + 1]].copy() for r in range(k)]
        self.lengths: List[int] = [int(x) for x in lengths[:k]]
        self._bs = fr['blocksize'].astype(np.int64)

    def emit(self, out, starts: Dict[int, int], mono: bool = True):
        """Decodes recording r into out[starts[r] : + lengths[r]] (mono: np.mean's float32 order over the channels, i.e.
        to_mono(decode_flac(...).T)) or, with mono=False, out[starts[r] * channels : + lengths[r] * channels] interleaved
        [n, channels]; one some_flac_decode call for all of ``starts`` on the current stream.  Returns the device status
        word (0 unless a chained frame failed to decode)."""
        import torch
        from . import _lib
        assert out.dtype == torch.float32 and out.device == self.device
        idx, off = [], []
        for r, start in starts.items():
            ch = 1 if mono else self.records[r].channels
            assert 0 <= start and (start + self.lengths[r]) * ch <= out.numel(), 'recording outside its buffer'
            c = self.chains[r]
            idx.append(c)
            off.append(start + np.concatenate([[0], np.cumsum(self._bs[c])[:-1]]).astype(np.int64) if len(c) else
                       np.zeros(0, np.int64))
        status = torch.zeros(1, dtype=torch.int32, device=self.device)
        chain = np.concatenate(idx) if idx else np.zeros(0, np.int32)
        if not len(chain):
            return status
        ch_of = np.array([r.channels for r in self.records], np.int64)
        fr_stream = np.concatenate([np.full(len(c), r, np.int64) for r, c in zip(starts, idx)])
        slot = self._bs[chain] * ch_of[fr_stream]
        scratch_off = np.concatenate([[0], np.cumsum(slot)[:-1]]).astype(np.int64)
        meta = torch.from_numpy(np.stack([scratch_off, np.concatenate(off)])).to(self.device)
        chain_d = torch.from_numpy(chain).to(self.device)
        scratch = torch.empty(max(int(slot.sum()), 1), dtype=torch.int32, device=self.device)
        lib = _lib.load()
        _lib.check(lib.some_flac_decode(self.data.data_ptr(), self.streams.data_ptr(), self.frames.data_ptr(),
                                        chain_d.data_ptr(), meta[0].data_ptr(), meta[1].data_ptr(), len(chain),
                                        scratch.data_ptr(), out.data_ptr(), int(mono), status.data_ptr(),
                                        C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)), 'some_flac_decode')
        return status


def _check_status(status) -> None:
    if int(status.item()):
        raise RuntimeError(f'some_flac_decode: a chained frame failed to decode (status {int(status.item())})')


def _flac_device(rec: EncodedAudio, mono: bool):
    """(CUDA float32 tensor: [n] mono / single channel or [channels, n], FlacBatch) for one record."""
    import torch
    dev = torch.device('cuda', torch.cuda.current_device())
    fb = FlacBatch([rec], dev)
    n, ch = fb.lengths[0], (1 if mono else rec.channels)
    y = torch.empty(max(n * ch, 1), dtype=torch.float32, device=dev)
    status = fb.emit(y, {0: 0}, mono=mono)
    y = y[:n * ch]
    _check_status(status)
    return (y if ch == 1 else y.view(n, ch).t().contiguous()), fb


def decode_flac(path) -> Tuple[np.ndarray, int]:
    """(samples, native rate) of a FLAC file as libsndfile hands them to librosa.load, decoded on the GPU: float32 [n]
    (one channel) or [n, channels], x * 2^-(bps - 1)."""
    rec = read_encoded(path)
    y, _ = _flac_device(rec, mono=False)
    return (y.cpu().numpy() if y.ndim == 1 else y.t().contiguous().cpu().numpy()), rec.rate


# ---------------------------------------------------------------------------------------------- AIFF (device)
def _pcm_device(data: bytes, m, mono: bool):
    """The samples some_audio_info found in ``data`` (a WAV data or AIFF SSND chunk), decoded by one some_pcm_decode on the
    current stream: a CUDA float32 tensor, [n] (mono or one channel) or [channels, n]."""
    import torch
    from . import _lib
    lib = _lib.load()
    dev = torch.device('cuda', torch.cuda.current_device())
    n, ch = int(m.frames), (1 if mono else int(m.channels))
    raw = np.frombuffer(data, np.uint8, count=int(m.data_bytes), offset=int(m.data_offset))
    src = torch.from_numpy(raw.copy()).to(dev)
    y = torch.empty(max(n * ch, 1), dtype=torch.float32, device=dev)
    item = _lib.PcmItem(src.data_ptr(), n, int(m.channels), int(m.kind), int(mono), 0, y.data_ptr())
    desc = np.zeros(int(lib.some_pcm_decode_bytes(1)), np.uint8)
    _lib.check(lib.some_pcm_decode_pack(C.byref(item), 1, desc.ctypes.data), 'some_pcm_decode_pack')
    desc_d = torch.from_numpy(desc).to(dev)
    _lib.check(lib.some_pcm_decode(desc.ctypes.data, desc_d.data_ptr(),
                                   C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), 'some_pcm_decode')
    y = y[:n * ch]
    return y if ch == 1 else y.view(n, ch).t().contiguous()


def decode_aiff(path) -> Tuple[np.ndarray, int]:
    """(samples, native rate) of an AIFF / AIFF-C file as libsndfile hands them to librosa.load, decoded on the GPU: float32
    [n] (one channel) or [n, channels]."""
    from . import _lib
    with open(path, 'rb') as f:
        data = f.read()
    m = audio_info(data, str(path))
    if m.container != _lib.AUDIO_AIFF:
        raise ValueError(f'{path}: not an AIFF or AIFF-C file')
    y = _pcm_device(data, m, mono=False)
    return (y.cpu().numpy() if y.ndim == 1 else y.t().contiguous().cpu().numpy()), int(m.rate)


# ---------------------------------------------------------------------------------------------- librosa.load
def load(path, sr=22050, mono: bool = True):
    """librosa.load(path, sr=sr, mono=mono) (librosa 0.9, res_type='kaiser_best') for RIFF/WAVE, FLAC and AIFF files:
    (y, rate).  ``sr=None`` keeps the native rate; otherwise the decoded (and down-mixed) samples are resampled on the GPU.
    FLAC and AIFF files are decoded and down-mixed on the GPU too."""
    from . import _lib
    with open(path, 'rb') as f:
        data = f.read(4)
        if data != b'RIFF':                                  # scipy reads RIFF files itself
            data += f.read()
    if data == b'RIFF':
        x, native = decode_wav(path)
        y = x.T                                              # librosa's (channels, n)
        if mono:
            y = to_mono(y)
        if sr is not None and as_rate(sr) != native:
            return resample(np.ascontiguousarray(y), native, as_rate(sr)), as_rate(sr)
        return y, native
    m = audio_info(data, str(path))                          # FLAC or AIFF / AIFF-C; ValueError for anything else
    if m.container == _lib.AUDIO_FLAC:
        y, _ = _flac_device(_flac_record(data, str(path), m), mono)
    else:
        y = _pcm_device(data, m, mono)
    if sr is not None and as_rate(sr) != m.rate:
        return resample(y, m.rate, as_rate(sr)).cpu().numpy(), as_rate(sr)
    return y.cpu().numpy(), m.rate


def load_native(path, sr=None):
    """``load(path, sr=None)``: the mono recording at its own rate, as (waveform, rate).  The second argument is the rate
    the caller wants (batch.batch_infer_dataset passes it) and is ignored: a loader that returns (waveform, rate) has the
    dataset driver resample on the device, straight into the batch's wave buffer."""
    return load(path, sr=None)


# ---------------------------------------------------------------------------------------------- float32 audio on the device
def is_cuda_tensor(x) -> bool:
    """Whether ``x`` is a CUDA torch tensor (without importing torch when the caller has not)."""
    import sys
    torch = sys.modules.get('torch')
    return torch is not None and isinstance(x, torch.Tensor) and x.is_cuda


def device_layout(t, index: int, who: str) -> Tuple[int, int, int, int, int]:
    """(channels, frames, channel stride, frame stride, layout) of a float32 recording tensor, ``[n]`` or librosa's
    ``[channels, n]``, read from its shape and ``stride()`` (some_downmix_layout: mono, planar or interleaved).  Raises
    ValueError naming item ``index`` for another dtype, rank or stride pattern.  Host only: CPU tensors are mapped too."""
    import torch
    from . import _lib
    where = f'{who}: item {index}'
    if not isinstance(t, torch.Tensor):
        raise ValueError(f'{where}: a torch tensor expected, got {type(t).__name__}')
    if t.dtype != torch.float32:
        raise ValueError(f'{where}: float32 audio expected, got {t.dtype}')
    if t.dim() == 1:
        ch, n, cs, fs = 1, int(t.shape[0]), 0, int(t.stride(0))
    elif t.dim() == 2:
        (ch, n), (cs, fs) = (int(v) for v in t.shape), (int(v) for v in t.stride())
    else:
        raise ValueError(f'{where}: [n] or [channels, n] expected, got shape {tuple(t.shape)}')
    lib = _lib.load()
    layout = C.c_int()
    if lib.some_downmix_layout(ch, n, cs, fs, C.byref(layout)) != 0:
        raise ValueError(f'{where}: {lib.some_last_error().decode("utf8", "replace")}')
    return ch, n, cs, fs, layout.value


def device_audio(t, index: int, who: str, sample_rate: int):
    """The some_device_audio descriptor of CUDA float32 recording ``t`` (see device_layout) at ``sample_rate``, produced on
    the current stream of its device; ValueError naming item ``index`` for a CPU tensor or what device_layout refuses."""
    import torch
    from . import _lib
    ch, n, cs, fs, _ = device_layout(t, index, who)
    if not t.is_cuda:
        raise ValueError(f'{who}: item {index}: a CUDA tensor expected, got one on {t.device}')
    stream = torch.cuda.current_stream(t.device).cuda_stream
    return _lib.DeviceAudio(t.data_ptr() if n else None, t.device.index, n, ch, cs, fs, int(sample_rate), stream or None)


def downmix_into(items: Sequence[Tuple[object, object, int]], who: str = 'downmix_into') -> None:
    """One some_downmix launch on the current stream of the destinations' device: item (t, dst, at) writes np.mean(y,
    axis=0) in float32 of the CUDA float32 recording t ([n] or librosa's [channels, n], on dst's device) to dst[at : at +
    frames], bit for bit."""
    import torch
    from . import _lib
    if not items:
        return
    lib = _lib.load()
    dev = items[0][1].device
    arr = (_lib.DownmixItem * len(items))()
    for k, (t, dst, at) in enumerate(items):
        ch, n, cs, _, layout = device_layout(t, k, who)
        if t.device != dev or dst.device != dev or dst.dtype != torch.float32 or at < 0 or at + n > dst.numel():
            raise ValueError(f'{who}: item {k}: a recording on {t.device} into {dst.numel()} floats of {dst.device} at {at}')
        arr[k] = _lib.DownmixItem(t.data_ptr() if n else None, n, ch, layout, cs, dst.data_ptr() + 4 * at if n else None)
    desc = np.zeros(int(lib.some_downmix_bytes(len(items))), np.uint8)
    _lib.check(lib.some_downmix_pack(arr, len(items), desc.ctypes.data), 'some_downmix_pack')
    desc_d = torch.from_numpy(desc).to(dev)
    _lib.check(lib.some_downmix(desc.ctypes.data, desc_d.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
               'some_downmix')
