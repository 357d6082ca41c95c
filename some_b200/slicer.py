"""Silence slicer in front of the path (SURVEY.md §8f-1): the GPU counterpart of utils/slicer2.py.

The reference computes the short-time RMS with numpy (slicer2.py:5-38: ~53 M multiply-adds and a 200 MB temporary for a
5-minute recording) and then walks the RMS list frame by frame in Python (:84-127).  Here

* the RMS frames come from ``some_slicer_rms`` (csrc/slicer.cu), launched by ``rms_lists`` on recordings that are already
  on the device — they have to go to the GPU for the mel front end anyway — and the kernel reproduces numpy's float32
  pairwise summation bit for bit, so every threshold comparison and argmin sees the reference's numbers;
* the cuts are decided by the native slicer next to that kernel (``some_slicer_ranges``, csrc/slicer.cu), on the host with no
  CUDA call: per SILENT RUN instead of per frame, since the reference's loop only acts on the first voiced frame after a run
  of frames with ``rms < threshold``.  The native session, streaming and the C ABI use the same code, so the cut rules exist
  once;
* ``Engine.transcribe_resident`` cuts recordings with ``cut_ranges`` over ``rms_lists`` and runs the chunks where they lie in
  device memory (no second upload); ``Engine.infer_sliced`` and ``batch.transcribe_recordings`` upload into it.

``Slicer`` keeps the reference's constructor, derived attributes and ``slice()`` return value (list of
``{'offset': seconds, 'waveform': view}``), so ``infer.py``-style callers can use it unchanged.  There is no CPU path:
the RMS needs the CUDA library.  ``cut_ranges`` applies the cuts of any object with those attributes; ``slicer_params``,
``slicer_frames``, ``slicer_ranges`` and ``SlicerStream`` wrap the native slicer's C functions (ctypes).
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib


def slicer_params(threshold: float = -40., min_length: float = 5000, min_interval: float = 300, hop_size: float = 20,
                  max_sil_kept: float = 1000) -> _lib.SlicerParams:
    """Slicer constructor arguments (ms / dB) for the session; the defaults are infer.py's Slicer(sr, max_sil_kept=1000)."""
    return _lib.SlicerParams(threshold, min_length, min_interval, hop_size, max_sil_kept)


def slicer_frames(sample_rate: int, params: Optional[_lib.SlicerParams] = None) -> _lib.SlicerFrames:
    """some_slicer_derive: the frame counts the native slicer uses (host only)."""
    lib = _lib.load()
    out = _lib.SlicerFrames()
    _lib.check(lib.some_slicer_derive(int(sample_rate), C.byref(params) if params is not None else None, C.byref(out)),
               'some_slicer_derive')
    return out


def slicer_ranges(rms: np.ndarray, num_samples: int, frames: _lib.SlicerFrames) -> List[Tuple[int, int]]:
    """some_slicer_ranges: the native slicer's chunk ranges for an RMS list (host only, no CUDA call)."""
    lib = _lib.load()
    rms = np.ascontiguousarray(rms, dtype=np.float32)
    cap = rms.shape[0] // 2 + 2
    out = np.zeros(2 * cap, dtype=np.int64)
    count = C.c_int()
    _lib.check(lib.some_slicer_ranges(rms.ctypes.data, int(rms.shape[0]), int(num_samples), C.byref(frames), out.ctypes.data,
                                      cap, C.byref(count)), 'some_slicer_ranges')
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(count.value)]


def rms_lists(waves_d: Sequence, frame_length: int, hop: int) -> List[np.ndarray]:
    """Short-time RMS lists of device-resident float32 recordings, bit-identical to the reference's get_rms
    (slicer2.py:5-38): one ``some_slicer_rms`` launch each into one buffer on the current stream, then one device-to-host
    copy and sync for all of them."""
    import torch
    counts = [1 + (int(w.numel()) + 2 * (frame_length // 2) - frame_length) // hop for w in waves_d]
    if not counts:
        return []
    lib = _lib.load()
    dev = waves_d[0].device
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    cuts = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(counts, out=cuts[1:])
    rms_d = torch.empty(int(cuts[-1]), dtype=torch.float32, device=dev)
    for w, a, n in zip(waves_d, cuts, counts):
        _lib.check(lib.some_slicer_rms(w.data_ptr(), int(w.numel()), frame_length, hop, rms_d[a:].data_ptr(), n, stream),
                   'some_slicer_rms')
    host = rms_d.cpu().numpy()
    return [host[a:b] for a, b in zip(cuts[:-1], cuts[1:])]


def one_chunk(slicer, num_samples: int) -> bool:
    """Whether ``slicer`` leaves a recording of ``num_samples`` samples whole without looking at its RMS: no more than
    min_length hops (slicer2.py:79-80)."""
    return (num_samples + slicer.hop_size - 1) // slicer.hop_size <= slicer.min_length


def cut_ranges(slicer, lengths: Sequence[int],
               rms_of: Callable[[List[int]], Sequence[np.ndarray]]) -> List[List[Tuple[int, int]]]:
    """[begin, end) sample ranges of the chunks of recordings of the given lengths, cut by ``slicer``: any object with the
    reference Slicer's attributes (threshold, hop_size, win_size, min_length, min_interval, max_sil_kept).  A recording
    that is ``one_chunk`` stays whole; ``rms_of(indices)`` returns the RMS lists of the others, in that order, and is called
    once, only if there is one, so that short recordings make no device call."""
    out = [[(0, int(n))] for n in lengths]
    need = [i for i, n in enumerate(lengths) if not one_chunk(slicer, n)]
    if need:
        frames = _lib.SlicerFrames(np.float32(slicer.threshold), slicer.hop_size, slicer.win_size, slicer.min_length,
                                   slicer.min_interval, slicer.max_sil_kept)
        for i, rms in zip(need, rms_of(need)):
            out[i] = slicer_ranges(rms, lengths[i], frames)
    return out


class SlicerStream:
    """some_slicer_stream_*: the slicer's decisions on an RMS list that arrives in pieces (host only, no CUDA call)."""

    handle = None

    def __init__(self, frames: _lib.SlicerFrames):
        self.lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self.lib.some_slicer_stream_create(C.byref(frames), C.byref(h)), 'some_slicer_stream_create')
        self.handle = h

    @staticmethod
    def _ranges(ptr, count) -> List[Tuple[int, int]]:
        if count.value == 0:
            return []
        a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int64)), (2 * count.value,))
        return [(int(a[2 * k]), int(a[2 * k + 1])) for k in range(count.value)]

    def feed(self, rms: np.ndarray, fixed: int) -> List[Tuple[int, int]]:
        """The next RMS frames and the samples fixed so far -> the [begin, end) sample ranges that became final."""
        rms = np.ascontiguousarray(rms, dtype=np.float32)
        ptr, count = C.c_void_p(), C.c_int()
        _lib.check(self.lib.some_slicer_stream_feed(self.handle, rms.ctypes.data, int(rms.shape[0]), int(fixed), C.byref(ptr),
                                                    C.byref(count)), 'some_slicer_stream_feed')
        return self._ranges(ptr, count)

    def finish(self, rms: np.ndarray, num_samples: int) -> List[Tuple[int, int]]:
        """The frames not fed yet and the final length -> the remaining ranges."""
        rms = np.ascontiguousarray(rms, dtype=np.float32)
        ptr, count = C.c_void_p(), C.c_int()
        _lib.check(self.lib.some_slicer_stream_finish(self.handle, rms.ctypes.data, int(rms.shape[0]), int(num_samples),
                                                      C.byref(ptr), C.byref(count)), 'some_slicer_stream_finish')
        return self._ranges(ptr, count)

    def keep_from(self) -> Tuple[int, int, int]:
        """(sample a range not returned yet begins at or after, unless it lies within [0, head); head; RMS values held)."""
        a, h, b = C.c_longlong(), C.c_longlong(), C.c_longlong()
        _lib.check(self.lib.some_slicer_stream_keep_from(self.handle, C.byref(a), C.byref(h), C.byref(b)),
                   'some_slicer_stream_keep_from')
        return a.value, h.value, b.value

    def close(self):
        if self.handle is not None:
            self.lib.some_slicer_stream_destroy(self.handle)
            self.handle = None

    def __del__(self):
        self.close()


class Slicer:
    """Drop-in for utils.slicer2.Slicer (same arguments, same derived attributes, same ``slice`` result)."""

    def __init__(self, sr: int, threshold: float = -40., min_length: int = 5000, min_interval: int = 300,
                 hop_size: int = 20, max_sil_kept: int = 5000, device=None):
        if not min_length >= min_interval >= hop_size:
            raise ValueError('The following condition must be satisfied: min_length >= min_interval >= hop_size')
        if not max_sil_kept >= hop_size:
            raise ValueError('The following condition must be satisfied: max_sil_kept >= hop_size')
        interval = sr * min_interval / 1000
        self.sr = sr
        self.threshold = 10 ** (threshold / 20.)
        self.hop_size = round(sr * hop_size / 1000)
        self.win_size = min(round(interval), 4 * self.hop_size)
        self.min_length = round(sr * min_length / 1000 / self.hop_size)
        self.min_interval = round(interval / self.hop_size)
        self.max_sil_kept = round(sr * max_sil_kept / 1000 / self.hop_size)
        self.device = device

    # ------------------------------------------------------------------ device part
    def rms(self, samples: np.ndarray) -> np.ndarray:
        """RMS list of a mono float32 waveform, computed on the GPU (bit-identical to get_rms, slicer2.py:5-38)."""
        import torch
        if not torch.cuda.is_available():
            raise _lib.SomeB200Error('some_b200.slicer needs a CUDA device (no CPU path)')
        dev = torch.device(self.device if self.device is not None else 'cuda')
        with torch.cuda.device(dev):
            x = torch.from_numpy(np.ascontiguousarray(samples, dtype=np.float32)).to(dev)
            return rms_lists([x], self.win_size, self.hop_size)[0]

    # ------------------------------------------------------------------ reference API
    def ranges(self, waveform: np.ndarray) -> List[Tuple[int, int]]:
        samples = waveform.mean(axis=0) if waveform.ndim > 1 else waveform          # slicer2.py:75-78
        return cut_ranges(self, [int(samples.shape[0])], lambda _: [self.rms(samples)])[0]

    def slice(self, waveform: np.ndarray):
        ranges = self.ranges(waveform)
        if ranges == [(0, waveform.shape[-1])]:                     # one chunk: the input itself (slicer2.py:80, :135-136)
            return [{'offset': 0, 'waveform': waveform}]
        return [{'offset': begin / self.sr,                         # == begin_frame * hop_size / sr
                 'waveform': waveform[..., begin:end]} for begin, end in ranges]
