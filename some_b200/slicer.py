"""Silence slicer in front of the path (SURVEY.md §8f-1): the GPU counterpart of utils/slicer2.py.

The reference computes the short-time RMS with numpy (slicer2.py:5-38: ~53 M multiply-adds and a 200 MB temporary for a
5-minute recording) and then walks the RMS list frame by frame in Python (:84-127).  Here

* the RMS frames come from ``some_slicer_rms`` (csrc/slicer.cu): the recording is uploaded once — it has to go to the GPU
  for the mel front end anyway — and the kernel reproduces numpy's float32 pairwise summation bit for bit, so every
  threshold comparison and argmin below sees the reference's numbers;
* the decisions are taken per SILENT RUN instead of per frame: the reference's loop only acts on the first voiced frame
  after a run of frames with ``rms < threshold``, so the runs are extracted with vectorised numpy and the (sequential, because
  of ``clip_start``) rules are applied to a few dozen runs;
* ``Engine.infer_sliced`` then processes the chunks where they lie in device memory (no second upload).

``Slicer`` keeps the reference's constructor, derived attributes and ``slice()`` return value (list of
``{'offset': seconds, 'waveform': view}``), so ``infer.py``-style callers can use it unchanged.  There is no CPU path:
the RMS needs the CUDA library.
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np


def silence_tags(rms: np.ndarray, p) -> List[Tuple[int, int]]:
    """Frame ranges to remove (slicer2.py:82-133).  ``p`` carries threshold, min_length, min_interval, max_sil_kept (frames)."""
    total = int(rms.shape[0])
    silent = rms < p.threshold                       # float32 comparison, as the reference's scalar `rms < self.threshold`
    edges = np.diff(silent.astype(np.int8), prepend=np.int8(0), append=np.int8(0))
    run_from = np.flatnonzero(edges == 1)
    run_to = np.flatnonzero(edges == -1)             # first voiced frame after the run (== total for a trailing run)
    keep = p.max_sil_kept
    tags: List[Tuple[int, int]] = []
    clip_from = 0

    def first_min(a: int, b: int) -> int:            # first-index argmin over frames [a, b)
        return int(rms[a:b].argmin()) + a

    for s, i in zip(run_from.tolist(), run_to.tolist()):
        if i == total:                               # trailing silence (slicer2.py:129-133)
            if total - s >= p.min_interval:
                tags.append((first_min(s, min(total, s + keep) + 1), total + 1))
            break
        leading = s == 0 and i > keep
        middle = i - s >= p.min_interval and i - clip_from >= p.min_length
        if not (leading or middle):
            continue
        span = i - s
        if span <= keep:
            cut = first_min(s, i + 1)
            tags.append((0, cut) if s == 0 else (cut, cut))
            clip_from = cut
        elif span <= 2 * keep:
            mid = first_min(i - keep, s + keep + 1)
            left = first_min(s, s + keep + 1)
            right = first_min(i - keep, i + 1)
            if s == 0:
                tags.append((0, right))
                clip_from = right
            else:
                tags.append((min(left, mid), max(right, mid)))
                clip_from = max(right, mid)
        else:
            left = first_min(s, s + keep + 1)
            right = first_min(i - keep, i + 1)
            tags.append((0, right) if s == 0 else (left, right))
            clip_from = right
    return tags


def chunk_ranges(tags: List[Tuple[int, int]], total_frames: int, hop_size: int, num_samples: int) -> List[Tuple[int, int]]:
    """[begin, end) SAMPLE ranges that remain after removing the tagged frames (slicer2.py:62-71,135-145)."""
    if not tags:
        return [(0, num_samples)]
    kept = []
    if tags[0][0] > 0:
        kept.append((0, tags[0][0]))
    kept.extend((a[1], b[0]) for a, b in zip(tags[:-1], tags[1:]))
    if tags[-1][1] < total_frames:
        kept.append((tags[-1][1], total_frames))
    return [(f0 * hop_size, min(num_samples, f1 * hop_size)) for f0, f1 in kept]


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
        from . import _lib
        lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.SomeB200Error('some_b200.slicer needs a CUDA device (no CPU path)')
        dev = torch.device(self.device if self.device is not None else 'cuda')
        with torch.cuda.device(dev):
            x = torch.from_numpy(np.ascontiguousarray(samples, dtype=np.float32)).to(dev)
            n = int(x.numel())
            n_frames = 1 + (n + 2 * (self.win_size // 2) - self.win_size) // self.hop_size
            out = torch.empty(n_frames, dtype=torch.float32, device=dev)
            import ctypes as C
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(lib.some_slicer_rms(x.data_ptr(), n, self.win_size, self.hop_size, out.data_ptr(), n_frames, stream),
                       'some_slicer_rms')
            return out.cpu().numpy()

    # ------------------------------------------------------------------ reference API
    def ranges(self, waveform: np.ndarray) -> List[Tuple[int, int]]:
        samples = waveform.mean(axis=0) if waveform.ndim > 1 else waveform          # slicer2.py:75-78
        n = int(samples.shape[0])
        if (n + self.hop_size - 1) // self.hop_size <= self.min_length:            # slicer2.py:79-80
            return [(0, n)]
        rms = self.rms(samples)
        return chunk_ranges(silence_tags(rms, self), rms.shape[0], self.hop_size, n)

    def slice(self, waveform: np.ndarray):
        n = waveform.shape[-1]
        if (n + self.hop_size - 1) // self.hop_size <= self.min_length:
            return [{'offset': 0, 'waveform': waveform}]
        chunks = []
        for begin, end in self.ranges(waveform):
            chunks.append({'offset': begin / self.sr,                               # == begin_frame * hop_size / sr
                           'waveform': waveform[..., begin:end]})
        return chunks
