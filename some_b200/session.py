"""ctypes wrapper of the native session (csrc/session.cu, include/some_b200.h): opens a model file written by
``python -m some_b200.export`` and transcribes with no torch on the path.  C / C++ hosts call the same functions directly
(examples/some_transcribe.c); this wrapper serves Python callers that want the same results, the tests and bench_session.py.
The slicer parameters of transcribe_sliced and stream are ``slicer_params(...)`` (defined in some_b200.slicer).

Results have the plugin's shape: one dict per clip / chunk with ``note_midi`` f32, ``note_dur`` in seconds
(``dur * timestep``, float64 as me_infer.py:95) and ``note_rest`` bool, plus ``note_frames`` (the durations in frames).

Every call takes ``frames=False``.  With ``frames=True`` it also returns the frame curves of every clip / chunk
(some_notes_get_frames), one ``Curves`` tuple ``(midi f32, rest bool, bound f32, note_index i32)`` per clip, as one more
element beside what it returns with frames off: ``transcribe`` returns ``(notes, curves)``, the calls that return
``(offsets, ranges, notes)`` return ``(offsets, ranges, notes, curves)``.  Frame t of a clip is centred at sample
``begin + t * hop``."""
from __future__ import annotations

import ctypes as C
import os
import weakref
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib, audio
# The slicer's parameters and host decisions are defined in some_b200.slicer; they stay importable from here because
# transcribe_sliced and stream take slicer_params(...), and existing callers import them with the session.
from .slicer import SlicerStream, slicer_frames, slicer_params, slicer_ranges  # noqa: F401


class Curves(NamedTuple):
    """The frame curves of one clip (some_notes_get_frames), T = 1 + samples // hop entries each."""
    midi: np.ndarray          # f32: the pitch value of each frame
    rest: np.ndarray          # bool: the frame is a rest
    bound: np.ndarray         # f32: the boundary probability
    note_index: np.ndarray    # i32: the 1-based note of the frame


def _label_call(fn, *args) -> Tuple[str, str]:
    """Runs some_label_write / some_notes_label (their leading arguments in ``args``): asks for the sizes, then fills."""
    lib = _lib.load()
    n_seq, n_dur = C.c_size_t(), C.c_size_t()
    _lib.check(getattr(lib, fn)(*args, None, 0, C.byref(n_seq), None, 0, C.byref(n_dur)), fn)
    seq, dur = C.create_string_buffer(n_seq.value), C.create_string_buffer(n_dur.value)
    _lib.check(getattr(lib, fn)(*args, seq, n_seq.value, C.byref(n_seq), dur, n_dur.value, C.byref(n_dur)), fn)
    return seq.value.decode('utf8'), dur.value.decode('utf8')


def label_write(offsets: Sequence[float], segments: Sequence[Dict[str, np.ndarray]], timestep: float, ph_dur: str, ph_num: str,
                round_midi: bool = False) -> Tuple[str, str]:
    """some_label_write: the ``note_seq`` / ``note_dur`` fields of transcriptions.csv for one item, what
    ``batch.row_notes(ph_dur, ph_num, batch.note_timeline(offsets, segments), round_midi)`` returns for segments whose
    ``note_dur`` is ``note_frames * timestep`` (each segment's ``note_frames``, int32, are the durations passed)."""
    counts = np.array([len(sg['note_frames']) for sg in segments] or [0], dtype=np.int32)
    midi = np.ascontiguousarray(np.concatenate([sg['note_midi'] for sg in segments] or [[]]), dtype=np.float32)
    frames = np.ascontiguousarray(np.concatenate([sg['note_frames'] for sg in segments] or [[]]), dtype=np.int32)
    rest = np.ascontiguousarray(np.concatenate([sg['note_rest'] for sg in segments] or [[]]), dtype=np.uint8)
    offs = np.ascontiguousarray(np.asarray(offsets, dtype=np.float64).reshape(-1))
    if offs.shape[0] != len(segments):
        raise ValueError(f'label_write: {offs.shape[0]} offsets for {len(segments)} segments')
    return _label_call('some_label_write', len(segments), offs.ctypes.data, counts.ctypes.data, midi.ctypes.data,
                       frames.ctypes.data, rest.ctypes.data, float(timestep), ph_dur.encode('utf8'), ph_num.encode('utf8'),
                       int(bool(round_midi)))


class Notes:
    """A caller-owned result object (some_notes_create / some_notes_destroy).  A session call that fills it records the
    session's sample rate and timestep on it, for label()."""

    handle = None
    _frames = False
    sample_rate = None
    timestep = None

    def __init__(self):
        self.lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self.lib.some_notes_create(C.byref(h)), 'some_notes_create')
        self.handle = h

    def set_frames(self, on: bool):
        """some_notes_set_frames: whether the calls that fill this object also fill frame curves.  The native object starts
        with frames off, and only a change is passed on, so a call with frames=False makes no extra native call."""
        if bool(on) != self._frames:
            _lib.check(self.lib.some_notes_set_frames(self.handle, int(bool(on))), 'some_notes_set_frames')
            self._frames = bool(on)

    def curves(self) -> List[Curves]:
        """The frame curves of every clip, copied out of the native object (it must have been filled with frames on)."""
        n = self.lib.some_notes_clips(self.handle)
        if n < 0:
            _lib.check(n, 'some_notes_clips')
        out = []
        t, pm, pr, pb, pn = C.c_int(), C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        def copy(p, dtype):              # a buffer copy: np.ctypeslib.as_array costs several times more per array
            size = t.value * np.dtype(dtype).itemsize
            return np.frombuffer((C.c_char * size).from_address(p.value), dtype).copy() if size else np.zeros(0, dtype)

        for i in range(n):
            _lib.check(self.lib.some_notes_get_frames(self.handle, i, C.byref(t), C.byref(pm), C.byref(pr), C.byref(pb),
                                                      C.byref(pn)), 'some_notes_get_frames')
            out.append(Curves(copy(pm, np.float32), copy(pr, np.uint8).view(bool), copy(pb, np.float32), copy(pn, np.int32)))
        return out

    def close(self):
        if self.handle is not None:
            self.lib.some_notes_destroy(self.handle)
            self.handle = None

    def __del__(self):
        self.close()

    def label(self, ph_dur: str, ph_num: str, round_midi: bool = False) -> Tuple[str, str]:
        """some_notes_label: the ``note_seq`` / ``note_dur`` fields of transcriptions.csv for the recording whose chunks this
        object holds, with its row's ``ph_dur`` / ``ph_num`` fields: ``batch.row_notes(ph_dur, ph_num,
        batch.note_timeline(offsets, segments), round_midi)`` of the same notes."""
        if self.sample_rate is None:
            raise ValueError('Notes.label: not filled by a session call')
        return _label_call('some_notes_label', self.handle, int(self.sample_rate), float(self.timestep), ph_dur.encode('utf8'),
                           ph_num.encode('utf8'), int(bool(round_midi)))

    def results(self, timestep: float) -> Tuple[List[Tuple[int, int]], List[Dict[str, np.ndarray]]]:
        """(sample range of every clip, notes of every clip) copied out of the native object."""
        n = self.lib.some_notes_clips(self.handle)
        if n < 0:
            _lib.check(n, 'some_notes_clips')
        ranges, out = [], []
        cnt, nm, nd, nr = C.c_int(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        a, b = C.c_int64(), C.c_int64()
        for i in range(n):
            _lib.check(self.lib.some_notes_get(self.handle, i, C.byref(cnt), C.byref(nm), C.byref(nd), C.byref(nr), C.byref(a),
                                               C.byref(b)), 'some_notes_get')
            k = cnt.value
            midi = np.ctypeslib.as_array(C.cast(nm, C.POINTER(C.c_float)), (k,)).copy() if k else np.zeros(0, np.float32)
            dur = np.ctypeslib.as_array(C.cast(nd, C.POINTER(C.c_int32)), (k,)).copy() if k else np.zeros(0, np.int32)
            rest = np.ctypeslib.as_array(C.cast(nr, C.POINTER(C.c_uint8)), (k,)).copy() if k else np.zeros(0, np.uint8)
            ranges.append((a.value, b.value))
            out.append({'note_midi': midi, 'note_dur': dur * timestep, 'note_rest': rest.astype(bool), 'note_frames': dur})
        return ranges, out


def shard_clips(lengths: Sequence[int], replicas: int) -> List[int]:
    """some_shard_clips: the replica (or rank) of every clip, by the longest-processing-time rule a multi-device session and
    some_b200.dist use."""
    lib = _lib.load()
    lens = np.ascontiguousarray(np.asarray(lengths, dtype=np.int64).reshape(-1))
    owner = np.zeros(max(lens.shape[0], 1), dtype=np.int32)
    _lib.check(lib.some_shard_clips(lens.ctypes.data, int(lens.shape[0]), int(replicas), owner.ctypes.data), 'some_shard_clips')
    return owner[:lens.shape[0]].tolist()


class Session:
    """some_session_open(path, device) ... some_session_close.  `device` is one device index, or a sequence of them
    (some_session_open_devices): a replica of the model on each, with the chunks of every call spread over them and the same
    results as a session on the first."""

    handle = None

    def __init__(self, path, device: Union[int, Sequence[int]] = 0):
        self.lib = _lib.load()
        h = C.c_void_p()
        if isinstance(device, (int, np.integer)):
            _lib.check(self.lib.some_session_open(os.fsencode(os.fspath(path)), int(device), C.byref(h)), 'some_session_open')
        else:
            devs = [int(d) for d in device]
            arr = (C.c_int * max(len(devs), 1))(*devs)
            _lib.check(self.lib.some_session_open_devices(os.fsencode(os.fspath(path)), arr, len(devs), C.byref(h)),
                       'some_session_open_devices')
        self.handle = h
        self._streams = weakref.WeakSet()      # closed before the session: a stream uses the session's device state
        info = _lib.SessionInfo()
        _lib.check(self.lib.some_session_get_info(h, C.byref(info)), 'some_session_get_info')
        self.sample_rate, self.hop, self.outdim = info.sample_rate, info.hop, info.outdim
        self.quantized, self.bias_corrected, self.timestep = bool(info.quantized), bool(info.bias_corrected), info.timestep
        prec = C.c_int()
        _lib.check(self.lib.some_session_get_precision(h, C.byref(prec)), 'some_session_get_precision')
        self.precision = {0: 'bf16', 1: 'fp32'}[prec.value]    # of the model file: every call runs at it

    def close(self):
        """Closes the session and, first, every stream still open on it."""
        if self.handle is not None:
            for st in list(self._streams):
                st.close()
            self.lib.some_session_close(self.handle)
            self.handle = None

    def __del__(self):
        self.close()

    @property
    def devices(self) -> List[int]:
        """some_session_get_devices: the device of every replica, in order."""
        n = C.c_int()
        _lib.check(self.lib.some_session_get_devices(self.handle, None, 0, C.byref(n)), 'some_session_get_devices')
        arr = (C.c_int * max(n.value, 1))()
        _lib.check(self.lib.some_session_get_devices(self.handle, arr, n.value, C.byref(n)), 'some_session_get_devices')
        return list(arr[:n.value])

    def load(self) -> List[Tuple[int, int]]:
        """some_session_get_load: (chunks, frames) each replica ran in the session's last completed step."""
        n = C.c_int()
        _lib.check(self.lib.some_session_get_load(self.handle, None, None, 0, C.byref(n)), 'some_session_get_load')
        chunks, frames = (C.c_int64 * max(n.value, 1))(), (C.c_int64 * max(n.value, 1))()
        _lib.check(self.lib.some_session_get_load(self.handle, chunks, frames, n.value, C.byref(n)), 'some_session_get_load')
        return list(zip(chunks[:n.value], frames[:n.value]))

    def stats(self) -> Dict[str, int]:
        """some_session_get_stats: totals since open (``calls``, ``steps``, ``max_calls``: the most calls one step held) and
        the calls ``queued`` at this moment.  The library is loaded with ctypes.CDLL, which releases the GIL around every
        call, so Python threads that share a session queue together and their calls can share a step."""
        st = _lib.SessionStats()
        _lib.check(self.lib.some_session_get_stats(self.handle, C.byref(st)), 'some_session_get_stats')
        return {name: getattr(st, name) for name, _ in _lib.SessionStats._fields_}

    def transcribe(self, waveforms: Sequence[np.ndarray], notes: Optional[Notes] = None, frames: bool = False):
        """some_session_transcribe: mono float32 clips at the model's rate -> one dict per clip, in input order (frames=True:
        and one Curves per clip)."""
        waves = [np.ascontiguousarray(w, dtype=np.float32) for w in waveforms]
        ptrs = (C.c_void_p * max(len(waves), 1))(*[w.ctypes.data for w in waves])
        lens = np.array([w.shape[0] for w in waves] or [0], dtype=np.int64)
        own = notes is None
        notes = notes or Notes()
        try:
            notes.set_frames(frames)
            _lib.check(self.lib.some_session_transcribe(self.handle, ptrs, lens.ctypes.data, len(waves), notes.handle),
                       'some_session_transcribe')
            res = notes.results(self.timestep)[1]
            return (res, notes.curves()) if frames else res
        finally:
            if own:
                notes.close()

    def transcribe_sliced(self, samples: np.ndarray, sample_rate: Optional[int] = None,
                          params: Optional[_lib.SlicerParams] = None, notes: Optional[Notes] = None, frames: bool = False):
        """some_session_transcribe_sliced: one mono recording (any integer rate) -> (chunk offsets in seconds, chunk sample
        ranges, per-chunk notes), as Engine.infer_sliced returns offsets and notes."""
        x = np.ascontiguousarray(samples, dtype=np.float32)
        own = notes is None
        notes = notes or Notes()
        try:
            notes.set_frames(frames)
            _lib.check(self.lib.some_session_transcribe_sliced(
                self.handle, x.ctypes.data, int(x.shape[0]), int(sample_rate or self.sample_rate),
                C.byref(params) if params is not None else None, notes.handle), 'some_session_transcribe_sliced')
            return self._results(notes, frames)
        finally:
            if own:
                notes.close()

    def _results(self, notes: Notes, frames: bool):
        """(offsets in seconds, ranges, notes), and the curves when `frames`."""
        notes.sample_rate, notes.timestep = self.sample_rate, self.timestep
        ranges, res = notes.results(self.timestep)
        offsets = [a / self.sample_rate for a, _ in ranges]
        return (offsets, ranges, res, notes.curves()) if frames else (offsets, ranges, res)

    def transcribe_encoded(self, items: Sequence, params: Optional[_lib.SlicerParams] = None, frames: bool = False,
                           notes: Optional[Sequence[Notes]] = None):
        """some_session_transcribe_encoded: WAV, FLAC or AIFF files (bytes, or paths to read) -> one (chunk offsets in seconds, chunk
        sample ranges, per-chunk notes) per item, what transcribe_sliced returns for audio.load(file, sr=None, mono=True).
        The files are decoded, resampled, sliced and transcribed in one GPU step.  ``notes``: one caller-owned Notes per item
        to fill (and keep, e.g. for Notes.label); by default the call uses its own."""
        datas = []
        for it in items:
            if isinstance(it, (bytes, bytearray, memoryview)):
                datas.append(bytes(it))
            else:
                with open(os.fspath(it), 'rb') as f:
                    datas.append(f.read())
        k = len(datas)
        bufs = [C.create_string_buffer(d, len(d)) if d else None for d in datas]
        enc = (_lib.Encoded * max(k, 1))(*[_lib.Encoded(C.cast(b, C.c_void_p) if b is not None else None, len(d))
                                           for b, d in zip(bufs, datas)])
        own = notes is None
        if not own and len(notes) != k:
            raise ValueError(f'transcribe_encoded: {k} items, {len(notes)} Notes')
        notes = [Notes() for _ in range(k)] if own else list(notes)
        try:
            for n in notes:
                n.set_frames(frames)
            outs = (C.c_void_p * max(k, 1))(*[n.handle for n in notes])
            _lib.check(self.lib.some_session_transcribe_encoded(self.handle, enc, k, C.byref(params) if params is not None else None,
                                                                outs), 'some_session_transcribe_encoded')
            return [self._results(n, frames) for n in notes]
        finally:
            if own:
                for n in notes:
                    n.close()

    def transcribe_device(self, tensors: Sequence, rates: Optional[Sequence[Optional[int]]] = None,
                          params: Optional[_lib.SlicerParams] = None, frames: bool = False,
                          notes: Optional[Sequence[Notes]] = None):
        """some_session_transcribe_device: CUDA float32 recordings, ``[n]`` or librosa's ``[channels, n]`` (the layout is read
        from ``stride()``: planar, or the ``[channels, n]`` view of an ``[n, channels]`` array) -> one (chunk offsets in
        seconds, chunk sample ranges, per-chunk notes) per recording, what transcribe_sliced returns for
        ``np.mean(y, axis=0)`` of its host copy, with no host copy.  ``rates``: each recording's rate (default: the model's).
        Each tensor is read after the work its device's current stream holds at the call; when the call returns the
        session no longer reads them.  Other dtypes, CPU tensors and other stride patterns raise ValueError naming the
        index."""
        k = len(tensors)
        if rates is None:
            rates = [None] * k
        if len(rates) != k:
            raise ValueError(f'transcribe_device: {k} recordings, {len(rates)} rates')
        descs = [audio.device_audio(t, i, 'transcribe_device', int(r or self.sample_rate))
                 for i, (t, r) in enumerate(zip(tensors, rates))]
        arr = (_lib.DeviceAudio * max(k, 1))(*descs)
        own = notes is None
        if not own and len(notes) != k:
            raise ValueError(f'transcribe_device: {k} recordings, {len(notes)} Notes')
        notes = [Notes() for _ in range(k)] if own else list(notes)
        try:
            for n in notes:
                n.set_frames(frames)
            outs = (C.c_void_p * max(k, 1))(*[n.handle for n in notes])
            _lib.check(self.lib.some_session_transcribe_device(self.handle, arr, k,
                                                               C.byref(params) if params is not None else None, outs),
                       'some_session_transcribe_device')
            return [self._results(n, frames) for n in notes]
        finally:
            if own:
                for n in notes:
                    n.close()

    def push_device_many(self, items: Sequence[Tuple['Stream', object]], finish: Optional[Sequence[bool]] = None,
                         frames: bool = False):
        """some_stream_push_device_many: push_many with CUDA float32 tensors (as Stream.push takes them) in place of host
        samples; each tensor is at its stream's rate."""
        k = len(items)
        descs = [audio.device_audio(t, i, 'push_device_many', st.rate) for i, (st, t) in enumerate(items)]
        arr = (_lib.DeviceAudio * max(k, 1))(*descs)
        streams = (C.c_void_p * max(k, 1))(*[st.handle for st, _ in items])
        outs = (C.c_void_p * max(k, 1))(*[st.notes.handle for st, _ in items])
        fin = None if finish is None else np.array([bool(f) for f in finish] or [0], dtype=np.int32)
        if fin is not None and len(finish) != k:
            raise ValueError(f'push_device_many: {k} items, {len(finish)} finish flags')
        for st, _ in items:
            st.notes.set_frames(frames)
        _lib.check(self.lib.some_stream_push_device_many(streams, arr, None if fin is None else fin.ctypes.data, k, outs),
                   'some_stream_push_device_many')
        return [st._results(frames=frames) for st, _ in items]

    def label_dataset(self, dataset, csv=None, round_midi: bool = False, overwrite: bool = False, budget: Optional[int] = None,
                      params: Optional[_lib.SlicerParams] = None, report: Optional[dict] = None):
        """some_session_label_dataset: batch_infer.py's command on a DiffSinger dataset (``transcriptions.csv`` and ``wavs/``),
        writing ``csv`` (default: the dataset's own transcriptions.csv) byte for byte as
        ``batch.batch_infer_dataset(..., load_audio=audio.load_native)`` does, and printing its warning for every missing
        audio file.  ``budget``: frames per GPU step (default SOME_SESSION_STEP_SAMPLES / hop); the output does not depend on
        it.  ``report``: a dict to receive the call's counts and times (some_label_report).  Returns the output path."""
        import pathlib

        def missing(path, _user):
            print(f"WARNING: audio file does not exist: '{os.fsdecode(path)}'")

        cb = _lib.LABEL_MISSING_FN(missing)
        lp = _lib.LabelParams(C.pointer(params) if params is not None else None, int(budget or 0))
        rep = _lib.LabelReport()
        _lib.check(self.lib.some_session_label_dataset(self.handle, os.fsencode(os.fspath(dataset)),
                                                       None if csv is None else os.fsencode(os.fspath(csv)), int(bool(round_midi)),
                                                       int(bool(overwrite)), C.byref(lp), cb, None, C.byref(rep)),
                   'some_session_label_dataset')
        if report is not None:
            report.update({name: getattr(rep, name) for name, _ in _lib.LabelReport._fields_})
        return pathlib.Path(csv) if csv is not None else pathlib.Path(dataset) / 'transcriptions.csv'

    def stream(self, sample_rate: Optional[int] = None, params: Optional[_lib.SlicerParams] = None) -> 'Stream':
        """some_stream_open: a recording pushed while it arrives (see Stream)."""
        return Stream(self, sample_rate, params)

    def stream_encoded(self, params: Optional[_lib.SlicerParams] = None) -> 'EncodedStream':
        """some_stream_open_encoded: a WAV, FLAC or AIFF file pushed as its bytes arrive (see EncodedStream)."""
        return EncodedStream(self, params)

    def push_bytes_many(self, items: Sequence[Tuple['EncodedStream', bytes]], finish: Optional[Sequence[bool]] = None,
                        frames: bool = False):
        """some_stream_push_bytes_many: push_many for encoded streams, with bytes in place of samples.  When a stream is refused
        on its content, the others still complete their step: the StreamRefused raised carries every item's results."""
        k = len(items)
        datas = [bytes(b) for _, b in items]
        bufs = [C.create_string_buffer(d, len(d)) if d else None for d in datas]
        streams = (C.c_void_p * max(k, 1))(*[st.handle for st, _ in items])
        ptrs = (C.c_void_p * max(k, 1))(*[C.cast(b, C.c_void_p) if b is not None else None for b in bufs])
        lens = np.array([len(d) for d in datas] or [0], dtype=np.int64)
        outs = (C.c_void_p * max(k, 1))(*[st.notes.handle for st, _ in items])
        fin = None if finish is None else np.array([bool(f) for f in finish] or [0], dtype=np.int32)
        if fin is not None and len(finish) != k:
            raise ValueError(f'push_bytes_many: {k} items, {len(finish)} finish flags')
        for st, _ in items:
            st.notes.set_frames(frames)
        rc = self.lib.some_stream_push_bytes_many(streams, ptrs, lens.ctypes.data, None if fin is None else fin.ctypes.data, k,
                                                  outs)
        if rc == _lib.STREAM_REFUSED:          # the other streams' chunks are in their Notes: hand them over with the refusal
            msg = self.lib.some_last_error().decode('utf8', 'replace')
            raise _lib.StreamRefused(f'some_stream_push_bytes_many failed ({rc}): {msg}',
                                     [st._results(frames=frames) for st, _ in items])
        _lib.check(rc, 'some_stream_push_bytes_many')
        return [st._results(frames=frames) for st, _ in items]

    def push_many(self, items: Sequence[Tuple['Stream', np.ndarray]], finish: Optional[Sequence[bool]] = None,
                  frames: bool = False):
        """some_stream_push_many: pushes samples to many streams of this session in one step, and finishes those with a true
        entry in `finish`.  Returns one (offsets, ranges, notes) per item, what Stream.push (then Stream.finish) would return;
        each stream's results go through its own Notes."""
        k = len(items)
        xs = [np.ascontiguousarray(x, dtype=np.float32) for _, x in items]
        streams = (C.c_void_p * max(k, 1))(*[st.handle for st, _ in items])
        ptrs = (C.c_void_p * max(k, 1))(*[x.ctypes.data for x in xs])
        lens = np.array([x.shape[0] for x in xs] or [0], dtype=np.int64)
        outs = (C.c_void_p * max(k, 1))(*[st.notes.handle for st, _ in items])
        fin = None if finish is None else np.array([bool(f) for f in finish] or [0], dtype=np.int32)
        if fin is not None and len(finish) != k:
            raise ValueError(f'push_many: {k} items, {len(finish)} finish flags')
        for st, _ in items:
            st.notes.set_frames(frames)
        _lib.check(self.lib.some_stream_push_many(streams, ptrs, lens.ctypes.data, None if fin is None else fin.ctypes.data, k,
                                                  outs), 'some_stream_push_many')
        return [st._results(frames=frames) for st, _ in items]

    def peek_many(self, streams: Sequence['Stream'], frames: bool = False):
        """some_stream_peek_many: the provisional notes of many streams of this session (PCM or encoded) in one step.  Returns
        one (offsets, ranges, notes) per stream, what Stream.peek returns."""
        k = len(streams)
        handles = (C.c_void_p * max(k, 1))(*[st.handle for st in streams])
        outs = (C.c_void_p * max(k, 1))(*[st._peek_notes(frames).handle for st in streams])
        _lib.check(self.lib.some_stream_peek_many(handles, k, outs), 'some_stream_peek_many')
        return [st._results(st.peeked, frames) for st in streams]


class Stream:
    """some_stream_*: push samples as they arrive; push() and finish() return the chunks that became final, in the shape
    transcribe_sliced returns them (offsets in seconds, sample ranges at the model's rate, notes).  Concatenated over all calls
    they equal transcribe_sliced on the whole recording.  Also a context manager (close() on exit)."""

    handle = None
    notes = None
    peeked = None
    rate = 0                  # of the pushed samples (an encoded stream's comes from its header)

    def __init__(self, session: Session, sample_rate: Optional[int] = None, params: Optional[_lib.SlicerParams] = None):
        self.lib, self.session = session.lib, session
        h = C.c_void_p()
        _lib.check(self.lib.some_stream_open(session.handle, int(sample_rate or session.sample_rate),
                                             C.byref(params) if params is not None else None, C.byref(h)), 'some_stream_open')
        self.handle = h
        self.rate = int(sample_rate or session.sample_rate)
        self.notes = Notes()
        session._streams.add(self)

    def _results(self, notes: Optional[Notes] = None, frames: bool = False):
        return self.session._results(notes or self.notes, frames)

    def _peek_notes(self, frames: bool = False) -> Notes:
        if self.peeked is None:
            self.peeked = Notes()
        self.peeked.set_frames(frames)
        return self.peeked

    def peek(self, frames: bool = False):
        """some_stream_peek: the provisional notes of the part of the recording the slicer has not closed yet, from the first
        sample no delivered chunk covers to the last fixed sample: zero or one clip, in the shape push() returns, with what
        transcribe() gives for those samples.  The stream does not change, and the results of the last push stay as they were
        (a peek has its own Notes)."""
        _lib.check(self.lib.some_stream_peek(self.handle, self._peek_notes(frames).handle), 'some_stream_peek')
        return self._results(self.peeked, frames)

    def push(self, samples: np.ndarray, frames: bool = False):
        """some_stream_push; a CUDA float32 tensor (``[n]`` or librosa's ``[channels, n]``, at the stream's rate) goes to
        some_stream_push_device instead: its down-mix is pushed, read on the device after the work its device's current
        stream holds at the call."""
        if audio.is_cuda_tensor(samples):
            a = audio.device_audio(samples, 0, 'Stream.push', self.rate)
            self.notes.set_frames(frames)
            _lib.check(self.lib.some_stream_push_device(self.handle, C.byref(a), self.notes.handle), 'some_stream_push_device')
            return self._results(frames=frames)
        x = np.ascontiguousarray(samples, dtype=np.float32)
        self.notes.set_frames(frames)
        _lib.check(self.lib.some_stream_push(self.handle, x.ctypes.data, int(x.shape[0]), self.notes.handle), 'some_stream_push')
        return self._results(frames=frames)

    def finish(self, frames: bool = False):
        self.notes.set_frames(frames)
        _lib.check(self.lib.some_stream_finish(self.handle, self.notes.handle), 'some_stream_finish')
        return self._results(frames=frames)

    def info(self) -> Dict[str, int]:
        i = _lib.StreamInfo()
        _lib.check(self.lib.some_stream_get_info(self.handle, C.byref(i)), 'some_stream_get_info')
        return {'received': i.received, 'fixed': i.fixed, 'held': i.held}

    def close(self):
        if self.handle is not None:
            self.lib.some_stream_close(self.handle)
            self.handle = None
        if self.notes is not None:
            self.notes.close()
        if self.peeked is not None:
            self.peeked.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        self.close()


class EncodedStream(Stream):
    """some_stream_open_encoded: push(bytes) takes the next bytes of a WAV, FLAC or AIFF file; push() and finish() return the chunks
    that became final, as Stream does.  Concatenated they equal Session.transcribe_encoded on the whole file."""

    def __init__(self, session: Session, params: Optional[_lib.SlicerParams] = None):
        self.lib, self.session = session.lib, session
        h = C.c_void_p()
        _lib.check(self.lib.some_stream_open_encoded(session.handle, C.byref(params) if params is not None else None,
                                                     C.byref(h)), 'some_stream_open_encoded')
        self.handle = h
        self.notes = Notes()
        session._streams.add(self)

    def push(self, data: bytes, frames: bool = False):
        d = bytes(data)
        self.notes.set_frames(frames)
        _lib.check(self.lib.some_stream_push_bytes(self.handle, d, len(d), self.notes.handle), 'some_stream_push_bytes')
        return self._results(frames=frames)

    def meta(self) -> Dict[str, int]:
        """some_stream_get_meta: the file's metadata (container 0 until the header is complete), the bytes pushed and the
        bytes held on the host."""
        m, got, held = _lib.AudioMeta(), C.c_longlong(), C.c_longlong()
        _lib.check(self.lib.some_stream_get_meta(self.handle, C.byref(m), C.byref(got), C.byref(held)), 'some_stream_get_meta')
        out = {name: getattr(m, name) for name, _ in _lib.AudioMeta._fields_ if name != 'reserved'}
        out.update(bytes_received=got.value, bytes_held=held.value)
        return out
