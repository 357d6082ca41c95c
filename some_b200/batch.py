"""Dataset-level driver (SURVEY.md §8f-2): the GPU counterpart of batch_infer.py.

The reference transcribes a DiffSinger dataset strictly one file at a time (batch_infer.py:164-176: librosa.load -> Slicer ->
infer on that file's chunks, a handful of 5-15 s clips per launch sequence).  Here the chunks of MANY recordings form one
var-len batch: every recording is uploaded once into one device buffer (``stage_recordings``), then
``Engine.transcribe_resident`` -- the same step ``Engine.infer_sliced`` ends in -- brings the slicer's RMS lists of all of them
back in one copy, decides the cuts on the host and runs ONE mel -> trunk -> decode pass over all chunks where they lie; audio
files are read by a thread pool while the GPU works on the previous group.

Everything after the notes is host string / rounding work and is restated so that ``transcriptions.csv`` comes out BYTE-identical
to batch_infer.py for the same notes (pinned by tests/golden/host_rows.npz, produced by the unmodified reference):
``calc_seq`` (:37-46), the note timeline of ``infer`` (:56-81), ``get_word_durs`` (:84-94), ``midi_align`` (:97-110), the
overlap helpers (:113-135) and the per-word assembly of the command (:178-219).

Third-party, absent here and restated: ``librosa.midi_to_note`` (librosa<0.10, requirements.txt:10; C-major spelling with
sharps, ``unicode=False``) and ``librosa.load(path, sr=audio_sample_rate, mono=True)``:
- exact path: ``load_audio=audio.load_native`` returns each WAV file's decoded mono samples at their NATIVE rate; the recordings
  are uploaded as they are and ``transcribe_recordings(..., rates=...)`` resamples them on the device with resampy's
  ``kaiser_best`` filter (librosa's default ``res_type``), bit-identical to librosa.load, straight into the batch's wave
  buffer (some_b200/audio.py, csrc/resample.cu);
- FLAC: ``load_audio=audio.read_encoded`` returns each FLAC file's bytes and metadata (``audio.EncodedAudio``) without
  decoding them; ``transcribe_recordings`` uploads the bytes of all of them into one buffer and decodes them on the device
  (csrc/flac.cu), straight to mono at their native rate, bit-identical to librosa.load, into the batch's wave buffer or
  the resampler's input;
- default ``load_wav``: the same WAV decode, then scipy's polyphase resampling on the host.  Files that are already at
  ``audio_sample_rate`` give librosa's samples exactly; other rates go through a different filter from librosa's, so their
  notes may differ at the margin.
"""
from __future__ import annotations

import concurrent.futures
import contextlib
import pathlib
import re
from csv import DictReader, DictWriter
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import audio
from .slicer import Slicer

_NOTE_NAMES = ('C', 'C#', 'D', 'D#', 'E', 'F', 'F#', 'G', 'G#', 'A', 'A#', 'B')


# ---------------------------------------------------------------------------------------------- strings / rounding
def midi_to_note(midi: float, cents: bool = False) -> str:
    """librosa.midi_to_note(midi, cents=cents, unicode=False) for a scalar (octave on, key C:maj).  With ``cents`` the
    signed cent offset ``int(100 * np.around(midi - round(midi), 2))`` follows as ``{:+02d}`` (``C4+0``, ``A#3-25``).
    Restated from librosa 0.9 (not installed here): the cents form could not be checked against librosa itself."""
    num = int(np.round(midi))
    note = '{:s}{:0d}'.format(_NOTE_NAMES[num % 12], int(num / 12) - 1)
    if cents:
        note = '{:s}{:+02d}'.format(note, int(100 * np.around(midi - num, 2)))
    return note


_PITCH_CLASSES = {'C': 0, 'D': 2, 'E': 4, 'F': 5, 'G': 7, 'A': 9, 'B': 11}
_ACCIDENTALS = {'#': 1, '': 0, 'b': -1, '!': -1, '\u266f': 1, '\U0001d12a': 2, '\u266d': -1, '\U0001d12b': -2, '\u266e': 0}
_NOTE_RE = re.compile('^(?P<note>[A-Ga-g])(?P<accidental>[#\u266f\U0001d12ab!\u266d\U0001d12b\u266e]*)(?P<octave>[+-]?\\d+)?'
                      '(?P<cents>[+-]\\d+)?$')


def note_to_midi(note: str, round_midi: bool = True):
    """librosa.note_to_midi(note, round_midi=round_midi) for one note name: pitch class, any accidentals (``#``, ``b``,
    ``!`` and the unicode signs), optional octave (default 0) and optional signed cents, as
    ``12 * (octave + 1) + pitch + accidentals + cents * 1e-2`` (rounded half to even to an int with ``round_midi``).  Raises
    ValueError for a malformed name.  Restated from librosa 0.9 (not installed here) and not checked against librosa
    itself; the DiffSinger labels it reads use the plain forms (``C#4``, ``A3+25``, ``rest`` is the caller's)."""
    match = _NOTE_RE.match(note)
    if not match:
        raise ValueError(f'Improper note format: {note:s}')
    pitch = match.group('note').upper()
    offset = np.sum([_ACCIDENTALS[o] for o in match.group('accidental')])
    octave = match.group('octave')
    cents = match.group('cents')
    octave = int(octave) if octave else 0
    cents = int(cents) * 1e-2 if cents else 0
    note_value = 12 * (octave + 1) + _PITCH_CLASSES[pitch] + offset + cents
    if round_midi:
        note_value = int(np.round(note_value))
    return note_value


def calc_seq(note_midi: float, note_rest: bool) -> str:
    """Note name with a signed cent offset, or 'rest' (batch_infer.py:37-46)."""
    if note_rest:
        return 'rest'
    nearest = round(note_midi, 0)
    cent = int(round(note_midi - nearest, 2) * 100)      # NB int() truncates 28.999999999999996 -> 28, as the reference does
    suffix = f'+{cent}' if cent > 0 else ('' if cent == 0 else str(cent))
    return f'{midi_to_note(nearest)}{suffix}'


def note_timeline(offsets: Sequence[float], segments: Sequence[Dict[str, np.ndarray]]) -> List[dict]:
    """Chunk-relative notes -> absolute, non-overlapping note records rounded to 6 decimals (batch_infer.py:56-81)."""
    notes: List[dict] = []
    for offset, seg in zip(offsets, segments):
        offset = round(float(offset), 6)
        pitch, dur, rest = seg['note_midi'].tolist(), seg['note_dur'].tolist(), seg['note_rest'].tolist()
        assert len(pitch) == len(dur) == len(rest)
        elapsed = 0
        for p, d, r in zip(pitch, dur, rest):
            d = round(d, 6)
            elapsed = round(elapsed, 6)
            rec = {'start_time': round(offset + elapsed, 6), 'end_time': round(offset + elapsed + d, 6), 'note_seq': calc_seq(p, r)}
            if notes and rec['start_time'] < notes[-1]['end_time']:
                rec['start_time'] = notes[-1]['end_time']
            rec['note_dur'] = round(rec['end_time'] - rec['start_time'], 6)
            notes.append(rec)
            elapsed += d
    return notes


def word_durations(ph_durs: Sequence[float], ph_nums: Sequence[int]) -> List[Tuple[float, float]]:
    """(start, end) of every word from phoneme durations and per-word phoneme counts (batch_infer.py:84-94)."""
    spans, first, t = [], 0, 0
    for count in ph_nums:
        length = round(sum(ph_durs[first:first + count]), 6)
        spans.append((round(t, 6), round(t + length, 6)))
        first += count
        t += length
    return spans


def align_to_words(notes: List[dict], words: Sequence[Tuple[float, float]], tolerance: float = 0.05) -> List[dict]:
    """Snap note edges to word boundaries within ``tolerance`` and drop notes that collapse (batch_infer.py:97-110).
    Mutates the records, like the reference."""
    edges = [w[0] for w in words] + [words[-1][1]]
    kept = []
    for rec in notes:
        for e in edges:
            if e - tolerance <= rec['start_time'] <= e + tolerance:
                rec['start_time'] = e
            if e - tolerance <= rec['end_time'] <= e + tolerance:
                rec['end_time'] = e
        rec['note_dur'] = round(rec['end_time'] - rec['start_time'], 6)
        if rec['note_dur'] > 0:
            kept.append(rec)
    return kept


def notes_touching(span: Tuple[float, float], notes: Sequence[dict]) -> List[dict]:
    """batch_infer.py:113-122."""
    lo, hi = span
    return [n for n in notes
            if lo < n['start_time'] < hi or lo < n['end_time'] < hi or (n['start_time'] <= lo and hi <= n['end_time'])]


def dominant_note(span: Tuple[float, float], notes: Sequence[dict]) -> str:
    """The note with the largest overlap with the word, 'rest' if none overlaps (batch_infer.py:125-135)."""
    best, best_overlap = 'rest', 0
    for n in notes:
        overlap = max(0, min(span[1], n['end_time']) - max(span[0], n['start_time']))
        if overlap > best_overlap:
            best_overlap, best = overlap, n['note_seq']
    return best


def row_notes(ph_dur_field: str, ph_num_field: str, notes: List[dict], round_midi: bool) -> Tuple[str, str]:
    """The ``note_seq`` / ``note_dur`` CSV fields of one item (batch_infer.py:178-219)."""
    ph_dur = [round(float(x), 6) for x in ph_dur_field.split(' ')]
    ph_num = [int(x) for x in ph_num_field.split(' ')]
    words = word_durations(ph_dur, ph_num)
    notes = align_to_words(notes, words)
    seq: list = []
    dur: list = []
    for start, end in words:
        word_len = round(end - start, 6)
        if round_midi:
            seq.append(dominant_note((start, end), notes))
            dur.append(word_len)
            continue
        w_seq, w_dur = [], []
        for n in notes_touching((start, end), notes):
            w_seq.append(n['note_seq'])
            if n['start_time'] <= start:
                w_dur.append(round(min(end, n['end_time']) - start, 6))
            elif n['end_time'] >= end:
                w_dur.append(round(end - max(start, n['start_time']), 6))
            else:                                  # (the reference's third branch is unreachable: it is covered by the first)
                w_dur.append(round(n['note_dur'], 6))
        if not w_seq:
            w_seq.append('rest')
            w_dur.append(word_len)
        if round(sum(w_dur), 6) < word_len:
            w_seq.append('rest')
            w_dur.append(word_len - round(sum(w_dur), 6))
        seq.extend(w_seq)
        dur.extend(w_dur)
    assert len(seq) == len(dur)
    return ' '.join(str(x) for x in seq), ' '.join(str(round(x, 6)) for x in dur)


# ---------------------------------------------------------------------------------------------- GPU part
def stage_recordings(eng, target_sr: int, waveforms: Sequence, rates: Optional[Sequence[Optional[int]]]):
    """Uploads mono recordings (numpy arrays, or ``audio.EncodedAudio`` FLAC records) into ONE device buffer at
    ``target_sr``, as transcribe_recordings describes: recordings at another rate are resampled on the device, FLAC records
    decoded there, and CUDA float32 tensors (``[n]`` or librosa's ``[channels, n]``) down-mixed there by one some_downmix
    launch per destination, with no host copy.  Call on the engine's device.  Returns (wave_d, bases int64 [n + 1], lens, flac_status): recording i is
    wave_d[bases[i] : bases[i] + lens[i]]; the FLAC status words are checked with audio._check_status once the stream has
    passed them, as ``staged`` does."""
    import torch
    enc = {i: w for i, w in enumerate(waveforms) if isinstance(w, audio.EncodedAudio)}
    here = torch.empty(0, device=eng.device).device                            # with its index
    dev = {i: w for i, w in enumerate(waveforms) if audio.is_cuda_tensor(w)}    # on another device: copied to the engine's
    dev = {i: t if t.device == here else t.to(here) for i, t in dev.items()}
    dev_frames = {i: audio.device_layout(t, i, 'stage_recordings')[1] for i, t in dev.items()}
    waves = [None if i in enc or i in dev else np.ascontiguousarray(w, dtype=np.float32) for i, w in enumerate(waveforms)]
    for w in waves:
        assert w is None or w.ndim == 1, 'mono recordings expected (librosa.load(..., mono=True), batch_infer.py:51)'
    if rates is None:
        rates = [None] * len(waves)
    assert len(rates) == len(waves), 'one rate per recording'
    for i, rec in enc.items():
        if rates[i] is not None and audio.as_rate(rates[i]) != rec.rate:
            raise ValueError(f'{rec.name}: rate {rates[i]} given for a FLAC record of {rec.rate} Hz')
    rates = [enc[i].rate if i in enc else audio.as_rate(target_sr if r is None else r) for i, r in enumerate(rates)]
    flac = None
    if enc:                                                        # scan + chain: one device-to-host copy, one sync
        flac = audio.FlacBatch(list(enc.values()), eng.device)
    slot = {i: k for k, i in enumerate(enc)}                       # recording -> its index in the FlacBatch
    native_lens = [flac.lengths[slot[i]] if i in enc else dev_frames[i] if i in dev else int(w.shape[0])
                   for i, w in enumerate(waves)]
    lens = [audio.resampled_length(n, r, target_sr) for n, r in zip(native_lens, rates)]
    bases = np.zeros(len(waves) + 1, dtype=np.int64)
    np.cumsum([(n + 3) & ~3 for n in lens], out=bases[1:])
    wave_d = torch.empty(max(int(bases[-1]), 4), dtype=torch.float32, device=eng.device)
    for w, b, n, r in zip(waves, bases, lens, rates):
        if n and r == target_sr and w is not None:
            src = torch.from_numpy(w)
            wave_d[b:b + n].copy_(src, non_blocking=src.is_pinned())
    audio.downmix_into([(dev[i], wave_d, int(bases[i])) for i in dev if rates[i] == target_sr], 'stage_recordings')
    flac_status = []
    direct = {slot[i]: int(bases[i]) for i in enc if rates[i] == target_sr}
    if direct:
        flac_status.append(flac.emit(wave_d, direct))
    for r in sorted(set(rates) - {target_sr}):                # one resampling launch per native rate
        group = [i for i, ri in enumerate(rates) if ri == r]
        starts = np.zeros(len(group) + 1, dtype=np.int64)
        np.cumsum([native_lens[i] for i in group], out=starts[1:])
        native_d = torch.empty(max(int(starts[-1]), 1), dtype=torch.float32, device=eng.device)
        for i, a in zip(group, starts):
            if i not in enc and i not in dev:
                native_d[a:a + native_lens[i]].copy_(torch.from_numpy(waves[i]))
        audio.downmix_into([(dev[i], native_d, int(a)) for i, a in zip(group, starts) if i in dev], 'stage_recordings')
        to_decode = {slot[i]: int(a) for i, a in zip(group, starts) if i in enc}
        if to_decode:
            flac_status.append(flac.emit(native_d, to_decode))
        audio.resample_into(native_d, starts[:-1].tolist(), [native_lens[i] for i in group], wave_d,
                            [int(bases[i]) for i in group], r, target_sr)
    return wave_d, bases, lens, flac_status


@contextlib.contextmanager
def staged(infer_ins, waveforms: Sequence, rates: Optional[Sequence[Optional[int]]]):
    """``stage_recordings`` for a plugin instance at its ``audio_sample_rate``, yielding (wave_d, bases, lens).  The block
    runs under the instance's lock (if it has one: concurrent callers share one engine and its buffers) on the engine's
    device.  When the block ends normally, its work on the stream has passed the FLAC decode, whose status words are then
    checked (audio._check_status)."""
    import torch
    eng = infer_ins.model
    lock = getattr(infer_ins, '_lock', None)
    with (lock if lock is not None else contextlib.nullcontext()), torch.cuda.device(eng.device):
        wave_d, bases, lens, flac_status = stage_recordings(eng, int(infer_ins.config['audio_sample_rate']), waveforms, rates)
        yield wave_d, bases, lens
        for st in flac_status:
            audio._check_status(st)


def transcribe_recordings(infer_ins, waveforms: Sequence, slicer: Optional[Slicer] = None,
                          rates: Optional[Sequence[Optional[int]]] = None):
    """[(chunk offsets in seconds, per-chunk notes)] for several mono recordings, as ONE var-len batch.

    Equivalent to ``[ (offsets, infer_ins.infer(chunks)) for chunks in (Slicer.slice(w) for w in waveforms) ]``
    (batch_infer.py:50-54) but every recording is uploaded once (``stage_recordings``), and ``Engine.transcribe_resident``
    brings all RMS lists back in one copy and covers every chunk of every recording with a single mel -> trunk -> decode
    pass.

    ``rates``: each recording's native sample rate (default: all at ``audio_sample_rate``).  A recording at another rate is
    uploaded as it is and resampled on the device, grouped by rate, straight into the batch's wave buffer, exactly as
    librosa.load(sr=audio_sample_rate) would have resampled it (audio.resample); slicing and inference then run on the
    resampled samples.

    ``waveforms`` may also hold ``audio.EncodedAudio`` records (FLAC files read by ``audio.read_encoded``).  Their rates
    come from the records (a ``rates`` entry for one must be None or equal it); the bytes of all of them are uploaded into
    one buffer and decoded on the device, straight to mono at their native rate (audio.FlacBatch), into the wave buffer or
    the resampler's input."""
    slicer = slicer or Slicer(sr=int(infer_ins.config['audio_sample_rate']), max_sil_kept=1000)   # batch_infer.py:52
    with staged(infer_ins, waveforms, rates) as (wave_d, bases, lens):
        return infer_ins.model.transcribe_resident(wave_d, bases, lens, slicer, bool(getattr(infer_ins, 'quantized', False)),
                                                   getattr(infer_ins, 'precision', 'bf16'))


def load_wav(path, sr: int) -> np.ndarray:
    """Mono float32 waveform at ``sr`` from a RIFF/WAVE file: librosa.load's decode and down-mix, then scipy's polyphase
    resampling on the host (NOT librosa's filter; ``audio.load_native`` is the exact path, see the module docstring)."""
    x, rate = audio.decode_wav(path)
    if x.ndim > 1:
        x = x.mean(axis=1)
    if rate != sr:
        from math import gcd
        from scipy.signal import resample_poly
        g = gcd(int(rate), int(sr))
        x = resample_poly(x, sr // g, rate // g).astype(np.float32)
    return np.ascontiguousarray(x, dtype=np.float32)


def load_groups(todo: Sequence[Tuple[object, pathlib.Path]], load_audio: Callable, sr: int, max_frames_per_batch: int,
                workers: int):
    """Reads the audio of ``todo = [(key, path), ...]`` with ``load_audio(path, sr)`` on a thread pool and yields groups
    ``[(key, waveform or EncodedAudio, native rate or None), ...]`` of about ``max_frames_per_batch`` frames, in order, to be
    run as one var-len batch each: decoding overlaps the GPU work on the previous group.  Only a bounded window of decoded
    recordings is ever held (the reference streams one file at a time; an unbounded list of futures would keep the whole
    dataset's audio in host memory)."""
    import collections
    with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
        window = max(2 * workers, 4)
        pending: 'collections.deque' = collections.deque()
        it = iter(todo)

        def refill():
            while len(pending) < window:
                nxt = next(it, None)
                if nxt is None:
                    return
                pending.append((nxt[0], pool.submit(load_audio, nxt[1], sr)))

        group: List[tuple] = []
        frames = 0
        refill()
        while pending:
            key, fut = pending.popleft()
            wave = fut.result()
            if isinstance(wave, audio.EncodedAudio):                   # decoded on the device; its rate is its own
                rate, n = None, wave.length * int(sr) // wave.rate
            else:
                wave, rate = wave if isinstance(wave, tuple) else (wave, sr)
                n = audio.resampled_length(len(wave), audio.as_rate(rate), int(sr))
            refill()
            t = 1 + n // 512
            if group and frames + t > max_frames_per_batch:
                yield group
                group, frames = [], 0
            group.append((key, wave, rate))
            frames += t
        if group:
            yield group


def batch_infer_dataset(dataset, infer_ins, config: dict, round_midi: bool = False, csv=None, overwrite: bool = False,
                        load_audio: Callable = load_wav, max_frames_per_batch: int = 400_000, workers: int = 4) -> pathlib.Path:
    """batch_infer.py's command (:149-226) with dataset-level batching.  ``dataset`` = DiffSinger raw data dir with
    ``transcriptions.csv`` and ``wavs/``; writes ``csv`` (default: the dataset's own transcriptions.csv).

    ``load_audio(path, sr)`` returns the mono waveform at ``sr``, a ``(waveform, native_rate)`` pair, or an
    ``audio.EncodedAudio`` record: pairs are resampled on the device (transcribe_recordings(rates=...)), records are also
    decoded there.  ``load_audio=audio.load_native`` is librosa.load's exact result for WAV files and
    ``load_audio=audio.read_encoded`` for FLAC files; the default ``load_wav`` resamples with scipy on the host.  (Dataset
    items are still found as ``wavs/{name}.wav``, whatever the files hold.)"""
    data_path = pathlib.Path(dataset)
    csv_path = pathlib.Path(csv) if csv is not None else data_path / 'transcriptions.csv'
    if csv_path.exists() and not overwrite:
        raise FileExistsError(f'The CSV path \'{csv_path}\' already exists. Please re-try with --overwrite option.')
    with open(data_path / 'transcriptions.csv', 'r', encoding='utf8', newline='') as f:
        rows = list(DictReader(f))
    sr = config['audio_sample_rate']
    todo = []
    for row in rows:
        wav_path = data_path / 'wavs' / f"{row['name']}.wav"
        if not wav_path.exists():
            print(f'WARNING: audio file does not exist: \'{wav_path}\'')
            continue
        todo.append((row, wav_path))
    for group in load_groups(todo, load_audio, sr, max_frames_per_batch, workers):
        results = transcribe_recordings(infer_ins, [w for _, w, _ in group], rates=[r for _, _, r in group])
        for (row, _, _), (offsets, segments) in zip(group, results):
            row['note_seq'], row['note_dur'] = row_notes(row['ph_dur'], row['ph_num'], note_timeline(offsets, segments), round_midi)
    with open(csv_path, 'w', encoding='utf8', newline='') as f:
        writer = DictWriter(f, fieldnames=['name', 'ph_seq', 'ph_dur', 'ph_num', 'note_seq', 'note_dur'])
        writer.writeheader()
        writer.writerows(rows)
    return csv_path
