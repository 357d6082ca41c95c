"""Dataset-level driver (SURVEY.md §8f-2): the GPU counterpart of batch_infer.py.

The reference transcribes a DiffSinger dataset strictly one file at a time (batch_infer.py:164-176: librosa.load -> Slicer ->
infer on that file's chunks, a handful of 5-15 s clips per launch sequence).  Here the chunks of MANY recordings form one
var-len batch: every recording is uploaded once into one device buffer, the slicer's RMS lists of all of them come back in one
copy (csrc/slicer.cu), the cuts are decided on the host, and ONE mel -> trunk -> decode pass runs over all chunks where they lie
(Engine.enqueue(resident=...)); audio files are read by a thread pool while the GPU works on the previous group.

Everything after the notes is host string / rounding work and is restated so that ``transcriptions.csv`` comes out BYTE-identical
to batch_infer.py for the same notes (pinned by tests/golden/host_rows.npz, produced by the unmodified reference):
``calc_seq`` (:37-46), the note timeline of ``infer`` (:56-81), ``get_word_durs`` (:84-94), ``midi_align`` (:97-110), the
overlap helpers (:113-135) and the per-word assembly of the command (:178-219).

Third-party, absent here and restated: ``librosa.midi_to_note`` (librosa<0.10, requirements.txt:10; C-major spelling with
sharps, ``unicode=False``) and ``librosa.load`` (replaced by a WAV reader: scipy.io.wavfile + polyphase resampling — files
that are already 44.1 kHz decode to the same samples up to the int -> float scale librosa uses; other rates resample with a
different filter than librosa's, so their notes may differ at the margin).
"""
from __future__ import annotations

import concurrent.futures
import pathlib
from csv import DictReader, DictWriter
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from .slicer import Slicer, chunk_ranges, silence_tags

_NOTE_NAMES = ('C', 'C#', 'D', 'D#', 'E', 'F', 'F#', 'G', 'G#', 'A', 'A#', 'B')


# ---------------------------------------------------------------------------------------------- strings / rounding
def midi_to_note(midi: float) -> str:
    """librosa.midi_to_note(midi, unicode=False) for a scalar (octave on, cents off, key C:maj)."""
    num = int(np.round(midi))
    return '{:s}{:0d}'.format(_NOTE_NAMES[num % 12], int(num / 12) - 1)


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
def transcribe_recordings(infer_ins, waveforms: Sequence[np.ndarray], slicer: Optional[Slicer] = None):
    """[(chunk offsets in seconds, per-chunk notes)] for several mono recordings, as ONE var-len batch.

    Equivalent to ``[ (offsets, infer_ins.infer(chunks)) for chunks in (Slicer.slice(w) for w in waveforms) ]``
    (batch_infer.py:50-54) but every recording is uploaded once, all RMS lists come back in one copy, and a single
    mel -> trunk -> decode pass covers every chunk of every recording."""
    import torch
    eng = infer_ins.model
    slicer = slicer or Slicer(sr=infer_ins.config['audio_sample_rate'], max_sil_kept=1000)   # batch_infer.py:52
    quantized = bool(getattr(infer_ins, 'quantized', False))
    waves = [np.ascontiguousarray(w, dtype=np.float32) for w in waveforms]
    for w in waves:
        assert w.ndim == 1, 'mono recordings expected (librosa.load(..., mono=True), batch_infer.py:51)'
    lens = [int(w.shape[0]) for w in waves]
    bases = np.zeros(len(waves) + 1, dtype=np.int64)
    np.cumsum([(n + 3) & ~3 for n in lens], out=bases[1:])
    lock = getattr(infer_ins, '_lock', None)
    if lock is not None:
        lock.acquire()
    try:
        with torch.cuda.device(eng.device):
            wave_d = torch.empty(max(int(bases[-1]), 4), dtype=torch.float32, device=eng.device)
            for w, b, n in zip(waves, bases, lens):
                if n:
                    src = torch.from_numpy(w)
                    wave_d[b:b + n].copy_(src, non_blocking=src.is_pinned())
            need = [i for i, n in enumerate(lens) if (n + slicer.hop_size - 1) // slicer.hop_size > slicer.min_length]
            rms_lists = eng.rms_frames_many([wave_d[bases[i]:bases[i] + lens[i]] for i in need], slicer.win_size, slicer.hop_size)
            per_rec: List[List[Tuple[int, int]]] = [[(0, n)] for n in lens]               # slicer2.py:79-80 (short: one chunk)
            for i, rms in zip(need, rms_lists):
                per_rec[i] = chunk_ranges(silence_tags(rms, slicer), rms.shape[0], slicer.hop_size, lens[i])
            flat = [(int(bases[i]) + a, int(bases[i]) + b) for i, rs in enumerate(per_rec) for a, b in rs]
            results: List[Dict[str, np.ndarray]] = []
            if flat:
                slab, cu, layout, _ = eng.enqueue(None, quantized, resident=(wave_d, flat))
                host = slab.cpu().numpy()                                                    # one D2H + sync
                results = eng.unpack_slab(host, cu, layout)
    finally:
        if lock is not None:
            lock.release()
    out, k = [], 0
    for rs in per_rec:
        out.append(([a / slicer.sr for a, _ in rs], results[k:k + len(rs)]))
        k += len(rs)
    return out


def load_wav(path, sr: int) -> np.ndarray:
    """Mono float32 waveform at ``sr`` from a RIFF/WAVE file (stand-in for librosa.load, see the module docstring)."""
    from scipy.io import wavfile
    rate, data = wavfile.read(path)
    if data.dtype.kind == 'i':
        x = data.astype(np.float32) / float(1 << (8 * data.dtype.itemsize - 1))
    elif data.dtype.kind == 'u':
        x = (data.astype(np.float32) - 128.0) / 128.0
    else:
        x = data.astype(np.float32)
    if x.ndim > 1:
        x = x.mean(axis=1)
    if rate != sr:
        from math import gcd
        from scipy.signal import resample_poly
        g = gcd(int(rate), int(sr))
        x = resample_poly(x, sr // g, rate // g).astype(np.float32)
    return np.ascontiguousarray(x, dtype=np.float32)


def batch_infer_dataset(dataset, infer_ins, config: dict, round_midi: bool = False, csv=None, overwrite: bool = False,
                        load_audio: Callable = load_wav, max_frames_per_batch: int = 400_000, workers: int = 4) -> pathlib.Path:
    """batch_infer.py's command (:149-226) with dataset-level batching.  ``dataset`` = DiffSinger raw data dir with
    ``transcriptions.csv`` and ``wavs/``; writes ``csv`` (default: the dataset's own transcriptions.csv)."""
    data_path = pathlib.Path(dataset)
    csv_path = pathlib.Path(csv) if csv is not None else data_path / 'transcriptions.csv'
    if csv_path.exists() and not overwrite:
        raise FileExistsError(f'The CSV path \'{csv_path}\' already exists. Please re-try with --overwrite option.')
    with open(data_path / 'transcriptions.csv', 'r', encoding='utf8', newline='') as f:
        rows = list(DictReader(f))
    sr = config['audio_sample_rate']
    todo = []
    for row in rows:
        audio = data_path / 'wavs' / f"{row['name']}.wav"
        if not audio.exists():
            print(f'WARNING: audio file does not exist: \'{audio}\'')
            continue
        todo.append((row, audio))
    with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
        # decoding overlaps the GPU work below; only a bounded window of decoded recordings is ever held (the reference
        # streams one file at a time; an unbounded list of futures would keep the whole dataset's audio in host memory)
        import collections
        window = max(2 * workers, 4)
        pending: 'collections.deque' = collections.deque()
        it = iter(todo)

        def refill():
            while len(pending) < window:
                nxt = next(it, None)
                if nxt is None:
                    return
                pending.append((nxt[0], pool.submit(load_audio, nxt[1], sr)))

        group: List[Tuple[dict, np.ndarray]] = []
        frames = 0

        def flush():
            nonlocal group, frames
            if group:
                for (row, _), (offsets, segments) in zip(group, transcribe_recordings(infer_ins, [w for _, w in group])):
                    row['note_seq'], row['note_dur'] = row_notes(row['ph_dur'], row['ph_num'], note_timeline(offsets, segments), round_midi)
            group, frames = [], 0

        refill()
        while pending:
            row, fut = pending.popleft()
            wave = fut.result()
            refill()
            t = 1 + len(wave) // 512
            if group and frames + t > max_frames_per_batch:
                flush()
            group.append((row, wave))
            frames += t
        flush()
    with open(csv_path, 'w', encoding='utf8', newline='') as f:
        writer = DictWriter(f, fieldnames=['name', 'ph_seq', 'ph_dur', 'ph_num', 'note_seq', 'note_dur'])
        writer.writeheader()
        writer.writerows(rows)
    return csv_path
