"""Validation losses and MIDI accuracy of a checkpoint over labelled DiffSinger datasets, on the GPU.

The numbers are the ones SOME's trainer logs for its validation set: ``validation/midi_loss``, ``validation/bound_loss``,
``validation/total_loss`` and ``midi_acc`` (training/me_task.py:72-154 for the continuous task,
training/me_quant_task.py:43-120 for the quantized one, aggregated as training/base_task.py:285-313 does).

Host part (this module), restating the label half of the binarizer:
- ``load_labels``: MIDIExtractionBinarizer.load_meta_data (preprocessing/me_binarizer.py:49-106): items from
  ``transcriptions.csv``, labels from ``wavs/{name}.ds``, glide skipping, note-name normalisation, ``merge_slurs`` and
  ``merge_rests`` (utils/binarizer_utils.py:11-71);
- ``item_labels``: the label arrays of ``_process_item`` (me_binarizer.py:201-223; quantized: me_quant_binarizer.py:22-34):
  ``note_midi`` with rests filled by nearest-neighbour interpolation, ``note_rest`` and ``unit2note`` (get_mel2ph_torch +
  LengthRegulator, binarizer_utils.py:75-84, modules/commons/tts_modules.py:5-38).  Validation items are never key-shifted.

Device part: the trunk runs once per batch with the raw logits head; ``some_eval_clips`` (csrc/evaluate.cu) computes every
clip's loss sums and accuracy counts from the logits without materialising the target, and writes the activated head that
``some_decode_notes`` turns into the predicted notes, exactly as infer() would (bf16) or infer_accurate() would (fp32).

Why one item per clip is the task's own computation: validation batches hold one item (``max_val_batch_size: 1``,
configs/base.yaml), so there is no padding, and ``get_mel2ph_torch`` leaves ``unit2note > 0`` on every frame, so the task's
``mask = unit2note > 0`` (me_task.py:87) is all ones (asserted here, not assumed).  The model's masked_fill calls are then
identities and each clip of the var-len batch is exactly the task's per-item forward.
"""
from __future__ import annotations

import csv
import ctypes as C
import dataclasses
import json
import math
import pathlib
from typing import Callable, Dict, List, Optional, Sequence, Union

import numpy as np

from . import _lib, audio
from .batch import load_groups, midi_to_note, note_to_midi, staged
from .engine import check_precision

HOP = 512


# ---------------------------------------------------------------------------------------------- labels (host)
def merge_slurs(note_seq: list, note_dur: list, note_slur: list, tolerance=None):
    """utils/binarizer_utils.py:11-51: merge slurred notes of similar pitch (duration-weighted mean MIDI)."""
    note_midi = [note_to_midi(n, round_midi=False) if n != 'rest' else 'rest' for n in note_seq]
    prev_min = prev_max = None
    midis = [note_midi[0]]
    durs = [note_dur[0]]

    def can_be_merged(midi):
        if tolerance is None or midi == 'rest' or midis[-1] == 'rest':
            return midis[-1] == midi
        return (abs(midi - midis[-1]) <= tolerance
                and (prev_min is None or abs(midi - prev_min) <= tolerance)
                and (prev_max is None or abs(midi - prev_max) <= tolerance))

    def merged_midi(midi1, dur1, midi2, dur2):
        if midi1 == midi2:
            return midi1
        return (midi1 * dur1 + midi2 * dur2) / (dur1 + dur2)

    for i in range(1, len(note_seq)):
        if note_slur[i] and can_be_merged(note_midi[i]):
            prev_min = min(note_midi[i], midis[-1]) if prev_min is None else min(prev_min, note_midi[i])
            prev_max = max(note_midi[i], midis[-1]) if prev_max is None else max(prev_max, note_midi[i])
            midis[-1] = merged_midi(midis[-1], durs[-1], note_midi[i], note_dur[i])
            durs[-1] += note_dur[i]
        else:
            midis.append(note_midi[i])
            durs.append(note_dur[i])
            prev_min = prev_max = None
    return [midi_to_note(n, cents=True) if n != 'rest' else 'rest' for n in midis], durs


def merge_rests(note_seq: list, note_dur: list):
    """utils/binarizer_utils.py:54-71: merge runs of rests into one."""
    i, seq, durs = 0, [], []
    while i < len(note_seq):
        if note_seq[i] != 'rest':
            seq.append(note_seq[i])
            durs.append(note_dur[i])
            i += 1
        else:
            j, rest_dur = i, 0
            while j < len(note_seq) and note_seq[j] == 'rest':
                rest_dur += note_dur[j]
                j += 1
            seq.append('rest')
            durs.append(rest_dur)
            i = j
    return seq, durs


def binarization_options(config: dict, quantized: bool) -> dict:
    """The ``binarization_args`` the label pipeline reads.  Missing keys take the values of the stock task configs
    (configs/continuous.yaml, configs/discrete.yaml): skip_glide, merge_rest and merge_slur on, no slur tolerance; the
    quantized binarizer always rounds MIDI (me_quant_binarizer.py:22-25)."""
    args = config.get('binarization_args') or {}
    return {'skip_glide': bool(args.get('skip_glide', True)), 'merge_rest': bool(args.get('merge_rest', True)),
            'merge_slur': bool(args.get('merge_slur', True)), 'slur_tolerance': args.get('slur_tolerance'),
            'round_midi': True if quantized else bool(args.get('round_midi', False))}


def load_labels(raw_data_dir, config: dict, quantized: bool = False, ds_id: int = 0) -> List[dict]:
    """MIDIExtractionBinarizer.load_meta_data (me_binarizer.py:49-106) for one raw data directory.  Returns
    ``[{'name': f'{ds_id}:{item}', 'wav_fn', 'note_seq', 'note_dur'}, ...]`` in transcriptions.csv order; items with glides
    are skipped (with the reference's message) when ``skip_glide`` is set.  The reference's two asserts are ValueErrors
    naming the item."""
    raw = pathlib.Path(raw_data_dir)
    opts = binarization_options(config, quantized)
    if not (raw / 'transcriptions.csv').exists():
        raise FileNotFoundError(f'transcriptions.csv not found in {raw}.')
    items = []
    with open(raw / 'transcriptions.csv', 'r', encoding='utf-8') as f:
        rows = list(csv.DictReader(f))
    for row in rows:
        item_name = row['name']
        with open(raw / 'wavs' / f'{item_name}.ds', 'r', encoding='utf8') as f:
            ds = json.load(f)
        if isinstance(ds, list):
            ds = ds[0]
        if opts['skip_glide'] and ds.get('note_glide') is not None and any(g != 'none' for g in ds['note_glide'].split()):
            print(f'Item {ds_id}:{item_name} contains glide notes. Skipping.')
            continue
        note_seq = [midi_to_note(np.clip(note_to_midi(n, round_midi=opts['round_midi']), a_min=0, a_max=127),
                                 cents=not opts['round_midi']) if n != 'rest' else 'rest'
                    for n in ds['note_seq'].split()]
        note_slur = [bool(int(s)) for s in ds['note_slur'].split()]
        note_dur = [float(x) for x in ds['note_dur'].split()]
        if not len(note_seq) == len(note_slur) == len(note_dur):
            raise ValueError(f'Lengths of note_seq, note_slur and note_dur mismatch in \'{item_name}\'.')
        if not any(note != 'rest' for note in note_seq):
            raise ValueError(f'All notes are rest in \'{item_name}\'.')
        if opts['merge_slur']:
            note_seq, note_dur = merge_slurs(note_seq, note_dur, note_slur, tolerance=opts['slur_tolerance'])
        if opts['merge_rest']:
            note_seq, note_dur = merge_rests(note_seq, note_dur)
        items.append({'name': f'{ds_id}:{item_name}', 'wav_fn': raw / 'wavs' / f'{item_name}.wav',
                      'note_seq': note_seq, 'note_dur': note_dur})
    return items


def item_labels(item: dict, frames: int, timestep: float, quantized: bool = False) -> Dict[str, np.ndarray]:
    """The label arrays of ``_process_item`` (me_binarizer.py:201-223) for an item of ``frames`` mel frames:
    ``note_midi`` (float32; quantized: int64 with rests = 128, me_quant_binarizer.py:28), ``note_rest`` (bool),
    ``note_dur`` (frames, int64) and ``unit2note`` (int64 [frames], 1-based).  The duration arithmetic runs in torch on the
    CPU, as the binarizer's does."""
    import torch
    from scipy import interpolate
    name = item['name']
    note_midi = np.array([(note_to_midi(n, round_midi=quantized) if n != 'rest' else -1) for n in item['note_seq']],
                         dtype=np.int64 if quantized else np.float32)
    note_rest = note_midi < 0
    if note_rest.all():
        raise ValueError(f'All notes are rest in \'{name}\'.')
    interp_func = interpolate.interp1d(np.where(~note_rest)[0], note_midi[~note_rest], kind='nearest',
                                       fill_value='extrapolate')
    note_midi[note_rest] = interp_func(np.where(note_rest)[0])
    if min(item['note_dur']) < 0:
        raise ValueError(f'Negative note duration in \'{name}\'.')
    durs = torch.FloatTensor(item['note_dur'])
    acc = torch.round(torch.cumsum(durs, dim=0) / timestep + 0.5).long()
    note_dur = torch.diff(acc, dim=0, prepend=torch.LongTensor([0])).numpy()
    # LengthRegulator: frame i belongs to the note whose [cumsum_prev, cumsum) holds i; pad with the last index or truncate
    unit2note = np.repeat(np.arange(1, len(note_dur) + 1, dtype=np.int64), note_dur)
    if unit2note.shape[0] == 0:
        raise ValueError(f'The notes of \'{name}\' last no frame.')
    if unit2note.shape[0] < frames:
        unit2note = np.concatenate([unit2note, np.full(frames - unit2note.shape[0], unit2note[-1], dtype=np.int64)])
    unit2note = unit2note[:frames]
    # the task's mask = unit2note > 0 (me_task.py:87) must be all ones for the per-clip evaluation to be the task's
    assert (unit2note > 0).all(), f'{name}: unit2note has unlabelled frames'
    if quantized:
        note_midi[note_rest] = 128
    return {'note_midi': note_midi, 'note_rest': note_rest, 'note_dur': note_dur, 'unit2note': unit2note}


# ---------------------------------------------------------------------------------------------- report
@dataclasses.dataclass
class EvalItem:
    name: str
    frames: int
    midi_loss: float
    bound_loss: float
    correct: int
    total: int
    note_midi: np.ndarray
    note_dur: np.ndarray
    note_rest: np.ndarray


@dataclasses.dataclass
class EvalReport:
    """``items``: one EvalItem per evaluated item (input order).  ``summary``: the trainer's validation numbers, aggregated
    as BaseTask does (base_task.py:285-313): each loss is a MeanMetric over the items with weight = batch size = 1
    (accumulated here in float64), ``total_loss`` sums the losses that ``use_midi_loss`` / ``use_bound_loss`` enable, and
    ``midi_acc`` = sum(correct) / sum(total).

    The trainer updates ``midi_acc`` only in the first ``num_valid_plots`` validation batches (me_task.py:109) and the losses
    over all of them; the per-item counts let a caller reproduce its number: sum the first ``num_valid_plots`` items in the
    validation loader's order."""
    items: List[EvalItem]
    summary: Dict[str, float]
    precision: str


def summarize(items: Sequence[EvalItem], config: dict) -> Dict[str, float]:
    n = len(items)
    midi = sum(it.midi_loss for it in items) / n if n else math.nan
    bound = sum(it.bound_loss for it in items) / n if n else math.nan
    use_midi, use_bound = config.get('use_midi_loss', True), config.get('use_bound_loss', True)
    total = (sum((it.midi_loss if use_midi else 0.0) + (it.bound_loss if use_bound else 0.0) for it in items) / n
             if n else math.nan)
    correct, frames = sum(it.correct for it in items), sum(it.total for it in items)
    out = {}
    if use_midi:
        out['midi_loss'] = midi
    if use_bound:
        out['bound_loss'] = bound
    out['total_loss'] = total
    out['midi_acc'] = correct / frames if frames else math.nan
    return out


# ---------------------------------------------------------------------------------------------- device part
class _Labels:
    """Device copies of a batch's labels for some_eval_clips, and its per-clip outputs."""

    def __init__(self, labels: Sequence[Dict[str, np.ndarray]], device):
        import torch
        self.cu_notes = torch.tensor(np.concatenate([[0], np.cumsum([len(l['note_midi']) for l in labels])]),
                                     dtype=torch.int32, device=device)
        self.unit2note = torch.from_numpy(np.concatenate([l['unit2note'] for l in labels]).astype(np.int32)).to(device)
        self.note_midi = torch.from_numpy(np.concatenate([l['note_midi'] for l in labels]).astype(np.float32)).to(device)
        self.note_rest = torch.from_numpy(np.concatenate([l['note_rest'] for l in labels]).astype(np.uint8)).to(device)
        b = len(labels)
        self.midi_loss = torch.empty(b, dtype=torch.float64, device=device)
        self.bound_loss = torch.empty(b, dtype=torch.float64, device=device)
        self.correct = torch.empty(b, dtype=torch.int32, device=device)


def eval_clips(eng, logits, bounds, cu_frames, lab: _Labels, c0: int, c1: int, row0: int, m: int, quantized: bool,
               head: int, probs=None):
    """Enqueues some_eval_clips for clips c0..c1 of ``lab`` whose frames are rows [0, m) of logits / bounds
    (chunk-relative ``cu_frames``; ``row0`` = the chunk's first frame in the batch)."""
    cfg = eng.config
    a = _lib.EvalArgs()
    a.logits, a.bounds, a.cu_frames = logits.data_ptr(), bounds.data_ptr(), cu_frames.data_ptr()
    a.unit2note = lab.unit2note.data_ptr() + 4 * row0
    a.cu_notes = lab.cu_notes.data_ptr() + 4 * c0
    a.note_midi, a.note_rest = lab.note_midi.data_ptr(), lab.note_rest.data_ptr()
    a.B, a.M, a.N, a.quantized, a.head = c1 - c0, m, eng.outdim, int(quantized), head
    a.vmin, a.vmax = float(cfg['midi_min']), float(cfg['midi_max'])
    a.deviation = float(cfg.get('midi_prob_deviation', 1.0))
    a.threshold = float(cfg.get('rest_threshold', 0.1))
    a.midi_loss = lab.midi_loss.data_ptr() + 8 * c0
    a.bound_loss = lab.bound_loss.data_ptr() + 8 * c0
    a.correct = lab.correct.data_ptr() + 4 * c0
    a.probs = _lib.ptr(probs)
    with eng._mark('some_eval_clips', m * (eng.outdim * 4.0 + 12.0)):
        _lib.check(eng.lib.some_eval_clips(C.byref(a), eng._stream), 'some_eval_clips')


def evaluate_recordings(infer_ins, waveforms: Sequence, labels: Sequence[Dict[str, np.ndarray]],
                        rates: Optional[Sequence[Optional[int]]] = None, precision: str = 'bf16', per_item: bool = False):
    """Evaluates whole recordings (no slicing: the task evaluates each item in one piece) against their label arrays
    (``item_labels`` for the recording's frame count).  ``waveforms`` / ``rates`` as in batch.transcribe_recordings.
    Returns per recording (midi_loss sum, bound_loss sum, correct, frames, notes dict).

    All recordings run as one var-len batch through the trunk of ``precision``.  ``per_item=True`` (fp32 only) runs them
    one at a time through the fp32 checker (Engine.accurate_clip, some_forward_f32) instead: the specification the batched
    fp32 path gives the same numbers as."""
    import torch
    eng = infer_ins.model
    quantized = bool(getattr(infer_ins, 'quantized', False))
    check_precision(precision)
    if per_item and precision != 'fp32':
        raise ValueError('per_item evaluation runs the fp32 checker: it needs precision=\'fp32\'')
    with staged(infer_ins, waveforms, rates) as (wave_d, bases, lens):
        frames = [1 + n // HOP for n in lens]
        for lab, t, it in zip(labels, frames, range(len(labels))):
            if lab['unit2note'].shape[0] != t:
                raise ValueError(f'recording {it}: labels for {lab["unit2note"].shape[0]} frames, audio has {t}')
        lab = _Labels(labels, eng.device)
        ranges = [(int(b), int(b) + n) for b, n in zip(bases, lens)]
        if per_item:
            notes = []
            for i, ((b0, _), n, t) in enumerate(zip(ranges, lens, frames)):
                start = torch.zeros(1, dtype=torch.int64, device=eng.device)
                length = torch.full((1,), n, dtype=torch.int64, device=eng.device)

                def hook(tt, cu_d, i=i, t=t):
                    eval_clips(eng, tt['probs'], tt['bounds'], cu_d, lab, i, i + 1, int(sum(frames[:i])), t, quantized,
                               _lib.EVAL_HEAD_F32, probs=tt['probs'])
                _, ws, k = eng.accurate_clip(wave_d[b0:] if n else wave_d, start, length, t, quantized, logits_hook=hook)
                notes.append({'note_midi': ws.note_midi[:k].cpu().numpy(),
                              'note_dur': ws.note_dur[:k].cpu().numpy().astype(np.int64) * eng.timestep,
                              'note_rest': ws.note_rest[:k].cpu().numpy().astype(bool)})
        else:
            head = _lib.EVAL_HEAD_TC if precision == 'bf16' else _lib.EVAL_HEAD_F32

            def hook(ws, c0, c1, mc, cu_d):
                eval_clips(eng, ws.probs, ws.bounds, cu_d, lab, c0, c1, int(cu[c0]), mc, quantized, head, probs=ws.probs)
            cu = np.zeros(len(ranges) + 1, dtype=np.int64)
            np.cumsum(frames, out=cu[1:])
            slab, cu_e, layout, _ = eng.enqueue(None, quantized, resident=(wave_d, ranges), logits_hook=hook,
                                                precision=precision)
            notes = eng.unpack_slab(slab.cpu().numpy(), cu_e, layout)
        midi_sum, bound_sum, correct = lab.midi_loss.cpu().numpy(), lab.bound_loss.cpu().numpy(), lab.correct.cpu().numpy()
    return [(float(ms), float(bs), int(c), t, nt) for ms, bs, c, t, nt in zip(midi_sum, bound_sum, correct, frames, notes)]


def evaluate_dataset(infer_ins, raw_data_dirs: Union[str, pathlib.Path, Sequence], config: dict, precision: str = 'bf16',
                     load_audio: Callable = audio.load_native, max_frames_per_batch: int = 400_000,
                     workers: int = 4, per_item: bool = False) -> EvalReport:
    """The trainer's validation numbers for a checkpoint (``infer_ins``, a plugin inference instance) over one or more
    DiffSinger raw data directories (``transcriptions.csv``, ``wavs/{name}.wav`` + ``wavs/{name}.ds``).

    Audio is read by ``load_audio(path, sr)`` on a thread pool and grouped into var-len batches of about
    ``max_frames_per_batch`` frames, as batch.batch_infer_dataset does; the default ``audio.load_native`` and
    ``audio.read_encoded`` (FLAC) give exactly librosa.load's samples, resampled / decoded on the device.

    ``precision='bf16'``: the product trunk (some_forward, bf16 tensor cores) once per batch; ``'fp32'``: the fp32 trunk
    (some_forward_f32_tiled) once per batch, whose logits are the fp32 checker's bit for bit, so every item's numbers are
    those of the trainer's fp32 validation as the checker computes them (``per_item=True`` runs the checker itself, one item
    at a time; see evaluate_recordings).  Either way some_eval_clips turns the logits into the losses, the accuracy counts
    and the probabilities the predicted notes are decoded from."""
    if isinstance(raw_data_dirs, (str, pathlib.Path)):
        raw_data_dirs = [raw_data_dirs]
    quantized = bool(getattr(infer_ins, 'quantized', False))
    sr = int(config['audio_sample_rate'])
    timestep = config['hop_size'] / config['audio_sample_rate']
    n_bins = int(config['midi_num_bins'])
    todo = []
    for ds_id, d in enumerate(raw_data_dirs):
        todo.extend((it, it['wav_fn']) for it in load_labels(d, config, quantized, ds_id))
    items: List[EvalItem] = []
    for group in load_groups(todo, load_audio, sr, max_frames_per_batch, workers):
        waves = [w for _, w, _ in group]
        rates = [r for _, _, r in group]
        labels = [item_labels(it, 1 + _resampled_len(w, r, sr) // HOP, timestep, quantized) for it, w, r in group]
        for (it, _, _), (ms, bs, c, t, nt) in zip(group, evaluate_recordings(infer_ins, waves, labels, rates, precision,
                                                                                       per_item)):
            midi = ms / t if quantized else ms / (t * n_bins)
            items.append(EvalItem(it['name'], t, midi, bs / t, c, t, nt['note_midi'], nt['note_dur'], nt['note_rest']))
    return EvalReport(items, summarize(items, config), precision)


def _resampled_len(wave, rate, sr: int) -> int:
    if isinstance(wave, audio.EncodedAudio):
        return audio.resampled_length(wave.length, wave.rate, sr)
    return audio.resampled_length(len(wave), audio.as_rate(rate if rate is not None else sr), sr)


def write_items_csv(report: EvalReport, path) -> None:
    """One row per item: name, frames, losses, accuracy counts and the predicted notes (space-separated)."""
    with open(path, 'w', encoding='utf8', newline='') as f:
        w = csv.writer(f)
        w.writerow(['name', 'frames', 'midi_loss', 'bound_loss', 'correct', 'total', 'note_midi', 'note_dur', 'note_rest'])
        for it in report.items:
            w.writerow([it.name, it.frames, repr(it.midi_loss), repr(it.bound_loss), it.correct, it.total,
                        ' '.join(repr(float(x)) for x in it.note_midi), ' '.join(repr(float(x)) for x in it.note_dur),
                        ' '.join(str(int(x)) for x in it.note_rest)])


def _main():
    import click

    @click.command(help='Score a checkpoint against labelled DiffSinger datasets: the trainer\'s validation losses and '
                        'MIDI accuracy')
    @click.option('--model', required=True, metavar='CKPT_PATH', help='Path to the model checkpoint (*.ckpt)')
    @click.option('--dataset', 'datasets', required=True, multiple=True, metavar='DIR',
                  help='Raw data directory with transcriptions.csv and wavs/*.wav + *.ds (repeatable)')
    @click.option('--fp32', is_flag=True, help='Use the fp32 trunk instead of the bf16 product path')
    @click.option('--items-csv', required=False, metavar='PATH', help='Write the per-item table to this CSV file')
    def evaluate(model, datasets, fp32, items_csv):
        import yaml

        from . import plugin
        model_path = pathlib.Path(model)
        with open(model_path.with_name('config.yaml'), 'r', encoding='utf8') as f:
            config = yaml.safe_load(f)
        cls = getattr(plugin, plugin.task_inference_mapping[config['task_cls']].rsplit('.', 1)[-1])
        infer_ins = cls(config=config, model_path=model_path)
        report = evaluate_dataset(infer_ins, list(datasets), config, precision='fp32' if fp32 else 'bf16')
        print(f'| {len(report.items)} items, {sum(it.frames for it in report.items)} frames, {report.precision}')
        for k, v in report.summary.items():
            print(f'validation/{k}: {v:.6f}' if k != 'midi_acc' else f'{k}: {v:.6f}')
        if items_csv:
            write_items_csv(report, items_csv)

    evaluate()


if __name__ == '__main__':
    _main()
