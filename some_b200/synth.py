"""Synthetic inputs shared by the tests and bench.py (SURVEY.md §8d): seeded "sung-note"
waveforms and a seeded random-weight checkpoint in the reference's on-disk layout
(``{'state_dict': {'model.' + k: v}}`` + flattened ``config.yaml`` beside it,
base_infer.py:27-33 / infer.py:21).  No pretrained weights or audio are obtainable offline.
"""
from __future__ import annotations

import copy
import pathlib
from collections import OrderedDict

import numpy as np
import yaml

from .config import model_param_shapes

SR = 44100

# Flattened configs of the three named model files (configs/base.yaml <- continuous.yaml <-
# two_head_model.yaml etc.), reduced to the keys inference reads (SURVEY.md §5 "Config / flags").
_EXTRACTOR = dict(dim=512, use_lay_skip=True, kernel_size=31, conv_drop=0.1, ffn_latent_drop=0.1,
                  ffn_out_drop=0.1, attention_drop=0.1, attention_heads=8, attention_heads_dim=64)
_COMMON = dict(hop_size=512, win_size=2048, audio_sample_rate=44100, fmin=40, fmax=8000,
               midi_min=0, midi_max=127, units_dim=80, units_encoder='mel',
               model_cls='modules.model.Gmidi_conform.midi_conforms',
               midi_prob_deviation=1.0, rest_threshold=0.1)
NAMED_CONFIGS = {
    'two_head': dict(_COMMON, task_cls='training.MIDIExtractionTask', midi_num_bins=128,
                     midi_extractor_args=dict(_EXTRACTOR, lay=3)),
    # quant_two_head_model.yaml lacks midi_prob_deviation / rest_threshold and the unmodified
    # reference raises KeyError (me_infer.py:26-27); the harness injects them (SURVEY.md §8d C3).
    'quant_two_head': dict(_COMMON, task_cls='training.QuantizedMIDIExtractionTask', midi_num_bins=129,
                           midi_extractor_args=dict(_EXTRACTOR, lay=3)),
    'midi_conformer': dict(_COMMON, task_cls='training.MIDIExtractionTask', midi_num_bins=128,
                           midi_extractor_args=dict(_EXTRACTOR, lay=8)),
}


def named_config(name: str, **overrides) -> dict:
    cfg = copy.deepcopy(NAMED_CONFIGS[name])
    for k, v in overrides.items():
        if k == 'lay':
            cfg['midi_extractor_args']['lay'] = v
        else:
            cfg[k] = v
    return cfg


def frames_of(num_samples: int, hop: int = 512) -> int:
    """T = 1 + floor(L / hop): pad 1024+1024, n_fft 2048, center=False (spec.py:48-60)."""
    return 1 + num_samples // hop


def synth_waveform(seed: int, seconds: float = None, num_samples: int = None, sr: int = SR,
                   silence_gaps: bool = False) -> np.ndarray:
    """Seeded "sung-note" signal: random-walk MIDI pitch in [48, 72], note length U(0.15, 0.8) s,
    15 % rests, 6 harmonics with 1/k amplitude, 5.5 Hz vibrato of +-30 cents, 10 ms raised-cosine
    note edges, peak 0.5, white noise at -50 dBFS; float32 mono."""
    rng = np.random.default_rng(seed)
    n = int(num_samples if num_samples is not None else round(seconds * sr))
    out = np.zeros(n, dtype=np.float64)
    t0 = 0
    pitch = float(rng.integers(55, 66))
    phase = np.zeros(6)
    next_gap = rng.uniform(6, 14) * sr if silence_gaps else None
    gaps = []
    while t0 < n:
        if silence_gaps and t0 >= next_gap:
            g = int(rng.uniform(0.5, 1.0) * sr)
            gaps.append((t0, min(n, t0 + g)))
            t0 += g
            next_gap = t0 + rng.uniform(6, 14) * sr
            continue
        ln = int(rng.uniform(0.15, 0.8) * sr)
        t1 = min(n, t0 + ln)
        m = t1 - t0
        is_rest = rng.random() < 0.15
        pitch = float(np.clip(pitch + rng.integers(-4, 5), 48, 72))
        if not is_rest and m > 0:
            tt = (np.arange(m) + t0) / sr
            cents = 30.0 * np.sin(2 * np.pi * 5.5 * tt)
            f = 440.0 * 2.0 ** ((pitch - 69.0 + cents / 100.0) / 12.0)
            dphi = 2 * np.pi * f / sr
            base = np.cumsum(dphi)
            seg = np.zeros(m)
            for k in range(1, 7):
                seg += np.sin(phase[k - 1] + k * base) / k
                phase[k - 1] = (phase[k - 1] + k * base[-1]) % (2 * np.pi)
            edge = min(int(0.010 * sr), m // 2)
            env = np.ones(m)
            if edge > 0:
                ramp = 0.5 - 0.5 * np.cos(np.pi * np.arange(edge) / edge)
                env[:edge] = ramp
                env[m - edge:] = ramp[::-1]
            out[t0:t1] = seg * env
        t0 = t1
    peak = np.abs(out).max()
    if peak > 0:
        out *= 0.5 / peak
    out += rng.standard_normal(n) * (10.0 ** (-50.0 / 20.0))
    for a, b in gaps:
        out[a:b] = 0.0  # digital silence so utils/slicer2 cuts there
    return out.astype(np.float32)


def edge_case_waveforms() -> 'OrderedDict[str, np.ndarray]':
    """Parity-only clips (SURVEY.md §8d): silence, full-scale sine, noise, ragged / tiny lengths."""
    rng = np.random.default_rng(7)
    t = np.arange(SR * 2) / SR
    return OrderedDict([
        ('zeros', np.zeros(SR, dtype=np.float32)),
        ('sine1k', np.sin(2 * np.pi * 1000.0 * t).astype(np.float32)),
        ('noise', (0.1 * rng.standard_normal(3 * SR)).astype(np.float32)),
        ('ragged', synth_waveform(11, num_samples=70001)),
        ('short', synth_waveform(12, num_samples=1500)),       # L < n_fft: T = 3
        ('one_frame', synth_waveform(13, num_samples=300)),    # T = 1
        ('empty', np.zeros(0, dtype=np.float32)),              # T = 1 (all padding)
    ])


def fabricate_state_dict(config: dict, seed: int = 1234):
    """Seeded weights in schema order.  Linear / conv: U(+-1/sqrt(fan_in)) like torch's default
    init; every LN / BN affine ~ U(0.8, 1.2) / N(0, 0.05); BN running_mean ~ N(0, 0.1),
    running_var ~ U(0.5, 1.5) so that folding bugs show (SURVEY.md §8d "Weights")."""
    import torch

    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    schema = model_param_shapes(config)
    for name, shape in schema.items():
        leaf = name.rsplit('.', 1)[-1]
        is_norm = '.norm' in name
        if leaf == 'num_batches_tracked':
            v = torch.tensor(0, dtype=torch.int64)
        elif leaf == 'running_mean':
            v = torch.randn(shape, generator=g) * 0.1
        elif leaf == 'running_var':
            v = torch.rand(shape, generator=g) + 0.5
        elif is_norm and leaf == 'weight':
            v = torch.rand(shape, generator=g) * 0.4 + 0.8
        elif is_norm and leaf == 'bias':
            v = torch.randn(shape, generator=g) * 0.05
        else:
            if leaf == 'weight':
                fan_in = int(np.prod(shape[1:]))
            else:  # bias: fan_in of the matching weight
                wshape = schema[name[:-4] + 'weight']
                fan_in = int(np.prod(wshape[1:]))
            bound = 1.0 / np.sqrt(fan_in)
            v = (torch.rand(shape, generator=g) * 2 - 1) * bound
        sd[name] = v.float() if v.dtype != torch.int64 else v
    return sd


def write_checkpoint(directory, config: dict, seed: int = 1234) -> pathlib.Path:
    """Writes ``model.ckpt`` + ``config.yaml`` the way train.py / simplify.py leave them."""
    import torch

    directory = pathlib.Path(directory)
    directory.mkdir(parents=True, exist_ok=True)
    sd = fabricate_state_dict(config, seed)
    path = directory / 'model.ckpt'
    torch.save({'state_dict': OrderedDict(('model.' + k, v) for k, v in sd.items())}, path)
    with open(directory / 'config.yaml', 'w', encoding='utf8') as f:
        yaml.safe_dump(config, f, sort_keys=False, allow_unicode=True)
    return path


def synth_labelled(seed: int, seconds: float, sr: int = SR):
    """Seeded sung-note waveform together with the DiffSinger labels the generator used: returns
    ``(waveform f32, {'note_seq': [...], 'note_dur': [...], 'note_slur': [...]})``.  Notes last U(0.12, 0.7) s (durations
    rounded to 0.1 ms, the last one cut so that they sum to ``seconds``), pitch is a random walk in [48, 72] MIDI with a
    cent offset on one note in four, one note in seven is a rest and one in five a slur of the note before it (within a
    semitone).  Rendering as in ``synth_waveform``: 6 harmonics, 5.5 Hz vibrato, 10 ms note edges, peak 0.5, noise at
    -50 dBFS."""
    from .batch import midi_to_note
    rng = np.random.default_rng(seed)
    names, durs, slurs, pitches = [], [], [], []
    total, pitch = 0.0, float(rng.integers(55, 66))
    while total < seconds - 1e-4:
        d = min(round(float(rng.uniform(0.12, 0.7)), 4), round(seconds - total, 4))
        slur = bool(names) and names[-1] != 'rest' and rng.random() < 0.2
        if slur:
            p = pitches[-1] + float(rng.choice([-1.0, -0.25, 0.0, 0.25, 1.0]))
        elif rng.random() < 1 / 7 and names and names[-1] != 'rest':
            p = None
        else:
            pitch = float(np.clip(pitch + rng.integers(-4, 5), 48, 72))
            p = pitch + (float(rng.choice([-0.25, 0.25, 0.4])) if rng.random() < 0.25 else 0.0)
        names.append('rest' if p is None else midi_to_note(p, cents=True))
        pitches.append(p)
        durs.append(d)
        slurs.append(int(slur))
        total = round(total + d, 4)
    n = int(round(seconds * sr))
    out = np.zeros(n, dtype=np.float64)
    phase = np.zeros(6)
    t0 = 0
    acc = 0.0
    for p, d in zip(pitches, durs):
        acc += d
        t1 = min(n, int(round(acc * sr)))
        m = t1 - t0
        if p is not None and m > 0:
            tt = (np.arange(m) + t0) / sr
            f = 440.0 * 2.0 ** ((p - 69.0 + 0.3 * np.sin(2 * np.pi * 5.5 * tt)) / 12.0)
            base = np.cumsum(2 * np.pi * f / sr)
            seg = np.zeros(m)
            for k in range(1, 7):
                seg += np.sin(phase[k - 1] + k * base) / k
                phase[k - 1] = (phase[k - 1] + k * base[-1]) % (2 * np.pi)
            edge = min(int(0.010 * sr), m // 2)
            env = np.ones(m)
            if edge > 0:
                ramp = 0.5 - 0.5 * np.cos(np.pi * np.arange(edge) / edge)
                env[:edge] = ramp
                env[m - edge:] = ramp[::-1]
            out[t0:t1] = seg * env
        t0 = t1
    peak = np.abs(out).max()
    if peak > 0:
        out *= 0.5 / peak
    out += rng.standard_normal(n) * (10.0 ** (-50.0 / 20.0))
    return out.astype(np.float32), {'note_seq': names, 'note_dur': durs, 'note_slur': slurs}


def write_wav16(path, samples: np.ndarray, sr: int = SR) -> np.ndarray:
    """Writes mono 16-bit PCM; returns the samples as librosa.load reads them back (int16 / 32768)."""
    import wave
    q = np.clip(np.round(np.asarray(samples, dtype=np.float64) * 32768.0), -32768, 32767).astype('<i2')
    with wave.open(str(path), 'wb') as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(int(sr))
        f.writeframes(q.tobytes())
    return (q.astype(np.float32) / np.float32(32768.0)).astype(np.float32)


def write_labelled_dataset(directory, items, sr: int = SR) -> pathlib.Path:
    """A DiffSinger raw data directory (``transcriptions.csv``, ``wavs/{name}.wav`` as 16-bit PCM, ``wavs/{name}.ds``) from
    ``items = [(name, waveform, labels), ...]`` with labels as ``synth_labelled`` returns them (extra keys, e.g.
    ``note_glide``, are written to the .ds as well)."""
    import csv
    import json
    directory = pathlib.Path(directory)
    (directory / 'wavs').mkdir(parents=True, exist_ok=True)
    with open(directory / 'transcriptions.csv', 'w', encoding='utf8', newline='') as f:
        w = csv.writer(f)
        w.writerow(['name', 'ph_seq', 'ph_dur', 'ph_num'])
        for name, wave_, lab in items:
            secs = sum(lab['note_dur'])
            w.writerow([name, 'SP', f'{secs:.4f}', '1'])
            write_wav16(directory / 'wavs' / f'{name}.wav', wave_, sr)
            ds = {k: ' '.join(str(x) for x in v) if isinstance(v, (list, tuple)) else v for k, v in lab.items()}
            with open(directory / 'wavs' / f'{name}.ds', 'w', encoding='utf8') as g:
                json.dump(ds, g)
    return directory
