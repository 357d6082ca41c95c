"""Export a checkpoint to one self-contained model file for hosts without Python (the counterpart of the reference's
``export.py`` + ``deployment/``, which write an ONNX graph).

    python -m some_b200.export --model CKPT [--out PATH] [--precision bf16|fp32]

reads ``config.yaml`` beside the checkpoint (export.py:53-55), builds the engine exactly as a default
``MIDIExtractionInference`` does (default launch sequence, load-time bias correction ``Engine.calibrate``: that step needs a
CUDA device) and writes the tensors that engine runs with: the device tensors ``build_c_model(w, ln_fold=False)`` points to,
biases corrected, plus the mel tables and resampy's float64 ``kaiser_best`` table.  ``--precision fp32`` writes the fp32
model instead (``weights.model_tensors_f32``: the checkpoint's own tensors, unrounded, as ``build_f32_model`` uploads them)
and records the precision in the header; a session that opens it runs ``some_forward_f32_tiled``, the notes of
``Engine.infer(..., precision='fp32')``.  ``some_session_open`` (csrc/session.cu)
is the only reader; the format is documented in INTEGRATION.md ("Deploying without Python").

The file is a pure function of the checkpoint: exporting the same checkpoint twice gives identical bytes.
"""
from __future__ import annotations

import argparse
import pathlib
import struct
from typing import Dict, List, Sequence, Tuple

import numpy as np

MAGIC = b'SOMEB200'
FORMAT_VERSION = 1
ABI_VERSION = 202
SUFFIX = '.somemodel'
HEADER = struct.Struct('<8sIIQQIiiiiiiffffiQi36x')     # 128 bytes; the int32 at byte 88 is the precision (0 in bf16 files)
PRECISIONS = {'bf16': 0, 'fp32': 1}                     # SOME_PRECISION_BF16 / SOME_PRECISION_FP32
ENTRY = struct.Struct('<64sII4QQQ8x')                   # 128 bytes
ALIGN = 256
DTYPES = {np.dtype('<f4'): 1, np.dtype('<u2'): 2, np.dtype('<i4'): 3, np.dtype('<f8'): 4}   # u2 = raw bfloat16
KAISER_TAPS = 32769
DIM, FFN, N_MELS, CONV_K, MEL_MAXW, MEL_TW, N_FFT, HOP = 512, 2048, 80, 31, 24, 1396, 2048, 512
# the tables of the front end, after the model's tensors (weights.model_tensors)
FRONT_END = [('mel_start', np.dtype('<i4'), (N_MELS,)), ('mel_count', np.dtype('<i4'), (N_MELS,)),
             ('mel_weights', np.dtype('<f4'), (N_MELS, MEL_MAXW)), ('twiddle', np.dtype('<f4'), (MEL_TW, 2)),
             ('window', np.dtype('<f4'), (N_FFT,)), ('kaiser_best', np.dtype('<f8'), (KAISER_TAPS,))]


def tensor_specs(lay: int, outdim: int, precision: str = 'bf16') -> List[Tuple[str, np.dtype, Tuple[int, ...]]]:
    """The tensors of a model file, in file order: (name, dtype, shape).  ``some_session_open`` expects exactly these."""
    from .weights import model_tensors, model_tensors_f32
    dims = {'outdim': outdim, 'outdim32': (outdim + 31) // 32 * 32}
    table = model_tensors_f32(lay) if precision == 'fp32' else model_tensors(lay)
    return [(t.key, t.dtype, tuple(dims.get(d, d) for d in t.shape)) for t in table] + FRONT_END


def write_model_file(path, scalars: dict, tensors: Dict[str, np.ndarray]) -> List[dict]:
    """Writes a model file (the only writer of the format).  ``scalars``: lay, outdim, quantized, audio_sample_rate,
    hop_size, win_size (512 / 2048: the mel kernel's), midi_min, midi_max, midi_prob_deviation, rest_threshold,
    bias_corrected, and optionally precision ('bf16', the default, or 'fp32').  ``tensors``: name -> array with the dtype and
    shape ``tensor_specs`` gives (bf16 as its raw uint16 bits).  Returns the directory as written: one dict per tensor with
    name, dtype code, shape, offset, nbytes and the byte offset of its directory entry."""
    if int(scalars['hop_size']) != HOP or int(scalars['win_size']) != N_FFT:
        raise ValueError(f"hop_size / win_size {scalars['hop_size']} / {scalars['win_size']}: the model file describes "
                         f'models of hop {HOP} and window {N_FFT} only')
    precision = scalars.get('precision', 'bf16')
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be 'bf16' or 'fp32', got {precision!r}")
    specs = tensor_specs(int(scalars['lay']), int(scalars['outdim']), precision)
    names = [n for n, _, _ in specs]
    if sorted(names) != sorted(tensors):
        raise ValueError(f'tensor set differs from the format: missing {sorted(set(names) - set(tensors))}, '
                         f'unexpected {sorted(set(tensors) - set(names))}')
    dir_off = HEADER.size
    data_off = (dir_off + ENTRY.size * len(specs) + ALIGN - 1) // ALIGN * ALIGN
    entries, off = [], data_off
    for i, (name, dt, shape) in enumerate(specs):
        a = tensors[name]
        if a.dtype != dt or tuple(a.shape) != shape:
            raise ValueError(f'{name}: {a.dtype} {tuple(a.shape)}, the format needs {dt} {shape}')
        entries.append({'name': name, 'dtype': DTYPES[dt], 'shape': shape, 'offset': off, 'nbytes': int(a.nbytes),
                        'entry_offset': dir_off + i * ENTRY.size})
        off = (off + a.nbytes + ALIGN - 1) // ALIGN * ALIGN
    file_size = off
    header = HEADER.pack(MAGIC, FORMAT_VERSION, ABI_VERSION, file_size, dir_off, len(specs), int(scalars['lay']),
                         int(scalars['outdim']), int(bool(scalars['quantized'])), int(scalars['audio_sample_rate']),
                         int(scalars['hop_size']), int(scalars['win_size']),
                         float(scalars['midi_min']), float(scalars['midi_max']), float(scalars['midi_prob_deviation']),
                         float(scalars['rest_threshold']), int(bool(scalars['bias_corrected'])), data_off,
                         PRECISIONS[precision])
    with open(path, 'wb') as f:
        f.write(header)
        for e in entries:
            shape4 = list(e['shape']) + [0] * (4 - len(e['shape']))
            f.write(ENTRY.pack(e['name'].encode('ascii'), e['dtype'], len(e['shape']), *shape4, e['offset'], e['nbytes']))
        for e in entries:
            f.write(b'\0' * (e['offset'] - f.tell()))
            f.write(np.ascontiguousarray(tensors[e['name']]).tobytes())
        f.write(b'\0' * (file_size - f.tell()))
    return entries


def engine_tensors(engine, precision: str = 'bf16') -> Dict[str, np.ndarray]:
    """The tensors of a built (and calibrated) engine, under the format's names, as host arrays: the device tensors of its
    bf16 model, or (``precision='fp32'``) the fp32 tensors of its checkpoint that Engine.model_f32 uploads."""
    import torch

    from .audio import kaiser_best_table
    from .weights import checkpoint_f32, model_tensors, model_tensors_f32, packed_tensor

    def host(t, f32=False):
        if isinstance(t, float):                    # b_cut, a host scalar of the engine
            return np.array([t], dtype='<f4')
        t = t.detach().contiguous().cpu()
        if f32:                                     # a checkpoint tensor of the fp32 model, as build_f32_model uploads it
            return t.to(torch.float32).numpy()
        return t.view(torch.uint16).numpy() if t.dtype == torch.bfloat16 else t.numpy()

    w = engine.w
    if precision == 'fp32':
        ck = checkpoint_f32(engine._state_dict, engine.config)
        out = {t.key: host(packed_tensor(ck, t), True) for t in model_tensors_f32(w.lay)}
    else:
        out = {t.key: host(packed_tensor(w, t)) for t in model_tensors(w.lay)}
    for k in ('mel_start', 'mel_count', 'mel_weights', 'twiddle', 'window'):
        out[k] = host(engine.mel[k])
    out['kaiser_best'] = np.asarray(kaiser_best_table(), dtype='<f8')
    return out


def export(model_path, out_path=None, device='cuda', precision: str = 'bf16') -> pathlib.Path:
    """Builds the default plugin for ``model_path`` (config.yaml beside it) on ``device`` and writes its model file to
    ``out_path`` (default: the checkpoint path with the suffix ``.somemodel``), of the bf16 model or the fp32 one."""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be 'bf16' or 'fp32', got {precision!r}")
    import yaml

    from .plugin import MIDIExtractionInference, QuantizedMIDIExtractionInference, task_inference_mapping
    model_path = pathlib.Path(model_path)
    with open(model_path.with_name('config.yaml'), 'r', encoding='utf8') as f:
        config = yaml.safe_load(f)
    cls_name = task_inference_mapping[config['task_cls']].rsplit('.', 1)[-1]
    cls = {'MIDIExtractionInference': MIDIExtractionInference,
           'QuantizedMIDIExtractionInference': QuantizedMIDIExtractionInference}[cls_name]
    ins = cls(config=config, model_path=model_path, device=device)
    eng = ins.model
    # calibrate() records every GEMM weight it has seen (and corrected the bias of): empty if it did not run
    corrected = bool(getattr(eng, '_corrected', None))
    scalars = {'lay': eng.w.lay, 'outdim': eng.outdim, 'quantized': cls.quantized,
               'audio_sample_rate': config['audio_sample_rate'], 'hop_size': config.get('hop_size', HOP),
               'win_size': config.get('win_size', N_FFT), 'midi_min': ins.midi_min, 'midi_max': ins.midi_max,
               'midi_prob_deviation': ins.midi_deviation, 'rest_threshold': ins.rest_threshold,
               'bias_corrected': corrected and precision == 'bf16', 'precision': precision}
    out_path = pathlib.Path(out_path) if out_path is not None else model_path.with_suffix(SUFFIX)
    write_model_file(out_path, scalars, engine_tensors(eng, precision))
    return out_path


def main(argv: Sequence[str] = None):
    ap = argparse.ArgumentParser(prog='python -m some_b200.export',
                                 description='Export a checkpoint to a self-contained model file for some_session_open')
    ap.add_argument('--model', required=True, metavar='CKPT_PATH', help='Path to the model checkpoint (*.ckpt)')
    ap.add_argument('--out', required=False, metavar='PATH', help=f'Path to the output model (default: CKPT{SUFFIX})')
    ap.add_argument('--precision', choices=sorted(PRECISIONS), default='bf16',
                    help='bf16: the product model (default); fp32: the unrounded fp32 model, run by some_forward_f32_tiled')
    args = ap.parse_args(argv)
    print(f'| exported \'{export(args.model, args.out, precision=args.precision)}\'')


if __name__ == '__main__':
    main()
