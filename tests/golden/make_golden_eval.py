"""Generates tests/golden/eval_labels.json and tests/golden/eval_{two_head,quant_two_head}.npz by EXECUTING THE UNMODIFIED
REFERENCE (/root/reference) on CPU through oracle/refshim.py.  Runs only in the build container (the reference is not on
the GPU box); the outputs are committed.

    python tests/golden/make_golden_eval.py

Reference code run: MIDIExtractionBinarizer.load_meta_data (with merge_slurs / merge_rests), get_mel2ph_torch +
LengthRegulator, the model forward (midi_conforms, seeded weights), the collaters of MIDIExtractionDataset /
QuantizedMIDIExtractionDataset, BCEWithLogitsLoss / CrossEntropyLoss, BinaryEMDLoss and decode_gaussian_blurred_probs.
librosa is absent: the shim's stub gets some_b200.batch's restated note_to_midi / midi_to_note.  torchmetrics is absent:
MIDIAccuracy.update's two counters are written out below, as me_task.py / me_quant_task.py feed them.

eval_labels.json: hand-written .ds items (slurs within and beyond the tolerance, runs of rests, glides, zero-length notes,
a list-form .ds) with the reference's load_meta_data output and unit2note, for both tasks.
eval_{cfg}.npz: labelled synthetic items (synth.synth_labelled(seed, seconds) written as 16-bit WAV): per item the label
arrays, the raw logits and bounds of the reference forward, the four numbers and the accuracy counts.
"""
import json
import pathlib
import sys
import tempfile

import numpy as np
import torch

HERE = pathlib.Path(__file__).resolve().parent
REPO = HERE.parent.parent
sys.path.insert(0, str(REPO))

from oracle import refshim  # noqa: E402
from some_b200 import batch, synth  # noqa: E402

LABEL_ITEMS = {
    'plain': {'note_seq': 'C4 D4 rest E4', 'note_dur': '0.3 0.25 0.2 0.4', 'note_slur': '0 0 0 0'},
    'slurs': {'note_seq': 'C4 C#4 C#4+30 A3 A3 rest rest G4 G#4+45 B4',
              'note_dur': '0.2 0.1 0.15 0.3 0.2 0.1 0.15 0.2 0.22 0.3', 'note_slur': '0 1 1 0 1 0 0 0 1 1'},
    'cents': {'note_seq': 'A4+25 Bb3-10 F#5 rest rest rest C2 B8 c4', 'note_dur': '0.1 0.2 0.3 0.05 0.05 0.1 0.2 0.2 0.1',
              'note_slur': '0 0 1 0 0 0 0 1 0'},
    'zero_len': {'note_seq': 'rest E4 F4 G4 rest A4', 'note_dur': '0.0 0.0052 0.0 0.4 0.001 0.3',
                 'note_slur': '0 0 0 0 0 0'},
    'glide': {'note_seq': 'C4 D4', 'note_dur': '0.3 0.3', 'note_slur': '0 0', 'note_glide': 'none up'},
    'glide_none': {'note_seq': 'C4 D4', 'note_dur': '0.3 0.3', 'note_slur': '0 0', 'note_glide': 'none none'},
    'as_list': [{'note_seq': 'G3 G3 rest', 'note_dur': '0.5 0.25 0.5', 'note_slur': '0 1 0'}],
}
FRAMES = {'plain': 120, 'slurs': 160, 'cents': 90, 'zero_len': 50, 'glide_none': 40, 'as_list': 150}
BIN_ARGS = {'continuous': dict(skip_glide=True, merge_rest=True, merge_slur=True, round_midi=False, slur_tolerance=0.5),
            'quantized': dict(skip_glide=True, merge_rest=True, merge_slur=True)}
AUDIO_ITEMS = ((311, 1.6), (312, 2.3))


def _install_note_functions():
    lib = sys.modules['librosa']
    lib.note_to_midi = lambda n, round_midi=True: batch.note_to_midi(n, round_midi=round_midi)
    lib.midi_to_note = lambda m, cents=False, unicode=True: batch.midi_to_note(m, cents=cents)


def _stub_attr(attr):
    if attr.startswith('__'):
        raise AttributeError(attr)
    return refshim._Anything


def _write_label_dataset(d: pathlib.Path):
    (d / 'wavs').mkdir(parents=True)
    with open(d / 'transcriptions.csv', 'w', encoding='utf8') as f:
        f.write('name,ph_seq,ph_dur,ph_num\n')
        for name, ds in LABEL_ITEMS.items():
            f.write(f'{name},SP,1,1\n')
            (d / 'wavs' / f'{name}.ds').write_text(json.dumps(ds), encoding='utf8')


def _binarizer(cls, args, round_midi):
    b = cls.__new__(cls)
    b.items = {}
    b.skip_glide, b.merge_rest, b.merge_slur = args['skip_glide'], args['merge_rest'], args['merge_slur']
    b.slur_tolerance = args.get('slur_tolerance')
    b.round_midi = round_midi
    return b


def _label_arrays(meta, length, timestep, int_midi, get_mel2ph_torch, lr, note_to_midi):
    """The label half of MIDIExtractionBinarizer._process_item (me_binarizer.py:201-223), line for line."""
    from scipy import interpolate
    note_midi = np.array([(note_to_midi(n, round_midi=int_midi) if n != 'rest' else -1) for n in meta['note_seq']],
                         dtype=np.int64 if int_midi else np.float32)
    note_rest = note_midi < 0
    interp_func = interpolate.interp1d(np.where(~note_rest)[0], note_midi[~note_rest], kind='nearest',
                                       fill_value='extrapolate')
    note_midi[note_rest] = interp_func(np.where(note_rest)[0])
    note_dur_sec = torch.FloatTensor(meta['note_dur'])
    note_acc = torch.round(torch.cumsum(note_dur_sec, dim=0) / timestep + 0.5).long()
    note_dur = torch.diff(note_acc, dim=0, prepend=torch.LongTensor([0]))
    unit2note = get_mel2ph_torch(lr, note_dur_sec, length, timestep)
    if int_midi:
        note_midi[note_rest] = 128                                                       # me_quant_binarizer.py:28
    return {'note_midi': note_midi, 'note_rest': note_rest, 'note_dur': note_dur.numpy(), 'unit2note': unit2note.numpy()}


def main():
    torch.set_num_threads(1)
    ref_inference = refshim.load_reference()
    _install_note_functions()
    for name in ('h5py', 'fairseq', 'fairseq.checkpoint_utils', 'matplotlib', 'matplotlib.pyplot', 'matplotlib.ticker',
                 'torchmetrics'):
        if name not in sys.modules:
            try:
                __import__(name)
            except ImportError:
                refshim._mod(name, __getattr__=_stub_attr)   # names only: never called here
    import modules.losses as ref_losses
    from modules.commons import LengthRegulator
    from preprocessing.me_binarizer import MIDIExtractionBinarizer
    from preprocessing.me_quant_binarizer import QuantizedMIDIExtractionBinarizer
    from training.me_quant_task import QuantizedMIDIExtractionDataset
    from training.me_task import MIDIExtractionDataset
    from utils.binarizer_utils import get_mel2ph_torch
    from utils.infer_utils import decode_gaussian_blurred_probs
    note_to_midi = sys.modules['librosa'].note_to_midi
    lr = LengthRegulator()
    timestep = 512 / 44100

    # ---------------------------------------------------------------- labels of hand-written items
    labels_out = {'items': LABEL_ITEMS, 'frames': FRAMES, 'binarization_args': BIN_ARGS}
    with tempfile.TemporaryDirectory() as d:
        d = pathlib.Path(d)
        _write_label_dataset(d)
        for task, cls in (('continuous', MIDIExtractionBinarizer), ('quantized', QuantizedMIDIExtractionBinarizer)):
            args = BIN_ARGS[task]
            b = _binarizer(cls, args, round_midi=True if task == 'quantized' else args['round_midi'])
            b.load_meta_data(d, 0)
            res = {}
            for key, meta in b.items.items():
                name = key.split(':', 1)[1]
                arr = _label_arrays(meta, FRAMES[name], timestep, task == 'quantized', get_mel2ph_torch, lr, note_to_midi)
                res[key] = {'note_seq': meta['note_seq'], 'note_dur_sec': meta['note_dur'],
                            **{k: v.tolist() for k, v in arr.items()}}
            labels_out[task] = res
    (HERE / 'eval_labels.json').write_text(json.dumps(labels_out, indent=1), encoding='utf8')
    print('eval_labels.json written', {t: list(labels_out[t]) for t in ('continuous', 'quantized')})

    # ---------------------------------------------------------------- labelled synthetic items through the model
    for cfg_name in ('two_head', 'quant_two_head'):
        quantized = cfg_name.startswith('quant')
        config = synth.named_config(cfg_name)
        with tempfile.TemporaryDirectory() as d:
            d = pathlib.Path(d)
            ckpt = synth.write_checkpoint(d / 'ckpt', config, seed=1234)
            cls = ref_inference.QuantizedMIDIExtractionInference if quantized else ref_inference.MIDIExtractionInference
            ins = cls(config=synth.named_config(cfg_name), model_path=ckpt, device='cpu')
            items = []
            for seed, secs in AUDIO_ITEMS:
                w, lab = synth.synth_labelled(seed, secs)
                items.append((f'item{seed}', w, lab))
            synth.write_labelled_dataset(d / 'data', items)
            task = 'quantized' if quantized else 'continuous'
            b = _binarizer(QuantizedMIDIExtractionBinarizer if quantized else MIDIExtractionBinarizer, BIN_ARGS[task],
                           round_midi=quantized or BIN_ARGS[task]['round_midi'])
            b.load_meta_data(d / 'data', 0)
            if quantized:
                ds = QuantizedMIDIExtractionDataset.__new__(QuantizedMIDIExtractionDataset)
            else:
                ds = MIDIExtractionDataset.__new__(MIDIExtractionDataset)
                ds.midi_min, ds.midi_max, ds.num_bins = config['midi_min'], config['midi_max'], config['midi_num_bins']
                ds.midi_deviation = config['midi_prob_deviation']
                ds.interval = (ds.midi_max - ds.midi_min) / (ds.num_bins - 1)
                ds.sigma = ds.midi_deviation / ds.interval
            out = {'seeds': np.array([s for s, _ in AUDIO_ITEMS]), 'seconds': np.array([t for _, t in AUDIO_ITEMS])}
            for i, (key, meta) in enumerate(b.items.items()):
                wave_ = (np.frombuffer((d / 'data' / 'wavs' / f'item{AUDIO_ITEMS[i][0]}.wav').read_bytes()[44:], '<i2')
                         .astype(np.float32) / 32768.0)
                sample = ins.preprocess(wave_)
                units = sample['units']
                length = units.shape[1]
                arr = _label_arrays(meta, length, timestep, quantized, get_mel2ph_torch, lr, note_to_midi)
                u = torch.from_numpy(arr['unit2note'])
                mask = (u > 0)[None]
                with torch.no_grad():
                    logits, bounds = ins.model(x=units, f0=sample['pitch'], mask=mask)
                s = {'units': units[0], 'pitch': sample['pitch'][0], 'note_midi': torch.from_numpy(arr['note_midi']),
                     'note_dur': torch.from_numpy(arr['note_dur']), 'unit2note': u}
                if not quantized:
                    s['note_rest'] = torch.from_numpy(arr['note_rest'])
                bt = ds.collater([s])
                def score(logits, bounds):
                    bound_loss = ref_losses.BinaryEMDLoss()(bounds, bt['bounds'])
                    if quantized:
                        midi_loss = torch.nn.CrossEntropyLoss(ignore_index=-1)(logits.transpose(1, 2), bt['midi_idx'])
                        probs = torch.softmax(logits, dim=2)
                        midi_pred = probs.argmax(dim=-1)
                        rest_pred = midi_pred == 128
                        midi_pred = midi_pred.float()
                        note_midi_gt = bt['note_midi'].float()
                        note_midi_gt[bt['note_midi'] == 128] = -torch.inf
                    else:
                        midi_loss = torch.nn.BCEWithLogitsLoss()(logits, bt['probs'])
                        midi_pred, rest_pred = decode_gaussian_blurred_probs(
                            torch.sigmoid(logits), vmin=config['midi_min'], vmax=config['midi_max'],
                            deviation=config['midi_prob_deviation'], threshold=config['rest_threshold'])
                        note_midi_gt = bt['note_midi'].clone()
                        note_midi_gt[bt['note_rest']] = -torch.inf
                    midi_pred[rest_pred] = -torch.inf
                    midi_gt = torch.gather(torch.nn.functional.pad(note_midi_gt, [1, 0], value=-torch.inf), 1, bt['unit2note'])
                    rest_gt = midi_gt < 0
                    masks = bt['unit2note'] > 0
                    overall = ~rest_pred & ~rest_gt & (torch.abs(midi_pred - midi_gt) <= 0.5) & (rest_pred == rest_gt) & masks
                    return midi_loss, bound_loss, overall, masks
                midi_loss, bound_loss, overall, masks = score(logits, bounds)
                # a confident model: logits that lean towards the labels, plus noise, so that the accuracy counts are not 0
                g = torch.Generator().manual_seed(1000 + i)
                noise = torch.randn(logits.shape, generator=g)
                if quantized:
                    lean = 6.0 * torch.nn.functional.one_hot(bt['midi_idx'], 129).float() + 2.0 * noise
                else:
                    lean = 10.0 * bt['probs'] - 6.0 + 1.5 * noise
                lean_bounds = (bt['bounds'] * 0.8 + 0.1 * torch.rand(bounds.shape, generator=g)).float()
                lean_scores = score(lean, lean_bounds)
                p = f'item{i}_'
                out[p + 'name'] = np.array(key)
                out[p + 'num_samples'] = np.int64(len(wave_))
                out[p + 'wave_sum'] = np.float64(wave_.astype(np.float64).sum())
                for k, v in arr.items():
                    out[p + k] = v
                out[p + 'logits'] = logits[0].numpy()
                out[p + 'bounds'] = bounds[0].numpy()
                out[p + 'midi_loss'] = np.float64(midi_loss.item())
                out[p + 'bound_loss'] = np.float64(bound_loss.item())
                out[p + 'correct'] = np.int64(overall.sum().item())
                out[p + 'total'] = np.int64(masks.sum().item())
                out[p + 'lean_logits'] = lean[0].numpy()
                out[p + 'lean_bounds'] = lean_bounds[0].numpy()
                out[p + 'lean_midi_loss'] = np.float64(lean_scores[0].item())
                out[p + 'lean_bound_loss'] = np.float64(lean_scores[1].item())
                out[p + 'lean_correct'] = np.int64(lean_scores[2].sum().item())
                print(cfg_name, key, length, float(midi_loss), float(bound_loss), int(overall.sum()), int(masks.sum()),
                      [float(x.sum()) for x in lean_scores])
        np.savez_compressed(HERE / f'eval_{cfg_name}.npz', **out)
        print(f'eval_{cfg_name}.npz written')


if __name__ == '__main__':
    main()
