"""CPU tests of the evaluator's host part (some_b200/evaluate.py) and of the oracle's losses (oracle/evaluate.py) against
tests/golden/eval_*.{json,npz}, which the unmodified reference produced (tests/golden/make_golden_eval.py): the label
pipeline (glide skipping, note-name normalisation, slur and rest merging, unit2note), the note-name functions, and the
refusals."""
import json

import numpy as np
import pytest

from oracle import evaluate as oev
from some_b200 import batch, evaluate, synth

TIMESTEP = 512 / 44100


@pytest.fixture(scope='module')
def golden_labels(golden_dir):
    return json.loads((golden_dir / 'eval_labels.json').read_text(encoding='utf8'))


def _write_ds(tmp_path, items):
    (tmp_path / 'wavs').mkdir(parents=True, exist_ok=True)
    with open(tmp_path / 'transcriptions.csv', 'w', encoding='utf8') as f:
        f.write('name,ph_seq,ph_dur,ph_num\n')
        for name, ds in items.items():
            f.write(f'{name},SP,1,1\n')
            (tmp_path / 'wavs' / f'{name}.ds').write_text(json.dumps(ds), encoding='utf8')
    return tmp_path


@pytest.mark.parametrize('task', ['continuous', 'quantized'])
def test_labels_equal_reference(task, golden_labels, tmp_path):
    data = _write_ds(tmp_path, golden_labels['items'])
    config = {'binarization_args': golden_labels['binarization_args'][task]}
    items = evaluate.load_labels(data, config, quantized=task == 'quantized')
    want = golden_labels[task]
    assert [it['name'] for it in items] == list(want)            # the glide item is skipped, glide 'none none' is kept
    for it in items:
        ref = want[it['name']]
        assert it['note_seq'] == ref['note_seq']
        assert it['note_dur'] == ref['note_dur_sec']              # exact: same float additions
        name = it['name'].split(':', 1)[1]
        arr = evaluate.item_labels(it, golden_labels['frames'][name], TIMESTEP, quantized=task == 'quantized')
        for k in ('unit2note', 'note_dur', 'note_rest'):
            np.testing.assert_array_equal(arr[k], np.asarray(ref[k]), err_msg=f'{it["name"]} {k}')
        np.testing.assert_array_equal(arr['note_midi'], np.asarray(ref['note_midi'], dtype=arr['note_midi'].dtype))
        assert arr['note_midi'].dtype == (np.int64 if task == 'quantized' else np.float32)
        assert (arr['unit2note'] > 0).all()


def test_slur_tolerance_and_rest_runs(golden_labels):
    cont = golden_labels['continuous']
    # C4 -> C#4 is a semitone (beyond the 0.5 tolerance): a new note; C#4+30 merges into C#4, duration-weighted
    assert cont['0:slurs']['note_seq'][:3] == ['C4+0', 'C#4+18', 'A3+0']
    assert cont['0:slurs']['note_seq'].count('rest') == 1        # two rests merged
    # without a tolerance (the quantized task's config) only equal pitches merge
    assert golden_labels['quantized']['0:slurs']['note_seq'][:3] == ['C4+0', 'C#4+0', 'A3+0']
    # zero-length notes survive the label pipeline; their indices never appear in unit2note
    z = cont['0:zero_len']
    assert 0.0 in z['note_dur_sec']
    assert len(set(z['unit2note'])) < len(z['note_seq'])


@pytest.mark.parametrize('cfg', ['two_head', 'quant_two_head'])
def test_audio_item_labels_and_oracle_losses(cfg, golden_dir, tmp_path):
    g = np.load(golden_dir / f'eval_{cfg}.npz')
    quantized = cfg.startswith('quant')
    config = synth.named_config(cfg)
    items = []
    for seed, secs in zip(g['seeds'], g['seconds']):
        w, lab = synth.synth_labelled(int(seed), float(secs))
        items.append((f'item{seed}', w, lab))
    data = synth.write_labelled_dataset(tmp_path, items)
    labels = evaluate.load_labels(data, config, quantized)
    for i, it in enumerate(labels):
        p = f'item{i}_'
        assert it['name'] == str(g[p + 'name'])
        wave = synth.write_wav16(tmp_path / 'x.wav', items[i][1])
        assert float(wave.astype(np.float64).sum()) == float(g[p + 'wave_sum'])
        t = g[p + 'unit2note'].shape[0]
        assert t == 1 + len(wave) // 512
        arr = evaluate.item_labels(it, t, TIMESTEP, quantized)
        for k in ('unit2note', 'note_midi', 'note_rest', 'note_dur'):
            np.testing.assert_array_equal(arr[k], g[p + k], err_msg=k)
        for pre in ('', 'lean_'):
            got = oev.losses(g[p + pre + 'logits'], g[p + pre + 'bounds'], arr, config, quantized)
            np.testing.assert_allclose(got['midi_loss'], g[p + pre + 'midi_loss'], rtol=1e-5)
            np.testing.assert_allclose(got['bound_loss'], g[p + pre + 'bound_loss'], rtol=1e-5)
            correct, total = oev.accuracy_counts(g[p + pre + 'logits'], arr, config, quantized)
            assert (correct, total) == (int(g[p + pre + 'correct']), int(g[p + 'total']))


@pytest.mark.parametrize('name,midi', [('C4', 60), ('C#4', 61), ('Db4', 61), ('A4+25', 69.25), ('B3-5', 58.95), ('C-1', 0),
                                       ('G9', 127), ('E#2', 41), ('Cb4', 59), ('c4', 60), ('F##3', 55)])
def test_note_names(name, midi):
    assert batch.note_to_midi(name, round_midi=False) == pytest.approx(midi, abs=1e-12)
    assert batch.note_to_midi(name) == int(np.round(midi))


@pytest.mark.parametrize('midi', [60.0, 61.25, 58.95, 69.5, 70.49, 0.0, 127.0, 64.333])
def test_note_name_round_trip_with_cents(midi):
    name = batch.midi_to_note(midi, cents=True)
    back = batch.note_to_midi(name, round_midi=False)
    assert abs(back - midi) <= 0.005 + 1e-9
    assert batch.midi_to_note(back, cents=True) == name
    assert batch.midi_to_note(midi) == batch.midi_to_note(midi, cents=False)


def test_cents_format():
    assert batch.midi_to_note(60.0, cents=True) == 'C4+0'
    assert batch.midi_to_note(61.25, cents=True) == 'C#4+25'
    assert batch.midi_to_note(58.95, cents=True) == 'B3-5'


@pytest.mark.parametrize('ds,match', [
    ({'note_seq': 'C4 D4', 'note_dur': '0.3', 'note_slur': '0 0'}, "mismatch in 'bad'"),
    ({'note_seq': 'rest rest', 'note_dur': '0.3 0.2', 'note_slur': '0 0'}, "All notes are rest in 'bad'"),
    ({'note_seq': 'H4 D4', 'note_dur': '0.3 0.2', 'note_slur': '0 0'}, 'Improper note format'),
])
def test_refusals(ds, match, tmp_path):
    data = _write_ds(tmp_path, {'bad': ds})
    with pytest.raises(ValueError, match=match):
        evaluate.load_labels(data, {}, quantized=False)


def test_refuses_missing_csv_and_empty_durations(tmp_path):
    with pytest.raises(FileNotFoundError):
        evaluate.load_labels(tmp_path, {}, False)
    item = {'name': '0:x', 'note_seq': ['C4'], 'note_dur': [0.0]}
    with pytest.raises(ValueError, match='last no frame'):
        evaluate.item_labels(item, 10, TIMESTEP)
    with pytest.raises(ValueError, match='Negative'):
        evaluate.item_labels({'name': '0:y', 'note_seq': ['C4', 'D4'], 'note_dur': [0.3, -0.1]}, 10, TIMESTEP)


def test_summary_aggregation():
    mk = lambda ml, bl, c, t: evaluate.EvalItem('x', t, ml, bl, c, t, np.zeros(0), np.zeros(0), np.zeros(0, bool))
    items = [mk(1.0, 2.0, 3, 10), mk(3.0, 4.0, 5, 30)]
    s = evaluate.summarize(items, {})
    assert s == {'midi_loss': 2.0, 'bound_loss': 3.0, 'total_loss': 5.0, 'midi_acc': 8 / 40}
    s = evaluate.summarize(items, {'use_bound_loss': False})
    assert s == {'midi_loss': 2.0, 'total_loss': 2.0, 'midi_acc': 8 / 40}
