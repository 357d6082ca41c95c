"""Dataset labelling on the H100: Session.label_dataset (some_session_label_dataset) on an exported model file writes the
transcriptions.csv bytes batch.batch_infer_dataset writes with load_audio=audio.load_native on the same checkpoint, for WAV
at several rates and widths and FLAC / AIFF bytes under .wav names, whatever the frame budget and the devices; Notes.label
equals row_notes(note_timeline(...)); a corrupt file stops the command with nothing written; examples/some_label writes the
same file."""
import pathlib
import shutil
import subprocess

import numpy as np
import pytest
import torch

from some_b200 import _lib, audio, batch, export, plugin, synth
from some_b200 import session as nsess

import test_gpu_aiff as ga
import test_gpu_encoded as ge

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent
EXAMPLE = REPO / 'examples' / 'some_label'
KINDS = {'two_head': plugin.MIDIExtractionInference, 'quant_two_head': plugin.QuantizedMIDIExtractionInference}


@pytest.fixture(scope='module', params=list(KINDS))
def model(request, tmp_path_factory):
    d = tmp_path_factory.mktemp(request.param)
    config = synth.named_config(request.param)
    ckpt = synth.write_checkpoint(d, config, seed=1234)
    path = export.export(ckpt)
    ins = KINDS[request.param](config=config, model_path=ckpt, device='cuda:0')
    sess = nsess.Session(path, 0)
    yield ins, config, path, sess
    sess.close()


def ph_fields(rng, seconds):
    """ph_dur / ph_num of a few words over `seconds`, six decimals as DiffSinger writes them."""
    n_ph = int(rng.integers(4, 16))
    cuts = np.sort(rng.uniform(0, seconds, size=n_ph - 1))
    durs = np.diff(np.concatenate([[0.0], cuts, [seconds]]))
    nums, left = [], n_ph
    while left:
        k = int(min(left, rng.integers(1, 4)))
        nums.append(k)
        left -= k
    return ' '.join(f'{d:.6f}' for d in durs), ' '.join(str(k) for k in nums)


@pytest.fixture(scope='module')
def dataset(tmp_path_factory):
    """A DiffSinger raw data directory: the labelled synthetic items of synth.write_labelled_dataset, then WAV at 48 kHz and
    22.05 kHz, 24-bit stereo WAV, FLAC and AIFF bytes under .wav names, a long item of several chunks and a missing file,
    with ph_dur / ph_num fields spread over each recording."""
    d = tmp_path_factory.mktemp('ds') / 'ds'
    items = []
    for i, secs in enumerate((6.0, 9.5)):
        w, lab = synth.synth_labelled(300 + i, seconds=secs)
        items.append((f'synth{i}', w, lab))
    synth.write_labelled_dataset(d, items)
    extra = {
        'wav48k': (ge.wav_file(synth.synth_waveform(61, seconds=12.0, sr=48000, silence_gaps=True), 48000, 's16'), 12.0),
        'wav22k': (ge.wav_file(synth.synth_waveform(62, seconds=10.0, sr=22050, silence_gaps=True), 22050, 's16'), 10.0),
        'wav24_stereo': (ge.wav_file(ge.stereo(63, 11.0, 44100), 44100, 's24'), 11.0),
        'flac_as_wav': (ge.flac_file(ge.stereo(64, 9.0, 44100), 44100, 16, channel_mode='mid_side'), 9.0),
        'aiff_as_wav': (ga.aiff_s16(ga.quantise16(synth.synth_waveform(65, seconds=8.0, sr=48000)), 48000.0), 8.0),
        'long, "many chunks"': (ge.wav_file(synth.synth_waveform(66, seconds=70.0, silence_gaps=True), 44100, 's16'), 70.0),
    }
    for name, (data, _) in extra.items():
        (d / 'wavs' / f'{name}.wav').write_bytes(data)
    rng = np.random.default_rng(77)
    import csv
    with open(d / 'transcriptions.csv', 'r', encoding='utf8', newline='') as f:
        rows = list(csv.DictReader(f))
    for r in rows:
        r['ph_dur'], r['ph_num'] = ph_fields(rng, float(sum(map(float, r['ph_dur'].split()))))
    for name, (_, secs) in extra.items():
        dur, num = ph_fields(rng, secs)
        rows.append({'name': name, 'ph_seq': 'a', 'ph_dur': dur, 'ph_num': num})
    rows.insert(3, {'name': 'missing', 'ph_seq': 'SP', 'ph_dur': '0.5', 'ph_num': '1'})
    with open(d / 'transcriptions.csv', 'w', encoding='utf8', newline='') as f:
        w = csv.DictWriter(f, fieldnames=['name', 'ph_seq', 'ph_dur', 'ph_num'])
        w.writeheader()
        w.writerows(rows)
    return d


def python_csv(ins, config, dataset, out, round_midi):
    batch.batch_infer_dataset(dataset, ins, config, round_midi=round_midi, csv=out, load_audio=audio.load_native)
    return out.read_bytes()


@pytest.mark.parametrize('round_midi', [False, True])
def test_label_dataset_equals_batch_infer_dataset(model, dataset, tmp_path, capsys, round_midi):
    ins, config, _, sess = model
    want = python_csv(ins, config, dataset, tmp_path / 'py.csv', round_midi)
    py_out = capsys.readouterr().out
    rep = {}
    sess.label_dataset(dataset, tmp_path / 'c.csv', round_midi=round_midi, report=rep)
    assert capsys.readouterr().out == py_out                    # the same warning for the missing file
    got = (tmp_path / 'c.csv').read_bytes()
    assert got == want
    assert rep['missing'] == 1 and rep['labelled'] == rep['rows'] - 1 and rep['chunks'] > rep['labelled']
    # one item per group: the same bytes
    sess.label_dataset(dataset, tmp_path / 'c1.csv', round_midi=round_midi, budget=1, report=rep)
    assert (tmp_path / 'c1.csv').read_bytes() == want and rep['groups'] == rep['labelled']


def test_two_devices_same_bytes(model, dataset, tmp_path, capsys):
    if torch.cuda.device_count() < 2:
        pytest.skip('one GPU visible')
    _, _, path, sess = model
    sess.label_dataset(dataset, tmp_path / 'one.csv')
    two = nsess.Session(path, [0, 1])
    try:
        two.label_dataset(dataset, tmp_path / 'two.csv', budget=20000)
    finally:
        two.close()
    assert (tmp_path / 'two.csv').read_bytes() == (tmp_path / 'one.csv').read_bytes()


def test_notes_label_equals_row_notes(model, dataset):
    ins, config, _, sess = model
    files = sorted((dataset / 'wavs').glob('*.wav'))
    notes = [nsess.Notes() for _ in files]
    try:
        res = sess.transcribe_encoded(files, notes=notes)
        rng = np.random.default_rng(5)
        for n, (offsets, _, segments) in zip(notes, res):
            secs = max([o + float(sg['note_dur'].sum()) for o, sg in zip(offsets, segments)] + [1.0])
            ph_dur, ph_num = ph_fields(rng, secs)
            for round_midi in (False, True):
                want = batch.row_notes(ph_dur, ph_num, batch.note_timeline(offsets, segments), round_midi)
                assert n.label(ph_dur, ph_num, round_midi) == want
    finally:
        for n in notes:
            n.close()


def test_corrupt_flac_stops_the_command(model, dataset, tmp_path):
    _, _, _, sess = model
    d = tmp_path / 'ds'
    shutil.copytree(dataset, d)
    data = bytearray((d / 'wavs' / 'flac_as_wav.wav').read_bytes())
    data[len(data) // 2] ^= 0x5A
    (d / 'wavs' / 'flac_as_wav.wav').write_bytes(bytes(data))
    before = (d / 'transcriptions.csv').read_bytes()
    for budget in (None, 1):
        with pytest.raises(_lib.SomeB200Error, match=r"flac_as_wav\.wav'"):
            sess.label_dataset(d, overwrite=True, budget=budget)
        assert (d / 'transcriptions.csv').read_bytes() == before
    with pytest.raises(_lib.SomeB200Error, match='already exists'):
        sess.label_dataset(d)


def test_some_label_example_writes_the_same_file(model, dataset, tmp_path):
    ins, config, path, _ = model
    assert EXAMPLE.is_file(), 'examples/some_label was not built'
    want = python_csv(ins, config, dataset, tmp_path / 'py.csv', False)
    r = subprocess.run([str(EXAMPLE), str(path), str(dataset), '--csv', str(tmp_path / 'ex.csv')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout == f"WARNING: audio file does not exist: '{dataset / 'wavs' / 'missing.wav'}'\n"
    assert (tmp_path / 'ex.csv').read_bytes() == want
    r = subprocess.run([str(EXAMPLE), str(path), str(dataset), '--csv', str(tmp_path / 'ex.csv')], capture_output=True, text=True)
    assert r.returncode == 1 and 'Please re-try with --overwrite option.' in r.stderr
