"""The native session on the H100 (csrc/session.cu): a checkpoint exported with ``python -m some_b200.export`` and run through
some_session_transcribe / some_session_transcribe_sliced gives BIT-identical notes to the Python plugin, for both model
kinds, and the C example transcribes a WAV file with no Python in the process."""
import pathlib
import subprocess
import threading

import numpy as np
import pytest

from some_b200 import audio, batch, export, plugin, synth
from some_b200 import session as nsess
from some_b200.slicer import Slicer

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent
EXAMPLE = REPO / 'examples' / 'some_transcribe'
KINDS = {'two_head': plugin.MIDIExtractionInference, 'quant_two_head': plugin.QuantizedMIDIExtractionInference}


@pytest.fixture(scope='module', params=list(KINDS))
def model(request, tmp_path_factory):
    """(kind, default plugin, exported model file, the bytes of a second export, open session)."""
    d = tmp_path_factory.mktemp(request.param)
    config = synth.named_config(request.param)
    ckpt = synth.write_checkpoint(d, config, seed=1234)
    path = export.export(ckpt)
    assert path == ckpt.with_suffix('.somemodel')
    second = export.export(ckpt, d / 'again.somemodel').read_bytes()
    ins = KINDS[request.param](config=config, model_path=ckpt, device='cuda:0')
    sess = nsess.Session(path, 0)
    yield request.param, ins, path, second, sess
    sess.close()


def assert_same_notes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g['note_midi'].shape == w['note_midi'].shape
        np.testing.assert_array_equal(g['note_midi'].view(np.uint32), w['note_midi'].view(np.uint32))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        assert g['note_dur'].dtype == np.float64
        np.testing.assert_array_equal(g['note_dur'].view(np.uint64), w['note_dur'].view(np.uint64))


def clips_30s(count):
    pool = [synth.synth_waveform(1000 + j, seconds=30.0) for j in range(4)]
    return [np.ascontiguousarray(np.roll(pool[i % 4], 4099 * (i // 4)) * np.float32(1.0 - 0.01 * (i % 7))) for i in range(count)]


def test_export_is_reproducible_and_describes_the_model(model):
    kind, ins, path, second, sess = model
    assert path.read_bytes() == second
    assert sess.sample_rate == 44100 and sess.hop == 512 and sess.timestep == ins.timestep
    assert sess.outdim == ins.model.outdim and sess.quantized == ins.quantized and sess.bias_corrected


def test_transcribe_equals_plugin(model):
    kind, ins, path, _, sess = model
    clips = [synth.synth_waveform(300 + i, seconds=s) for i, s in enumerate((0.4, 3.0, 7.3, 12.0, 1.1))]
    clips += list(synth.edge_case_waveforms().values())
    assert_same_notes(sess.transcribe(clips), ins.infer(clips))
    big = clips_30s(16) + clips                               # > 32 k frames: three pipeline chunks
    got = sess.transcribe(big)
    assert_same_notes(got, ins.infer(big))
    assert_same_notes(got[-len(clips):], sess.transcribe(clips))      # independent of the batch it came in
    assert sess.transcribe([]) == []


def test_sliced_equals_infer_sliced(model):
    kind, ins, path, _, sess = model
    wave = synth.synth_waveform(9002, seconds=300.0, silence_gaps=True)
    slicer = Slicer(44100, max_sil_kept=1000)
    offsets, ranges, got = sess.transcribe_sliced(wave)
    want_off, want = ins.model.infer_sliced(wave, slicer, quantized=ins.quantized)
    assert len(got) > 10
    assert offsets == list(want_off)
    assert ranges == slicer.ranges(wave)
    assert_same_notes(got, want)
    short = synth.synth_waveform(77, seconds=3.0)             # no longer than min_length: one chunk
    offsets, ranges, got = sess.transcribe_sliced(short)
    assert ranges == [(0, len(short))]
    assert_same_notes(got, ins.infer([short]))
    empty = np.zeros(0, np.float32)                           # one chunk of no samples
    offsets, ranges, got = sess.transcribe_sliced(empty)
    want_off, want = ins.model.infer_sliced(empty, slicer, quantized=ins.quantized)
    assert offsets == list(want_off) and ranges == [(0, 0)]
    assert_same_notes(got, want)


@pytest.mark.parametrize('rate', [48000, 22050])
def test_sliced_resamples_like_librosa_load(model, rate):
    kind, ins, path, _, sess = model
    wave = synth.synth_waveform(9002, seconds=300.0, sr=rate, silence_gaps=True)
    offsets, ranges, got = sess.transcribe_sliced(wave, rate)
    [(want_off, want)] = batch.transcribe_recordings(ins, [wave], rates=[rate])
    assert offsets == list(want_off) and len(got) > 10
    assert_same_notes(got, want)
    with pytest.raises(Exception, match='too small to resample'):
        sess.transcribe_sliced(np.zeros(1, np.float32), 96000)


def test_first_call_after_open_resamples_with_the_uploaded_table(model):
    """The weights and the resampling table go up on the session's own stream: a resampling call straight after opening, with
    no other host work in between, already gives the Python path's notes."""
    kind, ins, path, _, _ = model
    wave = synth.synth_waveform(6060, seconds=8.0, sr=48000)
    fresh = nsess.Session(path, 0)
    try:
        offsets, ranges, got = fresh.transcribe_sliced(wave, 48000)
    finally:
        fresh.close()
    [(want_off, want)] = batch.transcribe_recordings(ins, [wave], rates=[48000])
    assert offsets == list(want_off)
    assert_same_notes(got, want)


def test_threads_share_one_session(model):
    kind, ins, path, _, sess = model
    inputs = [[synth.synth_waveform(500 + 10 * t + i, seconds=2.0 + i) for i in range(6)] for t in range(2)]
    serial = [sess.transcribe(x) for x in inputs]
    results, errors = [[] for _ in inputs], []

    def work(t):
        notes = nsess.Notes()
        try:
            for _ in range(4):
                results[t].append(sess.transcribe(inputs[t], notes))
        except Exception as e:            # noqa: BLE001  (reported below)
            errors.append(e)
        finally:
            notes.close()

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(2):
        for r in results[t]:
            assert_same_notes(r, serial[t])


def test_c_example_transcribes_a_wav_file(model, tmp_path):
    kind, ins, path, _, sess = model
    if kind != 'two_head':
        pytest.skip('one model kind is enough for the example')
    assert EXAMPLE.is_file(), 'examples/some_transcribe is built with the library'
    linked = subprocess.run(['ldd', str(EXAMPLE)], capture_output=True, text=True, check=True).stdout
    assert 'libsome_b200' in linked and 'libpython' not in linked and 'libtorch' not in linked
    wav = tmp_path / 'rec.wav'
    synth.write_wav16(wav, synth.synth_waveform(4321, seconds=45.0, silence_gaps=True))
    run = subprocess.run([str(EXAMPLE), str(path), str(wav)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stderr
    samples, _ = audio.load(wav, sr=44100)
    offsets, notes = ins.model.infer_sliced(samples, Slicer(44100, max_sil_kept=1000))
    want = [f'{off:.17g} {m:.9g} {d:.17g} {int(r)}' for off, seg in zip(offsets, notes)
            for m, d, r in zip(seg['note_midi'].tolist(), seg['note_dur'].tolist(), seg['note_rest'].tolist())]
    assert len(want) > 20
    assert run.stdout.splitlines() == want
    import wave as wavmod
    stereo = tmp_path / 'stereo.wav'
    with wavmod.open(str(stereo), 'wb') as f:
        f.setnchannels(2)
        f.setsampwidth(2)
        f.setframerate(44100)
        f.writeframes(b'\0' * 4000)
    bad = subprocess.run([str(EXAMPLE), str(path), str(stereo)], capture_output=True, text=True, timeout=60)
    assert bad.returncode != 0 and 'mono' in bad.stderr
