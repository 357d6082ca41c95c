"""The native session on an fp32 model file (`python -m some_b200.export --precision fp32`): every call kind gives the notes,
ranges and frame curves of Engine's fp32 path (precision='fp32') on the same samples, bit for bit; several replicas and
coalesced threads give what one replica gives alone; a bf16 file still opens as bf16."""
import io
import threading

import numpy as np
import pytest
import scipy.io.wavfile

from some_b200 import audio, export, plugin, synth
from some_b200 import session as nsess
from some_b200.slicer import Slicer

pytestmark = pytest.mark.gpu
SR, HOP = 44100, 512
PLUGINS = {'two_head': plugin.MIDIExtractionInference, 'quant_two_head': plugin.QuantizedMIDIExtractionInference}


@pytest.fixture(scope='module', params=list(PLUGINS))
def model(request, tmp_path_factory):
    d = tmp_path_factory.mktemp(request.param)
    config = synth.named_config(request.param)
    ckpt = synth.write_checkpoint(d, config, seed=1234)
    ins = PLUGINS[request.param](config=config, model_path=ckpt, device='cuda:0')
    path = export.export(ckpt, d / 'f32.somemodel', precision='fp32')
    s = nsess.Session(path, 0)
    s.ins, s.path, s.ckpt = ins, path, ckpt
    yield s
    s.close()


def assert_same_notes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g['note_midi'].view(np.uint32), w['note_midi'].view(np.uint32))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        np.testing.assert_array_equal(np.asarray(g['note_dur']).view(np.uint64), np.asarray(w['note_dur']).view(np.uint64))


def recording(seed=7):
    return np.concatenate([synth.synth_waveform(seed, seconds=9.0), np.zeros(SR, np.float32),
                           synth.synth_waveform(seed + 1, seconds=7.5), np.zeros(SR // 2, np.float32),
                           synth.synth_waveform(seed + 2, seconds=6.0)]).astype(np.float32)


def wav_bytes(x):
    ints = np.clip(np.round(x.astype(np.float64) * 32767), -32768, 32767).astype(np.int16)
    b = io.BytesIO()
    scipy.io.wavfile.write(b, SR, ints)
    return b.getvalue()


def test_precision_and_file(model, tmp_path):
    assert model.precision == 'fp32' and not model.bias_corrected
    data = model.path.read_bytes()
    assert int.from_bytes(data[88:92], 'little') == 1
    bf = nsess.Session(export.export(model.ckpt, tmp_path / 'bf16.somemodel'), 0)
    try:
        assert bf.precision == 'bf16'
        assert (tmp_path / 'bf16.somemodel').read_bytes()[88:92] == b'\0\0\0\0'
    finally:
        bf.close()


def test_clips_and_curves_equal_engine_fp32(model):
    eng, q = model.ins.model, model.ins.quantized
    waves = [np.zeros(0, np.float32)] + [synth.synth_waveform(100 + i, num_samples=n)
                                         for i, n in enumerate([511, 512, 33 * HOP + 5, 30 * SR, 4 * SR])]
    want = eng.infer(waves, q, return_intermediates=True, precision='fp32')
    got, curves = model.transcribe(waves, frames=True)
    assert_same_notes(got, want)
    for c, w in zip(curves, want):
        np.testing.assert_array_equal(c.bound.view(np.uint32), w['bounds'].view(np.uint32))
    assert_same_notes(model.transcribe(waves), eng.infer(waves, q, precision='fp32'))


def test_sliced_encoded_and_streams_equal_engine_fp32(model):
    eng, q = model.ins.model, model.ins.quantized
    rec = recording()
    offs, notes = eng.infer_sliced(rec, Slicer(sr=SR, max_sil_kept=1000), q, precision='fp32')
    s_offs, ranges, s_notes = model.transcribe_sliced(rec)
    assert len(s_notes) > 1 and s_offs == offs
    assert_same_notes(s_notes, notes)
    # encoded: the WAV's samples as audio.load reads them
    data = wav_bytes(rec)
    p = model.path.with_name('rec.wav')
    p.write_bytes(data)
    y, _ = audio.load_native(p)
    e_offs, e_notes = eng.infer_sliced(y, Slicer(sr=SR, max_sil_kept=1000), q, precision='fp32')
    [(enc_offs, _, enc_notes)] = model.transcribe_encoded([data])
    assert enc_offs == e_offs
    assert_same_notes(enc_notes, e_notes)
    # a PCM stream, with a peek half way: the peek is the open region's notes, the chunks are transcribe_sliced's
    chunks, peeked = [], None
    with model.stream() as st:
        block = SR // 5
        for i in range(0, len(rec), block):
            chunks += st.push(rec[i:i + block])[2]
            if peeked is None and i >= 12 * SR:
                _, pr, pn = st.peek()
                if pr:
                    peeked = (pr[0], pn)
        chunks += st.finish()[2]
    assert_same_notes(chunks, s_notes)
    assert peeked is not None
    (a, b), pn = peeked
    assert_same_notes(pn, eng.infer([rec[a:b]], q, precision='fp32'))
    # a byte stream of the WAV: transcribe_encoded's chunks
    got = []
    with model.stream_encoded() as es:
        for i in range(0, len(data), 7919):
            got += es.push(data[i:i + 7919])[2]
        got += es.finish()[2]
    assert_same_notes(got, enc_notes)


def test_replicas_and_threads(model):
    waves = [synth.synth_waveform(300 + i, seconds=2.0 + 1.5 * i) for i in range(8)]
    want = model.transcribe(waves)
    two = nsess.Session(model.path, [0, 0])
    try:
        assert two.precision == 'fp32'
        assert_same_notes(two.transcribe(waves), want)
        alone = [model.transcribe(waves[k::4]) for k in range(4)]
        got, errs = [None] * 4, []

        def run(k):
            try:
                got[k] = two.transcribe(waves[k::4])
            except Exception as e:      # noqa: BLE001
                errs.append(e)
        ts = [threading.Thread(target=run, args=(k,)) for k in range(4)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errs, errs
        for g, w in zip(got, alone):
            assert_same_notes(g, w)
    finally:
        two.close()
