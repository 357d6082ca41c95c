"""GPU tests of some_flac_scan / some_flac_decode and some_b200.audio's FLAC path: the device decode equals the encoder's
input and the restated sequential decoder (oracle/flac.py) bit for bit over every feature the encoder can force, in one
call for a mixed batch too; the mono down-mix is np.mean's; false sync candidates are harmless; corrupt streams are
refused; and audio.load, transcribe_recordings and batch_infer_dataset give exactly what the oracle's librosa.load gives."""
import csv

import numpy as np
import pytest
import torch

from oracle import flac as of
from some_b200 import audio, batch, plugin, synth

pytestmark = pytest.mark.gpu

CASES = of.feature_cases()
REFUSAL = r'FLAC.*byte offset \d+'


def _write(tmp_path, name, data):
    p = tmp_path / f'{name}.flac'
    p.write_bytes(data)
    return p


@pytest.mark.parametrize('case', CASES, ids=lambda c: c[0])
def test_device_decode_equals_input_and_oracle(case, tmp_path):
    name, x, kw = case
    p = _write(tmp_path, name, of.encode(x, **kw))
    got, rate = audio.decode_flac(p)
    want, want_rate = of.decode_file(p)
    assert rate == want_rate == kw['rate'] and got.dtype == np.float32
    np.testing.assert_array_equal(got, want)
    ints = got.reshape(len(x), -1).astype(np.float64) * 2.0 ** (kw['bps'] - 1)     # exact: x * 2^-(bps-1)
    np.testing.assert_array_equal(ints, x)


def test_mixed_batch_in_one_call():
    recs = [audio.parse_flac(of.encode(x, **kw), name) for name, x, kw in CASES]
    dev = torch.device('cuda', 0)
    fb = audio.FlacBatch(recs, dev)
    assert fb.lengths == [len(x) for _, x, _ in CASES]
    # interleaved and mono into one buffer each, with a gap of 3 sentinel samples after every recording
    for mono in (False, True):
        width = [1 if mono else r.channels for r in recs]
        region = [-(-(n + 3) * w // 840) * 840 for n, w in zip(fb.lengths, width)]   # 840: a multiple of every width
        starts = np.concatenate([[0], np.cumsum(region)])
        out = torch.full((int(starts[-1]),), 7.0, device=dev)
        status = fb.emit(out, {r: int(starts[r]) // width[r] for r in range(len(recs))}, mono=mono)
        host = out.cpu().numpy()
        assert int(status.item()) == 0
        for r, (name, x, kw) in enumerate(CASES):
            f = x.astype(np.float32) * np.float32(2.0 ** -(kw['bps'] - 1))
            want = audio.to_mono(f.T) if mono else f.reshape(-1)
            a = int(starts[r])
            np.testing.assert_array_equal(host[a:a + want.size], want, err_msg=name)
            assert np.all(host[a + want.size:int(starts[r + 1])] == 7.0), name


def test_mono_downmix_equals_to_mono_for_1_to_8_channels(tmp_path):
    rng = np.random.default_rng(5)
    for ch in range(1, 9):
        x = rng.integers(-2 ** 23, 2 ** 23, size=(20000, ch))
        x[0] = 2 ** 23 - 1
        x[1] = -2 ** 23
        p = _write(tmp_path, f'noise{ch}', of.encode(x, 44100, 24))
        y, rate = audio.load(p, sr=None)
        f = x.astype(np.float32) * np.float32(2.0 ** -23)
        np.testing.assert_array_equal(y, audio.to_mono(f.T), err_msg=f'{ch} channels')
        np.testing.assert_array_equal(y, of.load(p, sr=None)[0])


def test_false_sync_inside_verbatim_samples_is_harmless(tmp_path):
    x = of.test_signal(6000, 1, 16, 9)
    real = of.encode(x[:4096], 44100, 16)
    head = real[42:42 + 6]                                  # a genuine, CRC-8-valid header of this stream (frame 0)
    fake = head[:-2] + bytes([0x01]) + bytes([of.crc8(head[:-2] + b'\x01')])   # frame number 1, CRC-8 recomputed
    words = np.frombuffer(fake, '>i2').astype(np.int64)
    y = x.copy()
    y[1000:1000 + len(words), 0] = words                    # VERBATIM samples whose bytes are that header
    data = of.encode(y, 44100, 16, subframe={'type': 'verbatim'})
    assert fake in data
    fb = audio.FlacBatch([audio.parse_flac(data)], torch.device('cuda', 0))
    assert fb.n_candidates > len(fb.chains[0])              # the fake header was found, parsed and never chained
    p = _write(tmp_path, 'fake', data)
    got, _ = audio.decode_flac(p)
    np.testing.assert_array_equal(got.astype(np.float64) * 2.0 ** 15, y[:, 0])


def _corrupt_streams():
    x = of.test_signal(12000, 2, 16, 8)
    good = of.encode(x, 44100, 16, blocksize=4096)
    crc = bytearray(good)
    end0 = of._frame(np.frombuffer(good, np.uint8), 42, len(good), 2, 16, 4096, np.zeros((2, 4096), np.int64), of.CRC8_T,
                     of.CRC16_T)[1]
    crc[end0 - 1] ^= 0x55                                   # frame 0's CRC-16
    return [('crc16', bytes(crc)), ('truncated_last_frame', good[:-7]),
            ('frame_gap', of.encode(x, 44100, 16, blocksize=4096, frame_numbers=[0, 2, 3]))]


@pytest.mark.parametrize('name,data', _corrupt_streams(), ids=lambda v: v if isinstance(v, str) else '')
def test_corrupt_streams_are_refused(name, data, tmp_path):
    p = _write(tmp_path, name, data)
    with pytest.raises(ValueError, match=REFUSAL):
        of.decode_file(p)
    with pytest.raises(ValueError, match=REFUSAL):
        audio.decode_flac(p)
    with pytest.raises(ValueError, match=REFUSAL):
        audio.load(p, sr=44100)
    ok = _write(tmp_path, 'ok', of.encode(of.test_signal(3000, 1, 16, 1), 44100, 16))
    assert audio.decode_flac(ok)[0].shape == (3000,)        # the device is fine afterwards


def _files(tmp_path):
    s = synth.synth_waveform(5, seconds=1.3, sr=48000)
    rng = np.random.default_rng(3)
    return [_write(tmp_path, 'stereo48', of.encode(np.round(np.stack([s, -0.5 * s], 1) * 32767).astype(np.int64), 48000, 16,
                                                      channel_mode='mid_side')),
            _write(tmp_path, 'mono44_24', of.encode(np.round(s[:40000, None] * 8e6).astype(np.int64), 44100, 24)),
            _write(tmp_path, 'six16k', of.encode(rng.integers(-2 ** 19, 2 ** 19, size=(9000, 6)), 16000, 20)),
            _write(tmp_path, 'id3_22k', of.encode(np.round(s[:20000, None] * 2000).astype(np.int64), 22050, 12,
                                                     id3=of.id3_tag()))]


def test_load_equals_the_restated_librosa_load(tmp_path):
    for p in _files(tmp_path):
        for sr in (44100, 22050, None):
            y, rate = audio.load(p, sr=sr)
            want, want_rate = of.load(p, sr=sr)
            assert rate == want_rate
            np.testing.assert_array_equal(y, want, err_msg=f'{p.name} sr={sr}')
        y, rate = audio.load(p, sr=None, mono=False)
        want, _ = of.load(p, sr=None, mono=False)
        np.testing.assert_array_equal(y, want)
        y, rate = audio.load_native(p, 44100)
        np.testing.assert_array_equal(y, of.load(p, sr=None)[0])


def _plugin(tmp_path, name='two_head'):
    config = synth.named_config(name)
    ckpt = synth.write_checkpoint(tmp_path, config)
    cls = plugin.QuantizedMIDIExtractionInference if name.startswith('quant') else plugin.MIDIExtractionInference
    return cls(config=config, model_path=ckpt, device='cuda:0'), config


def _same_notes(got, want):
    assert len(got) == len(want)
    for (go, gn), (wo, wn) in zip(got, want):
        assert go == wo and len(gn) == len(wn)
        for a, b in zip(gn, wn):
            for k in ('note_midi', 'note_dur', 'note_rest'):
                np.testing.assert_array_equal(a[k], b[k])


def test_transcribe_recordings_with_encoded_audio(tmp_path):
    ins, _ = _plugin(tmp_path)
    specs = [(48000, 2, 16, 9.0), (44100, 1, 16, 6.0), (22050, 2, 24, 7.5), (44100, 2, 24, 0.3), (32000, 3, 20, 5.0)]
    recs, decoded, rates, items, item_rates = [], [], [], [], []
    for i, (rate, ch, bps, secs) in enumerate(specs):
        w = synth.synth_waveform(70 + i, seconds=secs, sr=rate, silence_gaps=True)
        x = np.round(np.stack([w * (0.9 - 0.2 * c) for c in range(ch)], 1) * ((1 << (bps - 1)) - 1)).astype(np.int64)
        p = _write(tmp_path, f'r{i}', of.encode(x, rate, bps))
        rec = audio.read_encoded(p)
        mono, _ = of.load(p, sr=None)
        items += [rec, mono]                                  # encoded records mixed with numpy inputs
        item_rates += [None, rate]
        decoded += [mono, mono]
        rates += [rate, rate]
    got = batch.transcribe_recordings(ins, items, rates=item_rates)
    want = batch.transcribe_recordings(ins, decoded, rates=rates)
    _same_notes(got, want)
    with pytest.raises(ValueError, match='rate'):
        batch.transcribe_recordings(ins, [items[0]], rates=[44100])


def test_batch_infer_dataset_with_encoded_loader_writes_the_oracle_csv(tmp_path):
    ins, config = _plugin(tmp_path)
    data = tmp_path / 'raw'
    (data / 'wavs').mkdir(parents=True)
    rng = np.random.default_rng(8)
    rows = []
    for i, rate in enumerate([48000, 22050, 44100, 48000, 44100]):
        w = synth.synth_waveform(90 + i, seconds=float(rng.uniform(5, 10)), sr=rate, silence_gaps=True)
        x = np.round(np.stack([w, 0.7 * w], 1) * 32767).astype(np.int64)
        (data / 'wavs' / f'it{i}.wav').write_bytes(of.encode(x, rate, 16, channel_mode='mid_side'))   # FLAC bytes
        n_words = int(rng.integers(3, 8))
        ph_num = rng.integers(1, 4, size=n_words)
        secs = len(w) / rate
        durs = np.diff(np.concatenate([[0.0], np.sort(rng.uniform(0, secs, int(ph_num.sum()) - 1)), [secs]]))
        rows.append({'name': f'it{i}', 'ph_seq': ' '.join(['a'] * int(ph_num.sum())), 'ph_dur': ' '.join(f'{d:.6f}' for d in durs),
                     'ph_num': ' '.join(str(int(x)) for x in ph_num)})
    with open(data / 'transcriptions.csv', 'w', encoding='utf8', newline='') as f:
        wr = csv.DictWriter(f, fieldnames=['name', 'ph_seq', 'ph_dur', 'ph_num'])
        wr.writeheader()
        wr.writerows(rows)

    def oracle_loader(path, sr):
        return of.load(path, sr=sr)[0]

    a = batch.batch_infer_dataset(data, ins, config, csv=tmp_path / 'encoded.csv', load_audio=audio.read_encoded,
                                  max_frames_per_batch=1500)
    b = batch.batch_infer_dataset(data, ins, config, csv=tmp_path / 'oracle.csv', load_audio=oracle_loader,
                                  max_frames_per_batch=1500)
    assert a.read_bytes() == b.read_bytes()
    assert len(list(csv.DictReader(open(a, encoding='utf8', newline='')))) == len(rows)


def test_five_minute_recording(tmp_path):
    w = synth.synth_waveform(77, seconds=300.0, sr=44100, silence_gaps=True)
    x = np.round(np.stack([w, -0.6 * w], 1) * 32767).astype(np.int64)
    p = _write(tmp_path, 'long', of.encode(x, 44100, 16, channel_mode='mid_side'))
    got, rate = audio.decode_flac(p)
    assert rate == 44100 and got.shape == x.shape
    np.testing.assert_array_equal(got.astype(np.float64) * 2.0 ** 15, x)
    y, _ = audio.load(p, sr=None)
    np.testing.assert_array_equal(y, audio.to_mono(got.T))
