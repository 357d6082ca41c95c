"""AIFF and AIFF-C on the H100: some_pcm_decode equals oracle/aiff.py bit for bit for every new sample kind; audio.load and
decode_aiff equal the oracle (and audio.resample of it); the same samples stored as WAV, AIFF and AIFF-C give the same notes
through some_session_transcribe_encoded, alone or mixed with WAV and FLAC; encoded streams of AIFF bytes, split in any way
and mixed with other streams, equal the whole-file call; examples/some_infer and batch_infer_dataset read AIFF as they read
the equivalent WAV."""
import csv
import ctypes as C
import pathlib
import struct
import subprocess

import numpy as np
import pytest
import torch

from oracle import aiff as oa
from some_b200 import _lib, audio, batch, export, synth
from some_b200 import session as nsess

import test_gpu_audio as ga
import test_gpu_encoded as ge
import test_gpu_encoded_stream as gs

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent
EXAMPLE = REPO / 'examples' / 'some_infer'

NEW_KINDS = [  # (compression type, sampleSize): every kind the AIFF walk adds, and the little-endian ones through sowt
    (None, 8), (None, 12), (None, 16), (None, 20), (None, 24), (None, 32), (b'sowt', 8), (b'sowt', 16), (b'sowt', 24),
    (b'sowt', 32), (b'raw ', 8), (b'fl32', 32), (b'fl64', 64), (b'ulaw', 16), (b'alaw', 8)]


def quantise16(x: np.ndarray) -> np.ndarray:
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


def wav_s16(v: np.ndarray, rate: int) -> bytes:
    v = v if v.ndim == 2 else v[:, None]
    ch = v.shape[1]
    raw = v.astype('<i2').tobytes()
    fmt = struct.pack('<HHIIHH', 1, ch, rate, rate * ch * 2, ch * 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def aiff_s16(v: np.ndarray, rate: float, comp=None, **kw) -> bytes:
    v = v if v.ndim == 2 else v[:, None]
    raw = v.astype('<i2' if comp == b'sowt' else '>i2').tobytes()
    return oa.aiff_bytes(raw, v.shape[1], 16, rate, comp=comp, **kw)


# ---------------------------------------------------------------------------------------------- the PCM kernel
def test_pcm_decode_equals_oracle():
    """Every new kind at 1-8 and 12 channels, samples starting at odd byte offsets, all recordings in one launch, mono and
    interleaved, bit for bit (view as uint32)."""
    lib = _lib.load()
    rng = np.random.default_rng(11)
    files = []
    for comp, bits in NEW_KINDS:
        for ch in list(range(1, 9)) + [12]:
            n = int(rng.integers(0, 2500))
            kind = oa._kind_of(comp, bits)
            raw = bytearray(oa.raw_samples(kind, n, ch, int(rng.integers(1 << 30))))
            if kind in (oa.F32BE, oa.F64BE) and n > 1:
                sb = oa.SAMPLE_BYTES[kind] * ch
                raw[:2 * sb] = bytes(sb) + (b'\x80' + bytes(oa.SAMPLE_BYTES[kind] - 1)) * ch   # a +0.0 and a -0.0 frame
            data = oa.aiff_bytes(bytes(raw), ch, bits, 16000.0, comp=comp, offset=int(rng.integers(0, 5)))
            files.append((data, oa.walk(data)))
    blob, items = bytearray(), []
    for data, m in files:
        info = audio.audio_info(data)
        assert (info.kind, info.frames, info.data_offset) == (m['kind'], m['frames'], m['data_offset'])
        blob += bytes(1 + (len(blob) % 2 == 1))          # the next sample byte lands at an odd offset
        items.append((len(blob), m))
        blob += data[m['data_offset']:m['data_offset'] + m['data_bytes']]
    dev = torch.from_numpy(np.frombuffer(bytes(blob) + bytes(16), np.uint8).copy()).cuda()
    for mono in (0, 1):
        sizes = [m['frames'] * (1 if mono else m['channels']) for _, m in items]
        starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        out = torch.full((int(starts[-1]) + 1,), float('nan'), dtype=torch.float32, device='cuda')
        arr = (_lib.PcmItem * len(items))(*[
            _lib.PcmItem(dev.data_ptr() + off, m['frames'], m['channels'], m['kind'], mono, 0,
                         out.data_ptr() + 4 * int(starts[i])) for i, (off, m) in enumerate(items)])
        desc = np.zeros(lib.some_pcm_decode_bytes(len(items)), np.uint8)
        _lib.check(lib.some_pcm_decode_pack(arr, len(items), desc.ctypes.data), 'pack')
        desc_d = torch.from_numpy(desc).cuda()
        _lib.check(lib.some_pcm_decode(desc.ctypes.data, desc_d.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        got = out.cpu().numpy()
        for i, (data, m) in enumerate(files):
            x = oa.samples(data, m)
            w = oa.to_mono(x) if mono else x.reshape(-1)
            np.testing.assert_array_equal(got[starts[i]:starts[i + 1]].view(np.uint32), w.view(np.uint32),
                                          err_msg=f'item {i} kind {m["kind"]} channels {m["channels"]} mono={mono}')


def test_g711_every_code():
    """All 256 codes of both laws, as one recording each, through audio's decode path."""
    for comp, table in ((b'ulaw', oa.ULAW_TABLE), (b'alaw', oa.ALAW_TABLE)):
        data = oa.aiff_bytes(bytes(range(256)), 1, 8, 8000.0, comp=comp)
        y = audio._pcm_device(data, audio.audio_info(data), mono=False).cpu().numpy()
        np.testing.assert_array_equal(y * np.float32(32768), table.astype(np.float32))


# ---------------------------------------------------------------------------------------------- audio.load
LOAD_CASES = [('aiff_s16_2ch_48k', lambda: aiff_s16(quantise16(ge.stereo(41, 6.0, 48000)), 48000.0), 48000),
              ('aifc_s24_3ch_odd_rate', lambda: oa.aiff_bytes(oa.raw_samples(oa.S24BE, 22254 * 5, 3, 4), 3, 24, 22254.545454545454,
                                                             comp=b'NONE', offset=3), 22254),
              ('aifc_fl32_1ch_48k', lambda: oa.aiff_bytes((synth.synth_waveform(42, seconds=4.0, sr=48000) * 0.5).astype('>f4')
                                                         .tobytes(), 1, 32, 48000.0, comp=b'fl32'), 48000),
              ('aifc_ulaw_2ch_22k', lambda: oa.aiff_bytes(oa.raw_samples(oa.ULAW, 22050 * 3, 2, 5), 2, 16, 22050.0, comp=b'ulaw'),
               22050)]


@pytest.mark.parametrize('name,make,rate', LOAD_CASES, ids=[c[0] for c in LOAD_CASES])
def test_load_equals_oracle(tmp_path, name, make, rate):
    data = make()
    p = tmp_path / (name + '.aif')
    p.write_bytes(data)
    x = oa.samples(data, oa.walk(data))
    d, r = audio.decode_aiff(p)
    assert r == rate
    np.testing.assert_array_equal(d.reshape(x.shape).view(np.uint32), x.view(np.uint32))
    y, r = audio.load(p, sr=None)
    want, wr = oa.load(data, sr=None)
    assert r == wr == rate
    np.testing.assert_array_equal(y.view(np.uint32), want.view(np.uint32))
    y2, _ = audio.load(p, sr=None, mono=False)
    np.testing.assert_array_equal(y2.view(np.uint32), (x.T if x.shape[1] > 1 else x[:, 0]).view(np.uint32))
    y44, r44 = audio.load(p, sr=44100)
    assert r44 == 44100
    np.testing.assert_array_equal(y44.view(np.uint32), audio.resample(want, rate, 44100).view(np.uint32))
    yn, rn = audio.load_native(p, 44100)
    assert rn == rate and np.array_equal(yn.view(np.uint32), want.view(np.uint32))


def test_decode_wav_still_refuses_aiff(tmp_path):
    p = tmp_path / 'x.aif'
    p.write_bytes(aiff_s16(np.zeros(10, np.int16), 8000.0))
    with pytest.raises(ValueError, match='AIFF/IFF'):
        audio.decode_wav(p)
    q = tmp_path / 'x.wav'
    q.write_bytes(wav_s16(np.zeros(10, np.int16), 8000))
    with pytest.raises(ValueError, match='not an AIFF'):
        audio.decode_aiff(q)
    r = tmp_path / 'bad.aif'
    r.write_bytes(oa.aiff_bytes(bytes(20), 1, 16, 8000.0, comp=b'ima4'))
    with pytest.raises(ValueError, match="'ima4'"):
        audio.load(r)


# ---------------------------------------------------------------------------------------------- the session
@pytest.fixture(scope='module')
def sess(tmp_path_factory):
    d = tmp_path_factory.mktemp('aiff_model')
    config = synth.named_config('two_head')
    ckpt = synth.write_checkpoint(d, config, seed=1234)
    path = export.export(ckpt)
    s = nsess.Session(path, 0)
    s.path, s.ckpt, s.config = path, ckpt, config
    yield s
    s.close()


@pytest.fixture(scope='module')
def songs():
    """name: bytes.  The same int16 samples as WAV, AIFF and AIFF-C sowt, and other AIFF codings and rates."""
    v = quantise16(ge.stereo(51, 45.0, 48000))
    m = quantise16(synth.synth_waveform(52, seconds=40.0, sr=44100, silence_gaps=True) * np.float32(0.9))
    return {
        'wav': wav_s16(v, 48000),
        'aiff': aiff_s16(v, 48000.0, before=[(b'MARK', b'\0\0'), (b'COMT', b'abc')]),
        'aifc_sowt': aiff_s16(v, 48000.0, comp=b'sowt', name=b'sowt', offset=5),
        'aiff_mono_44k': aiff_s16(m, 44100.0),
        'aifc_fl64_22k': oa.aiff_bytes((ge.stereo(53, 35.0, 22050) * 0.7).astype('>f8').tobytes(), 2, 64, 22050.0,
                                       comp=b'fl64'),
        'aifc_alaw_odd_rate': oa.aiff_bytes(bytes(audio_alaw(synth.synth_waveform(54, seconds=38.0, sr=22254,
                                                                                  silence_gaps=True))), 1, 16,
                                            22254.545454545454, comp=b'alaw'),
        'flac': ge.flac_file(ge.stereo(55, 30.0, 44100), 44100, 16, channel_mode='mid_side'),
    }


def audio_alaw(x: np.ndarray) -> np.ndarray:
    """The A-law code nearest to each sample (a search over the 256 values)."""
    vals = oa.ALAW_TABLE.astype(np.float32) / np.float32(32768)
    order = np.argsort(vals)
    idx = np.clip(np.searchsorted(vals[order], x), 1, 255)
    lo, hi = order[idx - 1], order[idx]
    return np.where(np.abs(vals[lo] - x) <= np.abs(vals[hi] - x), lo, hi).astype(np.uint8)


def test_same_samples_same_notes_as_wav(sess, songs):
    got = sess.transcribe_encoded([songs['wav'], songs['aiff'], songs['aifc_sowt']])
    assert len(got[0][1]) > 2
    for g in got[1:]:
        assert g[:2] == got[0][:2]
        ge.assert_same_notes(g[2], got[0][2])
    y, rate = oa.load(songs['aiff'], sr=None)
    want = sess.transcribe_sliced(y, rate)
    assert got[1][0] == want[0] and got[1][1] == want[1]
    ge.assert_same_notes(got[1][2], want[2])


def test_mixed_call_equals_each_item_alone(sess, songs):
    names = list(songs)
    got = sess.transcribe_encoded([songs[n] for n in names])
    for name, g in zip(names, got):
        [alone] = sess.transcribe_encoded([songs[name]])
        assert alone[:2] == g[:2], name
        ge.assert_same_notes(alone[2], g[2])
        if name.startswith('aif'):
            y, rate = oa.load(songs[name], sr=None)
            want = sess.transcribe_sliced(y, rate)
            assert g[1] == want[1], name
            ge.assert_same_notes(g[2], want[2])


def test_stream_equals_transcribe_encoded(sess, songs):
    for name in ('aiff', 'aifc_sowt', 'aifc_alaw_odd_rate', 'aifc_fl64_22k'):
        data = songs[name]
        _, want_ranges, want_notes = sess.transcribe_encoded([data])[0]
        rng = np.random.default_rng(len(name))
        for sizes in (gs.byte_sizes(len(data), rng, small=200), [1] * 200 + [len(data) - 200], [len(data)]):
            with sess.stream_encoded() as st:
                calls = gs.push_all(st, data, sizes)
                meta = st.meta()
            ranges, notes = gs.flatten(calls)
            assert ranges == want_ranges, name
            ge.assert_same_notes(notes, want_notes)
            assert meta['container'] == _lib.AUDIO_AIFF and meta['bytes_received'] == len(data)


def test_push_bytes_many_mixes_aiff_wav_and_flac(sess, songs):
    names = list(songs)
    datas = [songs[n] for n in names]
    want = [r[1:] for r in sess.transcribe_encoded(datas)]
    rng = np.random.default_rng(9)
    streams = [sess.stream_encoded() for _ in names]
    got = [([], []) for _ in names]
    pos, done, tick = [0] * len(names), [False] * len(names), 0
    while not all(done):
        items, fin, idx = [], [], []
        for i, st in enumerate(streams):
            if done[i]:
                continue
            m = int(rng.integers(0, 1 << 17)) if tick else 40
            chunk = datas[i][pos[i]:pos[i] + m]
            pos[i] += len(chunk)
            f = pos[i] >= len(datas[i]) and rng.random() < 0.5
            items.append((st, chunk))
            fin.append(f)
            idx.append(i)
        for i, (_, r, nt) in zip(idx, sess.push_bytes_many(items, fin)):
            got[i][0].extend(r)
            got[i][1].extend(nt)
        for i, f in zip(idx, fin):
            done[i] = done[i] or f
        tick += 1
    for st in streams:
        st.close()
    for name, (gr, gn), (wr, wn) in zip(names, got, want):
        assert gr == wr, name
        ge.assert_same_notes(gn, wn)


def test_refused_aiff_stream_leaves_the_others(sess, songs):
    bad = oa.aiff_bytes(bytes(4000), 1, 16, 44100.0, comp=b'ima4')
    reason = gs._refusal(lambda: sess.transcribe_encoded([bad])).split('item 0: ', 1)[1]
    assert "'ima4'" in reason
    names = ['wav', 'aiff_mono_44k', 'flac']
    want = [r[1:] for r in sess.transcribe_encoded([songs[n] for n in names])]
    streams = [sess.stream_encoded() for _ in range(4)]
    datas = [songs[n] for n in names] + [bad]
    got = [([], []) for _ in datas]
    try:
        with pytest.raises(_lib.StreamRefused) as e:
            sess.push_bytes_many([(st, d[:100000]) for st, d in zip(streams, datas)])
        assert 'stream 3: ' + reason in str(e.value)
        assert e.value.results[3][1] == []
        for i in range(3):
            got[i][0].extend(e.value.results[i][1])
            got[i][1].extend(e.value.results[i][2])
        for i, (_, r, nt) in enumerate(sess.push_bytes_many([(streams[i], datas[i][100000:]) for i in range(3)], [1, 1, 1])):
            got[i][0].extend(r)
            got[i][1].extend(nt)
        for (gr, gn), (wr, wn) in zip(got[:3], want):
            assert gr == wr
            ge.assert_same_notes(gn, wn)
        rc = sess.lib.some_stream_push_bytes(streams[3].handle, b'x', 1, streams[3].notes.handle)
        assert rc != 0 and 'refused' in sess.lib.some_last_error().decode()
    finally:
        for st in streams:
            st.close()


# ---------------------------------------------------------------------------------------------- the example and the dataset
def test_some_infer_reads_aiff_as_wav(sess, songs, tmp_path):
    outs = {}
    for name, suffix in (('wav', '.wav'), ('aiff', '.aif'), ('aifc_sowt', '.aifc')):
        src = tmp_path / ('song' + suffix)
        src.write_bytes(songs[name])
        r = subprocess.run([str(EXAMPLE), str(sess.path), str(src)], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        outs[name] = src.with_suffix('.mid').read_bytes()
    assert outs['aiff'] == outs['wav'] == outs['aifc_sowt']
    assert len(outs['wav']) > 100


def test_batch_infer_dataset_reads_aiff_bytes(tmp_path):
    ins, config = ga._plugin(tmp_path)
    rng = np.random.default_rng(12)
    sets = {}
    for kind in ('wav', 'aiff'):
        data = tmp_path / kind
        (data / 'wavs').mkdir(parents=True)
        sets[kind] = data
    rows = []
    for i, rate in enumerate([48000, 22050, 44100]):
        v = quantise16(synth.synth_waveform(90 + i, seconds=float(rng.uniform(5, 9)), sr=rate, silence_gaps=True) * 0.9)
        (sets['wav'] / 'wavs' / f'it{i}.wav').write_bytes(wav_s16(v, rate))
        (sets['aiff'] / 'wavs' / f'it{i}.wav').write_bytes(aiff_s16(v, float(rate), comp=b'sowt' if i % 2 else None))
        n_words = int(rng.integers(3, 8))
        ph_num = rng.integers(1, 4, size=n_words)
        secs = len(v) / rate
        durs = np.diff(np.concatenate([[0.0], np.sort(rng.uniform(0, secs, int(ph_num.sum()) - 1)), [secs]]))
        rows.append({'name': f'it{i}', 'ph_seq': ' '.join(['a'] * int(ph_num.sum())),
                     'ph_dur': ' '.join(f'{d:.6f}' for d in durs), 'ph_num': ' '.join(str(int(x)) for x in ph_num)})
    out = {}
    for kind, data in sets.items():
        with open(data / 'transcriptions.csv', 'w', encoding='utf8', newline='') as f:
            wr = csv.DictWriter(f, fieldnames=['name', 'ph_seq', 'ph_dur', 'ph_num'])
            wr.writeheader()
            wr.writerows(rows)
        out[kind] = batch.batch_infer_dataset(data, ins, config, csv=tmp_path / f'{kind}.csv', load_audio=audio.load_native,
                                              max_frames_per_batch=1500).read_bytes()
    assert out['aiff'] == out['wav'] and len(out['wav']) > 100
