"""Encoded files on the H100: some_pcm_decode equals audio.decode_wav (and its to_mono) bit for bit; the FLAC emitter keeps
its bits with the shared down-mix; some_session_transcribe_encoded gives, for every WAV or FLAC item of one call, what
some_session_transcribe_sliced gives on audio.load(file, sr=None) and what Engine.infer_sliced gives on
audio.load(file, sr=44100), whatever else is in the call; and examples/some_infer writes the MIDI bytes of infer.py's flow."""
import ctypes as C
import pathlib
import re
import struct
import subprocess
import threading
import warnings

import numpy as np
import pytest
import torch

from oracle import flac as of
from some_b200 import _lib, audio, export, midi, plugin, synth
from some_b200 import session as nsess
from some_b200.slicer import Slicer

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent
EXAMPLE = REPO / 'examples' / 'some_infer'
KINDS = {'two_head': plugin.MIDIExtractionInference, 'quant_two_head': plugin.QuantizedMIDIExtractionInference}
PCM = {'u8': (1, 8, 1), 's16': (1, 16, 2), 's24': (1, 24, 3), 's32': (1, 32, 4), 'f32': (3, 32, 4), 'f64': (3, 64, 8)}


def wav_file(x: np.ndarray, rate: int, kind: str, extra=b'') -> bytes:
    """A RIFF/WAVE file of float samples x [n] or [n, ch] in [-1, 1) stored as `kind`."""
    x = x if x.ndim == 2 else x[:, None]
    n, ch = x.shape
    tag, bits, cb = PCM[kind]
    if kind == 'u8':
        raw = np.clip(np.round(x * 128 + 128), 0, 255).astype(np.uint8).tobytes()
    elif kind in ('s16', 's32'):
        full = 2 ** (bits - 1)
        raw = np.clip(np.round(x * full), -full, full - 1).astype('<i2' if bits == 16 else '<i4').tobytes()
    elif kind == 's24':
        v = np.clip(np.round(x * 2 ** 23), -2 ** 23, 2 ** 23 - 1).astype('<i4').reshape(-1)
        raw = np.stack([(v >> 8 * k) & 0xFF for k in range(3)], axis=1).astype(np.uint8).tobytes()
    else:
        raw = x.astype('<f4' if bits == 32 else '<f8').tobytes()
    fmt = struct.pack('<HHIIHH', tag, ch, rate, rate * ch * cb, ch * cb, bits)
    pad = b'\0' if len(raw) % 2 else b''
    body = b'WAVE' + extra + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw + pad
    return b'RIFF' + struct.pack('<I', len(body)) + body


def decode_wav_bytes(path: pathlib.Path, data: bytes):
    path.write_bytes(data)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return audio.decode_wav(path)


def stereo(seed, seconds, rate, silence_gaps=True, ch=2):
    cols = [synth.synth_waveform(seed + c, seconds=seconds, sr=rate, silence_gaps=silence_gaps) for c in range(ch)]
    return np.stack(cols, axis=1) * np.float32(0.9)


# ---------------------------------------------------------------------------------------------- the PCM kernel
def test_pcm_decode_equals_decode_wav(tmp_path):
    """Every sample kind at 1-8 channels (and 12: the pairwise sum's tail), data starting at odd byte offsets, all
    recordings in one launch, mono and interleaved."""
    lib = _lib.load()
    rng = np.random.default_rng(3)
    files, want_i, want_m = [], [], []
    for kind in PCM:
        for ch in list(range(1, 9)) + [12]:
            n = int(rng.integers(0, 3000))
            x = (rng.standard_normal((n, ch)) * 0.3).astype(np.float32)
            x[: n // 7] = np.float32(-0.0)
            data = wav_file(np.clip(x, -1, 0.999), 16000, kind, extra=b'LIST' + struct.pack('<I', 3) + b'abc\0')
            y, _ = decode_wav_bytes(tmp_path / 'x.wav', data)
            files.append((data, kind, ch, n))
            want_i.append(y.reshape(-1))
            want_m.append(audio.to_mono(y.T) if ch > 1 else y)
    # one byte buffer, every data chunk at an odd offset
    blob, items = bytearray(), []
    for data, kind, ch, n in files:
        m = _lib.AudioMeta()
        _lib.check(lib.some_audio_info(C.create_string_buffer(data, len(data)), len(data), C.byref(m)))
        assert m.frames == n and m.channels == ch
        blob += bytes(1 + (len(blob) % 2 == 1))          # the next data byte lands at an odd offset
        items.append((len(blob), m))
        blob += data[m.data_offset:m.data_offset + m.data_bytes]
    dev = torch.from_numpy(np.frombuffer(bytes(blob) + bytes(16), np.uint8).copy()).cuda()
    for mono in (0, 1):
        sizes = [m.frames * (1 if mono else m.channels) for _, m in items]
        starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        out = torch.full((int(starts[-1]) + 1,), float('nan'), dtype=torch.float32, device='cuda')
        arr = (_lib.PcmItem * len(items))(*[
            _lib.PcmItem(dev.data_ptr() + off, m.frames, m.channels, m.kind, mono, 0, out.data_ptr() + 4 * int(starts[i]))
            for i, (off, m) in enumerate(items)])
        desc = np.zeros(lib.some_pcm_decode_bytes(len(items)), np.uint8)
        _lib.check(lib.some_pcm_decode_pack(arr, len(items), desc.ctypes.data), 'pack')
        desc_d = torch.from_numpy(desc).cuda()
        _lib.check(lib.some_pcm_decode(desc.ctypes.data, desc_d.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        got = out.cpu().numpy()
        for i, w in enumerate(want_m if mono else want_i):
            np.testing.assert_array_equal(got[starts[i]:starts[i + 1]].view(np.uint32), w.astype(np.float32).view(np.uint32),
                                          err_msg=f'item {i} {files[i][1:]} mono={mono}')


def test_flac_emitter_keeps_its_bits():
    """The FLAC emitter through the shared down-mix: mono and interleaved output of the oracle's cases equal the oracle's
    decode, scaled and averaged in numpy's order, bit for bit."""
    for name, x, kw in of.feature_cases():
        if not (name.startswith('channels') or name.startswith('stereo') or name in ('bps8', 'bps24', 'variable', 'id3')):
            continue
        data = of.encode(x, **kw)
        rec = audio.parse_flac(data, name)
        want = of.scale(of.decode(data)[0], rec.bps)
        y, _ = audio._flac_device(rec, mono=False)
        got = y.cpu().numpy()
        np.testing.assert_array_equal(got.T.reshape(want.shape) if got.ndim == 2 else got.reshape(want.shape), want)
        m, _ = audio._flac_device(rec, mono=True)
        w = audio.to_mono(want.T) if want.ndim == 2 and want.shape[1] > 1 else want.reshape(-1)
        np.testing.assert_array_equal(m.cpu().numpy().view(np.uint32), w.astype(np.float32).view(np.uint32), err_msg=name)


# ---------------------------------------------------------------------------------------------- the session
@pytest.fixture(scope='module', params=list(KINDS))
def model(request, tmp_path_factory):
    d = tmp_path_factory.mktemp(request.param)
    config = synth.named_config(request.param)
    ckpt = synth.write_checkpoint(d, config, seed=1234)
    path = export.export(ckpt)
    ins = KINDS[request.param](config=config, model_path=ckpt, device='cuda:0')
    sess = nsess.Session(path, 0)
    yield request.param, ins, path, sess
    sess.close()


def assert_same_notes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g['note_midi'].view(np.uint32), np.asarray(w['note_midi'], np.float32).view(np.uint32))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        np.testing.assert_array_equal(g['note_dur'].view(np.uint64), np.asarray(w['note_dur'], np.float64).view(np.uint64))


def flac_file(x: np.ndarray, rate: int, bps: int, **kw) -> bytes:
    full = 2 ** (bps - 1)
    v = np.clip(np.round(x * full), -full, full - 1).astype(np.int64)
    return of.encode(v, rate=rate, bps=bps, subframe={'type': 'fixed', 'order': 2}, **kw)


@pytest.fixture(scope='module')
def mixed(tmp_path_factory):
    """About a dozen files of every kind the call mixes: (name, path)."""
    d = tmp_path_factory.mktemp('mixed')
    items = [
        ('wav_44k_s16_mono', wav_file(synth.synth_waveform(11, seconds=40.0, silence_gaps=True), 44100, 's16')),
        ('wav_48k_s24_stereo', wav_file(stereo(12, 35.0, 48000), 48000, 's24')),
        ('wav_22k_f32_stereo', wav_file(stereo(13, 30.0, 22050), 22050, 'f32')),
        ('wav_16k_s16_stereo', wav_file(stereo(14, 25.0, 16000), 16000, 's16')),
        ('wav_44k_f32_stereo', wav_file(stereo(15, 20.0, 44100), 44100, 'f32')),
        ('flac_48k_24_midside', flac_file(stereo(16, 30.0, 48000), 48000, 24, channel_mode='mid_side')),
        ('flac_44k_16_mono', flac_file(synth.synth_waveform(17, seconds=30.0, silence_gaps=True), 44100, 16)),
        ('flac_32k_12_leftside', flac_file(stereo(18, 20.0, 32000), 32000, 12, channel_mode='left_side', total_samples=0)),
        ('flac_44k_16_5min', flac_file(synth.synth_waveform(19, seconds=300.0, silence_gaps=True), 44100, 16,
                                       id3=of.id3_tag())),
        ('wav_short', wav_file(synth.synth_waveform(20, seconds=1.5), 48000, 's16')),
        ('wav_silent', wav_file(np.zeros((44100 * 8, 2), np.float32), 44100, 's16')),
        ('wav_empty', wav_file(np.zeros(0, np.float32), 44100, 's16')),
    ]
    out = []
    for name, data in items:
        p = d / (name + ('.flac' if name.startswith('flac') else '.wav'))
        p.write_bytes(data)
        out.append((name, p))
    return out


def test_one_mixed_call_equals_sliced_and_infer_sliced(model, mixed):
    kind, ins, path, sess = model
    got = sess.transcribe_encoded([p for _, p in mixed])
    slicer = Slicer(44100, max_sil_kept=1000)
    for (name, p), g in zip(mixed, got):
        y, rate = audio.load(p, sr=None)
        want = sess.transcribe_sliced(y, rate)
        assert g[0] == want[0] and g[1] == want[1], name
        assert_same_notes(g[2], want[2])
        y44, _ = audio.load(p, sr=44100)
        if len(y44):
            offs, notes = ins.model.infer_sliced(y44, slicer, quantized=ins.quantized)
            assert g[0] == list(offs), name
            assert_same_notes(g[2], notes)
    assert len(got[8][1]) > 10                                      # the 5-minute FLAC is cut into many chunks
    for (name, p), g in zip(mixed, got):                            # each item alone gives the same
        [alone] = sess.transcribe_encoded([p.read_bytes()])
        assert alone[:2] == g[:2], name
        assert_same_notes(alone[2], g[2])
    assert got[11][1] == [(0, 0)]                                   # the empty data chunk: one empty chunk, no upload
    assert sess.transcribe_encoded([]) == []


def test_refusals_name_the_item_and_leave_outputs_alone(model, mixed):
    kind, ins, path, sess = model
    lib = sess.lib
    good = mixed[0][1].read_bytes()
    notes = [nsess.Notes() for _ in range(3)]
    try:
        # sentinel results from files other than the ones the refused calls pass: a call that wrote any out[i] would show
        sentinel = [mixed[j][1].read_bytes() for j in (3, 6, 9)]
        keep = [C.create_string_buffer(d, len(d)) for d in sentinel]
        enc = (_lib.Encoded * 3)(*[_lib.Encoded(C.cast(b, C.c_void_p), len(d)) for b, d in zip(keep, sentinel)])
        _lib.check(lib.some_session_transcribe_encoded(sess.handle, enc, 3, None, (C.c_void_p * 3)(*[n.handle for n in notes])))
        before = [n.results(sess.timestep) for n in notes]
        assert all(b[0] for b in before)

        def untouched():
            for n, b in zip(notes, before):
                ranges, res = n.results(sess.timestep)
                assert ranges == b[0]
                assert_same_notes(res, b[1])

        def call(datas, handles):
            bufs = [C.create_string_buffer(d, max(len(d), 1)) for d in datas]
            e = (_lib.Encoded * len(datas))(*[_lib.Encoded(C.cast(b, C.c_void_p), len(d)) for b, d in zip(bufs, datas)])
            rc = lib.some_session_transcribe_encoded(sess.handle, e, len(datas), None, (C.c_void_p * len(handles))(*handles))
            return rc, lib.some_last_error().decode()

        h = [n.handle for n in notes]
        cases = [
            ([good, b''], h[:2], 'item 1 is NULL or empty'),
            ([good, good], [h[0], h[0]], 'item 1 shares its some_notes with item 0'),
            ([good, b'OggS' + bytes(60)], h[:2], r'item 1: not a RIFF/WAVE file \(Ogg\)'),
            ([good, good, wav_file(np.zeros(2, np.float32), 96000, 's16')], h, 'item 2: .*too small to resample'),
            ([good, wav_file(np.zeros(3000, np.float32), 2000000, 's16')], h[:2], 'item 1:'),
        ]
        for datas, handles, msg in cases:
            rc, err = call(datas, handles)
            assert rc != 0 and re.search(msg, err), (msg, err)
            untouched()
        # a corrupt FLAC stream: the item's index and FlacBatch's text, no output written; the next call succeeds
        flac = mixed[6][1].read_bytes()
        rec = audio.parse_flac(flac, 'f')
        bad = bytearray(flac)
        bad[rec.audio_offset + 5000] ^= 0x55
        with pytest.raises(ValueError) as py:
            audio.FlacBatch([audio.parse_flac(bytes(bad), 'f')], 'cuda')
        rc, err = call([good, bytes(bad), good], h)
        assert rc != 0 and err == 'some_session_transcribe_encoded: item 1: ' + str(py.value)[len('f: '):]
        untouched()
        [again] = sess.transcribe_encoded([sentinel[0]])
        assert again[1] == before[0][0]
        assert_same_notes(again[2], before[0][1])
    finally:
        for n in notes:
            n.close()


def test_threads_mix_encoded_calls_and_stream_pushes(model, mixed):
    kind, ins, path, sess = model
    files = [p for _, p in mixed[:6]]
    want = sess.transcribe_encoded(files)
    wave = synth.synth_waveform(5, seconds=20.0, silence_gaps=True)
    want_stream = sess.transcribe_sliced(wave)
    errors, results = [], {}

    def enc(t):
        try:
            for r in range(2):
                results[(t, r)] = sess.transcribe_encoded(files[t::2])
        except Exception as e:          # noqa: BLE001
            errors.append(e)

    def push():
        try:
            chunks = [[], [], []]
            with sess.stream() as st:
                for a in range(0, len(wave), 22050):
                    for k, v in enumerate(st.push(wave[a:a + 22050])):
                        chunks[k] += v
                for k, v in enumerate(st.finish()):
                    chunks[k] += v
            results['stream'] = chunks
        except Exception as e:          # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=enc, args=(0,)), threading.Thread(target=enc, args=(1,)), threading.Thread(target=push)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for t in (0, 1):
        for r in range(2):
            for g, w in zip(results[(t, r)], want[t::2]):
                assert g[:2] == w[:2]
                assert_same_notes(g[2], w[2])
    offs, ranges, notes = results['stream']
    assert ranges == want_stream[1]
    assert_same_notes(notes, want_stream[2])


# ---------------------------------------------------------------------------------------------- the example
def test_some_infer_writes_infer_py_midi(model, tmp_path):
    kind, ins, path, sess = model
    assert EXAMPLE.is_file()
    files = {'song.wav': wav_file(stereo(31, 40.0, 48000), 48000, 's24'),
             'song.take2.flac': flac_file(stereo(32, 30.0, 44100), 44100, 16, channel_mode='mid_side')}
    slicer = Slicer(44100, max_sil_kept=1000)
    for name, data in files.items():
        src = tmp_path / name
        src.write_bytes(data)
        r = subprocess.run([str(EXAMPLE), str(path), str(src)], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        out = src.with_suffix('.mid')
        assert r.stdout.strip() == f"MIDI file saved at: '{out}'"
        got = out.read_bytes()
        # infer.py's flow: librosa.load at the model's rate, the Slicer, plugin.infer, build_midi_file
        y, _ = audio.load(src, sr=44100)
        chunks = slicer.slice(y)
        offsets = [c['offset'] for c in chunks]
        segments = ins.infer([c['waveform'] for c in chunks])
        assert got == midi.build_midi_file(offsets, segments, 120).to_bytes()
        n = nsess.Notes()
        try:
            enc = (_lib.Encoded * 1)(_lib.Encoded(C.cast(C.create_string_buffer(data, len(data)), C.c_void_p), len(data)))
            _lib.check(sess.lib.some_session_transcribe_encoded(sess.handle, enc, 1, None, (C.c_void_p * 1)(n.handle)))
            size = C.c_size_t()
            _lib.check(sess.lib.some_notes_midi(n.handle, sess.sample_rate, sess.timestep, 120.0, None, 0, C.byref(size)))
            buf = (C.c_uint8 * size.value)()
            _lib.check(sess.lib.some_notes_midi(n.handle, sess.sample_rate, sess.timestep, 120.0, buf, size.value, C.byref(size)))
            assert bytes(buf) == got
        finally:
            n.close()
        r = subprocess.run([str(EXAMPLE), str(path), str(src), '--midi', str(tmp_path / 'o.mid'), '--tempo', '90.5'],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        assert (tmp_path / 'o.mid').read_bytes() == midi.build_midi_file(offsets, segments, 90.5).to_bytes()
