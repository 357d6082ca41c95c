"""Frame curves of the native session on the H100 (some_notes_set_frames / some_notes_get_frames, csrc/session.cu), bit for bit:
- against the decode the notes come from: the engine the model file was exported from gives the probabilities and bounds,
  and the oracle's restatements of decode_gaussian_blurred_probs / the quantized argmax and decode_bounds_to_alignment
  (pinned to the reference by tests/test_oracle_golden.py) give the curves;
- the curves decode, through the oracle's decode_note_sequence, to exactly the session's notes, in every test;
- frames off is unchanged: the same notes, and the step downloads the bytes it downloaded before;
- every call kind (clips, sliced, encoded WAV / FLAC / AIFF, PCM and encoded streams, peeks) at 44.1, 48 and 22.05 kHz,
  two replicas, threads mixing frames on and off, the refusals and the C example."""
import ctypes as C
import json
import pathlib
import subprocess
import threading
import time

import numpy as np
import pytest
import torch

from oracle import decode as odecode
from some_b200 import _lib, audio, export, plugin, synth
from some_b200 import session as nsess

import test_gpu_aiff as gaiff
import test_gpu_encoded as ge

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent
SR, HOP = 44100, 512
PLUGINS = {'two_head': plugin.MIDIExtractionInference, 'quant_two_head': plugin.QuantizedMIDIExtractionInference,
           'midi_conformer': plugin.MIDIExtractionInference}


def open_model(kind, d):
    config = synth.named_config(kind)
    ckpt = synth.write_checkpoint(d, config, seed=1234)
    s = nsess.Session(export.export(ckpt), 0)
    s.kind, s.path, s.config = kind, ckpt.with_suffix('.somemodel'), config
    s.ins = PLUGINS[kind](config=config, model_path=ckpt, device='cuda:0')
    return s


@pytest.fixture(scope='module', params=list(PLUGINS))
def every_model(request, tmp_path_factory):
    s = open_model(request.param, tmp_path_factory.mktemp(request.param))
    yield s
    s.close()


@pytest.fixture(scope='module', params=['two_head', 'quant_two_head'])
def sess(request, tmp_path_factory):
    s = open_model(request.param, tmp_path_factory.mktemp(request.param))
    yield s
    s.close()


def assert_same_notes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g['note_midi'].shape == w['note_midi'].shape
        np.testing.assert_array_equal(g['note_midi'].view(np.uint32), w['note_midi'].view(np.uint32))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        np.testing.assert_array_equal(np.asarray(g['note_dur']).view(np.uint64), np.asarray(w['note_dur']).view(np.uint64))


def assert_same_curves(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g.midi.view(np.uint32), w.midi.view(np.uint32))
        np.testing.assert_array_equal(g.rest, w.rest)
        np.testing.assert_array_equal(g.bound.view(np.uint32), w.bound.view(np.uint32))
        np.testing.assert_array_equal(g.note_index, w.note_index)


def check_consistent(s, notes, curves, lens=None):
    """Each clip's curves have 1 + len // hop frames and decode (decode_note_sequence) to exactly its notes."""
    assert len(notes) == len(curves)
    for k, (n, c) in enumerate(zip(notes, curves)):
        if lens is not None:
            assert c.midi.shape == c.rest.shape == c.bound.shape == c.note_index.shape == (1 + lens[k] // HOP,)
        values = c.midi.astype(np.int64) if s.quantized else c.midi
        midi, dur, mask = odecode.decode_note_sequence_vec(c.note_index.astype(np.int64), values, ~c.rest)
        np.testing.assert_array_equal(midi.view(np.uint32), n['note_midi'].view(np.uint32))
        np.testing.assert_array_equal(dur, n['note_frames'])
        np.testing.assert_array_equal(~mask, n['note_rest'])
        if c.note_index.size:           # the notes are the runs of equal note_index
            assert c.note_index[0] == 1 and np.all(np.diff(c.note_index) >= 0) and np.all(np.diff(c.note_index) <= 1)


def sliced_frames(s, ranges, curves, y, notes):
    """Every chunk's curves equal transcribe(frames=True) on its samples of y (the recording at the model's rate)."""
    for k in range(0, len(ranges), 64):
        want_n, want_c = s.transcribe([y[a:b] for a, b in ranges[k:k + 64]], frames=True)
        assert_same_notes(notes[k:k + 64], want_n)
        assert_same_curves(curves[k:k + 64], want_c)
    check_consistent(s, notes, curves, [b - a for a, b in ranges])


# ---------------------------------------------------------------------------------------------- 1, 2, 3: against the decode
def test_curves_equal_the_reference_decode(every_model):
    s = every_model
    cfg = s.config
    clips = [synth.synth_waveform(8100 + i, seconds=sec) for i, sec in enumerate((0.01, 1.7, 10.0, 30.0, 60.0))]
    clips.append(np.zeros(10 * SR, np.float32))
    assert 1 + clips[0].shape[0] // HOP == 1 and 1 + clips[4].shape[0] // HOP > 2048
    notes, curves = s.transcribe(clips, frames=True)
    want = s.ins.model.infer(clips, quantized=s.quantized, return_intermediates=True)
    assert_same_notes(notes, want)
    assert_same_notes(s.transcribe(clips), notes)                       # frames off: the same notes
    for c, w in zip(curves, want):
        probs, bounds = w['probs'], w['bounds']
        if s.quantized:                                                  # me_quant_infer.py:28-31
            arg = probs.argmax(axis=-1)
            values, rest = np.clip(arg, 0, 127).astype(np.float32), arg == 128
        else:
            values, rest = odecode.decode_gaussian_blurred_probs_vec(probs, cfg['midi_min'], cfg['midi_max'],
                                                                     cfg['midi_prob_deviation'], cfg['rest_threshold'])
        np.testing.assert_array_equal(c.midi.view(np.uint32), values.view(np.uint32))
        np.testing.assert_array_equal(c.rest, rest)
        np.testing.assert_array_equal(c.bound.view(np.uint32), bounds.view(np.uint32))
        np.testing.assert_array_equal(c.note_index, odecode.decode_bounds_to_alignment(bounds))
    check_consistent(s, notes, curves, [x.shape[0] for x in clips])
    assert s.transcribe([], frames=True) == ([], [])


def download_bytes(fn):
    """The device-to-host copy bytes of fn(), from a torch.profiler trace."""
    import tempfile
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = pathlib.Path(d) / 'trace.json'
        prof.export_chrome_trace(str(path))
        events = json.loads(path.read_text())['traceEvents']
    copies = [e for e in events if e.get('cat') == 'gpu_memcpy' and 'DtoH' in e.get('name', '')]
    return sum(int(e['args']['bytes']) for e in copies), len(copies)


def test_frames_off_downloads_what_it_did(sess):
    """One pipeline chunk of B clips and M frames: the notes slab is align16(4 B + 9 M) bytes in one copy, and the curves add
    align16(13 M) to that same copy only when asked for."""
    clips = [synth.synth_waveform(8200 + i, seconds=sec) for i, sec in enumerate((3.0, 10.0, 7.7))]
    m = sum(1 + x.shape[0] // HOP for x in clips)
    al = lambda b: (b + 15) & ~15
    sess.transcribe(clips, frames=True)                                  # the buffers are grown outside the traces
    off = download_bytes(lambda: sess.transcribe(clips))
    on = download_bytes(lambda: sess.transcribe(clips, frames=True))
    assert off == (al(4 * 3 + 9 * m), 1)
    assert on == (al(4 * 3 + 9 * m) + al(13 * m), 1)


# ---------------------------------------------------------------------------------------------- 4: every call kind
def model_rate(x, rate):
    return x if rate == SR else audio.resample(x, rate, SR)


@pytest.mark.parametrize('rate', [44100, 48000, 22050])
def test_sliced_and_streams(sess, rate):
    x = synth.synth_waveform(8300 + rate % 97, seconds=60.0, sr=rate, silence_gaps=True)
    y = model_rate(x, rate)
    offsets, ranges, notes, curves = sess.transcribe_sliced(x, rate, frames=True)
    assert len(ranges) > 5
    assert sess.transcribe_sliced(x, rate)[1] == ranges
    assert_same_notes(sess.transcribe_sliced(x, rate)[2], notes)
    sliced_frames(sess, ranges, curves, y, notes)
    # a PCM stream, with frame-enabled peeks after some pushes: its chunks are those of the sliced call, curves included,
    # and every peek's curves are transcribe's on its open region
    rng = np.random.default_rng(rate)
    got_r, got_n, got_c, peeks = [], [], [], []
    with sess.stream(rate) as st:
        a = 0
        while a < x.shape[0]:
            m = int(rng.integers(rate // 50, rate))
            _, r, n, c = st.push(x[a:a + m], frames=True)
            got_r += r
            got_n += n
            got_c += c
            a += m
            if rng.random() < 0.3:
                _, pr, pn, pc = st.peek(frames=True)
                peeks += list(zip(pr, pn, pc))
        _, r, n, c = st.finish(frames=True)
        got_r += r
        got_n += n
        got_c += c
    assert got_r == ranges
    assert_same_notes(got_n, notes)
    assert_same_curves(got_c, curves)
    assert len(peeks) > 3
    pr, pn, pc = zip(*peeks)
    sliced_frames(sess, list(pr), list(pc), y, list(pn))


@pytest.mark.parametrize('rate', [44100, 48000, 22050])
def test_encoded_files_and_byte_streams(sess, rate, tmp_path):
    x = synth.synth_waveform(8400 + rate % 89, seconds=40.0, sr=rate, silence_gaps=True) * np.float32(0.9)
    files = {'wav': ge.wav_file(x, rate, 's16'), 'flac': ge.flac_file(x, rate, 16),
             'aiff': gaiff.aiff_s16(gaiff.quantise16(x), rate)}
    results = sess.transcribe_encoded(list(files.values()), frames=True)
    plain = sess.transcribe_encoded(list(files.values()))
    for (name, data), (_, ranges, notes, curves), p in zip(files.items(), results, plain):
        assert p[1] == ranges and len(ranges) > 3
        assert_same_notes(p[2], notes)
        path = tmp_path / f'x.{name}'
        path.write_bytes(data)
        z, zr = audio.load(path, sr=None)
        sliced_frames(sess, ranges, curves, model_rate(z, zr), notes)
        # the same file pushed as bytes: the same chunks and curves; frame-enabled peeks do not change them
        got_r, got_n, got_c = [], [], []
        with sess.stream_encoded() as st:
            for a in range(0, len(data), 50000):
                _, r, n, c = st.push(data[a:a + 50000], frames=True)
                got_r += r
                got_n += n
                got_c += c
                st.peek(frames=True)
            _, r, n, c = st.finish(frames=True)
        assert got_r + r == ranges
        assert_same_notes(got_n + n, notes)
        assert_same_curves(got_c + c, curves)


def test_many_calls_mix_frames_on_and_off(sess):
    """push_many, push_bytes_many and peek_many: frames on gives the single calls' curves; frames off the same notes."""
    rates = [44100, 48000, 22050, 44100]
    xs = [synth.synth_waveform(8500 + k, seconds=30.0, sr=r, silence_gaps=True) for k, r in enumerate(rates)]
    logs = []
    for frames in (True, False):
        opened = [sess.stream(r) for r in rates]
        log = []
        try:
            for a in range(0, 30, 3):
                log.append(sess.push_many([(st, x[a * r:(a + 3) * r]) for st, x, r in zip(opened, xs, rates)], frames=frames))
                log.append(sess.peek_many(opened, frames=frames))
            log.append(sess.push_many([(st, x[:0]) for st, x in zip(opened, xs)], finish=[True] * 4, frames=frames))
        finally:
            for st in opened:
                st.close()
        logs.append(log)
    chunks = 0
    for on, off in zip(*logs):
        for a, b in zip(on, off):
            assert len(a) == 4 and len(b) == 3 and a[1] == b[1]
            assert_same_notes(a[2], b[2])
            check_consistent(sess, a[2], a[3], [q - p for p, q in a[1]])
            chunks += len(a[1])
    assert chunks > 20
    data = [ge.wav_file(x * np.float32(0.9), r, 's16') for x, r in zip(xs, rates)]
    encs = [sess.stream_encoded() for _ in data]
    try:
        got = [[] for _ in data]
        for a in range(0, max(map(len, data)), 1 << 18):
            for k, res in enumerate(sess.push_bytes_many([(st, d[a:a + (1 << 18)]) for st, d in zip(encs, data)], frames=True)):
                got[k].append(res)
        for k, res in enumerate(sess.push_bytes_many([(st, b'') for st in encs], finish=[True] * len(encs), frames=True)):
            got[k].append(res)
    finally:
        for st in encs:
            st.close()
    for k, (d, g) in enumerate(zip(data, got)):
        [(_, ranges, notes, curves)] = sess.transcribe_encoded([d], frames=True)
        assert [r for e in g for r in e[1]] == ranges
        assert_same_curves([c for e in g for c in e[3]], curves)


# ---------------------------------------------------------------------------------------------- 5: devices and threads
def test_two_replicas_give_the_one_replica_curves(sess):
    pair = nsess.Session(sess.path, [0, 0])
    try:
        clips = [synth.synth_waveform(8600 + i, seconds=4.0 + 3 * i) for i in range(12)]
        x = synth.synth_waveform(8650, seconds=120.0, silence_gaps=True)
        for s in (sess, pair):
            s.got = (s.transcribe(clips, frames=True), s.transcribe_sliced(x, frames=True))
            with s.stream(48000) as st:
                z = synth.synth_waveform(8651, seconds=20.0, sr=48000, silence_gaps=True)
                s.got += (st.push(z[:15 * 48000], frames=True), st.peek(frames=True), st.finish(frames=True))
        (n1, c1), *rest1 = sess.got
        (n2, c2), *rest2 = pair.got
        assert_same_notes(n1, n2)
        assert_same_curves(c1, c2)
        for a, b in zip(rest1, rest2):
            assert a[1] == b[1]
            assert_same_notes(a[2], b[2])
            assert_same_curves(a[3], b[3])
        assert len(rest1[0][1]) > 5
    finally:
        pair.close()


def test_threads_sharing_steps_get_what_they_get_alone(sess):
    n = 8
    inputs = [[synth.synth_waveform(8700 + 10 * t + i, seconds=2.0 + i) for i in range(4)] for t in range(n)]
    frames = [t % 2 == 0 for t in range(n)]
    want = [sess.transcribe(x, frames=f) for x, f in zip(inputs, frames)]
    got, errors = [None] * n, []

    def work(t):
        try:
            got[t] = sess.transcribe(inputs[t], frames=frames[t])
        except Exception as e:            # noqa: BLE001  (reported below)
            errors.append(e)

    before = sess.stats()
    holder = threading.Thread(target=sess.transcribe, args=([synth.synth_waveform(8799, seconds=600.0)] * 4,))
    holder.start()
    deadline = time.monotonic() + 120
    while sess.stats()['calls'] == before['calls']:
        assert time.monotonic() < deadline
        time.sleep(0.0005)
    threads = [threading.Thread(target=work, args=(t,)) for t in range(n)]
    for th in threads:
        th.start()
    for th in threads + [holder]:
        th.join()
    assert not errors, errors
    for t in range(n):
        if frames[t]:
            assert_same_notes(got[t][0], want[t][0])
            assert_same_curves(got[t][1], want[t][1])
        else:
            assert isinstance(got[t], list)
            assert_same_notes(got[t], want[t])
    after = sess.stats()
    assert after['max_calls'] > 1 and after['steps'] - before['steps'] < after['calls'] - before['calls']


# ---------------------------------------------------------------------------------------------- 6: refusals
def test_refusals(sess):
    lib = sess.lib
    notes = nsess.Notes()
    try:
        t, p = C.c_int(-1), C.c_void_p()
        get = lambda h, clip: _lib.check(lib.some_notes_get_frames(h, clip, C.byref(t), C.byref(p), None, None, None))
        sess.transcribe([synth.synth_waveform(8800, seconds=2.0)], notes)              # frames off
        assert lib.some_notes_clips(notes.handle) == 1
        with pytest.raises(_lib.SomeB200Error, match='filled with frames off'):
            get(notes.handle, 0)
        with pytest.raises(_lib.SomeB200Error, match='clip 1 out of range'):
            get(notes.handle, 1)
        notes.set_frames(True)                                                        # asks, but holds the frames-off fill
        with pytest.raises(_lib.SomeB200Error, match='filled with frames off'):
            get(notes.handle, 0)
        with pytest.raises(_lib.SomeB200Error, match='null pointer'):
            get(None, 0)
        assert t.value == -1
        sess.transcribe([synth.synth_waveform(8800, seconds=2.0)], notes, frames=True)
        get(notes.handle, 0)
        assert t.value == 1 + 2 * SR // HOP
        with pytest.raises(_lib.SomeB200Error, match='clip -1 out of range'):
            get(notes.handle, -1)
        assert _lib.check(lib.some_notes_get_frames(notes.handle, 0, None, None, None, None, None)) is None
    finally:
        notes.close()


# ---------------------------------------------------------------------------------------------- 7: the example
def test_c_example_prints_the_frames(sess, tmp_path):
    if sess.kind != 'two_head':
        pytest.skip('one model kind is enough for the example')
    example = REPO / 'examples' / 'some_stream'
    wav = tmp_path / 'rec.wav'
    synth.write_wav16(wav, synth.synth_waveform(8900, seconds=30.0, silence_gaps=True))
    data = wav.read_bytes()
    run = lambda *args: subprocess.run([str(example), *args, str(sess.path), '-'], input=data, capture_output=True,
                                       timeout=300)
    plain, framed, both = run(), run('--frames'), run('--frames', '--peek', '700')
    for r in (plain, framed, both):
        assert r.returncode == 0, r.stderr
    lines = framed.stdout.decode().splitlines()
    assert [ln for ln in lines if not ln.startswith('f ')] == plain.stdout.decode().splitlines()
    # the same pushes from Python: 64 KB reads, then the finish; a peek once another 700 ms is in
    want, want_peek, next_ms = [], [], 700

    def lines_of(ranges, curves, prefix):
        return ['%sf %.17g %.9g %d %.9g %d' % (prefix, (a + t * HOP) / SR, c.midi[t], c.rest[t], c.bound[t], c.note_index[t])
                for (a, _), c in zip(ranges, curves) for t in range(c.midi.shape[0])]

    with sess.stream_encoded() as st:
        for a in range(0, len(data), 1 << 16):
            _, r, _, c = st.push(data[a:a + (1 << 16)], frames=True)
            want += lines_of(r, c, '')
            received, rate = st.info()['received'], st.meta()['rate']
            if rate and received * 1000 >= next_ms * rate:
                _, pr, _, pc = st.peek(frames=True)
                want_peek += lines_of(pr, pc, '~ ')
                next_ms = (received * 1000 // rate // 700 + 1) * 700
        _, r, _, c = st.finish(frames=True)
        want += lines_of(r, c, '')
    got = [ln for ln in lines if ln.startswith('f ')]
    assert len(got) > 1000 and got == want
    for ln in got[:50]:
        _, tm, m, rest, b, k = ln.split()
        float(tm), float(m), int(rest), float(b), int(k)
    blines = both.stdout.decode().splitlines()
    assert [ln for ln in blines if ln.startswith('f ')] == want
    assert [ln for ln in blines if ln.startswith('~ f ')] == want_peek and len(want_peek) > 100
