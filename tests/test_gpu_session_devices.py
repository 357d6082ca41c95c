"""A native session on several devices, on the H100 (csrc/session.cu, some_session_open_devices): for every call, a session on
[0, 0] (two replicas on one GPU), and on [0, 1] and [1, 0] when two GPUs are visible, returns exactly what a session on the
first device returns: the same clips and chunks in the same order, the same sample ranges and bit-identical notes.  The
chunks of each call are split as some_shard_clips assigns them, every replica runs a share, threads may share the session,
and closing it joins its threads."""
import os
import pathlib
import struct
import subprocess
import threading

import numpy as np
import pytest
import torch

from oracle import aiff as oa
from oracle import flac as of
from some_b200 import _lib, export, synth
from some_b200 import session as nsess

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent
LISTS = [(0, 0), (0, 1), (1, 0)]


@pytest.fixture(scope='module', params=['two_head', 'quant_two_head'])
def model(request, tmp_path_factory):
    """(exported model file, a session on device 0)."""
    d = tmp_path_factory.mktemp(request.param)
    path = export.export(synth.write_checkpoint(d, synth.named_config(request.param), seed=1234))
    one = nsess.Session(path, 0)
    yield path, one
    one.close()


@pytest.fixture(scope='module', params=LISTS, ids=lambda d: ','.join(map(str, d)))
def pair(request, model):
    """(the session on the first device, a session on the listed devices)."""
    devices = list(request.param)
    if max(devices) >= torch.cuda.device_count():
        pytest.skip(f'{max(devices) + 1} GPUs needed, {torch.cuda.device_count()} visible')
    path, one = model
    first = one if devices[0] == 0 else nsess.Session(path, devices[0])
    many = nsess.Session(path, devices)
    yield first, many
    many.close()
    if first is not one:
        first.close()


def assert_same_notes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g['note_midi'].shape == w['note_midi'].shape
        np.testing.assert_array_equal(g['note_midi'].view(np.uint32), w['note_midi'].view(np.uint32))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        np.testing.assert_array_equal(g['note_frames'], w['note_frames'])


def assert_same(got, want):
    """(offsets, ranges, notes) triples."""
    assert got[0] == want[0] and got[1] == want[1]
    assert_same_notes(got[2], want[2])


def transcribe(sess, clips):
    notes = nsess.Notes()
    try:
        sess.transcribe(clips, notes)
        return notes.results(sess.timestep)
    finally:
        notes.close()


def assert_split(sess, lengths):
    """The last call's load: the split some_shard_clips makes of these chunk lengths, every replica busy when it can be."""
    r = len(sess.devices)
    owner = nsess.shard_clips(lengths, r)
    want = [(sum(1 for o in owner if o == k), sum(1 + n // 512 for n, o in zip(lengths, owner) if o == k)) for k in range(r)]
    assert sess.load() == want
    if len(lengths) >= r:
        assert all(c > 0 for c, _ in sess.load())


def test_devices(pair, model):
    first, many = pair
    assert len(many.devices) == 2 and many.devices[0] == first.devices[0]
    assert len(first.load()) == 1
    assert (many.sample_rate, many.outdim, many.quantized) == (first.sample_rate, first.outdim, first.quantized)


def test_transcribe(pair):
    first, many = pair
    clips = [synth.synth_waveform(300 + i, seconds=s) for i, s in enumerate((0.4, 3.0, 7.3, 12.0, 1.1, 30.0, 0.02))]
    clips += list(synth.edge_case_waveforms().values())
    clips += [np.zeros(0, np.float32), synth.synth_waveform(77, num_samples=2047), synth.synth_waveform(78, num_samples=513)]
    for batch in (clips, clips[:1], clips[-1:], clips[-3:-2], [clips[3]] * 5):
        want = transcribe(first, batch)
        assert_split(first, [len(c) for c in batch])
        got = transcribe(many, batch)
        assert got[0] == want[0]
        assert_same_notes(got[1], want[1])
        assert_split(many, [len(c) for c in batch])


@pytest.mark.parametrize('rate', [44100, 48000])
def test_transcribe_sliced(pair, rate):
    first, many = pair
    wave = synth.synth_waveform(9002, seconds=300.0, sr=rate, silence_gaps=True)
    want = first.transcribe_sliced(wave, rate)
    got = many.transcribe_sliced(wave, rate)
    assert len(want[1]) >= 20
    assert_same(got, want)
    assert_split(many, [b - a for a, b in want[1]])
    short = synth.synth_waveform(5, seconds=2.0, sr=rate)      # one chunk: one replica runs it
    assert_same(many.transcribe_sliced(short, rate), first.transcribe_sliced(short, rate))
    assert sorted(c for c, _ in many.load()) == [0, 1]


def wav16(x, rate):
    raw = np.clip(np.round(x * 32768), -32768, 32767).astype('<i2').tobytes()
    fmt = struct.pack('<HHIIHH', 1, 1, rate, rate * 2, 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def flac16(x, rate):
    v = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int64)
    return of.encode(v, rate=rate, bps=16, subframe={'type': 'fixed', 'order': 2})


def aiff16(x, rate):
    v = np.clip(np.round(x * 32768), -32768, 32767).astype('>i2').tobytes()
    return oa.aiff_bytes(v, 1, 16, float(rate))


def encoded_items():
    items = []
    for i in range(6):
        rate = (44100, 48000, 22050)[i % 3]
        x = synth.synth_waveform(700 + i, seconds=20.0 + 5 * i, sr=rate, silence_gaps=True) * np.float32(0.8)
        items.append((wav16, flac16, aiff16)[i % 3](x, rate))
    items.append(flac16(synth.synth_waveform(790, seconds=0.5, sr=48000), 48000))
    return items


def test_transcribe_encoded(pair):
    first, many = pair
    items = encoded_items()
    want = first.transcribe_encoded(items)
    got = many.transcribe_encoded(items)
    for g, w in zip(got, want):
        assert_same(g, w)
    assert_split(many, [b - a for _, ranges, _ in want for a, b in ranges])
    bad = items[:2] + [b'RIFF\x10\0\0\0WAVEjunkjunk'] + items[2:3]
    msgs = []
    for sess in (first, many):
        with pytest.raises(_lib.SomeB200Error) as e:
            sess.transcribe_encoded(bad)
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and 'item 2' in msgs[0]
    assert_same(many.transcribe_encoded(items[:1])[0], want[0])          # still usable


def pushes(sess, waves, rates, cuts):
    """Each wave pushed in the pieces its cuts make to a stream of its own, the streams advanced together with push_many and
    finished in the last tick; returns every tick's results."""
    pieces = [np.split(w, c) for w, c in zip(waves, cuts)]
    ticks = max(len(p) for p in pieces)
    streams = [sess.stream(r) for r in rates]
    try:
        return [sess.push_many([(st, p[k] if k < len(p) else p[-1][:0]) for st, p in zip(streams, pieces)],
                               [k == ticks - 1] * len(streams)) for k in range(ticks)]
    finally:
        for st in streams:
            st.close()


def test_streams(pair):
    first, many = pair
    rng = np.random.default_rng(3)
    rates = [44100, 48000, 22050, 44100, 32000]
    waves = [synth.synth_waveform(800 + i, seconds=float(rng.uniform(20, 60)), sr=r, silence_gaps=True)
             for i, r in enumerate(rates)]
    cuts = [sorted(int(x) for x in rng.integers(0, len(w), size=int(rng.integers(3, 12)))) for w in waves]
    want = pushes(first, waves, rates, cuts)
    got = pushes(many, waves, rates, cuts)
    for gt, wt in zip(got, want):
        for g, w in zip(gt, wt):
            assert_same(g, w)
    # one stream, pushed alone at random splits
    w = waves[0]
    outs = []
    for sess in (first, many):
        with sess.stream(44100) as st:
            res = [st.push(piece) for piece in np.split(w, cuts[0])] + [st.finish()]
        outs.append(res)
    for g, wt in zip(*outs[::-1]):
        assert_same(g, wt)


def test_encoded_streams(pair):
    first, many = pair
    items = encoded_items()[:3]
    rng = np.random.default_rng(4)
    cuts = [sorted(int(x) for x in rng.integers(1, len(d), size=6)) for d in items]
    outs = []
    for sess in (first, many):
        streams = [sess.stream_encoded() for _ in items]
        res = []
        try:
            for k in range(7):
                step = [(st, d[(c[k - 1] if k else 0):(c[k] if k < 6 else len(d))]) for st, d, c in zip(streams, items, cuts)]
                res.append(sess.push_bytes_many(step, [k == 6] * len(items)))
        finally:
            for st in streams:
                st.close()
        outs.append(res)
    for gt, wt in zip(*outs[::-1]):
        for g, w in zip(gt, wt):
            assert_same(g, w)


def test_threads_share_a_session(pair):
    first, many = pair
    inputs = [[synth.synth_waveform(500 + 10 * t + i, seconds=2.0 + i) for i in range(6)] for t in range(3)]
    want = [transcribe(first, x) for x in inputs]
    errors, results = [], [[] for _ in inputs]

    def work(t):
        try:
            for _ in range(3):
                results[t].append(transcribe(many, inputs[t]))
        except Exception as e:                                  # noqa: BLE001  (reported below)
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(len(inputs))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t, rs in enumerate(results):
        for r in rs:
            assert r[0] == want[t][0]
            assert_same_notes(r[1], want[t][1])


def thread_count():
    return len(os.listdir('/proc/self/task'))


def test_close_joins_threads_and_reopens(model):
    path, one = model
    clips = [synth.synth_waveform(40 + i, seconds=3.0) for i in range(4)]
    want = transcribe(one, clips)
    nsess.Session(path, [0, 0]).close()                        # the runtime's own threads exist from here on
    before = thread_count()
    for _ in range(2):
        s = nsess.Session(path, [0, 0])
        got = transcribe(s, clips)
        s.close()
        assert thread_count() == before
        assert got[0] == want[0]
        assert_same_notes(got[1], want[1])


def test_examples_take_a_device_list(model, tmp_path):
    path, _ = model
    wav = tmp_path / 'rec.wav'
    synth.write_wav16(wav, synth.synth_waveform(4321, seconds=30.0, silence_gaps=True))
    runs = {}
    for devices in ('0', '0,0'):
        run = subprocess.run([str(REPO / 'examples' / 'some_transcribe'), str(path), str(wav), devices], capture_output=True,
                             text=True, timeout=300)
        assert run.returncode == 0, run.stderr
        runs[devices] = run.stdout
    assert runs['0'] == runs['0,0'] and runs['0'].count('\n') > 10
    bad = subprocess.run([str(REPO / 'examples' / 'some_transcribe'), str(path), str(wav), '0,x'], capture_output=True,
                         text=True, timeout=60)
    assert bad.returncode != 0 and 'device' in bad.stderr
