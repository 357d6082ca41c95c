"""Calls from several threads on one native session, on the H100 (csrc/session.cu: submit / take_step).  Calls that queue
behind a running step run together as one GPU step, and each caller gets exactly what the same call gives alone on a fresh
session: the same chunks and ranges and bit-identical notes, for every kind of call, on [0], [0, 0] and, with two GPUs, [0, 1].
The merges themselves are checked with some_session_get_stats: a long call holds the session while short calls queue behind it,
and the waits poll the stats, so no test depends on how long anything takes."""
import struct
import threading
import time

import numpy as np
import pytest
import torch

from oracle import aiff as oa
from oracle import flac as of
from some_b200 import _lib, export, synth
from some_b200 import session as nsess
from some_b200.slicer import slicer_params

pytestmark = pytest.mark.gpu
LISTS = [(0,), (0, 0), (0, 1)]


@pytest.fixture(scope='module')
def path(tmp_path_factory):
    d = tmp_path_factory.mktemp('two_head')
    return export.export(synth.write_checkpoint(d, synth.named_config('two_head'), seed=1234))


@pytest.fixture(scope='module', params=LISTS, ids=lambda d: ','.join(map(str, d)))
def sess(request, path):
    devices = list(request.param)
    if max(devices) >= torch.cuda.device_count():
        pytest.skip(f'{max(devices) + 1} GPUs needed, {torch.cuda.device_count()} visible')
    s = nsess.Session(path, devices)
    yield s
    s.close()


def wav16(x, rate):
    raw = np.clip(np.round(x * 32768), -32768, 32767).astype('<i2').tobytes()
    fmt = struct.pack('<HHIIHH', 1, 1, rate, rate * 2, 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def flac16(x, rate, **kw):
    v = np.clip(np.round(x * 32768), -32768, 32767).astype(np.int64)
    return of.encode(v, rate=rate, bps=16, subframe={'type': 'fixed', 'order': 2}, **kw)


def aiff16(x, rate):
    v = np.clip(np.round(x * 32768), -32768, 32767).astype('>i2').tobytes()
    return oa.aiff_bytes(v, 1, 16, float(rate))


def same_notes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g['note_midi'].view(np.uint32), w['note_midi'].view(np.uint32))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        np.testing.assert_array_equal(g['note_frames'], w['note_frames'])


def same(got, want):
    """Results of one call: (offsets, ranges, notes) triples, or lists of them, or (ranges, notes) of a clip call."""
    if isinstance(got, list):
        assert len(got) == len(want)
        for g, w in zip(got, want):
            same(g, w)
        return
    assert len(got) == len(want)
    for g, w in zip(got[:-1], want[:-1]):
        assert g == w
    same_notes(got[-1], want[-1])


def clips_call(s, clips, notes=None):
    own = notes is None
    notes = notes or nsess.Notes()
    try:
        s.transcribe(clips, notes)
        return notes.results(s.timestep)
    finally:
        if own:
            notes.close()


def script(t, rng):
    """Thread t's calls: a list of functions of a session, each returning one call's results (a stream's calls share the stream
    they open)."""
    kind = t % 5
    if kind == 0:
        return [lambda s, c=[synth.synth_waveform(1000 * t + i, seconds=float(rng.uniform(0.3, 8))) for i in range(k)]:
                clips_call(s, c) for k in (1, int(rng.integers(2, 5)))]
    if kind == 1:
        calls = []
        for i in range(2):
            rate = (44100, 48000)[(t + i) % 2]
            params = None if (t // 5 + i) % 2 == 0 else slicer_params(threshold=-35., min_length=3000, max_sil_kept=500)
            x = synth.synth_waveform(1000 * t + i, seconds=float(rng.uniform(10, 40)), sr=rate, silence_gaps=True)
            calls.append(lambda s, x=x, rate=rate, params=params: s.transcribe_sliced(x, rate, params))
        return calls
    if kind == 2:
        calls = []
        for i in range(2):
            items = []
            for j in range(int(rng.integers(1, 5))):
                rate = (44100, 48000, 22050)[(t + j) % 3]
                x = synth.synth_waveform(1000 * t + 10 * i + j, seconds=float(rng.uniform(2, 25)), sr=rate, silence_gaps=True)
                items.append((wav16, flac16, aiff16)[(t + i + j) % 3](x * np.float32(0.8), rate))
            calls.append(lambda s, items=items: s.transcribe_encoded(items))
        return calls
    rate = (44100, 48000)[t % 2]
    x = synth.synth_waveform(1000 * t, seconds=float(rng.uniform(15, 40)), sr=rate, silence_gaps=True)
    data = x if kind == 3 else (wav16, flac16, aiff16)[t % 3](x * np.float32(0.8), rate)
    cuts = np.sort(rng.integers(1, len(data), size=int(rng.integers(3, 9))))
    pieces = np.split(x, cuts) if kind == 3 else [data[a:b] for a, b in zip([0, *cuts], [*cuts, len(data)])]
    state = {}

    def push(s, k):
        if k == 0:
            state[s] = s.stream(rate) if kind == 3 else s.stream_encoded()
        return state[s].push(pieces[k])

    def finish(s):
        st = state.pop(s)
        try:
            return st.finish()
        finally:
            st.close()
    return [lambda s, k=k: push(s, k) for k in range(len(pieces))] + [finish]


def run_threads(s, scripts):
    """Each script on a thread of its own, all started together; returns every thread's results."""
    results, errors = [None] * len(scripts), []
    go = threading.Barrier(len(scripts))

    def work(t):
        try:
            go.wait()
            results[t] = [call(s) for call in scripts[t]]
        except Exception as e:                                  # noqa: BLE001  (reported below)
            errors.append(e)
    threads = [threading.Thread(target=work, args=(t,)) for t in range(len(scripts))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    return results


@pytest.mark.parametrize('n_threads', [8, 32])
def test_threads_get_what_each_call_gives_alone(sess, path, n_threads):
    rng = np.random.default_rng(n_threads)
    scripts = [script(t, rng) for t in range(n_threads)]
    alone = nsess.Session(path, 0)
    try:
        want = [[call(alone) for call in sc] for sc in scripts]
    finally:
        alone.close()
    before = sess.stats()
    got = run_threads(sess, scripts)
    for g, w in zip(got, want):
        same(g, w)
    after = sess.stats()
    assert after['calls'] - before['calls'] == sum(len(sc) for sc in scripts)
    assert after['steps'] <= after['calls'] and after['queued'] == 0


# ---- merges, observed through the stats: a long call holds the session while the calls under test queue behind it

def wait_for(s, pred, what, timeout=120.0):
    end = time.monotonic() + timeout
    while not pred(s.stats()):
        assert time.monotonic() < end, f'timed out waiting for {what}: {s.stats()}'
        time.sleep(0.0005)


@pytest.fixture(scope='module')
def long_wave():
    return synth.synth_waveform(4242, seconds=1200.0, silence_gaps=True)


@pytest.fixture(scope='module')
def long_items(long_wave):
    """Three 20-minute WAV files: one encoded call that keeps a step running while other calls queue."""
    return [wav16(long_wave * np.float32(0.8), 44100)] * 3


class Behind:
    """Runs the long call on a thread, then each queued call on a thread of its own, in order: each one is started once the
    previous one shows in stats['queued'].  join() returns every call's result or exception and the stats before and after."""

    def __init__(self, s, long_items):
        self.s, self.threads, self.out = s, [], {}
        self.before = s.stats()
        self._start('long', lambda: s.transcribe_encoded(long_items))
        wait_for(s, lambda st: st['calls'] == self.before['calls'] + 1 and st['queued'] == 0, 'the long call to run')
        self.queued = 0

    def _start(self, name, fn):
        def work():
            try:
                self.out[name] = fn()
            except Exception as e:                              # noqa: BLE001  (returned to the test)
                self.out[name] = e
        th = threading.Thread(target=work)
        th.start()
        self.threads.append(th)

    def queue(self, name, fn):
        self._start(name, fn)
        self.queued += 1
        wait_for(self.s, lambda st, q=self.queued: st['queued'] == q, f'call {name} to queue')

    def join(self):
        for th in self.threads:
            th.join()
        return self.out, self.before, self.s.stats()


def short_items(n):
    return [[wav16(synth.synth_waveform(60 + i, seconds=6.0 + i, silence_gaps=True), 44100)] for i in range(n)]


def test_calls_queued_behind_a_step_share_the_next(sess, path, long_items):
    n = 6
    items = short_items(n)
    want = [sess.transcribe_encoded(it) for it in items]
    x = synth.synth_waveform(77, seconds=30.0, sr=48000, silence_gaps=True)
    want_sliced = sess.transcribe_sliced(x, 48000)
    b = Behind(sess, long_items)
    for i in range(n):
        b.queue(i, lambda it=items[i]: sess.transcribe_encoded(it))
    b.queue('sliced', lambda: sess.transcribe_sliced(x, 48000))   # a sliced call joins encoded calls
    out, before, after = b.join()
    assert after['steps'] - before['steps'] == 2
    assert after['max_calls'] >= n + 1
    for i in range(n):
        same(out[i], want[i])
    same(out['sliced'], want_sliced)


def test_clip_and_stream_calls_merge(sess, long_items):
    clips = [[synth.synth_waveform(90 + i, seconds=1.0 + i)] for i in range(4)]
    want = [clips_call(sess, c) for c in clips]
    waves = [synth.synth_waveform(95 + i, seconds=12.0, silence_gaps=True) for i in range(4)]
    want_streams = []
    for w in waves:
        with sess.stream() as st:
            want_streams.append([st.push(w[:300000]), st.finish()])
    streams = [sess.stream() for _ in waves]
    try:
        for st, w in zip(streams, waves):
            st.push(w[:300000])
        b = Behind(sess, long_items)
        for i, c in enumerate(clips):
            b.queue(('clip', i), lambda c=c: clips_call(sess, c))
        for i, st in enumerate(streams):
            b.queue(('stream', i), st.finish)
        out, before, after = b.join()
    finally:
        for st in streams:
            st.close()
    assert after['steps'] - before['steps'] == 3               # the long call, the clip calls, the stream calls
    for i in range(4):
        same(out[('clip', i)], want[i])
        same(out[('stream', i)], want_streams[i][1])


def test_a_refused_call_fails_alone(sess, long_items):
    good = short_items(3)
    want = [sess.transcribe_encoded(it) for it in good]
    flac = flac16(synth.synth_waveform(31, seconds=20.0, silence_gaps=True), 44100)
    bad = bytearray(flac)
    bad[len(flac) // 2] ^= 0x55
    bad = bytes(bad)
    odd_rate = wav16(np.zeros(3000, np.float32), 2000000)
    alone = {}
    for name, items in (('bad', [good[0][0], bad]), ('rate', [odd_rate])):
        with pytest.raises(_lib.SomeB200Error) as e:
            sess.transcribe_encoded(items)
        alone[name] = str(e.value)
    assert 'item 1:' in alone['bad'] and 'item 0:' in alone['rate']
    b = Behind(sess, long_items)
    b.queue(0, lambda: sess.transcribe_encoded(good[0]))
    b.queue('bad', lambda: sess.transcribe_encoded([good[0][0], bad]))
    b._start('rate', lambda: sess.transcribe_encoded([odd_rate]))  # refused before it queues
    b.queue(1, lambda: sess.transcribe_encoded(good[1]))
    b.queue(2, lambda: sess.transcribe_encoded(good[2]))
    out, before, after = b.join()
    assert after['steps'] - before['steps'] == 2 and after['calls'] - before['calls'] == 5
    assert isinstance(out['bad'], _lib.SomeB200Error) and str(out['bad']) == alone['bad']
    assert isinstance(out['rate'], _lib.SomeB200Error) and str(out['rate']) == alone['rate']
    for i in range(3):
        same(out[i], want[i])
    same(sess.transcribe_encoded(good[1]), want[1])               # still usable


def push_into(st, x, notes):
    """some_stream_push into a Notes of the caller's: two threads pushing one stream each read their own result."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    _lib.check(st.lib.some_stream_push(st.handle, x.ctypes.data, int(x.shape[0]), notes.handle), 'some_stream_push')
    ranges, res = notes.results(st.session.timestep)
    return [a / st.session.sample_rate for a, _ in ranges], ranges, res


def test_calls_on_one_stream_or_one_notes_never_share_a_step(sess, long_items):
    w = synth.synth_waveform(55, seconds=30.0, silence_gaps=True)
    other = synth.synth_waveform(56, seconds=30.0, silence_gaps=True)
    blocks = np.split(w, [400000, 800000])
    with sess.stream() as st:
        want = [st.push(blocks[0]), st.push(blocks[1]), st.push(blocks[2]), st.finish()]
    with sess.stream() as st:
        want_other = st.push(other)
    clips = [synth.synth_waveform(57, seconds=3.0)], [synth.synth_waveform(58, seconds=4.0)]
    want_clips = [clips_call(sess, c) for c in clips]
    st, st2 = sess.stream(), sess.stream()
    shared, n1, n2 = nsess.Notes(), nsess.Notes(), nsess.Notes()
    try:
        got = [st.push(blocks[0])]
        b = Behind(sess, long_items)
        b.queue('s1', lambda: push_into(st, blocks[1], n1))
        b.queue('t', lambda: st2.push(other))
        b.queue('s2', lambda: push_into(st, blocks[2], n2))       # the same stream: a later step, in order
        b.queue('c1', lambda: clips_call(sess, clips[0], shared))
        b.queue('c2', lambda: clips_call(sess, clips[1], shared))  # the same some_notes: a later step
        out, before, after = b.join()
        got += [out['s1'], out['s2'], st.finish()]
        # long; s1 + t; s2; c1; c2 (clips after streams: kinds run as consecutive steps)
        assert after['steps'] - before['steps'] == 5
        same(out['t'], want_other)
        same(got, want)
        same(out['c2'], want_clips[1])
    finally:
        st.close(), st2.close()
        shared.close(), n1.close(), n2.close()


def test_size_bound_and_unknown_length(sess, long_items, long_wave):
    small = short_items(2)
    want = [sess.transcribe_encoded(it) for it in small]
    x = synth.synth_waveform(33, seconds=8.0, silence_gaps=True)
    unknown = flac16(x, 44100, total_samples=0)
    want_unknown = sess.transcribe_encoded([unknown])
    # a call over SOME_SESSION_STEP_SAMPLES (40 minutes at 44.1 kHz) takes no joiner: the step is as large as it is
    big = np.concatenate([long_wave, long_wave])
    assert len(big) > 64 * 30 * 44100
    short = synth.synth_waveform(34, seconds=8.0, silence_gaps=True)
    want_short = sess.transcribe_sliced(short)
    b = Behind(sess, long_items)
    b.queue('big', lambda: sess.transcribe_sliced(big))
    b.queue(0, lambda: sess.transcribe_sliced(short))
    out, before, after = b.join()
    assert after['steps'] - before['steps'] == 3
    same(out[0], want_short)
    # an unknown length takes no joiner and joins no step
    b = Behind(sess, long_items)
    b.queue('unknown', lambda: sess.transcribe_encoded([unknown]))
    b.queue(0, lambda: sess.transcribe_encoded(small[0]))
    b.queue('unknown2', lambda: sess.transcribe_encoded([unknown]))
    b.queue(1, lambda: sess.transcribe_encoded(small[1]))
    out, before, after = b.join()
    assert after['steps'] - before['steps'] == 4                  # long; unknown; 0 + 1; unknown2
    same(out['unknown'], want_unknown), same(out['unknown2'], want_unknown)
    same(out[0], want[0]), same(out[1], want[1])


def test_pdl_settings_do_not_share_a_step(sess, long_items):
    items = short_items(2)
    want = [sess.transcribe_encoded(it) for it in items]
    lib = _lib.load()

    def with_pdl(on, it):
        was = lib.some_set_pdl(on)
        try:
            return sess.transcribe_encoded(it)
        finally:
            lib.some_set_pdl(was)
    b = Behind(sess, long_items)
    b.queue(0, lambda: with_pdl(1, items[0]))
    b.queue(1, lambda: with_pdl(0, items[1]))
    out, before, after = b.join()
    assert after['steps'] - before['steps'] == 3
    same(out[0], want[0]), same(out[1], want[1])
