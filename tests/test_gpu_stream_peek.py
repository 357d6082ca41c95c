"""Stream peeks on the H100 (some_stream_peek*, csrc/session.cu): the provisional notes of a stream's open region [a, b)
equal some_session_transcribe on those model-rate samples bit for bit, for PCM streams at the model's and other rates and for
encoded WAV and FLAC streams; peeks change no chunk; the region never goes back, never overlaps a delivered chunk and no later
chunk begins before it (except the all-silent recording's one chunk); peek_many equals one peek per stream; threads, refusals,
two replicas and the C example."""
import ctypes as C
import pathlib
import subprocess
import threading
import time

import numpy as np
import pytest

from some_b200 import _lib, audio, export, synth
from some_b200 import session as nsess

import test_gpu_encoded as ge

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent
SR = 44100


@pytest.fixture(scope='module', params=['two_head', 'quant_two_head'])
def sess(request, tmp_path_factory):
    d = tmp_path_factory.mktemp(request.param)
    ckpt = synth.write_checkpoint(d, synth.named_config(request.param), seed=1234)
    s = nsess.Session(export.export(ckpt), 0)
    s.kind, s.path = request.param, ckpt.with_suffix('.somemodel')
    yield s
    s.close()


def assert_same_notes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g['note_midi'].shape == w['note_midi'].shape
        np.testing.assert_array_equal(g['note_midi'].view(np.uint32), w['note_midi'].view(np.uint32))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        np.testing.assert_array_equal(g['note_dur'].view(np.uint64), w['note_dur'].view(np.uint64))


def push_sizes(n, rate, rng):
    """A few 1-sample pushes, then 1 ms to 1 s."""
    sizes = [1, 1, 1, 2, 3]
    while sum(sizes) < n:
        sizes.append(int(rng.integers(max(1, rate // 1000), rate + 1)))
    return sizes


def byte_sizes(n, rng):
    """Single bytes over the header, then 1 byte to 128 KB."""
    sizes = [1] * min(300, n)
    while sum(sizes) < n:
        sizes.append(int(rng.integers(1, 1 << 17)))
    return sizes


def pieces_of(x, sizes):
    out, a = [], 0
    for m in sizes:
        out.append(x[a:a + m])
        a += m
    return out


def run(st, pieces, peek=True):
    """Pushes the pieces (a peek right after open and after every push when `peek`), then finishes.  Returns the log: per
    push and for the finish ('chunks', ranges, notes); per peek ('peek', ranges, notes, fixed)."""
    log = []

    def peek_now():
        _, r, nt = st.peek()
        log.append(('peek', r, nt, st.info()['fixed']))

    if peek:
        peek_now()
    for p in pieces:
        _, r, nt = st.push(p)
        log.append(('chunks', r, nt))
        if peek:
            peek_now()
    _, r, nt = st.finish()
    log.append(('chunks', r, nt))
    return log


def chunks_of(log):
    return [e for e in log if e[0] == 'chunks']


def flat(log):
    ranges, notes = [], []
    for e in chunks_of(log):
        ranges += e[1]
        notes += e[2]
    return ranges, notes


def check_peeks_transcribe(sess, log, y):
    """Every peek: one clip [a, fixed) with transcribe's notes for y[a:fixed], or zero clips when nothing is fixed."""
    regions, got = [], []
    for e in log:
        if e[0] != 'peek':
            continue
        _, r, nt, fixed = e
        assert (len(r) == 0) == (fixed == 0), (r, fixed)
        if r:
            [(a, b)] = r
            assert b == fixed and 0 <= a < b <= y.shape[0]
            regions.append((a, b))
            got += nt
    for k in range(0, len(regions), 64):
        want = sess.transcribe([y[a:b] for a, b in regions[k:k + 64]])
        assert_same_notes(got[k:k + 64], want)
    return regions


def check_region(log, keep_samples):
    """a never decreases, is never before the end of a delivered chunk, and no later chunk begins before it; the one
    exception: the all-silent recording's one chunk [0, e), e <= max_sil_kept hops, from the finish."""
    a_max, end_max, exceptions = 0, 0, 0
    all_chunks = [c for e in chunks_of(log) for c in e[1]]
    for i, e in enumerate(log):
        if e[0] == 'peek':
            if not e[1]:
                continue
            a = e[1][0][0]
            assert a >= a_max, 'a went back'
            assert a >= end_max, 'a before a delivered chunk'
            a_max = a
        else:
            for b, c in e[1]:
                if b < a_max:
                    assert i == len(log) - 1 and all_chunks == [(b, c)] and b == 0 and c <= keep_samples, (b, c, a_max)
                    exceptions += 1
                end_max = max(end_max, c)
    return exceptions


def keep_samples():
    f = nsess.slicer_frames(SR)
    return f.max_sil_kept * f.hop_size


def wav_bytes(x, rate):
    return ge.wav_file(x, rate, 's16')


def flac_bytes(x, rate):
    return ge.flac_file(x, rate, 16)


def model_rate(sess, data, tmp_path, name):
    """audio.load(file, sr=None), resampled to the model's rate."""
    p = tmp_path / name
    p.write_bytes(data)
    y, rate = audio.load(p, sr=None)
    return audio.resample(y, rate, SR) if rate != SR else y


def inputs(kind, seed, seconds, tmp_path, sess):
    """(open a stream, its pieces, y at the model's rate, what the whole-recording call gives) for one input kind."""
    rng = np.random.default_rng(seed)
    if kind.startswith('pcm'):
        rate = int(kind[3:])
        x = synth.synth_waveform(seed, seconds=seconds, sr=rate, silence_gaps=True)
        y = x if rate == SR else audio.resample(x, rate, SR)
        return (lambda: sess.stream(rate)), pieces_of(x, push_sizes(x.shape[0], rate, rng)), y, sess.transcribe_sliced(x, rate)
    rate = {'wav': 48000, 'flac': 44100}[kind]
    x = synth.synth_waveform(seed, seconds=seconds, sr=rate, silence_gaps=True) * np.float32(0.9)
    data = (wav_bytes if kind == 'wav' else flac_bytes)(x, rate)
    y = model_rate(sess, data, tmp_path, f'{kind}{seed}.{kind}')
    want = sess.transcribe_encoded([data])[0]
    return sess.stream_encoded, pieces_of(data, byte_sizes(len(data), rng)), y, want


KINDS = ['pcm44100', 'pcm48000', 'pcm22050', 'wav', 'flac']


@pytest.mark.parametrize('kind', KINDS)
def test_peek_equals_transcribe_and_changes_nothing(sess, kind, tmp_path):
    open_stream, pieces, y, want = inputs(kind, 7100 + KINDS.index(kind), 45.0, tmp_path, sess)
    with open_stream() as st:
        peeked = run(st, pieces)
    with open_stream() as st:
        plain = run(st, pieces, peek=False)
    regions = check_peeks_transcribe(sess, peeked, y)
    assert len(regions) > 20
    # the chunks of every push and of the finish are the same with and without peeks, and equal the whole-recording call
    for p, q in zip(chunks_of(peeked), chunks_of(plain)):
        assert p[1] == q[1]
        assert_same_notes(p[2], q[2])
    assert len(chunks_of(peeked)) == len(chunks_of(plain))
    ranges, notes = flat(peeked)
    assert ranges == want[1] and len(ranges) > 3
    assert_same_notes(notes, want[2])
    assert check_region(peeked, keep_samples()) == 0


def test_region_properties(sess):
    """During a leading silence longer than max_sil_kept, inside a silence long enough for early delivery, and for a
    recording no longer than min_length; and the one exception, a recording that stays silent."""
    rng = np.random.default_rng(5)
    noise = (0.0005 * rng.standard_normal(8 * SR)).astype(np.float32)            # -66 dBFS: silent for the slicer
    t = np.arange(7 * SR) / SR
    p1 = (0.5 * synth.synth_waveform(71, seconds=7.0) + 0.2 * np.sin(2 * np.pi * 220.0 * t)).astype(np.float32)
    silent = noise.copy()
    silent[int(0.4 * SR):int(0.6 * SR)] *= np.float32(0.1)   # the trailing rule cuts the all-silent recording in this dip
    waves = {'leading': np.concatenate([noise, synth.synth_waveform(79, seconds=12.0)]),
             'early': np.concatenate([p1, np.zeros(3 * SR, np.float32), synth.synth_waveform(72, seconds=6.5)]),
             'short': synth.synth_waveform(77, seconds=3.0),
             'silent': silent}
    for name, x in waves.items():
        with sess.stream() as st:
            log = run(st, pieces_of(x, [4410] * (x.shape[0] // 4410 + 1)))
        check_peeks_transcribe(sess, log, x)
        exceptions = check_region(log, keep_samples())
        ranges, notes = flat(log)
        want = sess.transcribe_sliced(x)
        assert ranges == want[1]
        assert_same_notes(notes, want[2])
        assert exceptions == (1 if name == 'silent' else 0), name
        peeks = [e[1][0] for e in log if e[0] == 'peek' and e[1]]
        if name == 'short':
            assert all(a == 0 for a, _ in peeks)
        if name in ('leading', 'silent'):       # the region follows the silence: it starts past sample 0 before the end
            assert max(a for a, _ in peeks) > 4 * SR
        if name == 'early':                     # a peek after the early delivery begins past the delivered chunk
            first = next(i for i, e in enumerate(log) if e[0] == 'chunks' and e[1])
            assert first < len(log) - 1 and log[first + 1][1][0][0] >= log[first][1][-1][1]


def test_empty_region(sess):
    with sess.stream() as st, sess.stream(48000) as s48, sess.stream_encoded() as enc:
        assert st.peek() == ([], [], [])                     # right after open
        assert enc.peek() == ([], [], [])
        enc.push(ge.wav_file(np.zeros(100, np.float32), 44100, 's16')[:20])     # the header is not complete yet
        assert enc.peek() == ([], [], [])
        s48.push(np.zeros(1, np.float32))                    # one input sample fixes no model-rate sample
        assert s48.info()['fixed'] == 0 and s48.peek() == ([], [], [])
        x = synth.synth_waveform(3, seconds=2.0)
        st.push(x)
        _, r, _ = st.peek()
        assert r == [(0, x.shape[0])] and sess.load() == [(1, 1 + x.shape[0] // 512)]
        assert s48.peek() == ([], [], []) and sess.load() == [(0, 0)]     # no GPU work
        # a peek keeps its own Notes: the last push's results stay
        assert st._results()[1] == [] and st.peek()[1] == r


def test_peek_many_equals_each_peek(sess, tmp_path):
    opened, feeds, ys = [], [], []
    try:
        for k, kind in enumerate(KINDS):
            open_stream, pieces, y, _ = inputs(kind, 7200 + k, 25.0, tmp_path, sess)
            opened.append(open_stream())
            feeds.append(pieces)
            ys.append(y)
        steps = max(len(p) for p in feeds)
        for i in range(0, steps, max(1, steps // 12)):
            for st, pieces in zip(opened, feeds):
                for p in pieces[i:i + max(1, steps // 12)]:
                    st.push(p)
            alone = [st.peek() for st in opened]
            before = sess.stats()
            many = sess.peek_many(opened)
            assert sess.stats()['steps'] == before['steps'] + 1
            for a, m in zip(alone, many):
                assert a[0] == m[0] and a[1] == m[1]
                assert_same_notes(a[2], m[2])
        assert sum(len(m[1]) for m in many) >= 4
    finally:
        for st in opened:
            st.close()
    assert sess.peek_many([]) == []


def test_threads_peek_and_push_disjoint_streams(sess):
    n = 6
    rates = [44100, 48000, 22050, 44100, 48000, 44100]
    xs = [synth.synth_waveform(7300 + t, seconds=30.0, sr=rates[t], silence_gaps=True) for t in range(n)]
    feeds = [pieces_of(x, push_sizes(x.shape[0], r, np.random.default_rng(t))) for t, (x, r) in enumerate(zip(xs, rates))]

    def one(t):
        with sess.stream(rates[t]) as st:
            return run(st, feeds[t])

    want = [one(t) for t in range(n)]
    got, errors = [None] * n, []

    def work(t):
        try:
            got[t] = one(t)
        except Exception as e:                # noqa: BLE001  (reported below)
            errors.append(e)

    # a long call holds the session while every thread's first peek queues behind it: they share the next step
    long_clip = [synth.synth_waveform(7399, seconds=600.0)] * 4
    before = sess.stats()
    holder = threading.Thread(target=sess.transcribe, args=(long_clip,))
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
    for g, w in zip(got, want):
        assert len(g) == len(w)
        for p, q in zip(g, w):
            assert p[0] == q[0] and p[1] == q[1]
            assert_same_notes(p[2], q[2])
    after = sess.stats()
    assert after['max_calls'] > 1 and after['steps'] - before['steps'] < after['calls'] - before['calls']


def test_refusals(sess):
    lib = sess.lib
    x = synth.synth_waveform(7400, seconds=40.0, silence_gaps=True)
    pieces = pieces_of(x, [SR // 2] * 80)
    other = nsess.Session(sess.path, 0)
    st, st2, fin, bad = sess.stream(), sess.stream(), sess.stream(), sess.stream_encoded()
    o = other.stream()
    try:
        first = [('chunks', *st.push(p)[1:]) for p in pieces[:30]]
        st2.push(pieces[0])
        fin.finish()
        with pytest.raises(_lib.SomeB200Error):
            bad.push(b'RIFF\x10\x00\x00\x00NOTAWAVEFILE....' * 4)
        before = st.peek()

        def many(streams, notes, count=None):
            hs = (C.c_void_p * max(len(streams), 1))(*[s.handle if s is not None else None for s in streams])
            ns = (C.c_void_p * max(len(notes), 1))(*[n.handle for n in notes])
            _lib.check(lib.some_stream_peek_many(hs, len(streams) if count is None else count, ns))

        n1, n2 = nsess.Notes(), nsess.Notes()
        with pytest.raises(_lib.SomeB200Error, match='bad arguments'):
            _lib.check(lib.some_stream_peek_many(None, 1, (C.c_void_p * 1)(n1.handle)))
        with pytest.raises(_lib.SomeB200Error, match='bad arguments'):
            many([st], [n1], count=-1)
        with pytest.raises(_lib.SomeB200Error, match='stream 1 is NULL'):
            many([st, None], [n1, n2])
        with pytest.raises(_lib.SomeB200Error, match='stream 1 belongs to another session'):
            many([st, o], [n1, n2])
        with pytest.raises(_lib.SomeB200Error, match=r'stream 1 appears twice \(also at 0\)'):
            many([st, st], [n1, n2])
        with pytest.raises(_lib.SomeB200Error, match='stream 1 has finished'):
            many([st, fin], [n1, n2])
        with pytest.raises(_lib.SomeB200Error, match='stream 1 was refused'):
            many([st, bad], [n1, n2])
        with pytest.raises(_lib.SomeB200Error, match='stream 1 shares its some_notes with stream 0'):
            many([st, st2], [n1, n1])
        with pytest.raises(_lib.SomeB200Error, match='has finished'):
            fin.peek()
        with pytest.raises(_lib.SomeB200Error, match='was refused'):
            bad.peek()
        assert nsess.Notes.results(n1, sess.timestep) == ([], [])      # no out changed
        after = st.peek()
        assert before[1] == after[1]
        assert_same_notes(before[2], after[2])
        ranges, notes = flat(first + run(st, pieces[30:], peek=False))
        want = sess.transcribe_sliced(x)
        assert ranges == want[1] and len(ranges) > 1
        assert_same_notes(notes, want[2])
        n1.close(), n2.close()
    finally:
        for s in (st, st2, fin, bad, o):
            s.close()
        other.close()


def test_two_replicas_peek_as_one_device(sess, tmp_path):
    pair = nsess.Session(sess.path, [0, 0])
    try:
        logs = []
        for s in (sess, pair):
            opened = [s.stream(), s.stream(48000)]
            xs = [synth.synth_waveform(7500, seconds=30.0, silence_gaps=True),
                  synth.synth_waveform(7501, seconds=30.0, sr=48000, silence_gaps=True)]
            log = []
            for a in range(0, 30, 2):
                for st, x, r in zip(opened, xs, (SR, 48000)):
                    st.push(x[a * r:(a + 2) * r])
                log.append(s.peek_many(opened))
            for st in opened:
                st.close()
            logs.append(log)
        for p, q in zip(*logs):
            for a, b in zip(p, q):
                assert a[1] == b[1]
                assert_same_notes(a[2], b[2])
        assert any(len(a[1]) for a in logs[1][-1])
    finally:
        pair.close()


def test_c_example_peeks(sess, tmp_path):
    if sess.kind != 'two_head':
        pytest.skip('one model kind is enough for the example')
    example = REPO / 'examples' / 'some_stream'
    wav = tmp_path / 'rec.wav'
    synth.write_wav16(wav, synth.synth_waveform(4322, seconds=40.0, silence_gaps=True))
    data = wav.read_bytes()
    plain = subprocess.run([str(example), str(sess.path), '-'], input=data, capture_output=True, timeout=300)
    assert plain.returncode == 0, plain.stderr
    ms = 500
    run_ = subprocess.run([str(example), '--peek', str(ms), str(sess.path), '-'], input=data, capture_output=True, timeout=300)
    assert run_.returncode == 0, run_.stderr
    lines = run_.stdout.decode().splitlines()
    final = [ln for ln in lines if not ln.startswith('~ ')]
    assert len(final) > 20 and final == plain.stdout.decode().splitlines()
    # the same peeks from Python, at the same push boundaries: 64 KB reads, a peek once another `ms` of audio is in
    want, next_ms = [], ms
    with sess.stream_encoded() as st:
        for a in range(0, len(data), 1 << 16):
            st.push(data[a:a + (1 << 16)])
            received, rate = st.info()['received'], st.meta()['rate']
            if rate and received * 1000 >= next_ms * rate:
                offsets, _, notes = st.peek()
                for off, nt in zip(offsets, notes):
                    for m, d, r in zip(nt['note_midi'], nt['note_dur'], nt['note_rest']):
                        want.append('~ %.17g %.9g %.17g %d' % (off, m, d, 1 if r else 0))
                next_ms = (received * 1000 // rate // ms + 1) * ms
    provisional = [ln for ln in lines if ln.startswith('~ ')]
    assert len(provisional) > 20 and provisional == want
