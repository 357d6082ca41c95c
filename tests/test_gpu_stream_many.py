"""Many streams of one session advanced together (some_stream_push_many, Session.push_many): every stream's chunks equal
some_session_transcribe_sliced on its whole recording, arrive in the call in which a single push would deliver them, and
chunks closed in several streams at once come from one batch.  The many-window kernels behind the step
(some_resample_kaiser_windows, some_slicer_rms_windows) equal one single-window launch per window bit for bit."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from some_b200 import _lib, audio, export, synth
from some_b200 import session as nsess
from some_b200.slicer import Slicer

pytestmark = pytest.mark.gpu
SR = 44100
RATES = [44100, 48000, 32000, 22050, 16000]


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


def assert_same(got, want):
    assert got[0] == want[0] and got[1] == want[1]
    assert_same_notes(got[2], want[2])


def stream_current():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_windows(lib, kind, windows):
    """Packs the windows, copies the descriptors to the device and makes the one launch."""
    Win, nbytes, pack, launch = {
        'resample': (_lib.ResampleWindow, lib.some_resample_windows_bytes, lib.some_resample_windows_pack,
                     lib.some_resample_kaiser_windows),
        'rms': (_lib.RmsWindow, lib.some_slicer_rms_windows_bytes, lib.some_slicer_rms_windows_pack, lib.some_slicer_rms_windows),
    }[kind]
    arr = (Win * len(windows))(*windows)
    desc = np.zeros(nbytes(len(windows)), np.uint8)
    _lib.check(pack(arr, len(windows), desc.ctypes.data), kind)
    desc_d = torch.from_numpy(desc).cuda()
    _lib.check(launch(desc.ctypes.data, desc_d.data_ptr(), stream_current()), kind)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- kernels
def test_many_window_resampling_equals_single_windows():
    """Windows at random positions of recordings at three rate pairs (up, down, a larger down ratio), open and final, and
    empty ones, in one launch; each equals its own some_resample_kaiser_window launch bit for bit."""
    lib = _lib.load()
    rng = np.random.default_rng(5)
    t_end, x_first = C.c_longlong(), C.c_longlong()
    windows, keep, want = [], [], []
    for j in range(18):
        rate = [22050, 48000, 96000][j % 3]
        table = audio._device_table(rate, SR, 'cuda')
        x = synth.synth_waveform(40 + j, seconds=6.0, sr=rate, silence_gaps=True)
        received = int(rng.integers(1, x.shape[0] + 1)) if j % 6 else x.shape[0]
        final = int(j % 4 == 0 or received == x.shape[0])
        _lib.check(lib.some_resample_window_plan(received, final, 0, rate, SR, int(table.numel()), C.byref(t_end),
                                                 C.byref(x_first)))
        fixed = t_end.value
        t_begin = int(rng.integers(0, fixed + 1))
        t_stop = t_begin if j % 5 == 2 else int(rng.integers(t_begin, fixed + 1))    # some empty windows
        _lib.check(lib.some_resample_window_plan(received, final, t_begin, rate, SR, int(table.numel()), C.byref(t_end),
                                                 C.byref(x_first)))
        xf = max(0, x_first.value - int(rng.integers(0, 300)))
        buf = torch.from_numpy(x[xf:received].copy()).cuda()
        y_first = t_begin - int(rng.integers(0, 100))
        n_y = max(1, t_stop - y_first + 64)
        y_many = torch.full((n_y,), float('nan'), device='cuda')
        y_one = torch.full((n_y,), float('nan'), device='cuda')
        args = [buf.data_ptr(), xf, received, final, None, y_first, t_begin, t_stop, rate, SR, table.data_ptr(),
                int(table.numel())]
        _lib.check(lib.some_resample_kaiser_window(*args[:4], y_one.data_ptr(), *args[5:], stream_current()))
        args[4] = y_many.data_ptr()
        windows.append(_lib.ResampleWindow(*args))
        keep += [buf, table, y_many]
        want.append((y_one, y_many, t_stop - t_begin))
    assert sum(n == 0 for _, _, n in want) >= 3 and sum(w.final for w in windows) >= 3
    launch_windows(lib, 'resample', windows)
    for y_one, y_many, n in want:
        a, b = y_one.cpu().numpy(), y_many.cpu().numpy()
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))       # NaN where nothing was written, in both
    # a window whose outputs are not fixed yet is refused, and named
    bad = _lib.ResampleWindow(*[getattr(windows[1], f) for f, _ in _lib.ResampleWindow._fields_])
    bad.final, bad.t_end = 0, bad.received * 10
    arr = (_lib.ResampleWindow * 3)(windows[0], windows[2], bad)
    desc = np.zeros(lib.some_resample_windows_bytes(3), np.uint8)
    with pytest.raises(_lib.SomeB200Error, match='window 2'):
        _lib.check(lib.some_resample_windows_pack(arr, 3, desc.ctypes.data))


def test_many_window_rms_equals_single_windows():
    lib = _lib.load()
    rng = np.random.default_rng(6)
    sl = Slicer(SR, max_sil_kept=1000)
    win, hop, half = sl.win_size, sl.hop_size, sl.win_size // 2
    windows, keep, want = [], [], []
    for j in range(20):
        wave = synth.synth_waveform(60 + j, seconds=float(rng.uniform(1.0, 12.0)), silence_gaps=True)
        n = wave.shape[0]
        total = 1 + (n + 2 * half - win) // hop
        f0 = int(rng.integers(0, total))
        f1 = f0 if j % 7 == 3 else int(rng.integers(f0 + 1, min(total, f0 + 600) + 1))
        lo, hi = max(0, f0 * hop - half), (f1 - 1) * hop - half + win
        final = hi > n or j % 3 == 0                                   # open windows only where the frames allow it
        hi = min(hi, n) if final else hi
        lo = max(0, lo - int(rng.integers(0, 200)))
        if f1 == f0:                                                   # an empty window over some buffer
            hi = min(n, lo + 1000)
        buf = torch.from_numpy(wave[lo:hi].copy()).cuda()
        one = torch.full((max(1, f1 - f0),), float('nan'), device='cuda')
        many = torch.full((max(1, f1 - f0),), float('nan'), device='cuda')
        args = [buf.data_ptr(), lo, hi - lo, n if final else -1, win, hop, None, f0, f1]
        _lib.check(lib.some_slicer_rms_window(*args[:6], one.data_ptr(), *args[7:], stream_current()))
        args[6] = many.data_ptr()
        windows.append(_lib.RmsWindow(*args))
        keep.append(buf)
        want.append((one, many))
    assert sum(w.n_samples >= 0 for w in windows) >= 3 and sum(w.n_samples < 0 for w in windows) >= 3
    launch_windows(lib, 'rms', windows)
    for one, many in want:
        np.testing.assert_array_equal(one.cpu().numpy().view(np.uint32), many.cpu().numpy().view(np.uint32))
    bad = _lib.RmsWindow(*[getattr(windows[1], f) for f, _ in _lib.RmsWindow._fields_])
    bad.held, bad.n_samples = 0, -1
    arr = (_lib.RmsWindow * 2)(windows[0], bad)
    desc = np.zeros(lib.some_slicer_rms_windows_bytes(2), np.uint8)
    if bad.f_end > bad.f_begin:
        with pytest.raises(_lib.SomeB200Error, match='window 1.*buffer holds'):
            _lib.check(lib.some_slicer_rms_windows_pack(arr, 2, desc.ctypes.data))


# ------------------------------------------------------------------------------------------------- streams
def recordings(rng):
    """(rate, waveform, params) of 24 streams: seeded synth recordings at mixed rates, a leading silence longer than
    max_sil_kept, a recording shorter than min_length, an all-silent one and an empty one."""
    out = []
    for i in range(20):
        rate = RATES[i % len(RATES)]
        params = nsess.slicer_params(max_sil_kept=500, min_interval=200) if i % 4 == 3 else None
        out.append((rate, synth.synth_waveform(3000 + i, seconds=float(rng.uniform(8.0, 40.0)), sr=rate, silence_gaps=True),
                    params))
    noise = (0.0005 * rng.standard_normal(6 * 48000)).astype(np.float32)              # -66 dBFS: silent for the slicer
    out.append((48000, np.concatenate([noise, synth.synth_waveform(3100, seconds=12.0, sr=48000)]), None))
    out.append((22050, synth.synth_waveform(3101, seconds=3.0, sr=22050), None))      # shorter than min_length: one chunk
    out.append((32000, (0.0005 * rng.standard_normal(12 * 32000)).astype(np.float32), None))  # all silent
    out.append((44100, np.zeros(0, np.float32), None))                                # empty
    return out


def blocks(n, rate, rng):
    """Random block sizes that cover n samples: 0 and 1 sample, up to half a second."""
    sizes = []
    while sum(sizes) < n:
        r = rng.random()
        sizes.append(0 if r < 0.08 else 1 if r < 0.14 else int(rng.integers(2, rate // 2)))
    return sizes


def run_ticks(sess, streams, waves, sizes, finish_at, rng=None, single=()):
    """Advances the streams tick by tick: at tick k, stream i pushes its block sizes[i][k] (if any is left) and finishes at
    tick finish_at[i].  Streams in `single` use Stream.push / Stream.finish instead, on odd ticks (push_many on even ones).
    Returns each stream's (offsets, ranges, notes) concatenated, and the ranges each tick delivered to each stream."""
    got = [([], [], []) for _ in streams]
    ticks = [[] for _ in streams]
    pos = [0] * len(streams)
    done = [False] * len(streams)
    k = 0
    while not all(done):
        items, idx, fin = [], [], []
        for i, st in enumerate(streams):
            if done[i]:
                continue
            m = sizes[i][k] if k < len(sizes[i]) else 0
            part = waves[i][pos[i]:pos[i] + m]
            pos[i] += part.shape[0]
            f = k >= finish_at[i]
            if i in single and k % 2:
                res = [st.push(part)]
                if f:
                    res.append(st.finish())
                res = tuple(sum((r[j] for r in res), []) for j in range(3))
                for acc, p in zip(got[i], res):
                    acc += p
                ticks[i].append(res[1])
            else:
                items.append((st, part)), idx.append(i), fin.append(f)
            if f:
                done[i] = True
        if items:
            for i, res in zip(idx, sess.push_many(items, fin)):
                for acc, p in zip(got[i], res):
                    acc += p
                ticks[i].append(res[1])
        k += 1
    return got, ticks


def test_streams_equal_transcribe_sliced(sess):
    rng = np.random.default_rng(24)
    recs = recordings(rng)
    want = [sess.transcribe_sliced(w, r, p) for r, w, p in recs]
    assert any(len(w[2]) > 3 for w in want) and want[-1][1] == [(0, 0)] and len(want[-3][1]) == 1
    streams = [sess.stream(r, p) for r, _, p in recs]
    sizes = [blocks(w.shape[0], r, rng) for r, w, _ in recs]
    # finish at different ticks: some with their last samples, some a few ticks later
    finish_at = [len(s) - 1 + int(rng.integers(0, 4)) * (i % 2) for i, s in enumerate(sizes)]
    finish_at = [max(0, f) for f in finish_at]
    got, _ = run_ticks(sess, streams, [w for _, w, _ in recs], sizes, finish_at)
    for i in range(len(recs)):
        assert_same(got[i], want[i])
        st = streams[i].info()
        assert st['received'] == recs[i][1].shape[0]
        streams[i].close()


def test_chunks_of_several_streams_close_in_one_call(sess):
    """Identical recordings in lockstep: a call that delivers a chunk to one delivers the same chunk, with the same notes, to
    all; and in the call in which Stream.push with the same blocks delivers it."""
    rng = np.random.default_rng(31)
    rate = 48000
    wave = synth.synth_waveform(3200, seconds=50.0, sr=rate, silence_gaps=True)
    sizes = blocks(wave.shape[0], rate, rng)
    streams = [sess.stream(rate) for _ in range(4)]
    per_call = []
    pos = 0
    for k, m in enumerate(sizes + [0]):
        final = k == len(sizes)
        res = sess.push_many([(st, wave[pos:pos + m]) for st in streams], [final] * 4)
        pos += m
        for r in res[1:]:
            assert r[1] == res[0][1]
            assert_same_notes(r[2], res[0][2])
        per_call.append(res[0][1])
    for st in streams:
        st.close()
    assert sum(bool(r) for r in per_call) > 3
    alone = []
    with sess.stream(rate) as st:
        pos = 0
        for m in sizes:
            alone.append(st.push(wave[pos:pos + m])[1])
            pos += m
        alone.append(st.finish()[1])
    assert per_call == alone
    assert sum(per_call, []) == sess.transcribe_sliced(wave, rate)[1]


def test_mixing_push_and_push_many_and_threads(sess):
    rng = np.random.default_rng(41)
    rates = [44100, 48000, 22050, 32000, 16000, 44100, 48000]
    waves = [synth.synth_waveform(3300 + i, seconds=25.0, sr=r, silence_gaps=True) for i, r in enumerate(rates)]
    want = [sess.transcribe_sliced(w, r) for w, r in zip(waves, rates)]
    # one thread: streams 0 and 1 alternate Stream.push and push_many
    streams = [sess.stream(r) for r in rates[:3]]
    sizes = [blocks(w.shape[0], r, rng) for w, r in zip(waves[:3], rates[:3])]
    got, _ = run_ticks(sess, streams, waves[:3], sizes, [len(s) for s in sizes], single=(0, 1))
    for i in range(3):
        assert_same(got[i], want[i])
        streams[i].close()
    # two threads with push_many on disjoint streams, a third with Stream.push
    results, errors = {}, []

    def many(ids, seed):
        try:
            r = np.random.default_rng(seed)
            sts = [sess.stream(rates[i]) for i in ids]
            sz = [blocks(waves[i].shape[0], rates[i], r) for i in ids]
            g, _ = run_ticks(sess, sts, [waves[i] for i in ids], sz, [len(s) for s in sz])
            for i, res, st in zip(ids, g, sts):
                results[i] = res
                st.close()
        except Exception as e:            # noqa: BLE001  (reported below)
            errors.append(e)

    def single(i):
        try:
            r = np.random.default_rng(i)
            got = ([], [], [])
            with sess.stream(rates[i]) as st:
                pos = 0
                for m in blocks(waves[i].shape[0], rates[i], r):
                    for acc, p in zip(got, st.push(waves[i][pos:pos + m])):
                        acc += p
                    pos += m
                for acc, p in zip(got, st.finish()):
                    acc += p
            results[i] = got
        except Exception as e:            # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=many, args=([0, 2, 4], 1)), threading.Thread(target=many, args=([1, 3, 5], 2)),
               threading.Thread(target=single, args=(6,))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for i in range(len(rates)):
        assert_same(results[i], want[i])


def call_raw(sess, streams, samples, n, finish, notes, count=None):
    lib = sess.lib
    k = len(streams)
    arr = (C.c_void_p * max(k, 1))(*streams)
    ptrs = (C.c_void_p * max(k, 1))(*samples)
    lens = (C.c_longlong * max(k, 1))(*n)
    outs = (C.c_void_p * max(k, 1))(*notes)
    fin = None if finish is None else (C.c_int * max(k, 1))(*finish)
    _lib.check(lib.some_stream_push_many(arr, ptrs, lens, fin, k if count is None else count, outs), 'some_stream_push_many')


def test_refusals_change_nothing(sess):
    rng = np.random.default_rng(51)
    rates = [44100, 48000, 22050]
    waves = [synth.synth_waveform(3400 + i, seconds=20.0, sr=r, silence_gaps=True) for i, r in enumerate(rates)]
    streams = [sess.stream(r) for r in rates]
    got = [([], [], []) for _ in streams]
    pos = [0, 0, 0]

    def step(fin=None):
        items = []
        for i, st in enumerate(streams):
            m = int(rng.integers(0, rates[i]))
            items.append((st, waves[i][pos[i]:pos[i] + m]))
            pos[i] += items[-1][1].shape[0]
        for acc3, res in zip(got, sess.push_many(items, fin)):
            for acc, p in zip(acc3, res):
                acc += p

    step()
    other = nsess.Session(sess.path, 0)
    foreign = other.stream()
    done = sess.stream()
    done.finish()
    short = sess.stream(96000)
    short.push(np.zeros(1, np.float32))
    x = np.ones(10, np.float32)
    h = [st.handle for st in streams]
    nt = [st.notes.handle for st in streams]
    cases = [
        ([(streams[0], x), (streams[1], x), (streams[0], x)], None, 'stream 2 appears twice'),
        ([(streams[0], x), (foreign, x)], None, 'stream 1 belongs to another session'),
        ([(streams[0], x), (streams[1], x), (done, x)], None, 'stream 2 has finished'),
        ([(streams[0], x), (short, np.zeros(0, np.float32))], [False, True], 'stream 1: Input signal length=1 is too small'),
    ]
    infos = lambda: [st.info() for st in streams + [short]]          # noqa: E731
    before = infos()
    for items, fin, msg in cases:
        with pytest.raises(_lib.SomeB200Error, match=msg):
            sess.push_many(items, fin)
        assert infos() == before
    raw = [
        ((h, [x.ctypes.data] * 3, [10, 10, 10], None, [nt[0], nt[1], nt[0]]), 'stream 2 shares its some_notes with stream 0'),
        ((h, [x.ctypes.data] * 3, [10, -1, 10], None, nt), 'stream 1: -1 samples'),
        ((h, [x.ctypes.data, None, x.ctypes.data], [10, 5, 10], None, nt), 'stream 1: 5 samples'),
        ((h, [x.ctypes.data] * 3, [10, 10, 10], None, nt, -1), 'bad arguments'),
        (([h[0], None], [x.ctypes.data] * 2, [10, 10], None, nt[:2]), 'stream 1 is NULL'),
    ]
    for args, msg in raw:
        with pytest.raises(_lib.SomeB200Error, match=msg):
            call_raw(sess, *args)
        assert infos() == before
    call_raw(sess, h, [x.ctypes.data] * 3, [10, 10, 10], None, nt, 0)   # count 0: nothing happens
    assert infos() == before
    # the next valid calls still give the one-shot result
    while any(p < w.shape[0] for p, w in zip(pos, waves)):
        step()
    step([True, True, True])
    for i in range(3):
        assert_same(got[i], sess.transcribe_sliced(waves[i], rates[i]))
        streams[i].close()
    for st in (foreign, done, short):
        st.close()
    other.close()


@pytest.mark.parametrize('rate', [44100, 48000])
def test_leading_silence_keeps_memory_bounded(sess, rate):
    """A stream advanced only through push_many keeps the bound a single stream keeps during a long leading silence."""
    rng = np.random.default_rng(77)
    f = nsess.slicer_frames(SR)
    noise = (0.0005 * rng.standard_normal(40 * rate)).astype(np.float32)
    voice = synth.synth_waveform(79, seconds=20.0, sr=rate)
    waves = [np.concatenate([noise, voice]), noise]
    streams = [sess.stream(rate) for _ in waves]
    other = sess.stream(22050)                                      # a neighbour in every call
    other_wave = synth.synth_waveform(80, seconds=70.0, sr=22050, silence_gaps=True)
    infos = [[] for _ in waves]
    got = [([], [], []) for _ in waves]
    pos, opos, k = [0, 0], 0, 0
    while any(p < w.shape[0] for p, w in zip(pos, waves)):
        items = []
        for i, w in enumerate(waves):
            m = int(rng.integers(rate // 1000, rate + 1))
            items.append((streams[i], w[pos[i]:pos[i] + m]))
            pos[i] += items[-1][1].shape[0]
        items.append((other, other_wave[opos:opos + 22050 // 2]))
        opos += 22050 // 2
        for i, res in enumerate(sess.push_many(items)[:2]):
            for acc, p in zip(got[i], res):
                acc += p
            infos[i].append((items[i][1].shape[0], streams[i].info()))
        k += 1
    for i, res in enumerate(sess.push_many([(st, np.zeros(0, np.float32)) for st in streams], [True, True])):
        for acc, p in zip(got[i], res):
            acc += p
    silent_fixed = 40 * SR - 4 * f.hop_size
    bound = (2 * f.max_sil_kept + 2) * f.hop_size + f.win_size
    for i in range(2):
        assert_same(got[i], sess.transcribe_sliced(waves[i], rate))
        late = [(m, inf) for m, inf in infos[i] if (f.min_length + 60) * f.hop_size < inf['fixed'] < silent_fixed]
        assert len(late) > 20
        assert all(inf['held'] <= bound + m * SR // rate + 512 for m, inf in late), max(inf['held'] - m for m, inf in late)
        streams[i].close()
    other.close()
