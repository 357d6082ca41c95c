"""Streaming on the H100 (some_stream_*, csrc/session.cu): a recording pushed in any pieces gives, chunk by chunk, exactly
what some_session_transcribe_sliced gives for the whole recording (ranges and bit-identical notes), delivers a chunk by the
delivery bound, keeps its device buffer bounded, and serves several threads on one session.  The windowed kernels behind it
(some_resample_kaiser_window, some_slicer_rms_window) equal the whole-recording kernels bit for bit."""
import ctypes as C
import pathlib
import subprocess
import threading

import numpy as np
import pytest
import torch

from some_b200 import _lib, audio, export, synth
from some_b200 import session as nsess
from some_b200.slicer import Slicer

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


def stream_all(sess, wave, rate, sizes, params=None, infos=None):
    offsets, ranges, notes = [], [], []
    with sess.stream(rate, params) as st:
        a = 0
        for m in sizes:
            o, r, nt = st.push(wave[a:a + m])
            a += m
            offsets += o
            ranges += r
            notes += nt
            if infos is not None:
                infos.append((m, st.info()))
        o, r, nt = st.finish()
        offsets += o
        ranges += r
        notes += nt
    return offsets, ranges, notes


def assert_same(got, want):
    assert got[0] == want[0] and got[1] == want[1]
    assert_same_notes(got[2], want[2])


# ------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize('rate', [48000, 22050])
def test_windowed_resampling_equals_whole(rate):
    lib = _lib.load()
    rng = np.random.default_rng(rate)
    x = synth.synth_waveform(31, seconds=20.0, sr=rate, silence_gaps=True)
    whole = audio.resample(x, rate, SR)
    table = audio._device_table(rate, SR, 'cuda')
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    got = np.full(whole.shape[0], np.nan, np.float32)
    received = fixed = 0
    t_end, x_first = C.c_longlong(), C.c_longlong()
    while True:
        received = min(x.shape[0], received + int(rng.integers(1, 30000)))
        final = int(received == x.shape[0])
        _lib.check(lib.some_resample_window_plan(received, final, fixed, rate, SR, int(table.numel()), C.byref(t_end),
                                                 C.byref(x_first)))
        buf = torch.from_numpy(x[x_first.value:received].copy()).cuda()
        y = torch.empty(max(1, t_end.value - fixed), device='cuda')
        _lib.check(lib.some_resample_kaiser_window(buf.data_ptr(), x_first.value, received, final, y.data_ptr(), fixed, fixed,
                                                   t_end.value, rate, SR, table.data_ptr(), int(table.numel()), stream),
                   'some_resample_kaiser_window')
        got[fixed:t_end.value] = y[:t_end.value - fixed].cpu().numpy()
        fixed = t_end.value
        if final:
            break
    assert fixed == whole.shape[0]
    np.testing.assert_array_equal(got.view(np.uint32), whole.view(np.uint32))
    # outputs whose right wing reaches past the received input are refused
    _lib.check(lib.some_resample_window_plan(1000, 0, 0, rate, SR, int(table.numel()), C.byref(t_end), C.byref(x_first)))
    buf = torch.from_numpy(x[:1000].copy()).cuda()
    with pytest.raises(_lib.SomeB200Error, match='right wings'):
        _lib.check(lib.some_resample_kaiser_window(buf.data_ptr(), 0, 1000, 0, y.data_ptr(), 0, 0, t_end.value + 1, rate, SR,
                                                   table.data_ptr(), int(table.numel()), stream))


def test_windowed_rms_equals_whole():
    lib = _lib.load()
    rng = np.random.default_rng(3)
    sl = Slicer(SR, max_sil_kept=1000)
    wave = synth.synth_waveform(32, seconds=60.0, silence_gaps=True)
    n = wave.shape[0]
    whole = sl.rms(wave)
    win, hop, half = sl.win_size, sl.hop_size, sl.win_size // 2
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    f0 = 0
    while f0 < whole.shape[0]:
        f1 = min(whole.shape[0], f0 + int(rng.integers(1, 400)))
        lo, hi = max(0, f0 * hop - half), (f1 - 1) * hop - half + win
        final = hi > n                                            # frames that read past the end need the final length
        hi = min(hi, n)
        buf = torch.from_numpy(wave[lo:hi].copy()).cuda()
        out = torch.empty(f1 - f0, device='cuda')
        _lib.check(lib.some_slicer_rms_window(buf.data_ptr(), lo, hi - lo, n if final else -1, win, hop, out.data_ptr(), f0, f1,
                                              stream), 'some_slicer_rms_window')
        np.testing.assert_array_equal(out.cpu().numpy().view(np.uint32), whole[f0:f1].view(np.uint32))
        f0 = f1
    with pytest.raises(_lib.SomeB200Error, match='buffer holds'):
        _lib.check(lib.some_slicer_rms_window(buf.data_ptr(), lo, hi - lo - 1, -1, win, hop, out.data_ptr(), f1 - 1, f1, stream))


# ------------------------------------------------------------------------------------------------- streams
def test_stream_equals_transcribe_sliced(sess):
    rng = np.random.default_rng(9002)
    wave = synth.synth_waveform(9002, seconds=300.0, silence_gaps=True)
    want = sess.transcribe_sliced(wave)
    assert len(want[2]) > 10
    infos = []
    assert_same(stream_all(sess, wave, SR, push_sizes(wave.shape[0], SR, rng), infos=infos), want)
    assert_same(stream_all(sess, wave, SR, [wave.shape[0]]), want)
    # memory: the longest chunk, 2 max_sil_kept frames and the RMS window, plus the push in progress
    f = nsess.slicer_frames(SR)
    longest = max(b - a for a, b in want[1])
    bound = longest + 2 * f.max_sil_kept * f.hop_size + f.win_size
    assert all(info['held'] <= bound + m for m, info in infos), max(info['held'] - m for m, info in infos)
    assert max(info['held'] for _, info in infos) < wave.shape[0] // 4
    assert infos[-1][1]['received'] == infos[-1][1]['fixed'] == wave.shape[0]


@pytest.mark.parametrize('rate', [44100, 48000])
def test_leading_silence_keeps_memory_bounded(sess, rate):
    """A stream opened before the singer starts, and one that stays silent: during the leading silence the device keeps the
    first and the last max_sil_kept frames (and the RMS window), not everything since the stream opened."""
    rng = np.random.default_rng(77)
    f = nsess.slicer_frames(SR)
    noise = (0.0005 * rng.standard_normal(40 * rate)).astype(np.float32)            # -66 dBFS: silent for the slicer
    voice = synth.synth_waveform(79, seconds=20.0, sr=rate)
    for wave in (np.concatenate([noise, voice]), noise):
        infos = []
        assert_same(stream_all(sess, wave, rate, push_sizes(wave.shape[0], rate, rng), infos=infos), sess.transcribe_sliced(wave, rate))
        silent_fixed = 40 * SR - 4 * f.hop_size
        late = [(m, i) for m, i in infos if (f.min_length + 60) * f.hop_size < i['fixed'] < silent_fixed]   # pushes <= 1 s
        assert len(late) > 20
        bound = (2 * f.max_sil_kept + 2) * f.hop_size + f.win_size
        assert all(i['held'] <= bound + m * SR // rate + 512 for m, i in late), max(i['held'] - m for m, i in late)


@pytest.mark.parametrize('rate', [48000, 22050])
def test_stream_resamples_like_transcribe_sliced(sess, rate):
    rng = np.random.default_rng(rate)
    wave = synth.synth_waveform(9002, seconds=300.0, sr=rate, silence_gaps=True)
    want = sess.transcribe_sliced(wave, rate)
    assert len(want[2]) > 10
    infos = []
    assert_same(stream_all(sess, wave, rate, push_sizes(wave.shape[0], rate, rng), infos=infos), want)
    last = infos[-1][1]
    max_taps = 32769 // int(min(1.0, SR / rate) * 512)              # the resampler's right wing, in input samples
    assert last['received'] == wave.shape[0] and 0 < wave.shape[0] * SR // rate - last['fixed'] <= (max_taps + 2) * SR / rate


def test_edge_cases(sess):
    rng = np.random.default_rng(1)
    short = synth.synth_waveform(77, seconds=3.0)                   # no longer than min_length: one chunk, at finish
    with sess.stream() as st:
        assert all(st.push(short[a:a + 4410])[1] == [] for a in range(0, short.shape[0], 4410))
        got = st.finish()
    assert got[1] == [(0, short.shape[0])]
    assert_same(got, sess.transcribe_sliced(short))
    empty = np.zeros(0, np.float32)
    assert_same(stream_all(sess, empty, SR, []), sess.transcribe_sliced(empty))
    phrase = synth.synth_waveform(78, seconds=8.0)
    for tail in (0.2, 4.0):                                         # ends inside a short and inside a long silence
        wave = np.concatenate([phrase, np.zeros(int(tail * SR), np.float32)])
        assert_same(stream_all(sess, wave, SR, push_sizes(wave.shape[0], SR, rng)), sess.transcribe_sliced(wave))
    with sess.stream(96000) as st:                                  # too short to resample: refused at finish, as resampy
        st.push(np.zeros(1, np.float32))
        with pytest.raises(_lib.SomeB200Error, match='too small to resample'):
            st.finish()
    with sess.stream() as st:
        st.finish()
        with pytest.raises(_lib.SomeB200Error, match='has finished'):
            st.push(phrase[:10])
    with pytest.raises(_lib.SomeB200Error, match='min_length >= min_interval'):
        sess.stream(params=nsess.slicer_params(min_length=100, min_interval=300))


def test_early_delivery(sess):
    """Two phrases separated by 3 s of zeros: the first chunk comes back once frame max(ss + 2 keep, ss + min_interval - 1,
    begin + min_length - 1) of the silence is known, long before the second phrase."""
    # the first phrase has a sustained tone under it: no silent run inside it, so its chunk ends in the 3 s gap
    t = np.arange(7 * SR) / SR
    p1 = (0.5 * synth.synth_waveform(71, seconds=7.0) + 0.2 * np.sin(2 * np.pi * 220.0 * t)).astype(np.float32)
    p2 = synth.synth_waveform(72, seconds=6.5)
    wave = np.concatenate([p1, np.zeros(3 * SR, np.float32), p2])
    want = sess.transcribe_sliced(wave)
    sl = Slicer(SR, max_sil_kept=1000)
    rms = sl.rms(wave)
    ss = (p1.shape[0] + SR) // sl.hop_size
    while rms[ss - 1] < np.float32(sl.threshold):
        ss -= 1
    [chunk] = [k for k, (a, b) in enumerate(want[1]) if ss * sl.hop_size <= b <= (ss + sl.max_sil_kept + 1) * sl.hop_size]
    begin = want[1][chunk][0] // sl.hop_size
    j = max(ss + 2 * sl.max_sil_kept, ss + sl.min_interval - 1, begin + sl.min_length - 1)
    need = j * sl.hop_size - sl.win_size // 2 + sl.win_size                  # samples that complete frame j
    assert need < p1.shape[0] + 3 * SR
    got = ([], [], [])
    with sess.stream() as st:
        for a in range(0, need, 4410):
            for acc, part in zip(got, st.push(wave[a:min(need, a + 4410)])):
                acc += part
        assert got[1] == want[1][:chunk + 1]
        assert_same_notes(got[2], want[2][:chunk + 1])
        for acc, part in zip(got, st.push(wave[need:])):
            acc += part
        for acc, part in zip(got, st.finish()):
            acc += part
    assert_same(got, want)


def test_closing_the_session_closes_its_streams(sess):
    fresh = nsess.Session(sess.path, 0)
    st = fresh.stream()
    st.push(np.zeros(SR, np.float32))
    fresh.close()
    assert st.handle is None
    with pytest.raises(_lib.SomeB200Error, match='bad arguments'):
        st.push(np.zeros(10, np.float32))


def test_threads_share_one_session(sess):
    rates = [44100, 48000, 44100, 22050]
    waves = [synth.synth_waveform(600 + t, seconds=60.0, sr=rates[t], silence_gaps=True) for t in range(4)]
    want = [sess.transcribe_sliced(w, r) for w, r in zip(waves, rates)]
    results, errors = [None] * 4, []

    def work(t):
        try:
            rng = np.random.default_rng(t)
            results[t] = stream_all(sess, waves[t], rates[t], push_sizes(waves[t].shape[0], rates[t], rng))
        except Exception as e:            # noqa: BLE001  (reported below)
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(4):
        assert_same(results[t], want[t])


def test_c_example_streams_stdin(sess, tmp_path):
    if sess.kind != 'two_head':
        pytest.skip('one model kind is enough for the example')
    example, batch_example = REPO / 'examples' / 'some_stream', REPO / 'examples' / 'some_transcribe'
    assert example.is_file(), 'examples/some_stream is built with the library'
    linked = subprocess.run(['ldd', str(example)], capture_output=True, text=True, check=True).stdout
    assert 'libsome_b200' in linked and 'libpython' not in linked and 'libtorch' not in linked
    model = sess.path
    wav = tmp_path / 'rec.wav'
    samples = synth.write_wav16(wav, synth.synth_waveform(4321, seconds=45.0, silence_gaps=True))
    pcm = np.ascontiguousarray(samples, dtype='<f4').tobytes()
    run = subprocess.run([str(example), str(model), str(SR)], input=pcm, capture_output=True, timeout=300)
    assert run.returncode == 0, run.stderr
    want = subprocess.run([str(batch_example), str(model), str(wav)], capture_output=True, text=True, timeout=300)
    assert want.returncode == 0, want.stderr
    lines = run.stdout.decode().splitlines()
    assert len(lines) > 20 and lines == want.stdout.splitlines()
